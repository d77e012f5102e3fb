"""GPU suite (-m gpu): the resident chain's decode-ahead instantiation (chain_kernel<..., kChainAhead>, tmac_chain.cuh), which
decodes the first quads of each weight block while the warp waits for its chunk's input, against the instantiation without it
(debug knob chain_ahead = 0), which runs the whole block step after the input wait.

Decode-ahead moves only work that reads the weight block; the integer lookups are exact and the fp32 order is unchanged, so every
output must be bit for bit the same.  A sequence whose clusters need more than 3 CTAs per SM cannot run the decode-ahead
instantiation (bounded to 3 CTAs per SM for its registers): its build takes the other one, and it must still be the chain.
kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
import numpy as np
import pytest

import tmac_b200 as tb
from seq_util import TIGHT_TOL, glu, inputs, mk, oracle_gemv, run_form, same_bits, step, stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def run(steps, ext, ahead):
    """Builds the sequence as the resident chain, with (ahead = 1) or without decode-ahead, and launches it twice; returns
    (info, outputs)."""
    try:
        tb.debug_set("chain_ahead", ahead)
        return run_form("flow", steps, ext, launches=2)
    finally:
        tb.debug_set("chain_ahead", 1)


def same_both_ways(steps, ext):
    """The chain with and without decode-ahead: same ring, bit-identical outputs.  Returns the outputs."""
    info_a, got_a = run(steps, ext, 1)
    info_p, got_p = run(steps, ext, 0)
    assert info_a == info_p
    for i, (a, p) in enumerate(zip(got_a, got_p)):
        assert np.isfinite(a).all(), "op %d" % i
        assert same_bits(a, p), "op %d differs with decode-ahead" % i
    return got_a


def check(oracle, steps, xs, got, ops=None):
    for i, (o, src, off, *_) in enumerate(steps):
        if ops is not None and i not in ops:
            continue
        x = xs[src] if isinstance(src, str) else got[src][off:off + o.cfg.K].astype(np.float32)
        ref = oracle_gemv(oracle, o.cfg, o.A, o.S, x)
        err = np.abs(got[i] - ref).max() / np.abs(ref).max()
        assert err <= TIGHT_TOL, "op %d (%dx%d W%d): rel err %.3g" % (i, o.cfg.Mout, o.cfg.K, o.cfg.bits, err)


def test_bench_chain(oracle, mk):
    """The bench shape (11008x4096 W2 g128 zp, 2 blocks per warp), 8 dependent ops (the bench runs 32 of them)."""
    base = mk(11008, 4096, 2, zp=True, seed=1)
    steps = [step(base, "x")]
    for i in range(1, 8):
        steps.append(step(mk(11008, 4096, 2, zp=True, seed=1 + i), i - 1))
    xs, ext = inputs(np.random.default_rng(1), x=4096)
    got = same_both_ways(steps, ext)
    check(oracle, steps, xs, got, ops=(0, 1, 7))


def test_glu_chain(oracle, mk):
    """A SwiGLU FFN: gate and up, then down reading silu(gate) * up (the GLU instantiation)."""
    steps = [step(mk(2048, 1024, 2, zp=True, seed=11), "x"), step(mk(2048, 1024, 2, zp=True, seed=12), "x"),
             step(mk(1024, 2048, 2, zp=True, seed=13), glu(0, 0, 1, 0))]
    xs, ext = inputs(np.random.default_rng(2), x=1024)
    got = same_both_ways(steps, ext)
    check(oracle, steps, xs, got, ops=(0, 1))


@pytest.mark.parametrize("bits,g,ags", [(2, 128, 64), (4, 128, 128), (1, 64, 32), (3, 32, 32)])
def test_one_two_and_six_blocks_per_warp(oracle, mk, bits, g, ags):
    """Ops with 1, 2 and 6 blocks per warp at the bench grouping (K = 2048, 4096, 11008 over 128-wide chunks), and the same
    chain at groupings with fewer quads per chunk than the instantiation decodes ahead (g32: 2 quads).  At W3 / W4 the 11008-row
    op has 172 clusters (688 CTAs, 6 per SM on 132 SMs): both builds take the instantiation without decode-ahead, which must keep
    fitting 6 CTAs per SM."""
    kw = dict(g=g, ags=ags, zp=bits in (2, 3))
    steps = [step(mk(11008, 2048, bits, seed=21, **kw), "x"), step(mk(4096, 11008, bits, seed=22, **kw), 0),
             step(mk(512, 4096, bits, seed=23, **kw), 1)]
    xs, ext = inputs(np.random.default_rng(bits), x=2048)
    got = same_both_ways(steps, ext)
    check(oracle, steps, xs, got)


def test_sequence_too_large_for_three_ctas_per_sm(oracle, mk, stream):
    """18944 rows (the Qwen2-7B FFN width): 148 clusters, 592 CTAs -- more than 3 per SM on an H100's 132 SMs.  The build falls
    back to the instantiation without decode-ahead and the sequence is still the resident chain, correct and the same bits."""
    if 3 * torch.cuda.get_device_properties(0).multi_processor_count >= 592:
        pytest.skip("592 CTAs fit at 3 per SM on this device")
    steps = [step(mk(18944, 2048, 2, zp=True, seed=31), "x"), step(mk(512, 2048, 2, zp=True, seed=32), 0)]
    xs, ext = inputs(np.random.default_rng(3), x=2048)
    got = same_both_ways(steps, ext)
    check(oracle, steps, xs, got)
