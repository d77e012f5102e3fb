"""GPU suite (-m gpu): decode sequences over a batch of 2..4 activation rows (tmac_b200_seq_set_batch), in both forms of the resident
chain kernel, from small chains at every chunking to a decoder layer's half after attention at Llama-2-7B shapes and the bench chain.

The batch kernel decodes each weight block once and runs each row's table part, folds and scales in the one-row kernel's order, so
every check is first bit for bit: row t of every output must equal the same sequence built with one row and fed row t.  Rows are
also checked against the oracle.  kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
from types import SimpleNamespace

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from seq_util import (A_CASES, A_IDS, TIGHT_TOL, device, expect_kernel, fetch, form, glu, host, kc, mk, norm, norm_weight,
                      oracle_gemv, run_form, same_bits, sequence, step, stream)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def row_of(hx, t):
    """The one-row inputs of row t: per-row vectors ([n][len]) give their row t, norm weights ([len]) stay."""
    return {k: (v[t] if v.ndim == 2 else v) for k, v in hx.items()}


def run(name, steps, hx, n, explicit=False):
    """Builds and launches the sequence in form `name` on the host inputs hx; asserts that the resident chain serves it.  Returns
    the outputs as numpy arrays, [n][Mout] for n > 1."""
    return run_form(name, steps, device(hx), chained=True, n=n, explicit_batch=explicit)[1]


def singles(name, steps, hx, n):
    """[row t][op]: the one-row sequence fed row t."""
    return [run(name, steps, row_of(hx, t), 1) for t in range(n)]


def check_rows(got, ones, what):
    for t in range(got[0].shape[0]):
        for i, g in enumerate(got):
            assert same_bits(g[t], ones[t][i]), "%s: op %d row %d differs from the one-row sequence fed that row" % (what, i, t)


def check_oracle(oracle, steps, hx, got):
    """Plain ops of every row against the oracle, on the input the GPU op saw."""
    for t in range(got[0].shape[0]):
        for i, (o, src, off, res, f16) in enumerate(steps):
            if res is not None or not isinstance(src, (str, int)):
                continue
            x = hx[src][t] if isinstance(src, str) else got[src][t][off:off + o.cfg.K].astype(np.float32)
            ref = oracle_gemv(oracle, o.cfg, o.A, o.S, x)
            err = np.abs(got[i][t] - ref).max() / np.abs(ref).max()
            assert err <= TIGHT_TOL, "op %d row %d (%dx%d W%d): rel err %.3g" % (i, t, o.cfg.Mout, o.cfg.K, o.cfg.bits, err)


# ---- 1: every chunking, offset consumer and fan-out, both chain forms ------------------------------------------------------------
def chunking_chain(mk, g, ags, bits, zp):
    ck = min(g, 128)
    kw = dict(g=g, ags=ags, zp=zp)
    return [
        step(mk(768, 20 * ck, bits, seed=1, **kw), "x0"),       # 20 chunks: some warps hold 2 blocks, some 1
        step(mk(640, 512, bits, seed=2, **kw), 0),              # fewer rows than op 0: idle clusters
        step(mk(512, 512, bits, seed=3, **kw), 1, off=128),     # offset consumer
        step(mk(384 // bits, 256, bits, seed=4, **kw), 0, off=4),   # fan-out of op 0; ragged rows; 256/ck < 16 chunks
    ]


@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_every_chunking(oracle, mk, g, ags, bits, zp):
    steps = chunking_chain(mk, g, ags, bits, zp)
    hx = host(np.random.default_rng(g + ags + bits), x0=(4, steps[0].op.cfg.K))
    for name in ("flow", "barrier"):
        ones = singles(name, steps, hx, 4)
        for n in (2, 3, 4):
            got = run(name, steps, {"x0": hx["x0"][:n]}, n)
            check_rows(got, ones, "%s n=%d" % (name, n))
            if name == "flow":
                check_oracle(oracle, steps, {"x0": hx["x0"][:n]}, got)


# ---- 2: a decoder layer's half after attention -------------------------------------------------------------------------------------
def half_layer(mk, hidden, F, seed, f16=False):
    kw = dict(g=128, ags=64, zp=True)
    return [step(mk(hidden, hidden, 2, seed=seed, **kw), "att", res="x"),
            step(mk(F, hidden, 2, seed=seed + 1, **kw), norm(0, "w")),
            step(mk(F, hidden, 2, seed=seed + 2, **kw), norm(0, "w")),
            step(mk(hidden, F, 2, seed=seed + 3, **kw), glu(1, 0, 2, 0), res=0, f16=f16)]


def layer_inputs(rng, n, hidden):
    return dict(host(rng, att=(n, hidden), x=(n, hidden)), w=norm_weight(rng, hidden))


@pytest.mark.parametrize("name", ["flow", "barrier"])
def test_layer_half(mk, name):
    steps = half_layer(mk, 512, 768, seed=21)
    hx = layer_inputs(np.random.default_rng(22), 4, 512)
    ones = singles(name, steps, hx, 4)
    for n in (2, 3, 4):
        got = run(name, steps, {k: (v[:n] if v.ndim == 2 else v) for k, v in hx.items()}, n)
        check_rows(got, ones, "%s n=%d" % (name, n))


def test_llama2_7b_layer_half(mk):
    """[o(att) + x, gate(rmsnorm), up(rmsnorm), down(glu) + h] at Llama-2-7B shapes, W2 g128 zp, 4 rows: the resident chain serves it
    (run asserts ring_slots == -kChainCS) and every row equals its one-row sequence."""
    steps = half_layer(mk, 4096, 11008, seed=31)
    hx = layer_inputs(np.random.default_rng(32), 4, 4096)
    got = run("auto", steps, hx, 4)
    check_rows(got, singles("auto", steps, hx, 4), "auto n=4")


# ---- 3: rows stay independent ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["flow", "barrier"])
def test_rows_stay_independent(mk, name):
    """Rows 2^10 apart in magnitude and an all-zero row (its norm input is 0 * inv): swapping two input rows swaps the output rows
    bit for bit and leaves the others alone."""
    steps = half_layer(mk, 512, 768, seed=41)
    hx = layer_inputs(np.random.default_rng(42), 4, 512)
    for k in ("att", "x"):
        hx[k][1] *= 1024.0
        hx[k][2] = 0.0
        hx[k][3] /= 1024.0
    got = run(name, steps, hx, 4)
    check_rows(got, singles(name, steps, hx, 4), name)
    assert np.all(got[0][2] == 0) and np.all(got[3][2] == 0), "the all-zero row"
    for a, b in ((0, 1), (2, 3)):
        sw = {k: (v[[b if t == a else a if t == b else t for t in range(4)]] if v.ndim == 2 else v) for k, v in hx.items()}
        got2 = run(name, steps, sw, 4)
        for i in range(len(steps)):
            for t in range(4):
                u = b if t == a else a if t == b else t
                assert same_bits(got2[i][t], got[i][u]), "op %d: swapping rows %d and %d moved row %d" % (i, a, b, t)


# ---- 4: inputs that change between launches, fp16 C -------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["flow", "barrier"])
def test_inputs_change_between_launches(stream, mk, name, graph):
    """Every launch (or replay of one captured launch) gets new rows, written in place; a row that accepted a word of the previous
    launch would differ from its one-row sequence.  The last op stores fp16."""
    n = 3
    steps = half_layer(mk, 512, 768, seed=51, f16=True)
    rng = np.random.default_rng(52)
    ext = {"att": torch.zeros((n, 512), device="cuda"), "x": torch.zeros((n, 512), device="cuda"), "w": torch.zeros(512, device="cuda")}
    with form(name), sequence(steps, ext, n) as (seq, outs):
        expect_kernel(seq.info(), True)
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                seq.launch()
        try:
            for _ in range(3):
                hx = layer_inputs(rng, n, 512)
                for k, v in ext.items():
                    v.copy_(torch.from_numpy(hx[k]))             # current stream = the library stream: ordered before the launch
                if graph:
                    g.replay()
                else:
                    seq.launch()
                seq.status()
                got = fetch(outs)
                assert got[3].dtype == np.float16
                check_rows(got, singles(name, steps, hx, n), name)
        finally:
            if g is not None:
                torch.cuda.synchronize()
                g.reset()


# ---- 5: the bench chain ----------------------------------------------------------------------------------------------------------
def test_bench_chain(stream, oracle):
    """32 distinct 11008x4096 W2 g128 zp tensors, op i + 1 reading the first 4096 outputs of op i, at 4 rows: the resident chain
    serves it and every row equals its one-row sequence; the first two ops of every row against the oracle."""
    cfg = T.Config(11008, 4096, 2, kfactor=16, act_group_size=64, zero_point=True).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=61)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    base = tb.upload_plain(kc(cfg), w, sc, z)
    wts = [base] + [tb.clone(base) for _ in range(31)]
    try:
        steps = [step(SimpleNamespace(wt=wt, cfg=cfg, A=A, S=S), "x0" if i == 0 else i - 1) for i, wt in enumerate(wts)]
        hx = host(np.random.default_rng(62), x0=(4, 4096))
        got = run("auto", steps, hx, 4)
        check_rows(got, singles("auto", steps, hx, 4), "bench chain")
        check_oracle(oracle, steps[:2], hx, got[:2])      # later ops grow past fp32 range with these random weights
    finally:
        for wt in wts:
            wt.free()


# ---- 6: rejections, and n = 1 given explicitly ------------------------------------------------------------------------------------
def test_rejections(mk):
    p, q = mk(768, 512, 2, zp=True, seed=71), mk(512, 512, 2, zp=True, seed=72)
    lib = tb.load()
    x = torch.zeros((2, 512), device="cuda")
    for n in (0, 5, -1):
        with pytest.raises(tb.TMACError):
            tb.Sequence(n)
    seq = tb.Sequence()
    try:                                                    # after an op
        seq.add(p.wt, x=x)
        assert lib.tmac_b200_seq_set_batch(seq.h, 2) < 0
        seq.add(q.wt, in_op=0)
        seq.build()                                         # after the build
        assert lib.tmac_b200_seq_set_batch(seq.h, 2) < 0
        assert lib.tmac_b200_seq_set_batch(seq.h, 1) < 0
    finally:
        seq.free()
    peer, out = torch.zeros((2, 512), device="cuda"), torch.zeros((2, 512), device="cuda")

    def build(name, peers=False):
        with form(name):
            s = tb.Sequence(2)
            try:
                s.add(p.wt, x=x)
                s.add(q.wt, in_op=0, out=out)
                if peers:
                    s.peer_outputs(1, [peer.data_ptr()])
                s.build()
            finally:
                s.free()
    build("flow")                                           # the sequence itself qualifies
    with pytest.raises(tb.TMACError, match="peer outputs"):
        build("flow", peers=True)
    for name in ("streamk", "streamk_g7", "auto_g7"):
        with pytest.raises(tb.TMACError, match="resident chain"):
            build(name)


def test_explicit_single_row_is_the_default(mk):
    steps = chunking_chain(mk, 128, 64, 2, True)
    hx = host(np.random.default_rng(81), x0=(1, steps[0].op.cfg.K))
    for name in ("flow", "barrier"):
        a = run(name, steps, hx, 1, explicit=True)
        b = run(name, steps, hx, 1)
        for i, (u, v) in enumerate(zip(a, b)):
            assert same_bits(u, v), "%s op %d" % (name, i)


@pytest.mark.parametrize("bits", [3, 4])
def test_w3_w4_11008_rows_do_not_qualify(stream, bits):
    """An 11008-row W3 / W4 op is 172 clusters (688 CTAs): 6 CTAs per SM, which the batch kernels (bounded to 3, at 119-162
    registers) cannot keep resident, so a batch build fails instead of taking the stream-K kernel."""
    cfg = T.Config(11008, 4096, bits, kfactor=16, act_group_size=64).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=91)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    x = torch.zeros((2, 4096), device="cuda")
    s = tb.Sequence(2)
    try:
        s.add(wt, x=x)
        with pytest.raises(tb.TMACError, match="does not qualify"):
            s.build()
    finally:
        s.free()
        wt.free()
