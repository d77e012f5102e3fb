"""GPU suite (-m gpu): the GLU op of the decode sequences (tmac_b200_seq_add_gemv_glu) -- the down projection of a SwiGLU FFN
reading silu(gate) * up of two earlier ops -- in both sequence kernels and both forms of the resident chain.

The gated activation a = silu(g) * u is restated on the device with torch from the sequence's own gate and up outputs, in fp32
(g / (1 + exp(-g)) * u, eager, one op after the other: the rounding the library documents).  The GLU op must then be bit for bit
the op of the same sequence whose input is the external vector a, and within the oracle's tolerance of the oracle run on a.
kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from seq_util import (DENSE_NMSE, TIGHT_TOL, expect_kernel, fetch, form, glu, host, inputs, mk, oracle_gemv, run_form, same_bits,
                      sequence, step, stream)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def restate(got, src, K):
    """The GLU op's input, restated on the device from the sequence's own gate and up outputs."""
    _, gi, go, ui, uo = src
    g, u = (torch.from_numpy(got[i][off:off + K]).cuda() for i, off in ((gi, go), (ui, uo)))
    return g / (1 + torch.exp(-g)) * u


def check(oracle, steps, xs, got, dense=True):
    """Every op against the oracle on the input the GPU op saw (a GLU op: the restated activation), and against the float64
    dense dequantised GEMV.  Returns the restated GLU inputs {step: device vector}."""
    acts = {}
    for i, (o, src, off, *_) in enumerate(steps):
        K = o.cfg.K
        if isinstance(src, str):
            x = xs[src]
        elif isinstance(src, tuple):
            acts[i] = restate(got, src, K)
            x = acts[i].cpu().numpy()
        else:
            x = got[src][off:off + K]
        ref = oracle_gemv(oracle, o.cfg, o.A, o.S, x)
        err = np.abs(got[i] - ref).max() / np.abs(ref).max()
        assert err <= TIGHT_TOL, "op %d (%dx%d W%d): rel err %.3g" % (i, o.cfg.Mout, o.cfg.K, o.cfg.bits, err)
        if dense:
            e = T.nmse(T.dense_reference(o.w, o.sc, o.z, x, o.cfg)[0], got[i])
            assert e <= DENSE_NMSE, "op %d: NMSE %.3g against the dense dequantised GEMV" % (i, e)
    return acts


def check_against_plain(name, steps, ext, outs, acts, chained=None):
    """Each GLU op equals, bit for bit, the same op of the same sequence (same form, same ops: stream-K's shares depend on all of
    them) whose input is the external restated activation."""
    plain = [step(s.op, "glu%d" % i) if i in acts else s for i, s in enumerate(steps)]
    _, pouts = run_form(name, plain, dict(ext, **{"glu%d" % i: a.contiguous() for i, a in acts.items()}), chained)
    for i in range(len(steps)):
        assert same_bits(outs[i], pouts[i]), "%s: op %d differs from the op fed with the restated activation" % (name, i)


def ffn(mk, hidden, F, bits, g, ags, zp, seed):
    kw = dict(g=g, ags=ags, zp=zp)
    return [step(mk(F, hidden, bits, seed=seed, **kw), "x"), step(mk(F, hidden, bits, seed=seed + 1, **kw), "x"),
            step(mk(hidden, F, bits, seed=seed + 2, **kw), glu(0, 0, 1, 0))]


# ---- 1: every form and chunking ----------------------------------------------------------------------------------------------------
CASES = [("w2zp-g128-a64", 2, 128, 64, True), ("w4-g128", 4, 128, 64, False), ("w3", 3, 128, 64, True), ("w1", 1, 128, 64, False),
         ("w2-g32-a32", 2, 32, 32, True), ("w2-g64-a64", 2, 64, 64, False)]


@pytest.mark.parametrize("bits,g,ags,zp", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_ffn_block_in_every_form(oracle, mk, bits, g, ags, zp):
    steps = ffn(mk, 512, 768, bits, g, ags, zp, seed=bits * 10 + ags)
    xs, ext = inputs(np.random.default_rng(bits + g + ags), x=512)
    got = {}
    for name in ("flow", "barrier", "streamk", "streamk_g7"):
        info, got[name] = run_form(name, steps, ext)
        assert (info["quads_per_chunk"], info["quads_per_act_group"]) == (min(g, 128) // 16, ags // 16), info
        acts = check(oracle, steps, xs, got[name], dense=name == "flow")
        check_against_plain(name, steps, ext, got[name], acts)
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), "op %d: the chain forms differ" % i


# ---- 2: offsets and sources --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["flow", "barrier", "streamk"])
def test_fused_gate_up_tensor(oracle, mk, name):
    """Gate and up as the two halves of one 2F-row op."""
    F = 768
    steps = [step(mk(2 * F, 512, 2, zp=True, seed=101), "x"), step(mk(512, F, 2, zp=True, seed=102), glu(0, 0, 0, F))]
    xs, ext = inputs(np.random.default_rng(1), x=512)
    _, outs = run_form(name, steps, ext)
    acts = check(oracle, steps, xs, outs)
    check_against_plain(name, steps, ext, outs, acts)


def depth_chain(mk, gate_off, up_off):
    kw = dict(zp=True)
    return [
        step(mk(1024, 512, 2, seed=111, **kw), "x0"),
        step(mk(1024, 1024, 2, seed=112, **kw), 0),           # gate: three ops before the GLU op
        step(mk(768, 512, 2, seed=113, **kw), "x1"),
        step(mk(1024, 768, 2, seed=114, **kw), 2),            # up
        step(mk(512, 768, 2, seed=115, **kw), glu(1, gate_off, 3, up_off)),
        step(mk(256, 512, 2, seed=116, **kw), 4),             # a plain op reading the GLU op
    ]


@pytest.mark.parametrize("name", ["flow", "barrier", "streamk", "streamk_g7"])
def test_sources_at_different_depths(oracle, mk, name):
    steps = depth_chain(mk, 4, 128)
    xs, ext = inputs(np.random.default_rng(2), x0=512, x1=512)
    _, outs = run_form(name, steps, ext)
    acts = check(oracle, steps, xs, outs, dense=name == "flow")
    check_against_plain(name, steps, ext, outs, acts)


def test_offsets_the_barrier_form_refuses(oracle, mk):
    """Offsets that are 2 mod 4: the barrier form's float4 loads refuse them, auto_barrier falls back to stream-K and computes
    what stream-K computes; the data-flow form takes them."""
    steps = depth_chain(mk, 2, 254)
    xs, ext = inputs(np.random.default_rng(3), x0=512, x1=512)
    with pytest.raises(tb.TMACError):
        with form("barrier"), sequence(steps, ext):
            pass
    _, fb = run_form("auto_barrier", steps, ext, chained=False)
    _, sk = run_form("streamk", steps, ext)
    for i, (a, b) in enumerate(zip(fb, sk)):
        assert same_bits(a, b), i
    check(oracle, steps, xs, fb, dense=False)
    _, fl = run_form("flow", steps, ext)
    acts = check(oracle, steps, xs, fl)
    check_against_plain("flow", steps, ext, fl, acts)


# ---- 3: inputs that change between launches ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["flow", "streamk"])
def test_inputs_change_between_launches(stream, oracle, mk, name, graph):
    """A GLU op that accepted a word of the previous launch would compute on stale gate or up rows: every launch (or replay of one
    captured launch) gets new inputs, written in place, and every op is checked against that round's inputs."""
    steps = depth_chain(mk, 4, 128)
    rng = np.random.default_rng(4)
    ext = {"x0": torch.zeros(512, device="cuda"), "x1": torch.zeros(512, device="cuda")}
    with form(name), sequence(steps, ext) as (seq, outs):
        expect_kernel(seq.info(), name == "flow")
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                seq.launch()
        try:
            for _ in range(3):
                xs = host(rng, **{k: v.numel() for k, v in ext.items()})
                for k, v in ext.items():
                    v.copy_(torch.from_numpy(xs[k]))           # current stream = the library stream: ordered before the launch
                if graph:
                    g.replay()
                else:
                    seq.launch()
                seq.status()
                check(oracle, steps, xs, fetch(outs), dense=False)
        finally:
            if g is not None:
                torch.cuda.synchronize()
                g.reset()


# ---- 4: full size ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp,chained", [(2, True, True), (4, False, False)], ids=["w2zp-chain", "w4-streamk"])
def test_llama2_7b_ffn(oracle, mk, bits, zp, chained):
    """The Llama-2-7B FFN (gate / up 11008 x 4096, down 4096 x 11008, g128): W2 zp is held by the resident chain, W4 (172
    clusters of gate / up) by stream-K.  Every row of down against the oracle on the restated activation."""
    steps = ffn(mk, 4096, 11008, bits, 128, 64, zp, seed=120 + bits)
    xs, ext = inputs(np.random.default_rng(5), x=4096)
    _, outs = run_form("auto", steps, ext, chained=chained)
    check(oracle, steps, xs, outs, dense=False)


# ---- 5: rejections -----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    gate, up = mk(768, 512, 2, zp=True, seed=131), mk(768, 512, 2, zp=True, seed=132)
    down, wide = mk(512, 768, 2, zp=True, seed=133), mk(512, 1024, 2, zp=True, seed=134)
    _, ext = inputs(np.random.default_rng(6), x=512)
    seq = tb.Sequence()
    try:
        seq.add(gate.wt, x=ext["x"]); seq.add(up.wt, x=ext["x"])
        bad = [
            dict(gate_op=0, gate_offset=0, up_op=2, up_offset=0),       # a later op (the GLU op itself would be op 2)
            dict(gate_op=5, gate_offset=0, up_op=1, up_offset=0),       # no such op
            dict(gate_op=-1, gate_offset=0, up_op=1, up_offset=0),
            dict(gate_op=0, gate_offset=2, up_op=1, up_offset=0),       # [2, 770) beyond the producer's 768 rows
            dict(gate_op=0, gate_offset=0, up_op=1, up_offset=-2),
            dict(gate_op=0, gate_offset=0, up_op=1, up_offset=1),       # odd offset
        ]
        for kw in bad:
            with pytest.raises(tb.TMACError):
                seq.add_glu(down.wt, **kw)
        with pytest.raises(tb.TMACError):
            seq.add_glu(wide.wt, 0, 0, 1, 0)                             # K = 1024 > 768 rows
        host = np.zeros(512, np.float32)
        with pytest.raises(tb.TMACError):
            seq.add_glu(down.wt, 0, 0, 1, 0, out=host)                  # C must be a device pointer
        assert seq.add_glu(down.wt, 0, 0, 1, 0) == 2                     # the rejected calls added nothing
    finally:
        seq.free()


# ---- 6: the decode harness ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_harness_layer_with_ffn_sequence(stream, bits, zp):
    from decode_harness import DecodeLayer
    hidden, ffn_, heads, ctx = 1024, 2816, 8, 64
    layer = DecodeLayer(hidden, ffn_, heads, bits, zp, seed=3, ffn_sequence=True)
    try:
        hd = hidden // heads
        kcache = torch.randn((heads, ctx, hd), device="cuda") * 0.3; vcache = torch.randn((heads, ctx, hd), device="cuda") * 0.3
        kc2, vc2 = kcache.clone(), vcache.clone()
        pos = ctx - 1
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
        x = torch.randn((1, hidden), device="cuda")
        got = layer.forward(x, kcache, vcache, pos, cos, sin).clone()
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.forward(x, kc2, vc2, pos, cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T)).clone()
        torch.cuda.synchronize()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= DENSE_NMSE, nmse
    finally:
        layer.free()


def test_harness_graphed_token_step_with_ffn_sequence(stream):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=3, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=32, ffn_sequence=True)
    try:
        with torch.cuda.stream(stream):
            m.step()
        torch.cuda.synchronize()
        eager = m.y.clone()
        m.capture(stream)
        m.y.zero_()
        m.graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.y, eager)
    finally:
        m.free()
