"""GPU suite (-m gpu): the RMS-norm input (tmac_b200_seq_add_gemv_rmsnorm) and the residual output (tmac_b200_seq_residual) of the
decode sequences, in both sequence kernels and both forms of the resident chain, up to a decoder layer's whole half after attention
[o(att) + x, gate(rmsnorm(h) * w), up(rmsnorm(h) * w), down(silu(gate) * up) + h] at Llama-2-7B shapes.

Every check is first bit for bit: the sequence is restated as the same ops (same form, same tensors: stream-K's shares depend on all
of them) without norm inputs or residuals -- a norm op reads the external vector a, computed in numpy float32 in the documented
order from the sequence's own producer output, a plain op reads its producer's output as an external vector -- and each op must
equal the restated op plus, for a residual, a numpy float32 add (an fp16 C rounded once, at the store).
kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from seq_util import (DENSE_NMSE, EPS, FORMS, TIGHT_TOL, device, expect_kernel, fetch, form, glu, host, mk, norm, norm_weight,
                      oracle_gemv, rms_input, run_form, same_bits, sequence, step, stream)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ALL = ["flow", "barrier", "streamk", "streamk_g7", "auto"]


def restated(steps, got, hext):
    """The same ops without norm inputs and residuals: a norm op reads a (rms_input of its producer's output in `got`), a plain op
    reads its producer's output as an external vector, a GLU op stays (its producers compute the same bits).  All outputs fp32."""
    plain, pext = [], {}
    for i, (o, src, *_) in enumerate(steps):
        name = "in%d" % i
        if isinstance(src, str):
            pext[name] = hext[src]
        elif isinstance(src, int):
            pext[name] = got[src][:o.cfg.K].astype(np.float32)
        elif src[0] == "norm":
            pext[name] = rms_input(got[src[1]], hext[src[2]], src[3])[0]
        plain.append(step(o, src if name not in pext else name))
    return plain, pext


def check_restated(name, steps, hext, got, chained=None):
    """Every op bit for bit against the restated sequence (plus the residual, in numpy float32); returns the restated inputs."""
    plain, pext = restated(steps, got, hext)
    _, pgot = run_form(name, plain, device(pext), chained)
    for i, (o, src, off, res, f16) in enumerate(steps):
        want = pgot[i]
        if res is not None:
            want = want + (hext[res] if isinstance(res, str) else got[res].astype(np.float32))
        if f16:
            want = want.astype(np.float16)
        assert same_bits(want, got[i]), \
            "%s: op %d differs from the restated op%s" % (name, i, " plus its residual" if res is not None else "")
    return pext


def check_norm_oracle(oracle, steps, pext, got):
    for i, (o, src, off, res, f16) in enumerate(steps):
        if isinstance(src, tuple) and src[0] == "norm":
            ref = oracle_gemv(oracle, o.cfg, o.A, o.S, pext["in%d" % i])
            if res is not None:
                continue
            err = np.abs(got[i] - ref).max() / np.abs(ref).max()
            assert err <= TIGHT_TOL, "norm op %d: rel err %.3g against the oracle on a" % (i, err)


# ---- 1: residuals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f16", [False, True], ids=["c32", "c16"])
@pytest.mark.parametrize("name", ALL)
def test_residual(mk, name, f16):
    """An external residual on a middle op that others read, and an earlier op's output as the residual of the last op."""
    a, b, c = mk(512, 512, 2, zp=True, seed=1), mk(512, 512, 2, zp=True, seed=2), mk(512, 512, 2, zp=True, seed=3)
    steps = [step(a, "x"), step(b, 0, res="r"), step(c, 1, res=0, f16=f16)]
    hx = host(np.random.default_rng(11), x=512, r=512)
    _, got = run_form(name, steps, device(hx), chained=FORMS[name][0] != 0)
    check_restated(name, steps, hx, got, chained=FORMS[name][0] != 0)


# ---- 2: norm inputs ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,g,ags,zp", [(2, 128, 64, True), (4, 128, 64, False), (2, 32, 32, True)], ids=["w2zp", "w4", "w2-g32"])
@pytest.mark.parametrize("name", ALL)
def test_norm_op(oracle, mk, name, bits, g, ags, zp):
    """Two norm ops over one producer (with different weights, one of them read by a later op) and a norm op at a depth."""
    kw = dict(g=g, ags=ags, zp=zp)
    steps = [step(mk(768, 512, bits, seed=21, **kw), "x"), step(mk(512, 768, bits, seed=22, **kw), norm(0, "w0")),
             step(mk(256, 768, bits, seed=23, **kw), norm(0, "w1", 1e-3)), step(mk(768, 512, bits, seed=24, **kw), norm(1, "w2"))]
    rng = np.random.default_rng(12)
    hx = dict(host(rng, x=512), w0=norm_weight(rng, 768), w1=norm_weight(rng, 768), w2=norm_weight(rng, 512))
    chained = FORMS[name][0] != 0
    _, got = run_form(name, steps, device(hx), chained)
    pext = check_restated(name, steps, hx, got, chained)
    check_norm_oracle(oracle, steps, pext, got)


# ---- 3: a decoder layer's half after attention ------------------------------------------------------------------------------------
def half_layer(mk, hidden, F, bits, zp, seed):
    kw = dict(g=128, ags=64, zp=zp)
    return [step(mk(hidden, hidden, bits, seed=seed, **kw), "att", res="x"),
            step(mk(F, hidden, bits, seed=seed + 1, **kw), norm(0, "w")),
            step(mk(F, hidden, bits, seed=seed + 2, **kw), norm(0, "w")),
            step(mk(hidden, F, bits, seed=seed + 3, **kw), glu(1, 0, 2, 0), res=0)]


def dense_half_layer(steps, hx):
    """fp64 dense dequantised layer: h = o(att) + x, a = rmsnorm(h) * w, out = down(silu(gate(a)) * up(a)) + h."""
    def lin(i, x):
        o = steps[i][0]
        return T.dense_reference(o.w, o.sc, o.z, np.asarray(x, np.float32)[None], o.cfg)[0].astype(np.float64)
    h = lin(0, hx["att"]) + hx["x"]
    a = h / np.sqrt(np.mean(h * h) + EPS) * hx["w"]
    gt, up = lin(1, a), lin(2, a)
    return lin(3, gt / (1 + np.exp(-gt)) * up) + h


@pytest.mark.parametrize("bits,zp,chained", [(2, True, True), (4, False, False)], ids=["w2zp-chain", "w4-streamk"])
def test_llama2_7b_half_layer(mk, bits, zp, chained):
    steps = half_layer(mk, 4096, 11008, bits, zp, seed=40 + bits)
    rng = np.random.default_rng(13)
    hx = dict(host(rng, att=4096, x=4096), w=(1.0 + 0.1 * rng.standard_normal(4096)).astype(np.float32))
    _, got = run_form("auto", steps, device(hx), chained=chained)
    check_restated("auto", steps, hx, got, chained=chained)
    e = T.nmse(dense_half_layer(steps, hx), got[3])
    assert e <= DENSE_NMSE, "NMSE %.3g against the dense dequantised layer" % e


def test_layer_chain_without_decode_ahead(mk):
    """The layer instantiation of the chain without decode-ahead (QD = 0, what the build falls back to when the decode-ahead one does
    not keep every cluster resident) computes the same bits as the one with it."""
    steps = half_layer(mk, 512, 768, 2, True, seed=45)
    rng = np.random.default_rng(16)
    hx = dict(host(rng, att=512, x=512), w=norm_weight(rng, 512))
    _, ahead = run_form("flow", steps, device(hx))
    try:
        tb.debug_set("chain_ahead", 0)
        _, plain = run_form("flow", steps, device(hx))
    finally:
        tb.debug_set("chain_ahead", 1)
    for i, (a, b) in enumerate(zip(ahead, plain)):
        assert same_bits(a, b), "op %d" % i
    check_restated("flow", steps, hx, plain)


# ---- 4: inputs that change between launches ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["flow", "barrier", "streamk"])
def test_inputs_change_between_launches(stream, mk, name, graph):
    """A norm op or a residual that accepted a word of the previous launch would compute on stale rows: every launch (or replay of
    one captured launch) gets new att, x and norm weights, written in place, and every op is checked against that round."""
    steps = half_layer(mk, 512, 768, 2, True, seed=50)
    rng = np.random.default_rng(14)
    ext = {"att": torch.zeros(512, device="cuda"), "x": torch.zeros(512, device="cuda"), "w": torch.zeros(512, device="cuda")}
    chained = FORMS[name][0] != 0
    with form(name), sequence(steps, ext) as (seq, outs):
        expect_kernel(seq.info(), chained)
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                seq.launch()
        try:
            for _ in range(3):
                hx = dict(host(rng, att=512, x=512), w=norm_weight(rng, 512))
                for k, v in ext.items():
                    v.copy_(torch.from_numpy(hx[k]))             # current stream = the library stream: ordered before the launch
                if graph:
                    g.replay()
                else:
                    seq.launch()
                seq.status()
                got = fetch(outs)
                with form(name):
                    check_restated(name, steps, hx, got, chained)
        finally:
            if g is not None:
                torch.cuda.synchronize()
                g.reset()


# ---- 5: edge rows -------------------------------------------------------------------------------------------------------------------
EDGES = [("zero_row", "zero", EPS), ("eps0", "normal", 0.0)] + [("act_" + k, k, EPS) for k in act_rows.KINDS]


@pytest.mark.parametrize("kind,eps", [e[1:] for e in EDGES], ids=[e[0] for e in EDGES])
@pytest.mark.parametrize("name", ALL)
def test_edge_rows(oracle, mk, name, kind, eps):
    """The producer's row h is set through its residual: h = gemv(x) + r with x = 0 (whose gemv is 0), so h = r takes the all-zero
    row (inv = 1 / sqrt(eps)), or an act_rows row; "normal" keeps x and r normal for eps = 0."""
    rng = np.random.default_rng(15)
    K = 512
    if kind == "zero":
        hx = {"x": np.zeros(K, np.float32), "r": np.zeros(K, np.float32)}
    elif kind == "normal":
        hx = host(rng, x=K, r=K)
    else:
        hx = {"x": np.zeros(K, np.float32), "r": act_rows.rows(rng, 1, K, 64, kinds=(kind,))[0]}
    hx["w"] = norm_weight(rng, K)
    steps = [step(mk(K, K, 2, zp=True, seed=61), "x", res="r"), step(mk(768, K, 2, zp=True, seed=62), norm(0, "w", eps))]
    chained = FORMS[name][0] != 0
    _, got = run_form(name, steps, device(hx), chained)
    if kind != "normal":
        assert np.array_equal(got[0], hx["r"]), "h = 0 + r"
    if kind == "zero":
        assert np.all(rms_input(got[0], hx["w"], eps) == 0)
    pext = check_restated(name, steps, hx, got, chained)
    if kind not in ("zero",):
        check_norm_oracle(oracle, steps, pext, got)


# ---- 6: rejections -----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    p, q = mk(768, 512, 2, zp=True, seed=71), mk(512, 512, 2, zp=True, seed=72)
    n768, n512 = mk(512, 768, 2, zp=True, seed=73), mk(256, 512, 2, zp=True, seed=74)
    x = torch.zeros(512, device="cuda")
    w = torch.ones(769, device="cuda")
    seq = tb.Sequence()
    try:
        seq.add(p.wt, x=x); seq.add(q.wt, x=x)                            # 0: 768 rows, 1: 512 rows
        bad = [
            (n512, 0, w[:768], EPS),                                      # K = 512 != the producer's 768 rows
            (n768, 1, w[:768], EPS),                                      # K = 768 > the producer's 512 rows
            (n768, 2, w[:768], EPS),                                      # not an earlier op
            (n768, -1, w[:768], EPS),
            (n768, 0, np.ones(768, np.float32), EPS),                     # host w
            (n768, 0, w[1:], EPS),                                        # misaligned w
            (n768, 0, w[:768], -1e-6),                                    # eps < 0 / not finite
            (n768, 0, w[:768], float("inf")),
            (n768, 0, w[:768], float("nan")),
        ]
        for wt, src, ww, eps in bad:
            with pytest.raises(tb.TMACError):
                seq.add_rmsnorm(wt.wt, src, ww, eps)
        assert seq.add_rmsnorm(n768.wt, 0, w[:768], EPS) == 2              # the rejected calls added nothing
        r = torch.zeros(513, device="cuda")
        for kw in [dict(op=2, r=r[1:]), dict(op=2, r=np.zeros(512, np.float32)), dict(op=1, r_op=1), dict(op=1, r_op=2),
                   dict(op=2, r_op=0), dict(op=2), dict(op=2, r=r[:512], r_op=1), dict(op=3, r=r[:512]), dict(op=-1, r=r[:512])]:
            with pytest.raises(tb.TMACError):
                seq.residual(**kw)                                        # misaligned / host r, r_op not earlier or another Mout
        seq.residual(2, r=r[:512])
        with pytest.raises(tb.TMACError):
            seq.residual(2, r_op=1)                                       # two residuals on one op
        seq.build()
        with pytest.raises(tb.TMACError):
            seq.residual(1, r=r[:512])
        with pytest.raises(tb.TMACError):
            seq.add_rmsnorm(n768.wt, 0, w[:768], EPS)
    finally:
        seq.free()


# ---- 7: the decode harness ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_harness_layer_with_post_attn_sequence(stream, bits, zp):
    from decode_harness import DecodeLayer
    hidden, ffn_, heads, ctx = 1024, 2816, 8, 64
    with pytest.raises(ValueError):
        DecodeLayer(hidden, ffn_, heads, bits, zp, seed=3, ffn_sequence=True, post_attn_sequence=True)
    layer = DecodeLayer(hidden, ffn_, heads, bits, zp, seed=3, post_attn_sequence=True)
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


def test_harness_graphed_token_step_with_post_attn_sequence(stream):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=3, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=32, post_attn_sequence=True)
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
