"""GPU suite (-m gpu): tmac_b200_gemv_rmsnorm_bias and tmac_b200_prefill_rmsnorm_bias, the q/k/v launches of a layer whose q/k/v
projections carry a bias (Qwen2), and the decode harness's qkv_bias layers.

Every check is bit for bit against the equivalence the header documents: each output equals the call without a bias
(gemv_rmsnorm at the same decomposition, prefill_rmsnorm on the same tile) with F32 outputs, followed by a numpy float32 add of the
bias, rounded once to fp16 for an F16 call."""
import types

import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from fused_util import knobs
from seq_util import DENSE_NMSE, EPS, kc, mk, norm_weight, rms_input, stream
from test_gpu_gemv_fused_io import dev, expect, nan_out

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

K = 1280                                        # 10 chunks of 128 K, 40 of 32 K
M = 768
PF16_TOL, INT8_TOL = 5e-4, 2e-5                 # the tiles' bounds against the oracle, max |got - ref| / max |ref| (DESIGN 3.3)


def biases(rng, count, m=M, big=True):
    """count fp32 [m] biases, device; normal values with a few +-0 and (big) large entries."""
    out = []
    for _ in range(count):
        b = rng.standard_normal(m).astype(np.float32)
        b[::37] = 0.0
        b[5::41] = -0.0
        if big:
            b[11::53] *= 1000.0
        out.append(dev(b))
    return out


# (bits, group, act group, zero points, one scale)
FORMATS = {"w2zp-g128-a64": (2, 128, 64, True, False), "w3zp-g128-a64": (3, 128, 64, True, False), "w4-g128-a64": (4, 128, 64, False, False),
           "w4-g32-a32": (4, 32, 32, False, False), "w1-g128-a64": (1, 128, 64, False, False), "w2-one-scale-a64": (2, 128, 64, False, True)}


@pytest.fixture
def make(mk):
    """make(fmt, count, seed): count tensors of one format, [M][K], freed after the test.  The one-scale format is a ternary W2
    tensor with activation groups of 64 (chunk 128 K), uploaded as the decode harness uploads BitNet's tensors."""
    made = []

    def f(fmt, count, seed):
        bits, g, ags, zp, one = FORMATS[fmt]
        if not one:
            return [mk(M, K, bits, g=g, ags=ags, zp=zp, seed=seed + i) for i in range(count)]
        for i in range(count):
            w = (np.random.default_rng(seed + i).integers(-1, 2, size=(M, K)) + 2).astype(np.uint8)
            made.append(tb.upload_plain(tb.make_kcfg(M, K, 2, 256, ags // 4, 128, ags, False, True), w, np.array([0.037], np.float32)))
        return [types.SimpleNamespace(wt=wt) for wt in made[-count:]]
    yield f
    for wt in made:
        wt.free()


def check(form, ref_form, ops, N, H, w, bias, dtype=torch.float32):
    """form (gemv_rmsnorm_bias / prefill_rmsnorm_bias) of ops on host rows H passed as dtype against ref_form (gemv_rmsnorm /
    prefill_rmsnorm) with F32 outputs on the same rows plus a float32 add of the bias; the two report the same launch.  Returns the
    F32 reference rows (numpy, without the bias) and the bias call's outputs."""
    f16 = dtype == torch.float16
    dH, dw = dev(H, dtype), dev(w)
    outs = [nan_out(N, M, dtype) for _ in ops]
    form([o.wt for o in ops], N, dH, dw, EPS, bias, outs, dtype=tb.F16 if f16 else tb.F32)
    launch = tb.last_launch()
    refs = [nan_out(N, M) for _ in ops]
    ref_form([o.wt for o in ops], N, dH.float(), dw, EPS, refs)
    assert tb.last_launch() == launch
    torch.cuda.synchronize()
    refs = [r.cpu().numpy() for r in refs]
    for i, (o, r, b) in enumerate(zip(outs, refs, bias)):
        expect(o, r, b.cpu().numpy(), f16, "%s tensor %d" % (form.__name__, i))
    return refs, outs


# ---- 1: decode form, bit for bit -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 3, 8])
@pytest.mark.parametrize("count", [1, 3])
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_decode_form(make, fmt, count, N):
    ops = make(fmt, count, seed=10 * count + N)
    rng = np.random.default_rng(N + count + len(fmt))
    ags = FORMATS[fmt][2]
    w, bias = norm_weight(rng, K), biases(rng, count)
    check(tb.gemv_rmsnorm_bias, tb.gemv_rmsnorm, ops, N, act_rows.rows(rng, N, K, ags), w, bias)
    check(tb.gemv_rmsnorm_bias, tb.gemv_rmsnorm, ops, N, act_rows.rows16(rng, N, K, ags), w, bias, dtype=torch.float16)


@pytest.mark.parametrize("cs,wpc", [(1, 8), (2, 4), (4, 2), (8, 1), (1, 1)])
def test_decode_decompositions(make, cs, wpc):
    """Forced cluster / warp decompositions: the bias call and gemv_rmsnorm at each one."""
    ops = make("w4-g128-a64", 3, seed=40)
    rng = np.random.default_rng(cs * 8 + wpc)
    w, bias = norm_weight(rng, K), biases(rng, 3)
    with knobs(cs=cs, wpc=wpc):
        for N in (1, 3):
            check(tb.gemv_rmsnorm_bias, tb.gemv_rmsnorm, ops, N, act_rows.rows(rng, N, K, 64), w, bias)
            launch = tb.last_launch()
            assert (launch["cluster"], launch["warps_per_cta"]) == (cs, wpc), launch


# ---- 2: prompt form, bit for bit and against the oracle --------------------------------------------------------------------------
PROMPT = ["w2zp-g128-a64", "w3zp-g128-a64", "w4-g128-a64", "w4-g32-a32", "w2-one-scale-a64"]


@pytest.mark.parametrize("t16", [0, 1], ids=["int8-tile", "prefill16"])
@pytest.mark.parametrize("N", [1, 31, 64, 300])
@pytest.mark.parametrize("fmt", PROMPT)
def test_prompt_form(make, oracle, fmt, N, t16):
    count = 3 if fmt == "w4-g128-a64" else 1
    ops = make(fmt, count, seed=20 + N)
    rng = np.random.default_rng(N + t16 + len(fmt))
    ags = FORMATS[fmt][2]
    w, bias = norm_weight(rng, K), biases(rng, count, big=False)     # the oracle's bound is relative to max |C|
    with knobs(prefill16=t16):
        H = act_rows.rows(rng, N, K, ags)
        _, outs = check(tb.prefill_rmsnorm_bias, tb.prefill_rmsnorm, ops, N, H, w, bias)
        launch = tb.last_launch()
        assert launch["batch"] == -N and launch["cluster"] == (16 if t16 and N >= 64 else 1), launch
        check(tb.prefill_rmsnorm_bias, tb.prefill_rmsnorm, ops, N, act_rows.rows16(rng, N, K, ags), w, bias, dtype=torch.float16)
    if FORMATS[fmt][4]:
        return                                   # one-scale tensors: the oracle of their twin is test_gpu_prefill_subnorm's
    # the float oracle on the first rows of tensor 0, with the bias: the tile's bound of max |C|
    op = ops[0]
    a = rms_input(H[:4], w, EPS)
    q, ls, lb = oracle.preprocessor(a, op.cfg.act_group_size)
    want = oracle.qgemm(op.cfg, op.A, op.S, q, ls, lb) + bias[0].cpu().numpy()
    got = outs[0].cpu().numpy()[:4]
    tol = PF16_TOL if t16 and N >= 64 else INT8_TOL
    assert np.abs(got - want).max() <= tol * np.abs(want).max()


# ---- 3: CUDA graphs ---------------------------------------------------------------------------------------------------------------
def test_graph_replay_gives_the_eager_outputs(stream, make):
    """Both forms: one eager call, then a capture; a replay into cleared outputs gives the eager outputs."""
    ops = make("w4-g128-a64", 3, seed=50)
    rng = np.random.default_rng(51)
    w, bias = dev(norm_weight(rng, K)), biases(rng, 3)
    h1, hp = dev(act_rows.rows(rng, 1, K, 64)), dev(act_rows.rows(rng, 130, K, 64))
    y1, yp = [nan_out(1, M) for _ in ops], [nan_out(130, M) for _ in ops]

    def calls():
        tb.gemv_rmsnorm_bias([o.wt for o in ops], 1, h1, w, EPS, bias, y1)
        tb.prefill_rmsnorm_bias([o.wt for o in ops], 130, hp, w, EPS, bias, yp)

    calls()
    torch.cuda.synchronize()
    eager = [y.clone() for y in y1 + yp]
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    for y in y1 + yp:
        y.fill_(float("nan"))
    cg.replay()
    torch.cuda.synchronize()
    for e, y in zip(eager, y1 + yp):
        assert torch.equal(e, y)


# ---- 4: rejections ---------------------------------------------------------------------------------------------------------------
def test_rejections(mk, make):
    op, op2 = make("w4-g128-a64", 2, seed=60)
    other = mk(2 * M, K, 4, seed=62)                 # another geometry
    w1 = mk(M, K, 1, seed=63)
    int_cfg = T.Config(320, 1280, 2, one_scale=True).resolved()
    wi, sci, zi, _ = T.make_problem(int_cfg, seed=64)
    A, S = T.pack_reference_layout(wi, sci, zi, int_cfg)
    int_wt = tb.upload_reference_layout(kc(int_cfg), A, S)
    try:
        x, xp, nw = nan_out(1, K), nan_out(100, K), torch.ones(K, device="cuda")
        x.normal_(); xp.normal_()
        out, outp = nan_out(1, M), nan_out(100, M)
        b, b2 = torch.zeros(M, device="cuda"), torch.zeros(M, device="cuda")
        big = torch.zeros(M + 4, device="cuda")
        xi, outi, bi = torch.randn((1, 1280), device="cuda"), nan_out(1, 320), torch.zeros(320, device="cuda")
        bad = []
        for f, N, xx, o in ((tb.gemv_rmsnorm_bias, 1, x, out), (tb.prefill_rmsnorm_bias, 100, xp, outp)):
            bad += [
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw, EPS, None, [o]),                   # null bias array
                lambda f=f, N=N, xx=xx, o=o: f([op.wt, op2.wt], N, xx, nw, EPS, [b, None], [o, o]),   # null entry
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw, EPS, [np.zeros(M, np.float32)], [o]),   # host bias
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw, EPS, [big[1:]], [o]),              # misaligned bias
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw, EPS, [o.view(-1)[:M]], [o]),       # bias overlaps C
                lambda f=f, N=N, xx=xx, o=o: f([op.wt, other.wt], N, xx, nw, EPS, [b, b2], [o, nan_out(N, 2 * M)]),   # geometry
                lambda f=f: f([int_wt], 1, xi, torch.ones(1280, device="cuda"), EPS, [bi], [outi]),   # integer path
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw[1:], EPS, [b], [o]),                # gemv_rmsnorm's own: w
                lambda f=f, N=N, xx=xx, o=o: f([op.wt], N, xx, nw, float("nan"), [b], [o]),           # and eps
            ]
        bad.append(lambda: tb.prefill_rmsnorm_bias([w1.wt], 100, xp, nw, EPS, [b], [outp]))     # W1 in the prompt form
        torch.cuda.synchronize()
        for i, call in enumerate(bad):
            for t in (out, outp, outi):
                t.fill_(float("nan"))
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all() and torch.isnan(outp).all() and torch.isnan(outi).all(), "rejected call %d launched" % i
        # an armed peer output makes either call fail, launching nothing, and is disarmed by it
        for f, N, xx, o in ((tb.gemv_rmsnorm_bias, 1, x, out), (tb.prefill_rmsnorm_bias, 100, xp, outp)):
            o.fill_(float("nan"))
            tb.peer_outputs([nan_out(1, M).data_ptr()])
            with pytest.raises(tb.TMACError):
                f([op.wt], N, xx, nw, EPS, [b], [o])
            torch.cuda.synchronize()
            assert torch.isnan(o).all()
            f([op.wt], N, xx, nw, EPS, [b], [o])
            torch.cuda.synchronize()
            assert not torch.isnan(o).any()
    finally:
        int_wt.free()


# ---- 5: the decode harness --------------------------------------------------------------------------------------------------------
def nmse(got, ref):
    return float(((got - ref) ** 2).mean() / (ref ** 2).mean())


@pytest.mark.parametrize("kv_heads", [2, 4], ids=["gqa-stacked", "mha-three"])
@pytest.mark.parametrize("fused", [False, True], ids=["per-linear", "fused_ops"])
@pytest.mark.parametrize("step", ["token", "prompt"])
def test_harness_layer(stream, step, fused, kv_heads):
    """A Qwen2-shaped layer (hidden 512, 4 heads of 128, W4, q/k/v biases) against the same layer with dense dequantised fp32 weights
    and the same biases, NMSE <= DENSE_NMSE, in the layer's output and in its q/k/v outputs, which without the biases are far off."""
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx, P = 512, 1408, 4, 64, 48
    layer = DecodeLayer(hidden, ffn, heads, 4, False, seed=7, fused_ops=fused, kv_heads=kv_heads, qkv_bias=True)
    try:
        assert layer.qkv_names == (("qkv",) if kv_heads == 2 else ("q", "k", "v"))
        hd = hidden // heads
        caches = [torch.randn((kv_heads, ctx, hd), device="cuda") * 0.3 for _ in range(2)]
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        lin = lambda n, inp, out: out.copy_(inp @ dense[n].T)
        if step == "token":
            pos = ctx - 1
            cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
            x = torch.randn((1, hidden), device="cuda")
            run = lambda **kw: layer.forward(x, *[c.clone() for c in caches], pos, cos, sin, **kw).clone()
        else:
            ang = torch.arange(P, device="cuda").float()[:, None] * inv[None, :]
            cos, sin = torch.cos(ang), torch.sin(ang)
            x = torch.randn((P, hidden), device="cuda")
            run = lambda **kw: layer.prompt(x, *[c.clone() for c in caches], cos, sin, **kw).clone()
        qkv = lambda: torch.cat([(layer.buf if step == "token" else layer.pbuf)[n] for n in layer.qkv_names], dim=1)
        got = run()
        got_qkv = qkv()
        ref = run(linear=lin)
        ref_qkv = qkv()
        bias = torch.cat([layer.qkv_b[n] for n in layer.qkv_names])
        torch.cuda.synchronize()
        assert nmse(got, ref) <= DENSE_NMSE, nmse(got, ref)
        # the q/k/v outputs themselves: the reference's, and far from it without the biases
        assert nmse(got_qkv, ref_qkv) <= DENSE_NMSE, nmse(got_qkv, ref_qkv)
        assert nmse(got_qkv, ref_qkv - bias) > 100 * DENSE_NMSE, nmse(got_qkv, ref_qkv - bias)
    finally:
        layer.free()
