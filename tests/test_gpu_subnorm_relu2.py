"""GPU suite (-m gpu): tmac_b200_gemv_subnorm_relu2 and tmac_b200_prefill_subnorm_relu2, the down projection of a squared-ReLU FFN
behind its ffn_sub_norm (BitNet b1.58 2B4T), and the 2B4T layer of the decode harness (ffn_act="relu2", kv_heads).

Every check is bit for bit against the equivalence the header documents: row n of the call equals row n of tmac_b200_gemv on the
same tensor fed a = rmsnorm(s) * w materialised in fp32, s = (r * r) * u with r = relu(g) (NaN kept), all in numpy float32 in the
documented order -- the decode form at the GEMV's own decomposition, the prompt form on the same tile (a one-scale tensor: on its
twin, the same codes with per-row scales all equal to its scale) -- plus a numpy float32 add of the residual, rounded once to fp16
for an F16 call."""
import contextlib
import types

import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from fused_util import bm_of, knobs, launched, serial_input, tdt
from seq_util import DENSE_NMSE, EPS, Op, norm_weight, rms_input, same_bits, stream
from test_gpu_gemv_fused_io import dev, expect, nan_out, normal

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SCALE0 = float(np.float32(np.float16(0.037)))
H2B, F2B = 2560, 6912                                   # BitNet b1.58 2B4T: hidden, FFN (the down projection is H2B x F2B)


@pytest.fixture
def tensors(stream):
    """one_scale(M, K, ags, seed): a ternary one-scale W2 tensor with activation groups of ags (chunk 128 K, as QLinear uploads it)
    and its twin (the same codes, per-row scales all SCALE0); per_row(M, K, bits, g, ags, zp, seed): an Op.  Freed after the test."""
    made = []

    def one_scale(M, K, ags, seed):
        w = (np.random.default_rng(seed).integers(-1, 2, size=(M, K)) + 2).astype(np.uint8)
        bm = bm_of(M, 2)
        one = tb.upload_plain(tb.make_kcfg(M, K, 2, bm, ags // 4, 128, ags, False, True), w, np.array([SCALE0], np.float32))
        made.append(one)
        sc = np.full((M, K // 128), SCALE0, np.float32)
        twin = tb.upload_plain(tb.make_kcfg(M, K, 2, bm, ags // 4, 128, ags, False, False), w, sc)
        made.append(twin)
        cfg = T.Config(M, K, 2, bm=bm, kfactor=ags // 4, group_size=128, act_group_size=ags).resolved()
        return types.SimpleNamespace(wt=one, twin=twin, w=w, sc=sc, z=None, cfg=cfg, M=M, K=K, ags=ags)

    def per_row(M, K, bits, g, ags, zp, seed):
        op = Op(M, K, bits, g=g, ags=ags, zp=zp, seed=seed)
        made.append(op.wt)
        return types.SimpleNamespace(wt=op.wt, twin=op.wt, w=op.w, sc=op.sc, z=op.z, cfg=op.cfg, M=M, K=K, ags=ags)
    yield types.SimpleNamespace(one_scale=one_scale, per_row=per_row)
    for wt in made:
        wt.free()


def relu2_np(g, u):
    """s = (r * r) * u in numpy float32, r = g where g > 0 or g is NaN, else +0 (torch's relu)."""
    g, u = np.asarray(g, np.float32), np.asarray(u, np.float32)
    r = np.where((g > 0) | np.isnan(g), g, np.float32(0.0)).astype(np.float32)
    return (r * r) * u


def relu2_input(dG, dU, w, eps=EPS):
    """The documented input a from the device rows G and U (fp16 widened): numpy float32 [N][K]."""
    with np.errstate(invalid="ignore", over="ignore"):
        return rms_input(relu2_np(dG.float().cpu().numpy(), dU.float().cpu().numpy()), w, eps)


def dense(wt, N, a, t16=None):
    """tmac_b200_gemv of the fp32 rows a: the GEMV (t16 None, N small) or the fp16 / int8 tile.  numpy float32 [N][Mout]."""
    out = nan_out(N, wt.cfg.M)
    if t16 is None:
        tb.gemv(wt, N, dev(a), out)
    else:
        with knobs(prefill_min_n=1, prefill16=int(t16)):
            tb.gemv(wt, N, dev(a), out)
            launched(t16, N)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def run(form, p, N, G, U, w, R=None, dtype=torch.float32, res="none", t16=None, eps=EPS):
    """form (gemv_subnorm_relu2 or prefill_subnorm_relu2) of p on host rows G, U passed as dtype, with no residual, R, or R == C
    (res "none" / "given" / "inplace"), checked against dense() on the materialised input.  Returns (output numpy, a)."""
    f16 = dtype == torch.float16
    dG, dU = dev(G, dtype), dev(U, dtype)
    dR = None if res == "none" else dev(R, dtype)
    out = dR.clone() if res == "inplace" else nan_out(N, p.M, dtype)
    with knobs(prefill16=int(bool(t16))) if t16 is not None else contextlib.nullcontext():
        form(p.wt, N, dG, dev(w), eps, out, U=dU, R=out if res == "inplace" else dR, dtype=tdt(dtype))
        if t16 is not None:
            launched(t16 and N >= 64, N)
    torch.cuda.synchronize()
    a = relu2_input(dG, dU, w, eps)
    ref = dense(p.wt, N, a) if t16 is None else dense(p.twin, N, a, bool(t16) and N >= 64)
    with np.errstate(invalid="ignore", over="ignore"):
        expect(out, ref, None if dR is None else dR.float().cpu().numpy(), f16, "%s (R %s, %s)" % (form.__name__, res, "F16" if f16 else "F32"))
    got = out.cpu().numpy()
    return got, a


def gate_rows(rng, N, K, ags, f16=False):
    """Gate rows of act_rows' kinds, every 5th activation negative and a few at +-0."""
    G = (act_rows.rows16 if f16 else act_rows.rows)(rng, N, K, ags)
    G[:, ::5] = -np.abs(G[:, ::5])
    G[:, 3::97] = 0.0
    G[:, 7::97] = -0.0
    return G


# ---- 1: per-row equality, decode form ------------------------------------------------------------------------------------------
DECODE = ["2b4t-down-w2-a64", "w4-g128-a64"]


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("kind", DECODE)
def test_decode_form(tensors, kind, N):
    """gemv_subnorm_relu2 against tmac_b200_gemv on a: F32 and F16, R absent, given and equal to C."""
    p = tensors.one_scale(H2B, F2B, 64, seed=1) if kind.startswith("2b4t") else tensors.per_row(768, 2560, 4, 128, 64, False, seed=2)
    rng = np.random.default_rng(N + p.K)
    w = norm_weight(rng, p.K)
    for dtype in (torch.float32, torch.float16):
        f16 = dtype == torch.float16
        for res in ("none", "given", "inplace"):
            R = normal(rng, N, p.M)
            if f16:
                R = R.astype(np.float16).astype(np.float32)
            U = normal(rng, N, p.K)
            if f16:
                U = U.astype(np.float16).astype(np.float32)
            got, _ = run(tb.gemv_subnorm_relu2, p, N, gate_rows(rng, N, p.K, p.ags, f16), U, w, R=R, dtype=dtype, res=res)
            assert not np.isnan(got.astype(np.float32)).any()


# ---- 2: per-row equality, prompt form -------------------------------------------------------------------------------------------
PROMPT = [(40, False), (130, False), (130, True)]


@pytest.mark.parametrize("N,t16", PROMPT, ids=["int8-n40", "int8-n130", "fp16-n130"])
@pytest.mark.parametrize("kind", DECODE)
def test_prompt_form(tensors, oracle, kind, N, t16):
    """prefill_subnorm_relu2 against the dense call on the same tile (a one-scale tensor: on its twin), F32 with R absent, given
    and equal to C, F16 with R; the first rows also against the float oracle within the tile's bound."""
    p = tensors.one_scale(H2B, F2B, 64, seed=3) if kind.startswith("2b4t") else tensors.per_row(768, 2560, 4, 128, 64, False, seed=4)
    rng = np.random.default_rng(N + p.K + t16)
    w = norm_weight(rng, p.K)
    for res in ("none", "given", "inplace"):
        got, a = run(tb.prefill_subnorm_relu2, p, N, gate_rows(rng, N, p.K, p.ags), normal(rng, N, p.K), w,
                     R=normal(rng, N, p.M), res=res, t16=t16)
        if res == "none":                                   # the float oracle on the twin's config, 4 rows
            A, S = T.pack_reference_layout(p.w, p.sc, p.z, p.cfg)
            q, ls, lb = oracle.preprocessor(a[:4], p.cfg.act_group_size)
            ref = oracle.qgemm(p.cfg, A, S, q, ls, lb)
            tol = 5e-4 if t16 and N >= 64 else 2e-5
            assert np.abs(got[:4] - ref).max() <= tol * np.abs(ref).max()
    h16 = lambda *s: act_rows.rows16(rng, *s, p.ags)
    run(tb.prefill_subnorm_relu2, p, N, h16(N, p.K), h16(N, p.K), w, R=normal(rng, N, p.M).astype(np.float16).astype(np.float32),
        dtype=torch.float16, res="given", t16=t16)


# ---- 3: the order is pinned -----------------------------------------------------------------------------------------------------
def pinned_rows(rng, K, ags):
    """G, U [6][K]: act_rows' fp32 and mixed gates, a two-magnitude row (one K-group of s near 2^17, the others near 1), a row of
    negative, +-0 and large gates, an all-negative row (with +-0), and a plain normal row (row 5, for the NaN test)."""
    fp32, mixed = act_rows.rows(rng, 2, K, ags, kinds=("fp32", "mixed"))
    g_two, u_two = np.abs(normal(rng, K)) + np.float32(4.0), np.float32(0.1) * normal(rng, K)
    u_two[:4] = 4096.0
    edge = normal(rng, K)
    edge[::3] = -np.abs(edge[::3])
    edge[1::7], edge[2::7] = 0.0, -0.0
    edge[5::11] *= np.float32(3000.0)                      # r * r near 1e7, s * s near 1e14: large, still finite
    neg = -np.abs(normal(rng, K)) - np.float32(0.01)
    neg[::9], neg[4::9] = 0.0, -0.0
    G = np.stack([fp32, mixed, g_two, edge, neg, normal(rng, K)])
    U = np.stack([normal(rng, K), mixed[::-1].copy(), u_two, normal(rng, K), normal(rng, K), normal(rng, K)])
    return G.astype(np.float32), U.astype(np.float32)


def test_order_is_pinned(tensors):
    """The rows tell the documented (r * r) * u from r * (r * u) and the documented sum of squares from a serial one; both forms
    equal the dense call on them; the all-negative row gives a = 0 and a zero output; a NaN in one token's gate makes that token's
    outputs NaN and leaves the other tokens' bits as they were."""
    p = tensors.one_scale(1024, 2560, 64, seed=5)
    rng = np.random.default_rng(6)
    G, U = pinned_rows(rng, p.K, 64)
    w = norm_weight(rng, p.K)
    for i in (0, 1, 3):
        r = np.maximum(G[i], np.float32(0.0))
        assert not np.array_equal((r * r) * U[i], r * (r * U[i])), "row %d no longer tells the product orders apart" % i
    s = relu2_np(G, U)
    assert not np.array_equal(rms_input(s[2], w, EPS)[0], serial_input(s[2], w, EPS)), \
        "the two-magnitude row no longer tells the documented sum of squares from a serial sum"
    for form, t16 in ((tb.gemv_subnorm_relu2, None), (tb.prefill_subnorm_relu2, False), (tb.prefill_subnorm_relu2, True)):
        N = 6 if t16 is None else 70                       # the prompt form: the pinned rows among normal rows, N >= 64
        Gn, Un = (G, U) if t16 is None else (np.concatenate([G, normal(rng, N - 6, p.K)]), np.concatenate([U, normal(rng, N - 6, p.K)]))
        got, a = run(form, p, N, Gn, Un, w, t16=t16)
        assert not np.any(a[4]) and not np.any(got[4]), "the all-negative gate row is not zero"
        Gnan = Gn.copy()
        Gnan[5, 17] = np.nan
        out = nan_out(N, p.M)
        with knobs(prefill16=int(bool(t16))) if t16 is not None else contextlib.nullcontext():
            form(p.wt, N, dev(Gnan), dev(w), EPS, out, U=dev(Un))
        torch.cuda.synchronize()
        nan = out.cpu().numpy()
        assert np.isnan(nan[5]).all(), "%s: the NaN gate's token is not NaN" % form.__name__
        keep = [n for n in range(N) if n != 5]
        assert same_bits(nan[keep], got[keep]), "%s: a NaN in one token changed another" % form.__name__


# ---- 4: rejections --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prompt", [False, True], ids=["gemv", "prefill"])
def test_rejections(tensors, prompt):
    from decode_harness import QLinear
    K, M, N = 1024, 512, 64
    p = tensors.per_row(M, K, 2, 128, 64, True, seed=80)
    w1 = tensors.per_row(M, K, 1, 128, 64, False, seed=81)
    ip = QLinear(M, K, 2, 128, False, seed=82, one_scale=True)   # the integer path
    form = tb.prefill_subnorm_relu2 if prompt else tb.gemv_subnorm_relu2
    cname = "tmac_b200_prefill_subnorm_relu2" if prompt else "tmac_b200_gemv_subnorm_relu2"
    try:
        rng = np.random.default_rng(83)
        G, U, R, w = dev(normal(rng, N, K)), dev(normal(rng, N, K)), dev(normal(rng, N, M)), dev(norm_weight(rng, K))
        out = nan_out(N, M)
        wbuf = torch.zeros(K + 4, device="cuda")
        lib = tb.load()
        call = lambda wt=p.wt, n=N, G_=G, U_=U, w_=w, eps=EPS, C=out, R_=R: form(wt, n, G_, w_, eps, C, U=U_, R=R_)
        bad = {
            "null U": lambda: call(U_=None),
            "integer path": lambda: call(wt=ip.wt),
            "host G": lambda: call(G_=G.cpu()),
            "host U": lambda: call(U_=U.cpu()),
            "host w": lambda: call(w_=w.cpu()),
            "host R": lambda: call(R_=R.cpu()),
            "host C": lambda: call(C=out.cpu()),
            "null G": lambda: tb.check(getattr(lib, cname)(p.wt.handle, N, tb.F32, None, tb.ptr(U), tb.ptr(w), EPS, None, tb.ptr(out)),
                                       "null G"),
            "null w": lambda: call(w_=None),
            "unaligned w": lambda: call(w_=wbuf[1:]),
            "negative eps": lambda: call(eps=-1e-5),
            "nan eps": lambda: call(eps=float("nan")),
            "inf eps": lambda: call(eps=float("inf")),
            "N 0": lambda: call(n=0),
        }
        if prompt:
            bad["w1"] = lambda: call(wt=w1.wt)
            bad["token tiles"] = lambda: call(n=1 << 25)           # more than 65535 token tiles; nothing is read
        msgs = {}
        for name, c in bad.items():
            out.fill_(float("nan"))
            torch.cuda.synchronize()
            try:
                c()
            except tb.TMACError as ex:
                msgs[name] = str(ex)
            else:
                pytest.fail("'%s' was not rejected" % name)
            torch.cuda.synchronize()
            assert torch.isnan(out).all(), "rejected call '%s' launched" % name
        if prompt:
            assert "use gemv_subnorm_relu2" in msgs["w1"], msgs["w1"]
            assert "too large" in msgs["token tiles"]
        # an armed peer output: the call fails, launches nothing and disarms it
        n1 = 1 if not prompt else N
        peer = nan_out(1, M)
        out.fill_(float("nan"))
        tb.peer_outputs([peer.data_ptr()])
        with pytest.raises(tb.TMACError):
            form(p.wt, n1, G[:n1], w, EPS, out[:n1], U=U[:n1])
        torch.cuda.synchronize()
        assert torch.isnan(out).all()
        tb.gemv(p.wt, 1, torch.zeros((1, K), device="cuda"), torch.zeros((1, M), device="cuda"))
        torch.cuda.synchronize()
        assert torch.isnan(peer).all(), "the peer output stayed armed"
    finally:
        ip.free()


# ---- 5: graph capture -----------------------------------------------------------------------------------------------------------
def test_graph_replays_follow_the_inputs(stream, tensors):
    """Both forms captured after one eager call, on buffers rewritten before every replay: each replay equals eager calls."""
    p = tensors.one_scale(H2B, F2B, 64, seed=7)
    rng = np.random.default_rng(8)
    w = dev(norm_weight(rng, F2B))
    N1, NP = 1, 130
    g1, u1, r1, y1 = nan_out(N1, F2B), nan_out(N1, F2B), nan_out(N1, H2B), nan_out(N1, H2B)
    gp, up, rp, yp = nan_out(NP, F2B), nan_out(NP, F2B), nan_out(NP, H2B), nan_out(NP, H2B)
    gen = torch.Generator(device="cuda").manual_seed(9)

    def calls():
        tb.gemv_subnorm_relu2(p.wt, N1, g1, w, EPS, y1, U=u1, R=r1)
        tb.prefill_subnorm_relu2(p.wt, NP, gp, w, EPS, yp, U=up, R=rp)

    def fill():
        for t in (g1, u1, r1, gp, up, rp):
            t.copy_(torch.randn(t.shape, device="cuda", generator=gen))

    fill(); calls(); torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    seen = []
    for _ in range(3):
        fill()
        cg.replay()
        torch.cuda.synchronize()
        replayed = [y1.clone(), yp.clone()]
        seen.append(gp.clone())
        calls()
        torch.cuda.synchronize()
        for a, b in zip(replayed, (y1, yp)):
            assert same_bits(a.cpu().numpy(), b.cpu().numpy())
            assert not torch.isnan(a).any()
    assert not torch.equal(seen[0], seen[1])


# ---- 6: the 2B4T layer of the decode harness -------------------------------------------------------------------------------------
def small_2b4t_layer(seed):
    """A relu2 GQA layer with 2B4T's head dim (128) and group ratio (4) at a small width: hidden 512, FFN 1408, 4 heads, 1 KV head."""
    from decode_harness import DecodeLayer
    layer = DecodeLayer(512, 1408, 4, 2, False, seed=seed, fused_ops=True, sub_norms=True, ffn_act="relu2", kv_heads=1)
    assert layer.hd == 128 and layer.lin["qkv"].mout == 768 and set(layer.lin) == {"qkv", "o", "gate", "up", "down"}
    return layer


def test_harness_relu2_token_step(stream):
    """The fused token step (gemv_rmsnorm([qkv]), gemv_subnorm(o), gemv_rmsnorm([gate, up]), gemv_subnorm_relu2(down)) against the
    dense fp32 reference layer, NMSE <= 5e-4."""
    layer = small_2b4t_layer(seed=10)
    try:
        ctx, hd = 64, 128
        kc, vc = torch.randn((1, ctx, hd), device="cuda") * 0.3, torch.randn((1, ctx, hd), device="cuda") * 0.3
        kc2, vc2 = kc.clone(), vc.clone()
        pos = ctx - 1
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
        x = torch.randn((1, 512), device="cuda")
        got = layer.forward(x, kc, vc, pos, cos, sin).clone()
        dense_w = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.forward(x, kc2, vc2, pos, cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense_w[n].T)).clone()
        torch.cuda.synchronize()
        assert torch.isfinite(got).all()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= DENSE_NMSE, nmse
    finally:
        layer.free()


@pytest.mark.parametrize("P", [16, 130])
def test_harness_relu2_prompt_step(stream, P):
    """The fused prompt step (prefill_rmsnorm([qkv]), prefill_subnorm(o), prefill_rmsnorm([gate, up]), prefill_subnorm_relu2(down))
    against the dense fp32 reference layer, NMSE <= 5e-4."""
    layer = small_2b4t_layer(seed=11)
    try:
        hd = 128
        torch.manual_seed(12)
        x = torch.randn((P, 512), device="cuda")
        ang = torch.arange(P, device="cuda").float()[:, None] / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(ang), torch.sin(ang)
        kc, vc = torch.zeros((1, P, hd), device="cuda"), torch.zeros((1, P, hd), device="cuda")
        got = layer.prompt(x, kc, vc, cos, sin).clone()
        assert tb.last_launch()["batch"] == -P, "the down projection did not run a tile"
        dense_w = {n: l.dense(torch) for n, l in layer.lin.items()}
        want = layer.prompt(x, kc.clone(), vc.clone(), cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense_w[n].T)).clone()
        nmse = float(((got - want) ** 2).mean() / (want ** 2).mean())
        assert nmse < DENSE_NMSE, nmse
    finally:
        layer.free()


def test_harness_2b4t_model(stream):
    """Two full-size 2B4T layers (hidden 2560, FFN 6912, 20 heads, 5 KV heads): one graphed token step and one prompt step, finite."""
    from decode_harness import DecodeModel
    m = DecodeModel(2, H2B, F2B, 20, 2, False, ctx=160, fused_ops=True, sub_norms=True, ffn_act="relu2", kv_heads=5, prompt_len=130)
    try:
        assert m.kc[0].shape == (5, 160, 128) and m.layers[0].lin["qkv"].mout == 3840
        m.capture(stream)
        m.graph.replay()
        m.prompt()
        torch.cuda.synchronize()
        assert torch.isfinite(m.y).all() and torch.isfinite(m.py).all()
    finally:
        m.free()
