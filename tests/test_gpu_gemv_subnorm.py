"""GPU suite (-m gpu): tmac_b200_gemv_subnorm, the GEMV behind the RMS norm of a row (BitNet's attn_sub_norm before o) or of its SwiGLU
(BitNet's ffn_sub_norm before down), with an optional residual, and the BitNet layer of the decode harness built on it.

Every check is bit for bit against the equivalence the header documents: the call equals tmac_b200_gemv_grouped on the same tensor fed
a = rmsnorm(X) * w materialised in fp32 -- X = G, or the GLU input g / (1 + exp(-g)) * u computed on the GPU, and the norm computed in
numpy float32 in the documented order -- plus a numpy float32 add of the residual, rounded once to fp16 for an F16 call."""
import types

import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from fused_util import serial_input
from seq_util import EPS, TIGHT_TOL, kc, mk, norm_weight, oracle_gemv, rms_input, same_bits, stream
from test_gpu_gemv_fused_io import dev, expect, glu_ref, grouped, nan_out

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def normal(rng, *shape):
    return rng.standard_normal(shape).astype(np.float32)


@pytest.fixture
def bitnet(stream):
    """bitnet(M, K, seed) uploads a ternary one-scale tensor with activation groups of 64 (BitNet-3B's grouping: the fp path, chunk
    128 where K allows it, else 64), through the decode harness's QLinear; every tensor made in the test is freed after it."""
    from decode_harness import QLinear
    made = []

    def make(M, K, seed):
        q = QLinear(M, K, 2, 128, False, seed, one_scale=True, act_group_size=64)
        made.append(q)
        return types.SimpleNamespace(wt=q.wt, cfg=types.SimpleNamespace(Mout=M, K=K))
    yield make
    for q in made:
        q.free()


def subnorm_input(dG, dU, w, eps):
    """The input a the call documents, from the device rows G (and U): numpy float32 [N][K]."""
    x = dG.float() if dU is None else glu_ref(dG, dU)
    return rms_input(x.cpu().numpy(), w, eps)


def check_subnorm(op, N, G, w, U=None, R=None, eps=EPS, dtype=torch.float32):
    """gemv_subnorm of op on host rows G (U, R; float32, passed as dtype) against gemv_grouped on the materialised input; returns a."""
    f16 = dtype == torch.float16
    dG = dev(G, dtype)
    dU = None if U is None else dev(U, dtype)
    dR = None if R is None else dev(R, dtype)
    out = nan_out(N, op.cfg.Mout, dtype)
    tb.gemv_subnorm(op.wt, N, dG, dev(w), eps, out, U=dU, R=dR, dtype=tb.F16 if f16 else tb.F32)
    torch.cuda.synchronize()
    a = subnorm_input(dG, dU, w, eps)
    expect(out, grouped([op], N, dev(a))[0], None if dR is None else dR.float().cpu().numpy(), f16,
           "gemv_subnorm (U %s, R %s, %s)" % (U is not None, R is not None, "F16" if f16 else "F32"))
    return a


def all_forms(op, N, K, rng, ags):
    """U null and given, R null and given, F32 and F16 (fp16-exact rows for F16)."""
    M = op.cfg.Mout
    for f16 in (False, True):
        rows = (lambda: act_rows.rows16(rng, N, K, ags)) if f16 else (lambda: act_rows.rows(rng, N, K, ags))
        res = (lambda: normal(rng, N, M).astype(np.float16).astype(np.float32)) if f16 else (lambda: normal(rng, N, M))
        dtype = torch.float16 if f16 else torch.float32
        w = norm_weight(rng, K)
        for with_u in (False, True):
            for with_r in (False, True):
                check_subnorm(op, N, rows(), w, U=rows() if with_u else None, R=res() if with_r else None, dtype=dtype)


# ---- 1: bit equality with gemv_grouped on the materialised input, every grouping -------------------------------------------------
GROUPINGS = [("w2zp-g128-a64", 2, 128, 64, True), ("w3zp-g128-a64", 3, 128, 64, True), ("w4-g128-a64", 4, 128, 64, False),
             ("w4-g32-a32", 4, 32, 32, False), ("w1-g128-a64", 1, 128, 64, False)]


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("name,bits,g,ags,zp", GROUPINGS, ids=[c[0] for c in GROUPINGS])
def test_every_grouping(mk, name, bits, g, ags, zp, N):
    K = 20 * min(g, 128)                          # 20 chunks: some warps hold 2 blocks, some 1
    op = mk(768, K, bits, g=g, ags=ags, zp=zp, seed=bits + g)
    all_forms(op, N, K, np.random.default_rng(g + ags + bits + N), ags)


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("M,K", [(768, 2560), (256, 8640)], ids=["chunk128", "chunk64-k8640"])
def test_bitnet_grouping(bitnet, M, K, N):
    """One weight scale, activation groups of 64: chunk 128 at K = 2560, chunk 64 at BitNet-3B's down K = 8640."""
    op = bitnet(M, K, seed=K + N)
    all_forms(op, N, K, np.random.default_rng(K + N), 64)


# ---- 2: the order of the sum of squares, and the zero row -----------------------------------------------------------------------
def test_order_and_zero_row(mk):
    """A row whose SwiGLU values have two magnitudes: one K-group of squares near 2^28 and 639 of squares near 1, each below half
    an ulp of the large one.  A serial sum of squares drops every small group; the documented order sums them per lane first and
    adds them in the butterfly, some hundred ulps more, so the row's inv tells the two orders apart.  Also a row of mixed
    magnitudes (U mixed), the plain mixed row for U = NULL, and an all-zero row (silu(0) = 0, so a = 0 whatever U holds): its
    output is +0, or R."""
    K, M, ags = 2560, 512, 64
    op = mk(M, K, 2, ags=ags, zp=True, seed=3)
    rng = np.random.default_rng(7)
    fp32, mixed = act_rows.rows(rng, 2, K, ags, kinds=("fp32", "mixed"))
    g_two, u_two = np.abs(normal(rng, K)) + np.float32(4.0), np.float32(0.1) * normal(rng, K)
    u_two[:4] = 4096.0
    G = np.stack([g_two, normal(rng, K), fp32, np.zeros(K, np.float32)])
    U = np.stack([u_two, mixed, normal(rng, K), normal(rng, K)])
    w = norm_weight(rng, K)
    a = check_subnorm(op, 4, G, w, U=U)
    s = glu_ref(dev(G), dev(U)).cpu().numpy()
    assert not np.array_equal(a[0], serial_input(s[0], w, EPS)), \
        "the two-magnitude SwiGLU row no longer tells the documented order from a serial sum"
    assert not np.any(a[3])
    G, U = G[1:], U[1:]
    a = check_subnorm(op, 2, np.stack([mixed, np.zeros(K, np.float32)]), w)
    assert not np.array_equal(a[0], serial_input(mixed, w, EPS)), "the mixed row no longer tells the documented order"
    # the zero row's output: +0 without a residual, R with one
    for R in (None, normal(rng, 1, M)):
        out = nan_out(1, M)
        tb.gemv_subnorm(op.wt, 1, dev(np.zeros((1, K))), dev(w), EPS, out, U=dev(U[2:]), R=None if R is None else dev(R))
        torch.cuda.synchronize()
        assert same_bits(out, np.zeros((1, M), np.float32) if R is None else R)
    check_subnorm(op, 2, G[:2], w, U=U[:2], eps=0.0)            # eps = 0 without the zero row, whose inv would be inf
    check_subnorm(op, 3, G, w, U=U, eps=0.5)


# ---- 3: against the float oracle -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_against_oracle(oracle, mk, bits, zp):
    K, M, N = 2560, 768, 2
    op = mk(M, K, bits, g=128, ags=64, zp=zp, seed=20 + bits)
    rng = np.random.default_rng(21 + bits)
    G, U, w = normal(rng, N, K), normal(rng, N, K), norm_weight(rng, K)
    for u in (None, U):
        out = nan_out(N, M)
        tb.gemv_subnorm(op.wt, N, dev(G), dev(w), EPS, out, U=None if u is None else dev(u))
        torch.cuda.synchronize()
        a = subnorm_input(dev(G), None if u is None else dev(u), w, EPS)
        got = out.cpu().numpy()
        for n in range(N):
            ref = oracle_gemv(oracle, op.cfg, op.A, op.S, a[n])
            err = np.abs(got[n] - ref).max() / np.abs(ref).max()
            assert err <= TIGHT_TOL, "row %d (U %s): rel err %.3g against the oracle on a" % (n, u is not None, err)


# ---- 4: forced decompositions ----------------------------------------------------------------------------------------------------
def test_forced_decompositions(mk, bitnet):
    """Under the cs / wpc knobs the call still equals gemv_grouped under the same knobs."""
    ops = [("w2zp", mk(512, 2560, 2, zp=True, seed=30), 2560), ("bitnet-k8640", bitnet(256, 8640, seed=31), 8640)]
    rng = np.random.default_rng(32)
    try:
        for _, op, K in ops:
            G, U, w, R = normal(rng, 2, K), normal(rng, 2, K), norm_weight(rng, K), normal(rng, 2, op.cfg.Mout)
            for cs, wpc in ((1, 1), (2, 3), (4, 8), (8, 2), (8, 8)):
                tb.debug_set("cs", cs); tb.debug_set("wpc", wpc)
                check_subnorm(op, 2, G, w, U=U, R=R)
                ll = tb.last_launch()
                assert (ll["cluster"], ll["warps_per_cta"]) == (cs, wpc), ll
                check_subnorm(op, 2, G, w)
    finally:
        tb.debug_set("cs", 0); tb.debug_set("wpc", 0)


# ---- 5: aliasing and graphs ------------------------------------------------------------------------------------------------------
def test_residual_in_place(mk, bitnet):
    K, N, M = 2560, 2, 512
    rng = np.random.default_rng(40)
    for op in (mk(M, K, 2, zp=True, seed=40), bitnet(M, K, seed=41)):
        for dtype, d in ((torch.float32, tb.F32), (torch.float16, tb.F16)):
            G, U, R, w = dev(normal(rng, N, K), dtype), dev(normal(rng, N, K), dtype), dev(normal(rng, N, M), dtype), dev(norm_weight(rng, K))
            for u in (None, U):
                sep = nan_out(N, M, dtype)
                tb.gemv_subnorm(op.wt, N, G, w, EPS, sep, U=u, R=R, dtype=d)
                inplace = R.clone()
                tb.gemv_subnorm(op.wt, N, G, w, EPS, inplace, U=u, R=inplace, dtype=d)
                torch.cuda.synchronize()
                assert same_bits(inplace, sep)


def test_graph_replay(stream, bitnet):
    """Both forms captured in one CUDA graph: the replay gives the eager outputs."""
    H, F = 640, 1728
    o, down = bitnet(H, H, seed=50), bitnet(H, F, seed=51)
    rng = np.random.default_rng(52)
    att, x, g, u = dev(normal(rng, 1, H)), dev(normal(rng, 1, H)), dev(normal(rng, 1, F)), dev(normal(rng, 1, F))
    w_as, w_fs = dev(norm_weight(rng, H)), dev(norm_weight(rng, F))
    h, y = nan_out(1, H), nan_out(1, H)

    def calls():
        tb.gemv_subnorm(o.wt, 1, att, w_as, EPS, h, R=x)
        tb.gemv_subnorm(down.wt, 1, g, w_fs, EPS, y, U=u, R=h)

    calls()                                       # eager, and warm-up: pointer tables, module load
    torch.cuda.synchronize()
    eager_h, eager_y = h.clone(), y.clone()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    h.fill_(float("nan")); y.fill_(float("nan"))
    cg.replay()
    torch.cuda.synchronize()
    assert same_bits(h, eager_h) and same_bits(y, eager_y)


# ---- 6: rejections -----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    K, M = 1024, 512
    op = mk(M, K, 2, zp=True, seed=70)
    # the integer path: one activation group over the whole row
    int_cfg = T.Config(320, 1280, 2, one_scale=True).resolved()
    w_, sc, z, _ = T.make_problem(int_cfg, seed=72)
    A, S = T.pack_reference_layout(w_, sc, z, int_cfg)
    int_wt = tb.upload_reference_layout(kc(int_cfg), A, S)
    try:
        x, nw, out, r = nan_out(1, K), torch.ones(K, device="cuda"), nan_out(1, M), torch.zeros((1, M), device="cuda")
        xi, nwi, outi = nan_out(1, 1280), torch.ones(1280, device="cuda"), nan_out(1, 320)
        hx, hout = np.zeros((1, K), np.float32), np.zeros((1, M), np.float32)
        bad = [
            lambda: tb.gemv_subnorm(int_wt, 1, xi, nwi, EPS, outi),                        # integer path
            lambda: tb.gemv_subnorm(int_wt, 1, xi, nwi, EPS, outi, U=xi),
            lambda: tb.gemv_subnorm(op.wt, 1, hx, nw, EPS, out),                           # host pointers
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, EPS, out, U=hx),
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw.cpu(), EPS, out),
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, EPS, out, R=hout),
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, EPS, hout),
            lambda: tb.gemv_subnorm(op.wt, 1, None, nw, EPS, out),                         # null G
            lambda: tb.gemv_subnorm(op.wt, 1, x, None, EPS, out),                          # null w
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw[1:], EPS, out),                        # w not 16-byte aligned
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, -1e-5, out),                          # eps negative / not finite
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, float("nan"), out),
            lambda: tb.gemv_subnorm(op.wt, 1, x, nw, float("inf"), out, U=x),
        ]
        torch.cuda.synchronize()
        for i, call in enumerate(bad):
            out.fill_(float("nan")); outi.fill_(float("nan"))
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all() and torch.isnan(outi).all(), "rejected call %d launched" % i
        # an armed peer output makes the call fail and is disarmed by it
        xf = torch.randn((1, K), device="cuda")
        for call in (lambda: tb.gemv_subnorm(op.wt, 1, xf, nw, EPS, out, R=r), lambda: tb.gemv_subnorm(op.wt, 1, xf, nw, EPS, out, U=xf)):
            tb.peer_outputs([nan_out(1, M).data_ptr()])
            out.fill_(float("nan"))
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all()
            call()
            torch.cuda.synchronize()
            assert not torch.isnan(out).any()
    finally:
        int_wt.free()


# ---- 7: the decode harness's BitNet layer ---------------------------------------------------------------------------------------
def test_harness_bitnet_layer_with_fused_ops(stream):
    """A sub_norms fused_ops layer against the same layer with dense dequantised fp32 weights and torch sub-norms, NMSE <= 5e-4 as in
    test_gpu_decode_harness.py."""
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx = 1024, 2816, 8, 64
    layer = DecodeLayer(hidden, ffn, heads, 2, False, seed=3, fused_ops=True, sub_norms=True)
    try:
        assert all(l.one_scale for l in layer.lin.values())
        hd = hidden // heads
        kc_, vc = torch.randn((heads, ctx, hd), device="cuda") * 0.3, torch.randn((heads, ctx, hd), device="cuda") * 0.3
        kc2, vc2 = kc_.clone(), vc.clone()
        pos = ctx - 1
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
        x = torch.randn((1, hidden), device="cuda")
        got = layer.forward(x, kc_, vc, pos, cos, sin).clone()
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.forward(x, kc2, vc2, pos, cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T)).clone()
        torch.cuda.synchronize()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= 5e-4, nmse
    finally:
        layer.free()


def test_harness_bitnet_model_graph(stream):
    """Two BitNet-3B-shaped layers (hidden 3200, FFN 8640, 32 heads) with fused_ops: the captured token step replays the eager one."""
    from decode_harness import DecodeModel
    m = DecodeModel(layers=2, hidden=3200, ffn=8640, heads=32, bits=2, zero_point=False, ctx=32, fused_ops=True, sub_norms=True)
    try:
        with torch.cuda.stream(stream):
            m.step()
        torch.cuda.synchronize()
        eager = m.y.clone()
        assert torch.isfinite(eager).all()
        m.capture(stream)
        m.y.zero_()
        m.graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.y, eager)
    finally:
        m.free()


@pytest.mark.parametrize("other", [{"ffn_sequence": True}, {"post_attn_sequence": True}, {"experts": 4, "fused_ops": True}],
                         ids=["ffn_sequence", "post_attn_sequence", "experts"])
def test_harness_rejects_sub_norms_with(stream, other):
    from decode_harness import DecodeLayer, DecodeModel
    with pytest.raises(ValueError):
        DecodeLayer(256, 512, 2, 2, False, seed=0, sub_norms=True, **other)
    with pytest.raises(ValueError):
        DecodeModel(1, 256, 512, 2, 2, False, ctx=8, sub_norms=True, **other)


def test_harness_bitnet_prompt_step(stream):
    """A sub_norms fused_ops layer's prompt step runs its linears as per-linear calls and matches the dense fp32 reference."""
    from decode_harness import DecodeLayer
    hidden, ffn, heads, P = 640, 1728, 8, 16
    layer = DecodeLayer(hidden, ffn, heads, 2, False, seed=5, fused_ops=True, sub_norms=True)
    try:
        hd = hidden // heads
        kc_, vc = torch.zeros((heads, P, hd), device="cuda"), torch.zeros((heads, P, hd), device="cuda")
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        ang = torch.arange(P, device="cuda").float()[:, None] * inv[None, :]
        cos, sin = torch.cos(ang), torch.sin(ang)
        x = torch.randn((P, hidden), device="cuda")
        got = layer.prompt(x, kc_, vc, cos, sin).clone()
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.prompt(x, kc_.clone(), vc.clone(), cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T)).clone()
        torch.cuda.synchronize()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= 5e-4, nmse
    finally:
        layer.free()
