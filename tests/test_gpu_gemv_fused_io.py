"""GPU suite (-m gpu): the GEMV launches with a transformed input or a residual output -- tmac_b200_gemv_rmsnorm (q/k/v, gate/up
behind an RMSNorm), tmac_b200_gemv_glu (down behind SiLU*mul, with or without a residual) and tmac_b200_gemv_residual (o + x).

Every check is bit for bit against the equivalence the header documents: the call equals tmac_b200_gemv_grouped on the same tensors
fed the transformed input materialised in fp32 -- the norm input computed in numpy float32 in the documented order, the GLU input as
g / (1 + exp(-g)) * u on the GPU -- plus a numpy float32 add of the residual, rounded once to fp16 for an F16 call.
kfactor = act_group_size / 4 everywhere, as in the sequence tests."""
import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from seq_util import A_CASES, A_IDS, EPS, kc, mk, norm_weight, rms_input, same_bits, stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def dev(x, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda().to(dtype)


def nan_out(N, M, dtype=torch.float32):
    return torch.full((N, M), float("nan"), device="cuda", dtype=dtype)


def grouped(ops, N, a):
    """gemv_grouped of the tensors on the fp32 input a (device [N][K]): the outputs as numpy float32."""
    outs = [nan_out(N, o.cfg.Mout) for o in ops]
    tb.gemv_grouped([o.wt for o in ops], N, a, outs)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in outs]


def glu_ref(G, U):
    """The GLU input on the GPU from device tensors G, U (fp32 or fp16, widened)."""
    g, u = G.float(), U.float()
    return g / (1 + torch.exp(-g)) * u


def expect(got, want32, res=None, f16=False, what=""):
    """got (device) == want32 (+ res, numpy float32), rounded to fp16 when f16."""
    want = want32 if res is None else want32 + np.asarray(res, np.float32)
    if f16:
        want = want.astype(np.float16)
    g = got.cpu().numpy()
    assert same_bits(g, want), "%s differs from the materialised-input launch (max |diff| %g)" % (
        what, float(np.nanmax(np.abs(g.astype(np.float32) - want.astype(np.float32)))))


def check_norm(ops, N, H, w, eps=EPS, dtype=torch.float32):
    """gemv_rmsnorm of the tensors on H (host [N][K] float32, passed as dtype) against gemv_grouped on rms_input."""
    f16 = dtype == torch.float16
    dH = dev(H, dtype)
    outs = [nan_out(N, o.cfg.Mout, dtype) for o in ops]
    tb.gemv_rmsnorm([o.wt for o in ops], N, dH, dev(w), eps, outs, dtype=tb.F16 if f16 else tb.F32)
    launch = tb.last_launch()
    torch.cuda.synchronize()
    a = rms_input(dH.float().cpu().numpy(), w, eps)
    for i, (o, ref) in enumerate(zip(outs, grouped(ops, N, dev(a)))):
        expect(o, ref, f16=f16, what="gemv_rmsnorm tensor %d" % i)
    return a, launch


def check_glu(op, N, G, U, R=None, dtype=torch.float32):
    f16 = dtype == torch.float16
    dG, dU = dev(G, dtype), dev(U, dtype)
    dR = None if R is None else dev(R, dtype)
    out = nan_out(N, op.cfg.Mout, dtype)
    tb.gemv_glu(op.wt, N, dG, dU, out, R=dR, dtype=tb.F16 if f16 else tb.F32)
    ref = grouped([op], N, glu_ref(dG, dU))[0]
    expect(out, ref, None if dR is None else dR.float().cpu().numpy(), f16, "gemv_glu")


def check_residual(op, N, B, R, dtype=torch.float32):
    f16 = dtype == torch.float16
    dB, dR = dev(B, dtype), dev(R, dtype)
    out = nan_out(N, op.cfg.Mout, dtype)
    tb.gemv_residual(op.wt, N, dB, dR, out, dtype=tb.F16 if f16 else tb.F32)
    ref = grouped([op], N, dB.float())[0]
    expect(out, ref, dR.float().cpu().numpy(), f16, "gemv_residual")


def normal(rng, *shape):
    return rng.standard_normal(shape).astype(np.float32)


# ---- 1: every chunking ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_every_chunking(mk, g, ags, bits, zp, N):
    K = 20 * min(g, 128)                          # 20 chunks: some warps hold 2 blocks, some 1
    ops = [mk(768, K, bits, g=g, ags=ags, zp=zp, seed=s) for s in (1, 2)]
    rng = np.random.default_rng(g + ags + bits + N)
    check_norm(ops, N, act_rows.rows(rng, N, K, ags), norm_weight(rng, K))
    check_glu(ops[0], N, act_rows.rows(rng, N, K, ags), normal(rng, N, K), R=normal(rng, N, 768))
    check_glu(ops[1], N, normal(rng, N, K), act_rows.rows(rng, N, K, ags))
    check_residual(ops[1], N, act_rows.rows(rng, N, K, ags), normal(rng, N, 768))


# ---- 2: the order of the norm's sum of squares ----------------------------------------------------------------------------------
def test_norm_order_and_row_edges(mk):
    """fp32 and mixed-magnitude rows (the mixed row's inv changes when its sum of squares is re-associated), a row 2^10 times the
    fp32 row, and an all-zero row (its input is 0 * inv, with eps only inside the root)."""
    K, ags = 2560, 64
    ops = [mk(512, K, 2, ags=ags, zp=True, seed=s) for s in (3, 4, 5)]
    rng = np.random.default_rng(7)
    fp32, mixed = act_rows.rows(rng, 2, K, ags, kinds=("fp32", "mixed"))
    H = np.stack([mixed, fp32, fp32 * np.float32(1024.0), np.zeros(K, np.float32)])
    g = mixed.reshape(-1, 4)
    q = (g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + (g[:, 2] * g[:, 2] + g[:, 3] * g[:, 3])
    serial = np.float32(0.0)
    for v in q:
        serial = np.float32(serial + v)
    w = norm_weight(rng, K)
    a, _ = check_norm(ops, 4, H, w)
    assert not np.array_equal(a[0], (mixed * (np.float32(1.0) / np.sqrt(serial / np.float32(K) + np.float32(EPS)))) * w), \
        "the mixed row no longer tells the documented order from a serial sum"
    assert not np.any(a[3])
    check_norm(ops[:1], 3, H[:3], w, eps=0.0)         # eps = 0 without the zero row, whose inv would be inf
    check_norm(ops[:1], 4, H, w, eps=0.5)


# ---- 3: groups ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 4, 40])
def test_groups(mk, N):
    """A 3-tensor group (q/k/v) and a 2-tensor group (gate/up); at N = 40 the call still runs the GEMV kernel."""
    K = 1024
    rng = np.random.default_rng(N)
    qkv = [mk(640, K, 2, zp=True, seed=10 + s) for s in range(3)]
    gu = [mk(1536, K, 4, seed=20 + s) for s in range(2)]
    for ops in (qkv, gu):
        _, launch = check_norm(ops, N, normal(rng, N, K), norm_weight(rng, K))
        assert launch["batch"] == len(ops), launch       # >= 0: not the prefill tile (batch -N)


# ---- 4: fp16 ----------------------------------------------------------------------------------------------------------------------
def test_fp16(mk):
    """fp16 inputs, residual and output: each call's C16 is the fp16 rounding of the same call in fp32 on the widened inputs."""
    K, N, M = 1024, 3, 768
    ops = [mk(M, K, bits, zp=bits == 2, seed=30 + bits) for bits in (2, 4)]
    rng = np.random.default_rng(31)
    h16 = lambda *s: act_rows.rows16(rng, s[0], s[1], 64)
    for op in ops:
        check_norm([op], N, h16(N, K), norm_weight(rng, K), dtype=torch.float16)
        check_glu(op, N, h16(N, K), h16(N, K), R=h16(N, M), dtype=torch.float16)
        check_glu(op, N, h16(N, K), h16(N, K), dtype=torch.float16)
        check_residual(op, N, h16(N, K), h16(N, M), dtype=torch.float16)
        # and C16 == fp16(C32) of the fp32 call on the same (fp16-exact) values
        G, U, R = h16(N, K), h16(N, K), h16(N, M)
        c32, c16 = nan_out(N, M), nan_out(N, M, torch.float16)
        tb.gemv_glu(op.wt, N, dev(G), dev(U), c32, R=dev(R))
        tb.gemv_glu(op.wt, N, dev(G, torch.float16), dev(U, torch.float16), c16, R=dev(R, torch.float16), dtype=tb.F16)
        torch.cuda.synchronize()
        assert same_bits(c16.cpu().numpy(), c32.cpu().numpy().astype(np.float16))


# ---- 5: in place, inputs that change, graphs ------------------------------------------------------------------------------------
def test_in_place_residual(mk):
    K, N, M = 1024, 2, 512
    op = mk(M, K, 2, zp=True, seed=40)
    rng = np.random.default_rng(41)
    for dtype, d in ((torch.float32, tb.F32), (torch.float16, tb.F16)):
        B, G, U, R = normal(rng, N, K), normal(rng, N, K), normal(rng, N, K), normal(rng, N, M)
        for call in (lambda out, r: tb.gemv_residual(op.wt, N, dev(B, dtype), r, out, dtype=d),
                     lambda out, r: tb.gemv_glu(op.wt, N, dev(G, dtype), dev(U, dtype), out, R=r, dtype=d)):
            sep = nan_out(N, M, dtype)
            call(sep, dev(R, dtype))
            inplace = dev(R, dtype)
            call(inplace, inplace)
            torch.cuda.synchronize()
            assert same_bits(inplace.cpu().numpy(), sep.cpu().numpy())


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_inputs_change_between_launches(stream, mk, graph):
    """The four calls of a layer on buffers rewritten before every launch (or CUDA-graph replay) give that launch's fresh outputs."""
    K, N = 1024, 1
    qkv = [mk(K, K, 2, zp=True, seed=50 + s) for s in range(3)]
    o, down = mk(K, K, 2, zp=True, seed=53), mk(K, 2048, 2, zp=True, seed=54)
    gu = [mk(2048, K, 2, zp=True, seed=55 + s) for s in range(2)]
    rng = np.random.default_rng(56)
    w1, w2 = dev(norm_weight(rng, K)), dev(norm_weight(rng, K))
    x, att, g, u = nan_out(N, K), nan_out(N, K), nan_out(N, 2048), nan_out(N, 2048)
    q = [nan_out(N, K) for _ in range(3)]; h = nan_out(N, K); gg = [nan_out(N, 2048) for _ in range(2)]; y = nan_out(N, K)

    def calls():
        tb.gemv_rmsnorm([t.wt for t in qkv], N, x, w1, EPS, q)
        tb.gemv_residual(o.wt, N, att, x, h)
        tb.gemv_rmsnorm([t.wt for t in gu], N, h, w2, EPS, gg)
        tb.gemv_glu(down.wt, N, g, u, y, R=h)

    def fill():
        for t, L in ((x, K), (att, K), (g, 2048), (u, 2048)):
            t.copy_(dev(normal(rng, N, L)))

    fill(); calls(); torch.cuda.synchronize()     # warm-up: pointer tables, module load
    cg = None
    if graph:
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=stream):
            calls()
    for _ in range(3):
        fill()
        if cg is not None:
            cg.replay()
        else:
            calls()
        torch.cuda.synchronize()
        hx, hatt = x.cpu().numpy(), att.cpu().numpy()
        a1 = rms_input(hx, w1.cpu().numpy(), EPS)
        for got, ref in zip(q, grouped(qkv, N, dev(a1))):
            expect(got, ref, what="q/k/v")
        expect(h, grouped([o], N, att)[0], hx, what="o + x")
        hh = h.cpu().numpy()
        for got, ref in zip(gg, grouped(gu, N, dev(rms_input(hh, w2.cpu().numpy(), EPS)))):
            expect(got, ref, what="gate/up")
        expect(y, grouped([down], N, glu_ref(g, u))[0], hh, what="down + h")
        assert np.array_equal(x.cpu().numpy(), hx) and np.array_equal(att.cpu().numpy(), hatt)


# ---- 6: Llama-2-7B shapes --------------------------------------------------------------------------------------------------------
def test_llama2_7b_shapes(mk):
    """W2 g128 zp, N = 1: q/k/v 4096x4096 behind a norm, gate/up 11008x4096 behind a norm, down 4096x11008 with GLU and a residual."""
    H, F = 4096, 11008
    qkv = [mk(H, H, 2, g=128, ags=64, zp=True, seed=60 + s) for s in range(3)]
    gu = [mk(F, H, 2, g=128, ags=64, zp=True, seed=63 + s) for s in range(2)]
    down = mk(H, F, 2, g=128, ags=64, zp=True, seed=65)
    rng = np.random.default_rng(66)
    check_norm(qkv, 1, normal(rng, 1, H), norm_weight(rng, H))
    check_norm(gu, 1, normal(rng, 1, H), norm_weight(rng, H))
    check_glu(down, 1, normal(rng, 1, F), normal(rng, 1, F), R=normal(rng, 1, H))


# ---- 7: rejections ----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    K, M = 1024, 512
    op = mk(M, K, 2, zp=True, seed=70)
    other = mk(2 * M, K, 2, zp=True, seed=71)
    # the integer path: one activation group over the whole row, wider than a chunk (the layout keeps every fp-path group inside one)
    int_cfg = T.Config(320, 1280, 2, one_scale=True).resolved()
    w, sc, z, _ = T.make_problem(int_cfg, seed=72)
    A, S = T.pack_reference_layout(w, sc, z, int_cfg)
    int_wt = tb.upload_reference_layout(kc(int_cfg), A, S)
    try:
        x, nw, out, r = nan_out(1, K), torch.ones(K, device="cuda"), nan_out(1, M), torch.zeros((1, M), device="cuda")
        xi, nwi, outi = nan_out(1, 1280), torch.ones(1280, device="cuda"), nan_out(1, 320)
        hx, hout = np.zeros((1, K), np.float32), np.zeros((1, M), np.float32)
        bad = [
            lambda: tb.gemv_rmsnorm([int_wt], 1, xi, nwi, EPS, [outi]),                    # integer path
            lambda: tb.gemv_glu(int_wt, 1, xi, xi, outi),
            lambda: tb.gemv_residual(int_wt, 1, xi, torch.zeros((1, 320), device="cuda"), outi),
            lambda: tb.gemv_rmsnorm([op.wt], 1, hx, nw, EPS, [out]),                       # host pointers
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw.cpu(), EPS, [out]),
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw, EPS, [hout]),
            lambda: tb.gemv_glu(op.wt, 1, hx, x, out),
            lambda: tb.gemv_glu(op.wt, 1, x, hx, out),
            lambda: tb.gemv_glu(op.wt, 1, x, x, out, R=hout),
            lambda: tb.gemv_residual(op.wt, 1, x, hout, out),
            lambda: tb.gemv_residual(op.wt, 1, x, r, hout),
            lambda: tb.gemv_rmsnorm([op.wt, other.wt], 1, x, nw, EPS, [out, nan_out(1, 2 * M)]),   # different geometry
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, None, EPS, [out]),                      # null w
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw[1:], EPS, [out]),                    # w not 16-byte aligned
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw, -1e-5, [out]),                      # eps negative / not finite
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw, float("nan"), [out]),
            lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw, float("inf"), [out]),
            lambda: tb.gemv_residual(op.wt, 1, x, None, out),                              # null R
            lambda: tb.gemv_glu(op.wt, 1, x, None, out),                                   # null U
        ]
        torch.cuda.synchronize()
        for i, call in enumerate(bad):
            out.fill_(float("nan")); outi.fill_(float("nan"))
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all() and torch.isnan(outi).all(), "rejected call %d launched" % i
        # an armed peer output makes the call fail and is disarmed by it, as for gemv_grouped
        for call in (lambda: tb.gemv_rmsnorm([op.wt], 1, x, nw, EPS, [out]), lambda: tb.gemv_residual(op.wt, 1, x, r, out),
                     lambda: tb.gemv_glu(op.wt, 1, x, x, out)):
            tb.peer_outputs([nan_out(1, M).data_ptr()])
            with pytest.raises(tb.TMACError):
                call()
            call()
    finally:
        int_wt.free()


# ---- 8: the decode harness ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_harness_layer_with_fused_ops(stream, bits, zp):
    """A fused_ops layer against the same layer with dense dequantised fp32 weights, NMSE <= 5e-4 as in test_gpu_decode_harness.py."""
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx = 1024, 2816, 8, 64
    layer = DecodeLayer(hidden, ffn, heads, bits, zp, seed=3, fused_ops=True)
    try:
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


def test_harness_graphed_token_step_with_fused_ops(stream):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=3, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=32, fused_ops=True)
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


@pytest.mark.parametrize("other", ["ffn_sequence", "post_attn_sequence"])
def test_harness_rejects_fused_ops_with_a_sequence(stream, other):
    from decode_harness import DecodeLayer, DecodeModel
    with pytest.raises(ValueError):
        DecodeLayer(256, 512, 2, 2, True, seed=0, fused_ops=True, **{other: True})
    with pytest.raises(ValueError):
        DecodeModel(1, 256, 512, 2, 2, True, ctx=8, fused_ops=True, **{other: True})
