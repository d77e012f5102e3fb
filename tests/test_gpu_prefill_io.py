"""GPU suite (-m gpu): the transformed-input calls at prefill sizes -- tmac_b200_prefill_rmsnorm (q/k/v, gate/up behind an RMSNorm,
all tensors in one tile launch), tmac_b200_prefill_glu (down behind SiLU*mul, with or without a residual) and
tmac_b200_prefill_residual (o + x), which run the routed wgmma tiles as one expert with the identity routing.

Every row is checked bit for bit against the equality the header documents: the dense tile call tmac_b200_gemv on the input
materialised in fp32 (the norm input in numpy float32 in the documented order, seq_util.rms_input; the GLU input on the GPU), forced
onto the same tile (prefill_min_n = 1; prefill16 = 0 for the int8 tile), plus a numpy float32 add of the residual, rounded once to
fp16 for an F16 call.  kfactor = act_group_size / 4 everywhere, as in the sequence tests."""
import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
from fused_util import dense_tile, knobs, tdt
from seq_util import A_CASES, A_IDS, EPS, mk, norm_weight, rms_input, same_bits, stream
from test_gpu_gemv_fused_io import dev, expect, glu_ref, nan_out, normal

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

PF16_TOL, INT8_TOL = 5e-4, 2e-5   # the tiles' bounds against the oracle, max |got - ref| / max |ref| (DESIGN 3.3)
TILES = [True, False]
TILE_IDS = ["fp16", "int8"]
TILE_CASES = [c for c in A_CASES if c[2] != 1]    # every fp grouping the tiles take, W2 / W3 / W4 (g256: 128-K chunks)
TILE_CASE_IDS = [i for c, i in zip(A_CASES, A_IDS) if c in TILE_CASES]


def takes16(prefill16, N):
    """The tile the prefill forms pick: the dense calls' rule."""
    return bool(prefill16) and N >= 64


def run_norm(wts, N, H, w, eps, prefill16, dtype=torch.float32):
    outs = [nan_out(N, wt.cfg.M, dtype) for wt in wts]
    with knobs(prefill16=int(prefill16)):
        tb.prefill_rmsnorm(wts, N, H, w, eps, outs, dtype=tdt(dtype))
        launch = tb.last_launch()
    torch.cuda.synchronize()
    return outs, launch


def check_norm(wts, N, H, w, prefill16, eps=EPS, dtype=torch.float32):
    """prefill_rmsnorm of the tensors on H (device, dtype) against the dense tile on rms_input; returns the materialised input."""
    t16 = takes16(prefill16, N)
    outs, launch = run_norm(wts, N, H, dev(w), eps, prefill16, dtype)
    assert launch["cluster"] == (16 if t16 else 1) and launch["batch"] == -N, launch
    a = rms_input(H.float().cpu().numpy(), w, eps)
    for i, (wt, o) in enumerate(zip(wts, outs)):
        expect(o, dense_tile(wt, dev(a), t16), f16=dtype == torch.float16, what="prefill_rmsnorm tensor %d" % i)
    return a


def check_glu(wt, N, G, U, prefill16, R=None, dtype=torch.float32):
    t16 = takes16(prefill16, N)
    out = nan_out(N, wt.cfg.M, dtype)
    with knobs(prefill16=int(prefill16)):
        tb.prefill_glu(wt, N, G, U, out, R=R, dtype=tdt(dtype))
        assert tb.last_launch()["cluster"] == (16 if t16 else 1)
    torch.cuda.synchronize()
    expect(out, dense_tile(wt, glu_ref(G, U), t16), None if R is None else R.float().cpu().numpy(), dtype == torch.float16, "prefill_glu")


def check_residual(wt, N, B, R, prefill16, dtype=torch.float32):
    t16 = takes16(prefill16, N)
    out = nan_out(N, wt.cfg.M, dtype)
    with knobs(prefill16=int(prefill16)):
        tb.prefill_residual(wt, N, B, R, out, dtype=tdt(dtype))
        assert tb.last_launch()["cluster"] == (16 if t16 else 1)
    torch.cuda.synchronize()
    expect(out, dense_tile(wt, B, t16), R.float().cpu().numpy(), dtype == torch.float16, "prefill_residual")


# ---- 1: every fp grouping, both tiles ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pf16", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("g,ags,bits,zp", TILE_CASES, ids=TILE_CASE_IDS)
def test_groupings(mk, g, ags, bits, zp, pf16):
    """N = 257: a ragged last token tile on either tile.  Two tensors in the norm launch."""
    K, M, N = 1024, 384, 257
    ops = [mk(M, K, bits, g=g, ags=ags, zp=zp, seed=s) for s in (1, 2)]
    rng = np.random.default_rng(g + ags + bits)
    check_norm([o.wt for o in ops], N, dev(act_rows.rows(rng, N, K, ags)), norm_weight(rng, K), pf16)
    check_glu(ops[0].wt, N, dev(act_rows.rows(rng, N, K, ags)), dev(normal(rng, N, K)), pf16, R=dev(normal(rng, N, M)))
    check_residual(ops[1].wt, N, dev(act_rows.rows(rng, N, K, ags)), dev(normal(rng, N, M)), pf16)


# ---- 2: N and count ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pf16", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("N", [1, 3, 63, 64, 257, 300])
def test_rows_and_counts(mk, N, pf16):
    """count = 1, 2 and 3 in the norm launch; the GLU form without a residual; N below, at and past the fp16 tile's 64 and past
    one and two token tiles."""
    K, M = 512, 640
    ops = [mk(M, K, 2, zp=True, seed=10 + s) for s in range(3)]
    rng = np.random.default_rng(N)
    w = norm_weight(rng, K)
    for count in (1, 2, 3):
        check_norm([o.wt for o in ops[:count]], N, dev(normal(rng, N, K)), w, pf16)
    check_glu(ops[0].wt, N, dev(normal(rng, N, K)), dev(normal(rng, N, K)), pf16)
    check_residual(ops[2].wt, N, dev(normal(rng, N, K)), dev(normal(rng, N, M)), pf16)


# ---- 3: fp16, in place, norm edges -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pf16", TILES, ids=TILE_IDS)
def test_fp16_inputs_and_outputs(mk, pf16):
    K, M, N = 1024, 512, 130
    ops = [mk(M, K, bits, zp=bits == 2, seed=20 + bits) for bits in (2, 4)]
    rng = np.random.default_rng(21)
    h16 = lambda *s: torch.from_numpy(act_rows.rows16(rng, s[0], s[1], 64)).cuda().half()
    for op in ops:
        check_norm([op.wt], N, h16(N, K), norm_weight(rng, K), pf16, dtype=torch.float16)
        check_glu(op.wt, N, h16(N, K), h16(N, K), pf16, R=h16(N, M), dtype=torch.float16)
        check_residual(op.wt, N, h16(N, K), h16(N, M), pf16, dtype=torch.float16)


@pytest.mark.parametrize("pf16", TILES, ids=TILE_IDS)
def test_in_place_residual(mk, pf16):
    K, N, M = 1024, 96, 512
    op = mk(M, K, 2, zp=True, seed=30)
    rng = np.random.default_rng(31)
    for dtype in (torch.float32, torch.float16):
        B, G, U, R = (dev(normal(rng, *s), dtype) for s in ((N, K), (N, K), (N, K), (N, M)))
        for call in (lambda out, r: tb.prefill_residual(op.wt, N, B, r, out, dtype=tdt(dtype)),
                     lambda out, r: tb.prefill_glu(op.wt, N, G, U, out, R=r, dtype=tdt(dtype))):
            sep = nan_out(N, M, dtype)
            inplace = R.clone()
            with knobs(prefill16=int(pf16)):
                call(sep, R)
                call(inplace, inplace)
            torch.cuda.synchronize()
            assert same_bits(inplace.cpu().numpy(), sep.cpu().numpy())


@pytest.mark.parametrize("pf16", TILES, ids=TILE_IDS)
def test_norm_order_and_row_edges(mk, pf16):
    """The rows of the GEMV form's norm-order test (a mixed-magnitude row whose inv changes when its sum of squares is re-associated,
    an fp32 row, that row times 2^10, an all-zero row) among 60 normal rows, so that both tiles see them; eps = 0 and 0.5."""
    K, ags, N = 2560, 64, 64
    ops = [mk(512, K, 2, ags=ags, zp=True, seed=s) for s in (40, 41, 42)]
    rng = np.random.default_rng(43)
    fp32, mixed = act_rows.rows(rng, 2, K, ags, kinds=("fp32", "mixed"))
    H = np.concatenate([np.stack([mixed, fp32, fp32 * np.float32(1024.0), np.zeros(K, np.float32)]), normal(rng, N - 4, K)])
    w = norm_weight(rng, K)
    a = check_norm([o.wt for o in ops], N, dev(H), w, pf16)
    assert not np.any(a[3])
    check_norm([ops[0].wt], N - 1, dev(H[[0, 1, 2] + list(range(4, N))]), w, pf16, eps=0.0)   # no zero row: its inv would be inf
    check_norm([ops[0].wt], N, dev(H), w, pf16, eps=0.5)


# ---- 4: graphs ---------------------------------------------------------------------------------------------------------------------
def test_inputs_change_between_graph_replays(stream, mk):
    """The four calls of a layer on buffers rewritten before every replay: each replay equals eager calls on the same inputs."""
    K, F, N = 1024, 2048, 200
    qkv = [mk(K, K, 2, zp=True, seed=50 + s) for s in range(3)]
    o, down = mk(K, K, 2, zp=True, seed=53), mk(K, F, 2, zp=True, seed=54)
    gu = [mk(F, K, 2, zp=True, seed=55 + s) for s in range(2)]
    rng = np.random.default_rng(56)
    w1, w2 = dev(norm_weight(rng, K)), dev(norm_weight(rng, K))
    x, att = nan_out(N, K), nan_out(N, K)
    q = [nan_out(N, K) for _ in range(3)]; h = nan_out(N, K); gg = [nan_out(N, F) for _ in range(2)]; y = nan_out(N, K)
    gen = torch.Generator(device="cuda").manual_seed(57)

    def calls():
        tb.prefill_rmsnorm([t.wt for t in qkv], N, x, w1, EPS, q)
        tb.prefill_residual(o.wt, N, att, x, h)
        tb.prefill_rmsnorm([t.wt for t in gu], N, h, w2, EPS, gg)
        tb.prefill_glu(down.wt, N, gg[0], gg[1], y, R=h)

    def fill():
        x.copy_(torch.randn((N, K), device="cuda", generator=gen))
        att.copy_(torch.randn((N, K), device="cuda", generator=gen))

    fill(); calls(); torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    seen = []
    for _ in range(3):
        fill()
        cg.replay()
        torch.cuda.synchronize()
        replayed = [t.clone() for t in q + [h] + gg + [y]]
        seen.append(x.clone())
        calls()
        torch.cuda.synchronize()
        for a, b in zip(replayed, q + [h] + gg + [y]):
            assert same_bits(a.cpu().numpy(), b.cpu().numpy())
    assert not torch.equal(seen[0], seen[1])


# ---- 5: reporting ------------------------------------------------------------------------------------------------------------------
def test_reports_the_tile_and_rows(mk):
    K, M = 512, 256
    op = mk(M, K, 2, zp=True, seed=60)
    rng = np.random.default_rng(61)
    w = dev(norm_weight(rng, K))
    for N, pf16, want in ((64, 1, 16), (63, 1, 1), (1, 1, 1), (300, 0, 1), (300, 1, 16)):
        _, launch = run_norm([op.wt], N, dev(normal(rng, N, K)), w, EPS, pf16)
        assert launch["cluster"] == want and launch["batch"] == -N, (N, pf16, launch)


# ---- 6: the Llama-2-7B shapes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_llama2_7b_layer_shapes(stream, bits, zp):
    """q/k/v, o, gate/up and down of Llama-2-7B (4096 / 11008) at N = 512, g128: bit for bit the dense tile, and within the
    tile's bound of the gemv_* forms on the same inputs."""
    from decode_harness import QLinear
    H, F, N = 4096, 11008, 512
    shapes = {"q": (H, H), "k": (H, H), "v": (H, H), "o": (H, H), "gate": (F, H), "up": (F, H), "down": (H, F)}
    lin = {n: QLinear(m, k, bits, 128, zp, seed=70 + i) for i, (n, (m, k)) in enumerate(shapes.items())}
    try:
        rng = np.random.default_rng(71)
        w = norm_weight(rng, H)
        x, att, R = dev(normal(rng, N, H)), dev(normal(rng, N, H)), dev(normal(rng, N, H))
        G, U = dev(normal(rng, N, F)), dev(normal(rng, N, F))
        for names, inp in ((("q", "k", "v"), x), (("gate", "up"), x)):
            wts = [lin[n].wt for n in names]
            check_norm(wts, N, inp, w, 1)
            outs, _ = run_norm(wts, N, inp, dev(w), EPS, 1)
            gem = [nan_out(N, wt.cfg.M) for wt in wts]
            tb.gemv_rmsnorm(wts, N, inp, dev(w), EPS, gem)
            torch.cuda.synchronize()
            for a, b in zip(outs, gem):
                assert float((a - b).abs().max()) <= (PF16_TOL + INT8_TOL) * float(b.abs().max())
        check_residual(lin["o"].wt, N, att, R, 1)
        check_glu(lin["down"].wt, N, G, U, 1, R=R)
        for pf, gm, args in ((tb.prefill_residual, tb.gemv_residual, (att, R)), (tb.prefill_glu, tb.gemv_glu, (G, U))):
            wt = lin["o" if pf is tb.prefill_residual else "down"].wt
            a, b = nan_out(N, H), nan_out(N, H)
            pf(wt, N, *args, a); gm(wt, N, *args, b)
            torch.cuda.synchronize()
            assert float((a - b).abs().max()) <= (PF16_TOL + INT8_TOL) * float(b.abs().max())
    finally:
        for l in lin.values():
            l.free()


# ---- 7: rejections -----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    from decode_harness import QLinear
    K, M, N = 1024, 512, 64
    op, other = mk(M, K, 2, zp=True, seed=80), mk(2 * M, K, 2, zp=True, seed=81)
    w1 = mk(M, K, 1, seed=82)
    k64 = mk(M, 1088, 2, g=64, ags=64, zp=True, seed=83)          # K % 128 == 64: a GEMV tensor the tiles do not take
    ip = QLinear(M, K, 2, 128, False, seed=84, one_scale=True)
    try:
        rng = np.random.default_rng(85)
        H, R, w = dev(normal(rng, N, K)), dev(normal(rng, N, M)), dev(norm_weight(rng, K))
        H64 = dev(normal(rng, N, 1088))
        out = nan_out(N, M)
        wbuf = torch.zeros(K + 4, device="cuda")
        lib = tb.load()
        huge = 1 << 25                                            # more than 65535 token tiles of either tile; nothing is read
        bad = {
            "w1 norm": lambda: tb.prefill_rmsnorm([w1.wt], N, H, w, EPS, [out]),
            "w1 glu": lambda: tb.prefill_glu(w1.wt, N, H, H, out),
            "w1 residual": lambda: tb.prefill_residual(w1.wt, N, H, R, out),
            "integer path norm": lambda: tb.prefill_rmsnorm([ip.wt], N, H, w, EPS, [out]),
            "K % 128 glu": lambda: tb.prefill_glu(k64.wt, N, H64, H64, out),
            "K % 128 residual": lambda: tb.prefill_residual(k64.wt, N, H64, R, out),
            "geometry": lambda: tb.prefill_rmsnorm([op.wt, other.wt], N, H, w, EPS, [out, out]),
            "host H": lambda: tb.prefill_rmsnorm([op.wt], N, H.cpu(), w, EPS, [out]),
            "host w": lambda: tb.prefill_rmsnorm([op.wt], N, H, w.cpu(), EPS, [out]),
            "host C": lambda: tb.prefill_rmsnorm([op.wt], N, H, w, EPS, [out.cpu()]),
            "host U": lambda: tb.prefill_glu(op.wt, N, H, H.cpu(), out),
            "host R": lambda: tb.prefill_residual(op.wt, N, H, R.cpu(), out),
            "null w": lambda: tb.prefill_rmsnorm([op.wt], N, H, None, EPS, [out]),
            "unaligned w": lambda: tb.prefill_rmsnorm([op.wt], N, H, wbuf[1:], EPS, [out]),
            "negative eps": lambda: tb.prefill_rmsnorm([op.wt], N, H, w, -1e-5, [out]),
            "nan eps": lambda: tb.prefill_rmsnorm([op.wt], N, H, w, float("nan"), [out]),
            "inf eps": lambda: tb.prefill_rmsnorm([op.wt], N, H, w, float("inf"), [out]),
            "null R": lambda: tb.check(lib.tmac_b200_prefill_residual(op.wt.handle, N, tb.F32, tb.ptr(H), None, tb.ptr(out)), "null R"),
            "null U": lambda: tb.check(lib.tmac_b200_prefill_glu(op.wt.handle, N, tb.F32, tb.ptr(H), None, None, tb.ptr(out)), "null U"),
            "N 0": lambda: tb.prefill_residual(op.wt, 0, H, R, out),
            "token tiles": lambda: tb.prefill_residual(op.wt, huge, H, R, out),
            "token tiles int8": lambda: tb.prefill_rmsnorm([op.wt], huge, H, w, EPS, [out]),
        }
        msgs = {}
        for name, call in bad.items():
            out.fill_(float("nan"))
            torch.cuda.synchronize()
            with knobs(prefill16=0 if name == "token tiles int8" else 1):
                try:
                    call()
                except tb.TMACError as ex:
                    msgs[name] = str(ex)
                else:
                    pytest.fail("'%s' was not rejected" % name)
            torch.cuda.synchronize()
            assert torch.isnan(out).all(), "rejected call '%s' launched" % name
        for name, form in (("w1 norm", "gemv_rmsnorm"), ("w1 glu", "gemv_glu"), ("w1 residual", "gemv_residual"),
                           ("integer path norm", "gemv_rmsnorm"), ("K % 128 glu", "gemv_glu"), ("K % 128 residual", "gemv_residual")):
            assert "use " + form in msgs[name], msgs[name]
        assert "too large" in msgs["token tiles"] and "too large" in msgs["token tiles int8"]
        # an armed peer output makes the call fail, launch nothing and be disarmed
        for call in (lambda: tb.prefill_rmsnorm([op.wt], N, H, w, EPS, [out]), lambda: tb.prefill_glu(op.wt, N, H, H, out),
                     lambda: tb.prefill_residual(op.wt, N, H, R, out)):
            peer = nan_out(1, M)
            out.fill_(float("nan"))
            tb.peer_outputs([peer.data_ptr()])
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all()
            tb.gemv(op.wt, 1, torch.zeros((1, K), device="cuda"), torch.zeros((1, M), device="cuda"))
            torch.cuda.synchronize()
            assert torch.isnan(peer).all(), "the peer output stayed armed"
            call()
    finally:
        ip.free()
