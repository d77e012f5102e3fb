"""GPU suite (-m gpu): the prefill tiles (N >= 32) on W4 and W3 weights.

Both wgmma tiles take the 4-plane stream layout: a 128-row tile is two 64-row super-blocks, one per consumer warpgroup, and the
producers expand a row's four plane codes into the 8 contraction entries S[e] = sum_b 2*alpha_b * sign * [j_b == e] (|S| <= 15;
the padded fourth plane of W3 weighs 0).  int8 tile (tmac_prefill.cuh): exact integer sums -> TIGHT_TOL.  fp16 tile
(tmac_prefill16.cuh): A = fp16(S * fp16(0.5 * scale)) -> P16_TOL, as for W2."""
import ctypes as C

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TIGHT_TOL = 2e-5    # int8 tile: the GEMV's integer sums, fp32 re-association only
P16_TOL = 5e-4      # fp16 tile: operands rounded to fp16, fp32 accumulation over K
CLUSTER = {"int8": 1, "fp16": 16}   # last_launch()["cluster"] marks which tile served the call


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; libtmac_b200 has no CPU fallback")
    lib = tb.load()
    tb.check(lib.tmac_b200_init(0), "init")
    st = torch.cuda.Stream()               # torch fills and library launches on one stream
    torch.cuda.set_stream(st)
    tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")
    yield lib
    torch.cuda.synchronize()
    tb.check(lib.tmac_b200_set_stream(None), "set_stream")


def kc(cfg):
    return tb.make_kcfg(cfg.Mout, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale)


def not_fp16(v):
    """Scales / zero points that fp16 cannot hold: the stream layout keeps them as fp32 (4 bytes each)."""
    return None if v is None else (v * np.float32(1 + 2 ** -13)).astype(np.float32)


def assert_tile(tile, N):
    ll = tb.last_launch()
    assert ll["batch"] == -N and ll["planes_per_word"] == 4 and ll["cluster"] == CLUSTER[tile], "expected the %s tile, got %r" % (tile, ll)


CASES = [(T.Config(256, 1024, 4, zero_point=True), 64, False),
         (T.Config(384, 2048, 4), 130, False),                    # ragged token tile
         (T.Config(192, 512, 4, zero_point=True), 300, False),    # 3 super-blocks: the last tile has no second one
         (T.Config(384, 1024, 3, zero_point=True), 96, False),
         (T.Config(320, 1024, 4, zero_point=True), 96, True),     # fp32 scales and zero points, 5 super-blocks
         (T.Config(384, 1024, 3), 64, True)]


@pytest.mark.parametrize("tile", ["int8", "fp16"])
@pytest.mark.parametrize("cfg,N,fp32_scales", CASES, ids=["w4zp_n64", "w4sym_n130", "w4zp_odd_n300", "w3zp_n96", "w4zp_f32s_n96", "w3sym_f32s_n64"])
def test_prefill_w34_tiles_match_oracle(lib, oracle, cfg, N, fp32_scales, tile):
    cfg = cfg.resolved()
    tol = TIGHT_TOL if tile == "int8" else P16_TOL
    w, sc, z, x = T.make_problem(cfg, seed=31, N=N)
    if fp32_scales:
        sc, z = not_fp16(sc), not_fp16(z)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if tile == "int8" else 1)
        tb.debug_set("prefill_min_n", 32)              # these few row tiles take the tile from N = 128 by default (tile_min_n)
        dx = torch.from_numpy(x).cuda()
        nag = cfg.K // cfg.act_group_size
        q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
        ls = torch.zeros((N, nag), device="cuda"); lb = torch.zeros_like(ls)
        out = torch.zeros((N, cfg.Mout), device="cuda")
        tb.preprocessor(cfg.K, N, cfg.act_group_size, dx, ls, lb, q)
        tb.qgemm_lut(wt, N, q, ls, lb, out)
        assert_tile(tile, N)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = out.cpu().numpy()
        assert np.abs(got - Co).max() <= tol * np.abs(Co).max()
        assert T.nmse(T.dense_reference(w, sc, z, x, cfg), got) <= 5e-4
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2)                       # the one-call form takes the same tile: bit-identical
        assert_tile(tile, N)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        tb.debug_set("prefill", 0)                     # tiles disabled: the GEMV kernel per activation row
        out3 = torch.zeros_like(out)
        tb.qgemm_lut(wt, N, q, ls, lb, out3)
        assert tb.last_launch()["batch"] >= 0, "the tile was supposed to be disabled"
        torch.cuda.synchronize()
        assert np.abs(out3.cpu().numpy() - got).max() <= (tol + TIGHT_TOL) * np.abs(Co).max()
    finally:
        tb.debug_set("prefill", 1); tb.debug_set("prefill16", 1); tb.debug_set("prefill_min_n", 0)
        wt.free()


@pytest.mark.parametrize("tile", ["int8", "fp16"])
def test_prefill_w4_fp16_activations_and_outputs(lib, oracle, tile):
    """fp16 activations in, fp16 C out: the tile's epilogue rounds its fp32 result once."""
    cfg = T.Config(256, 2048, 4, zero_point=True).resolved()
    N = 80
    w, sc, z, x = T.make_problem(cfg, seed=37, N=N)         # x is fp16-representable
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if tile == "int8" else 1)
        tb.debug_set("prefill_min_n", 32)
        dx = torch.from_numpy(x).cuda().half()
        nag = cfg.K // cfg.act_group_size
        q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
        ls = torch.zeros((N, nag), device="cuda"); lb = torch.zeros_like(ls)
        out = torch.zeros((N, cfg.Mout), dtype=torch.float16, device="cuda")
        tb.preprocessor(cfg.K, N, cfg.act_group_size, dx, ls, lb, q, dtype=tb.F16)
        tb.qgemm_lut(wt, N, q, ls, lb, out, dtype=tb.F16)
        assert_tile(tile, N)
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2, dtype=tb.F16)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = out.float().cpu().numpy()
        tol = (TIGHT_TOL if tile == "int8" else P16_TOL) + 2 ** -11     # + one fp16 rounding of the output
        assert np.abs(got - Co).max() <= tol * np.abs(Co).max()
    finally:
        tb.debug_set("prefill16", 1); tb.debug_set("prefill_min_n", 0)
        wt.free()


def test_prefill_w4_reference_dispatcher(lib, oracle):
    """preprocessor_int8 / qgemm_lut_int8 with a registered kcfg reach the whole-tensor launch, so W4 prefill takes the tile."""
    cfg = T.Config(512, 2048, 4, zero_point=True).resolved()
    N = 128                                                  # the automatic threshold of a tensor this small
    w, sc, z, x = T.make_problem(cfg, seed=41, N=N)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    k = kc(cfg)
    wt = tb.upload_reference_layout(k, A, S)                # the load-time registration of these reference buffers
    try:
        nag = cfg.K // cfg.act_group_size
        dx = torch.from_numpy(x).cuda()
        dq = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
        dls = torch.zeros((N, nag), device="cuda"); dlb = torch.zeros_like(dls)
        dC = torch.zeros((N, cfg.Mout), device="cuda")
        tb.check(lib.tmac_b200_register_kcfg(C.byref(k)), "register")
        tb.check(lib.preprocessor_int8(cfg.Mout * cfg.bits, cfg.K, N, cfg.bits, dx.data_ptr(), dls.data_ptr(), dlb.data_ptr(), dq.data_ptr()), "preprocessor_int8")
        tb.check(lib.qgemm_lut_int8(cfg.Mout * cfg.bits, cfg.K, N, cfg.bits, A.ctypes.data, dq.data_ptr(), S.ctypes.data, dls.data_ptr(), dlb.data_ptr(), dC.data_ptr()), "qgemm_lut_int8")
        assert_tile("fp16", N)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = dC.cpu().numpy()
        assert np.abs(got - Co).max() <= P16_TOL * np.abs(Co).max()
        assert T.nmse(T.dense_reference(w, sc, z, x, cfg), got) <= 5e-4
    finally:
        wt.free()


@pytest.mark.parametrize("shape,mode", [((4096, 4096, False, 256), "fp16_tile_per_cta"), ((4096, 4096, False, 256), "int8"),
                                        ((11008, 4096, True, 256), "fp16_tile_per_cta"), ((11008, 4096, True, 256), "fp16_streamk"),
                                        ((3584, 18944, True, 128), "fp16_tile_per_cta")],
                         ids=["llama4096_sym_fp16", "llama4096_sym_int8", "11008x4096_zp_fp16", "11008x4096_zp_streamk", "qwen2_3584x18944_zp_fp16"])
def test_prefill_w4_full_size(lib, oracle, shape, mode):
    """Llama-2-7B / Qwen2-7B W4 g128 layer shapes at full size: every row of 8 sampled tokens against the oracle; run twice and
    bit-identical (stream-K: partial tiles summed in a fixed order, flags clean for the next launch)."""
    Mout, K, zp, N = shape
    cfg = T.Config(Mout, K, 4, zero_point=zp).resolved()
    w, sc, z, x = T.make_problem(cfg, seed=43, N=N)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if mode == "int8" else 1)
        tb.debug_set("pf_streamk", 1 if mode == "fp16_streamk" else 0)
        dx = torch.from_numpy(x).cuda()
        out = torch.zeros((N, cfg.Mout), device="cuda"); out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out)
        assert_tile("int8" if mode == "int8" else "fp16", N)
        if mode.startswith("fp16"):
            assert tb.last_launch()["min_blocks"] == (1 if mode == "fp16_streamk" else 0)
        tb.gemv(wt, N, dx, out2)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        toks = [0, 1, 63, 64, 127, N // 2 + 3, N - 2, N - 1]
        qo, lso, lbo = oracle.preprocessor(x[toks], cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        tol = TIGHT_TOL if mode == "int8" else P16_TOL
        assert np.abs(out.cpu().numpy()[toks] - Co).max() <= tol * np.abs(Co).max()
    finally:
        tb.debug_set("prefill16", 1); tb.debug_set("pf_streamk", 0)
        wt.free()


@pytest.mark.parametrize("cfg,N", [(T.Config(512, 1024, 1), 64),
                                   (T.Config(256, 1024, 4, kfactor=8, group_size=32, act_group_size=32), 64),
                                   (T.Config(320, 1280, 2, one_scale=True), 64),
                                   (T.Config(256, 1024, 4, zero_point=True), 16),
                                   (T.Config(1024, 1024, 4, zero_point=True), 96)],
                         ids=["w1", "w4_act32", "bitnet_one_scale", "w4_n16", "w4_few_row_tiles_n96"])
def test_prefill_routing_keeps_gemv_outside_the_tiles(lib, oracle, cfg, N):
    """Shapes the tiles do not cover keep the GEMV kernel per activation row (batch >= 0), and stay exact.  A W4 tensor of fewer
    than 64 row tiles takes the tiles from N = 128 only (below that the GEMV is faster there)."""
    cfg = cfg.resolved()
    w, sc, z, x = T.make_problem(cfg, seed=47, N=N)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        dx = torch.from_numpy(x).cuda()
        nag = cfg.K // cfg.act_group_size
        q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
        ls = torch.zeros((N, nag), device="cuda"); lb = torch.zeros_like(ls)
        out = torch.zeros((N, cfg.Mout), device="cuda")
        tb.preprocessor(cfg.K, N, cfg.act_group_size, dx, ls, lb, q)
        tb.qgemm_lut(wt, N, q, ls, lb, out)
        assert tb.last_launch()["batch"] >= 0, tb.last_launch()
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2)
        assert tb.last_launch()["batch"] >= 0, tb.last_launch()
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = out.cpu().numpy()
        if cfg.one_scale:
            assert np.array_equal(got.view(np.uint32), Co.view(np.uint32))
        else:
            assert np.abs(got - Co).max() <= TIGHT_TOL * np.abs(Co).max()
        assert torch.equal(out, out2)
    finally:
        wt.free()
