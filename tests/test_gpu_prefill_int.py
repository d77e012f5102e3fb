"""GPU suite (-m gpu): the int8 prefill tile on the integer path (BitNet: one weight scale, one activation group per row).

The tile sums the exact int32 contraction S . T8 over the whole K and applies the token's LUT scale and bias and the tensor's scale
in one epilogue, in the GEMV's order: its output is the GEMV's and the reference's, bit for bit.  The fp16 tile is never taken here
(it is not exact)."""
import ctypes as C

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


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


def int_tile_min_n(mout):
    """The integer path's automatic threshold (DESIGN.md 3.3): 128 below 64 row tiles of 128 rows, else 64."""
    return 128 if (mout + 127) // 128 < 64 else 64


def assert_int8_tile(N):
    ll = tb.last_launch()
    assert ll["batch"] == -N and ll["cluster"] == 1, "expected the int8 tile, got %r" % ll


def bit_exact(got, Co):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(Co).view(np.uint32))


def problem(cfg, seed, N, full_range=False):
    """make_problem draws ternary codes for one-scale tensors; full_range draws every code of the bit width instead."""
    w, sc, z, x = T.make_problem(cfg, seed=seed, N=N)
    if full_range:
        w = np.random.default_rng(seed + 1).integers(0, 1 << cfg.bits, size=w.shape, dtype=np.uint8)
    return w, sc, z, x


def lut(cfg, N, dx, dtype=tb.F32):
    q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
    ls = torch.zeros((N, 1), device="cuda"); lb = torch.zeros_like(ls)      # [N][1]: one activation group per row
    tb.preprocessor(cfg.K, N, cfg.act_group_size, dx, ls, lb, q, dtype=dtype)
    return q, ls, lb


def check_three_ways(oracle, cfg, w, sc, x, N):
    """preprocessor + qgemm_lut on the tile, bit-exact against the oracle; gemv on the tile, equal; the GEMV per row, equal."""
    A, S = T.pack_reference_layout(w, sc, None, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, None)
    try:
        dx = torch.from_numpy(x).cuda()
        q, ls, lb = lut(cfg, N, dx)
        out = torch.zeros((N, cfg.Mout), device="cuda")
        tb.qgemm_lut(wt, N, q, ls, lb, out)
        assert_int8_tile(N)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert bit_exact(out.cpu().numpy(), Co), "integer-path tile must be bit exact"
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2)                       # the one-call form: preprocessor + the same tile
        assert_int8_tile(N)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        tb.debug_set("prefill", 0)                     # tiles disabled: the GEMV kernel per activation row
        out3 = torch.zeros_like(out)
        tb.qgemm_lut(wt, N, q, ls, lb, out3)
        assert tb.last_launch()["batch"] >= 0, "the tile was supposed to be disabled"
        torch.cuda.synchronize()
        assert torch.equal(out, out3)
    finally:
        tb.debug_set("prefill", 1)
        wt.free()


@pytest.fixture(autouse=True)
def default_knobs():
    yield
    tb.debug_set("prefill", 1); tb.debug_set("prefill16", 1); tb.debug_set("prefill_min_n", 0)


CASES = [(T.Config(640, 3200, 2, one_scale=True), 64, False),       # QCH 8
         (T.Config(384, 8640, 2, one_scale=True), 130, False),      # QCH 4 (K = 8640 is not a multiple of 128), ragged token tile
         (T.Config(320, 1280, 2, one_scale=True), 96, False),       # 320 rows: the last row tile holds 64
         (T.Config(384, 1024, 4, one_scale=True), 96, True),        # W4, every code
         (T.Config(192, 1024, 3, one_scale=True), 64, True)]        # W3, 3 super-blocks: the last tile has no second one


@pytest.mark.parametrize("cfg,N,full_range", CASES, ids=["w2_qch8_n64", "w2_qch4_n130", "w2_ragged_rows_n96", "w4_n96", "w3_odd_sb_n64"])
def test_int_tile_matches_oracle_bit_exact(lib, oracle, cfg, N, full_range):
    cfg = cfg.resolved()
    w, sc, _, x = problem(cfg, 61, N, full_range)
    tb.debug_set("prefill_min_n", 32)                 # these few row tiles take the tile from N = 128 by default
    check_three_ways(oracle, cfg, w, sc, x, N)


def test_int_path_never_takes_the_fp16_tile(lib, oracle):
    """prefill16 = 1 serves the fp path's N >= 64 with the fp16 tile; the integer path keeps the exact int8 tile."""
    cfg = T.Config(256, 2048, 4, one_scale=True).resolved()
    N = 128
    w, sc, _, x = problem(cfg, 67, N, full_range=True)
    tb.debug_set("prefill16", 1)
    tb.debug_set("prefill_min_n", 32)
    check_three_ways(oracle, cfg, w, sc, x, N)


def test_int_tile_row_edge_cases(lib, oracle):
    """Rows with different maxima, an all-zero row (scale 0 -> table 0 -> output 0) and a row scaled by 32."""
    cfg = T.Config(512, 3200, 2, one_scale=True).resolved()
    N = 64
    w, sc, _, x = problem(cfg, 71, N)
    x[1] *= 32.0
    x[2] = 0.0
    x[5] *= 0.25
    x[9, : cfg.K // 2] = 0.0
    tb.debug_set("prefill_min_n", 32)
    check_three_ways(oracle, cfg, w, sc, x, N)


def test_int_tile_fp16_activations_and_outputs(lib, oracle):
    """fp16 activations in, fp16 C out: the epilogue's fp32 result is rounded once at the store."""
    cfg = T.Config(640, 8640, 2, one_scale=True).resolved()
    N = 80
    w, sc, _, x = problem(cfg, 73, N)                  # x is fp16-representable
    A, S = T.pack_reference_layout(w, sc, None, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, None)
    try:
        tb.debug_set("prefill_min_n", 32)
        dx = torch.from_numpy(x).cuda().half()
        q, ls, lb = lut(cfg, N, dx, dtype=tb.F16)
        out = torch.zeros((N, cfg.Mout), dtype=torch.float16, device="cuda")
        tb.qgemm_lut(wt, N, q, ls, lb, out, dtype=tb.F16)
        assert_int8_tile(N)
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2, dtype=tb.F16)
        assert_int8_tile(N)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert np.array_equal(out.cpu().numpy(), Co.astype(np.float16))
        assert torch.equal(out, out2)
    finally:
        wt.free()


def test_int_tile_reference_dispatcher(lib, oracle):
    """preprocessor_int8 / qgemm_lut_int8 with a registered BitNet kcfg reach the whole-tensor launch and take the tile."""
    cfg = T.Config(640, 3200, 2, one_scale=True).resolved()
    N = int_tile_min_n(cfg.Mout)                       # the automatic threshold of this tensor
    w, sc, _, x = problem(cfg, 79, N)
    A, S = T.pack_reference_layout(w, sc, None, cfg)
    k = kc(cfg)
    wt = tb.upload_reference_layout(k, A, S)
    try:
        dx = torch.from_numpy(x).cuda()
        dq = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
        dls = torch.zeros((N, 1), device="cuda"); dlb = torch.zeros_like(dls)
        dC = torch.zeros((N, cfg.Mout), device="cuda")
        tb.check(lib.tmac_b200_register_kcfg(C.byref(k)), "register")
        tb.check(lib.preprocessor_int8(cfg.Mout * cfg.bits, cfg.K, N, cfg.bits, dx.data_ptr(), dls.data_ptr(), dlb.data_ptr(), dq.data_ptr()), "preprocessor_int8")
        tb.check(lib.qgemm_lut_int8(cfg.Mout * cfg.bits, cfg.K, N, cfg.bits, A.ctypes.data, dq.data_ptr(), S.ctypes.data, dls.data_ptr(), dlb.data_ptr(), dC.data_ptr()), "qgemm_lut_int8")
        assert_int8_tile(N)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert bit_exact(dC.cpu().numpy(), Co)
    finally:
        wt.free()


BITNET_3B = [(3200, 3200), (8640, 3200), (3200, 8640)]


@pytest.mark.parametrize("mout,k", BITNET_3B, ids=["%dx%d" % s for s in BITNET_3B])
def test_int_tile_bitnet_3b_full_size(lib, oracle, mout, k):
    """BitNet-3B layer shapes at N = 256 through tmac_b200_gemv with the automatic threshold: 8 sampled tokens bit-exact against
    the oracle, every token equal to the GEMV per row, two runs equal; the route agrees with the rule in DESIGN.md 3.3."""
    cfg = T.Config(mout, k, 2, one_scale=True).resolved()
    N = 256
    w, sc, _, x = problem(cfg, 83, N)
    A, S = T.pack_reference_layout(w, sc, None, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, None)
    try:
        dx = torch.from_numpy(x).cuda()
        out = torch.zeros((N, cfg.Mout), device="cuda"); out2 = torch.zeros_like(out); gemv = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out)
        on_tile = tb.last_launch()["batch"] == -N
        assert on_tile == (N >= int_tile_min_n(mout)), tb.last_launch()
        if on_tile:
            assert_int8_tile(N)
        tb.gemv(wt, N, dx, out2)
        tb.debug_set("prefill", 0)
        tb.gemv(wt, N, dx, gemv)
        assert tb.last_launch()["batch"] >= 0
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        assert torch.equal(out, gemv)
        toks = [0, 1, 63, 64, 127, N // 2 + 3, N - 2, N - 1]
        qo, lso, lbo = oracle.preprocessor(x[toks], cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert bit_exact(out.cpu().numpy()[toks], Co)
    finally:
        wt.free()


@pytest.mark.parametrize("cfg,N,w1", [(T.Config(256, 96, 2, kfactor=8, one_scale=True), 64, False),
                                      (T.Config(512, 1024, 1, one_scale=True), 64, True)],
                         ids=["k96_qch2", "w1"])
def test_int_path_outside_the_tile_keeps_the_gemv(lib, oracle, cfg, N, w1):
    """32-wide chunks (K not a multiple of 64) and W1 streams keep the GEMV kernel per activation row (batch >= 0), bit-exact."""
    cfg = cfg.resolved()
    w, sc, _, x = problem(cfg, 89, N)
    if w1:
        w = np.random.default_rng(90).integers(0, 2, size=w.shape, dtype=np.uint8)   # ternary codes do not fit one bit
    A, S = T.pack_reference_layout(w, sc, None, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, None)
    try:
        tb.debug_set("prefill_min_n", 32)
        dx = torch.from_numpy(x).cuda()
        q, ls, lb = lut(cfg, N, dx)
        out = torch.zeros((N, cfg.Mout), device="cuda"); out2 = torch.zeros_like(out)
        tb.qgemm_lut(wt, N, q, ls, lb, out)
        assert tb.last_launch()["batch"] >= 0, tb.last_launch()
        tb.gemv(wt, N, dx, out2)
        assert tb.last_launch()["batch"] >= 0, tb.last_launch()
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert bit_exact(out.cpu().numpy(), Co)
        assert torch.equal(out, out2)
    finally:
        wt.free()
