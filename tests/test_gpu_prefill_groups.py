"""GPU suite (-m gpu): the prefill tiles on every fp-path grouping besides chunk 128 / act group 64.

Both wgmma tiles take chunks ck of 128, 64 or 32 K and activation groups ags of 128, 64 or 32 K (ags <= ck, K % 128 == 0): the
producers stage a 128-K window of 128 / ck chunk blocks, the int8 tile folds its int32 accumulator once per activation group and
adds the bias / zero-point term once per chunk, the fp16 tile gives each A entry its own chunk's scale and each B entry its own
activation group's LUT scale.  ggml Q4_0 and GPTQ g32 tensors are (32, 32).  int8 tile: the GEMV's integer sums -> TIGHT_TOL;
fp16 tile: operands rounded to fp16 -> P16_TOL."""
import ctypes as C
import os

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


@pytest.fixture(autouse=True)
def default_knobs():
    yield
    tb.debug_set("prefill", 1); tb.debug_set("prefill16", 1); tb.debug_set("prefill_min_n", 0); tb.debug_set("pf_streamk", 0)


def kc(cfg):
    return tb.make_kcfg(cfg.Mout, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale)


def config(mout, k, bits, ck, ags, zp):
    """The reference's kfactor is ags / 4 for these groupings (16 for ags 64)."""
    return T.Config(mout, k, bits, kfactor=ags // 4, group_size=ck, act_group_size=ags, zero_point=zp).resolved()


def not_fp16(v):
    """Scales / zero points that fp16 cannot hold: the stream layout keeps them as fp32 (4 bytes each)."""
    return None if v is None else (v * np.float32(1 + 2 ** -13)).astype(np.float32)


def fp_tile_min_n(bits, mout, ck):
    """The fp path's automatic threshold (DESIGN.md 3.3): 32, but for a W3/W4 tensor of fewer than 64 row tiles 128, or 64 with a
    32-K chunk and at least 32 row tiles."""
    nrt = (mout + 127) // 128
    if bits >= 3 and nrt < 64:
        return 64 if ck == 32 and nrt >= 32 else 128
    return 32


def assert_tile(tile, N, bits):
    ll = tb.last_launch()
    assert ll["batch"] == -N and ll["cluster"] == CLUSTER[tile] and ll["planes_per_word"] == (2 if bits == 2 else 4), \
        "expected the %s tile, got %r" % (tile, ll)


def lut(cfg, N, dx, dtype=tb.F32):
    nag = cfg.K // cfg.act_group_size
    q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
    ls = torch.zeros((N, nag), device="cuda"); lb = torch.zeros_like(ls)
    tb.preprocessor(cfg.K, N, cfg.act_group_size, dx, ls, lb, q, dtype=dtype)
    return q, ls, lb


def check_tile(oracle, cfg, w, sc, z, x, N, tile):
    """preprocessor + qgemm_lut on the tile against the oracle; gemv on the same tile, bit for bit; the GEMV per row (prefill = 0)
    within tolerance of the tile."""
    tol = TIGHT_TOL if tile == "int8" else P16_TOL
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if tile == "int8" else 1)
        tb.debug_set("prefill_min_n", 32)              # small tensors: below the automatic threshold of W3/W4
        dx = torch.from_numpy(x).cuda()
        q, ls, lb = lut(cfg, N, dx)
        out = torch.zeros((N, cfg.Mout), device="cuda")
        tb.qgemm_lut(wt, N, q, ls, lb, out)
        assert_tile(tile, N, cfg.bits)
        torch.cuda.synchronize()
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = out.cpu().numpy()
        assert np.abs(got - Co).max() <= tol * np.abs(Co).max()
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2)                       # the one-call form takes the same tile: bit-identical
        assert_tile(tile, N, cfg.bits)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        tb.debug_set("prefill", 0)                     # tiles disabled: the GEMV kernel per activation row
        out3 = torch.zeros_like(out)
        tb.qgemm_lut(wt, N, q, ls, lb, out3)
        assert tb.last_launch()["batch"] >= 0, "the tile was supposed to be disabled"
        torch.cuda.synchronize()
        assert np.abs(out3.cpu().numpy() - got).max() <= (tol + TIGHT_TOL) * np.abs(Co).max()
    finally:
        tb.debug_set("prefill", 1)
        wt.free()


# (ck, ags): the five groupings besides (128, 64).  Shapes: W2 320 rows (the last row tile holds 64), W3/W4 192 or 320 rows (3 or
# 5 super-blocks: the last tile has no second one); ragged token counts; zero points in about half the cases.
GROUPINGS = [(32, 32), (64, 64), (64, 32), (128, 32), (128, 128)]
CASES = []
for _i, (_ck, _ags) in enumerate(GROUPINGS):
    for _j, _bits in enumerate((2, 4, 3) if _ck == 32 else (2, 4)):
        _mout = 320 if _bits == 2 else (192, 320)[_i % 2]
        _k = (1024, 1536)[(_i + _j) % 2]
        CASES.append(pytest.param(_mout, _k, _bits, _ck, _ags, (_i + _j) % 2 == 0, (96, 130, 300)[(_i + _j) % 3],
                                  id="w%d_g%d_a%d_%dx%d_n%d" % (_bits, _ck, _ags, _mout, _k, (96, 130, 300)[(_i + _j) % 3])))


@pytest.mark.parametrize("tile", ["int8", "fp16"])
@pytest.mark.parametrize("mout,k,bits,ck,ags,zp,N", CASES)
def test_grouping_tiles_match_oracle(lib, oracle, mout, k, bits, ck, ags, zp, N, tile):
    cfg = config(mout, k, bits, ck, ags, zp)
    w, sc, z, x = T.make_problem(cfg, seed=101 + ck + ags + bits, N=N)
    check_tile(oracle, cfg, w, sc, z, x, N, tile)


@pytest.mark.parametrize("tile", ["int8", "fp16"])
@pytest.mark.parametrize("ck,ags,bits", [(32, 32, 4), (64, 64, 2)], ids=["w4_g32_a32", "w2_g64_a64"])
def test_grouping_tiles_fp32_scales(lib, oracle, ck, ags, bits, tile):
    """Scales and zero points that are not fp16-exact: 4-byte scales, whose offsets in a block depend on both the chunk and sd."""
    cfg = config(320, 1024, bits, ck, ags, True)
    N = 96
    w, sc, z, x = T.make_problem(cfg, seed=113 + ck, N=N)
    check_tile(oracle, cfg, w, not_fp16(sc), not_fp16(z), x, N, tile)


def test_q4_0_through_the_hook_takes_the_tile(lib, oracle, golden_dir):
    """A ggml Q4_0 tensor (golden blocks from the reference's gguf-py) through ggml_tmac_b200_transform_tensor_typed, then
    preprocessor_int8 + qgemm_lut_int8 on host buffers for N = 64 tokens: the whole-tensor call takes a tile."""
    z = np.load(os.path.join(golden_dir, "ggml_blocks.npz"))
    q, deq, qt = np.ascontiguousarray(z["q4_0_bytes"]), z["q4_0_dequant"], int(z["q4_0_type"])
    rows, K = deq.shape
    bits, N = 4, 64
    cfg = config(rows, K, bits, 32, 32, False)
    k = kc(cfg)
    tb.check(lib.tmac_b200_register_kcfg(C.byref(k)), "register")
    extra = tb.TensorExtra()
    h = lib.ggml_tmac_b200_transform_tensor_typed(q.ctypes.data, qt, K, rows, C.byref(extra))
    tb.check(h, "transform_tensor_typed")
    try:
        tb.debug_set("prefill_min_n", 32)
        w = np.zeros((rows, K), np.uint8); sc = np.zeros((rows, K // 32), np.float32)
        assert lib.tmac_b200_debug_decode_ggml(qt, q.ctypes.data, K, rows, w.ctypes.data, sc.ctypes.data) == 32
        A, S = T.pack_reference_layout(w, sc, None, cfg)
        x = np.random.default_rng(7).standard_normal((N, K)).astype(np.float16).astype(np.float32)
        nag = K // 32
        ql = np.zeros((N, K // 4, 16), np.int8); ls = np.zeros((N, nag), np.float32); lb = np.zeros_like(ls)
        out = np.zeros((N, rows), np.float32)
        tb.check(lib.preprocessor_int8(rows * bits, K, N, bits, x.ctypes.data, ls.ctypes.data, lb.ctypes.data, ql.ctypes.data), "preprocessor_int8")
        tb.check(lib.qgemm_lut_int8(rows * bits, K, N, bits, extra.qweights, ql.ctypes.data, extra.scales, ls.ctypes.data, lb.ctypes.data,
                                    out.ctypes.data), "qgemm_lut_int8")
        ll = tb.last_launch()
        assert ll["batch"] == -N and ll["cluster"] in (1, 16) and ll["planes_per_word"] == 4, ll
        tol = TIGHT_TOL if ll["cluster"] == 1 else P16_TOL
        qo, lso, lbo = oracle.preprocessor(x, 32)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        assert np.abs(out - Co).max() <= tol * np.abs(Co).max()
        assert T.nmse(x @ deq.T, out) <= 5e-4               # the reference's dequantised weights
    finally:
        lib.tmac_b200_free_weights(h)


FULL = [(11008, 4096), (4096, 11008)]


@pytest.mark.parametrize("mode", ["fp16", "fp16_streamk", "int8"])
@pytest.mark.parametrize("mout,k", FULL, ids=["%dx%d" % s for s in FULL])
def test_q4_0_style_full_size(lib, oracle, mout, k, mode):
    """W4 g32 / a32 (Q4_0's grouping) at Llama-2-7B sizes, N = 256, through tmac_b200_gemv with the automatic threshold: the route
    follows the rule in DESIGN.md 3.3, every row of 8 sampled tokens against the oracle, two runs bit-identical."""
    cfg = config(mout, k, 4, 32, 32, False)
    N = 256
    w, sc, z, x = T.make_problem(cfg, seed=127, N=N)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if mode == "int8" else 1)
        tb.debug_set("pf_streamk", 1 if mode == "fp16_streamk" else 0)
        dx = torch.from_numpy(x).cuda()
        out = torch.zeros((N, cfg.Mout), device="cuda"); out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out)
        on_tile = tb.last_launch()["batch"] == -N
        assert on_tile == (N >= fp_tile_min_n(4, mout, 32)), tb.last_launch()
        tile = "int8" if mode == "int8" else "fp16"
        if on_tile:
            assert_tile(tile, N, 4)
            if tile == "fp16":
                assert tb.last_launch()["min_blocks"] == (1 if mode == "fp16_streamk" else 0)
        tb.gemv(wt, N, dx, out2)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        toks = [0, 1, 63, 64, 127, N // 2 + 3, N - 2, N - 1]
        qo, lso, lbo = oracle.preprocessor(x[toks], cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        tol = (TIGHT_TOL if tile == "int8" else P16_TOL) if on_tile else TIGHT_TOL
        assert np.abs(out.cpu().numpy()[toks] - Co).max() <= tol * np.abs(Co).max()
    finally:
        wt.free()


@pytest.mark.parametrize("N", [48, 64])
def test_q4_0_style_threshold_at_32_row_tiles(lib, N):
    """W4 g32 / a32 at 4096 x 4096 (32 row tiles) takes the tiles from N = 64 (DESIGN.md 3.3) and agrees with the GEMV per row."""
    cfg = config(4096, 4096, 4, 32, 32, False)
    w, sc, z, x = T.make_problem(cfg, seed=139, N=N)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        dx = torch.from_numpy(x).cuda()
        out = torch.zeros((N, cfg.Mout), device="cuda"); gemv = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out)
        assert (tb.last_launch()["batch"] == -N) == (N >= fp_tile_min_n(4, 4096, 32)), tb.last_launch()
        tb.debug_set("prefill", 0)
        tb.gemv(wt, N, dx, gemv)
        torch.cuda.synchronize()
        ref = gemv.cpu().numpy()
        assert np.abs(out.cpu().numpy() - ref).max() <= (P16_TOL + TIGHT_TOL) * np.abs(ref).max()
    finally:
        wt.free()


@pytest.mark.parametrize("tile,ck,ags,bits", [("int8", 64, 32, 2), ("fp16", 128, 128, 4)], ids=["int8_w2_g64_a32", "fp16_w4_g128_a128"])
def test_grouping_fp16_activations_and_outputs(lib, oracle, tile, ck, ags, bits):
    """fp16 activations in, fp16 C out: the tile's epilogue rounds its fp32 result once."""
    cfg = config(320, 1024, bits, ck, ags, True)
    N = 80
    w, sc, z, x = T.make_problem(cfg, seed=131, N=N)         # x is fp16-representable
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    try:
        tb.debug_set("prefill16", 0 if tile == "int8" else 1)
        tb.debug_set("prefill_min_n", 32)
        dx = torch.from_numpy(x).cuda().half()
        q, ls, lb = lut(cfg, N, dx, dtype=tb.F16)
        out = torch.zeros((N, cfg.Mout), dtype=torch.float16, device="cuda")
        tb.qgemm_lut(wt, N, q, ls, lb, out, dtype=tb.F16)
        assert_tile(tile, N, bits)
        out2 = torch.zeros_like(out)
        tb.gemv(wt, N, dx, out2, dtype=tb.F16)
        assert_tile(tile, N, bits)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
        Co = oracle.qgemm(cfg, A, S, qo, lso, lbo)
        got = out.float().cpu().numpy()
        tol = (TIGHT_TOL if tile == "int8" else P16_TOL) + 2 ** -11     # + one fp16 rounding of the output
        assert np.abs(got - Co).max() <= tol * np.abs(Co).max()
    finally:
        wt.free()


@pytest.mark.parametrize("cfg,N", [(T.Config(256, 1056, 4, kfactor=8, group_size=32, act_group_size=32), 64),
                                   (T.Config(512, 1024, 1, group_size=64, act_group_size=64, zero_point=True), 64)],
                         ids=["w4_g32_k1056", "w1_g64"])
def test_groupings_outside_the_tiles_keep_the_gemv(lib, oracle, cfg, N):
    """A g32 tensor whose K is not a multiple of 128 and a W1 g64 tensor keep the GEMV kernel per activation row (batch >= 0)."""
    cfg = cfg.resolved()
    w, sc, z, x = T.make_problem(cfg, seed=137, N=N)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
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
        assert np.abs(out.cpu().numpy() - Co).max() <= TIGHT_TOL * np.abs(Co).max()
        assert torch.equal(out, out2)
    finally:
        wt.free()
