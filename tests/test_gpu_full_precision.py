"""GPU suite (-m gpu): the bit-exact gates on full-precision fp32 activations and at activation-value edges.

The rest of the suite draws fp16-rounded activations, whose short fp32 sums are almost all exact: there a kernel that built its LUT
in another order than the reference's (DESIGN.md section 1) would still give the oracle's bytes, scales and biases.  Here every row
comes from tests/act_rows.py -- fp32, mixed-magnitude, zero / -0.0 groups, outliers, round-half-even ties, and an fp16 variant with
subnormals, values near +-2**15 and a kind built to show the abs-sum order.  On the fp32 and mixed rows a re-associated abs-sum,
entry, addv8 or block sum changes the LUT scale or bias of 10 % or more of the activation groups; on the fp16_order rows a
re-associated abs-sum changes every LUT scale (tests/test_lut_order_cpu.py keeps both so).

Configs that go through oracle.qgemm on the fp path use kfactor = act_group_size / 4: the oracle (like the reference) is only the
reference then.  One-scale (BitNet) configs keep the kfactor test_gpu_parity.py uses."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from act_rows import KINDS, KINDS16, rows, rows16
from seq_util import CHAIN_RING, kc, same_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TIGHT_TOL = 2e-5        # fp path: max |got - oracle| / max |oracle|, per activation row
P16_TOL = 5e-4          # the fp16-operand prefill tile (test_gpu_parity.py)
DENSE_NMSE = 5e-4       # against the float64 dense dequantised GEMV


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; libtmac_b200 has no CPU fallback")
    lib = tb.load()
    tb.check(lib.tmac_b200_init(0), "init")
    st = torch.cuda.Stream()                # torch fills and library launches on one stream
    torch.cuda.set_stream(st)
    tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")
    yield lib
    torch.cuda.synchronize()
    tb.check(lib.tmac_b200_set_stream(None), "set_stream")
    torch.cuda.set_stream(torch.cuda.default_stream())


@pytest.fixture(autouse=True)
def default_knobs(lib):
    yield
    for k, v in (("prefill", 1), ("prefill16", 1), ("prefill_min_n", 0), ("fused", 1), ("seq_impl", 2), ("chain_flags", 0),
                 ("chain_ahead", 1), ("seq_grid", 0), ("seq_handover", 1)):
        tb.debug_set(k, v)
    tb.check(lib.tmac_b200_set_lut_mode(0), "set_lut_mode")


def raw(a):
    """The bytes of a numpy array or tensor as unsigned integers of its element size."""
    a = np.ascontiguousarray(a.cpu().numpy() if hasattr(a, "cpu") else a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def assert_rows_close(got, ref, tol, what):
    """Each activation row against the oracle, relative to that row's largest output (a zero row must give exact zeros)."""
    ref = np.asarray(ref, np.float64)
    got = np.asarray(got, np.float64).reshape(ref.shape)
    for n in range(ref.shape[0]):
        err, bound = np.abs(got[n] - ref[n]).max(), tol * np.abs(ref[n]).max()
        assert err <= bound, "%s: row %d: max |got - oracle| = %.3g > %.3g" % (what, n, err, bound)


def oracle_out(oracle, cfg, A, S, x):
    qo, lso, lbo = oracle.preprocessor(x, cfg.act_group_size)
    return oracle.qgemm(cfg, A, S, qo, lso, lbo)


def fp_cfg(Mout, K, bits, ck, ags, zp):
    return T.Config(Mout, K, bits, kfactor=ags // 4, group_size=ck, act_group_size=ags, zero_point=zp).resolved()


def int_cfg(Mout, K):
    return T.Config(Mout, K, 2, kfactor=8 if K % 64 else 16, one_scale=True).resolved()


class Tensor:
    """One uploaded tensor and the problem it was made from."""

    def __init__(self, cfg, seed, zero_rows=None):
        self.cfg = cfg
        self.w, self.sc, self.z, _ = T.make_problem(cfg, seed=seed)
        if zero_rows is not None:                   # rows with weight scale 0 and zero point 0: their outputs are 0
            self.sc[zero_rows] = 0.0
            self.z[zero_rows] = 0.0
        self.A, self.S = T.pack_reference_layout(self.w, self.sc, self.z, cfg)
        self.wt = tb.upload_plain(kc(cfg), self.w, self.sc, self.z)

    def oracle(self, oracle, x):
        return oracle_out(oracle, self.cfg, self.A, self.S, x)


@pytest.fixture
def mk(lib):
    made = []

    def make(cfg, seed, zero_rows=None):
        made.append(Tensor(cfg, seed, zero_rows))
        return made[-1]
    yield make
    for t in made:
        t.wt.free()


def lut_dev(cfg, x, dtype=tb.F32):
    """preprocessor into fresh device buffers: (QLUT, LUT scales, LUT biases)."""
    N = x.shape[0]
    q = torch.zeros((N, cfg.K // 4, 16), dtype=torch.int8, device="cuda")
    ls = torch.zeros((N, cfg.K // cfg.act_group_size), device="cuda"); lb = torch.zeros_like(ls)
    tb.preprocessor(cfg.K, N, cfg.act_group_size, x, ls, lb, q, dtype=dtype)
    return q, ls, lb


# ---- 1: G1 (QLUT bytes, LUT scales, LUT biases) on full-precision rows -----------------------------------------------------------
G1_CASES = [(K, ags) for K in (256, 3200, 4096, 8640, 18944) for ags in (32, 64, 128, K) if K % ags == 0]


def preprocess(x, ags, dtype, device):
    """tmac_b200_preprocessor on rows x (F16: x is fp16-representable and goes in as fp16); the outputs start as garbage."""
    N, K = x.shape
    xin = np.ascontiguousarray(x.astype(np.float16) if dtype == tb.F16 else x)
    if device:
        q = torch.full((N, K // 4, 16), 0x5a, dtype=torch.int8, device="cuda")
        ls = torch.full((N, K // ags), float("nan"), device="cuda"); lb = ls.clone()
        tb.preprocessor(K, N, ags, torch.from_numpy(xin).cuda(), ls, lb, q, dtype=dtype)
        torch.cuda.synchronize()
        return q.cpu().numpy(), ls.cpu().numpy(), lb.cpu().numpy()
    q = np.full((N, K // 4, 16), 0x5a, np.int8)
    ls = np.full((N, K // ags), np.nan, np.float32); lb = ls.copy()
    tb.preprocessor(K, N, ags, xin, ls, lb, q, dtype=dtype)
    return q, ls, lb


def assert_g1(got, want, what):
    for name, g, w in zip(("QLUT bytes", "LUT scales", "LUT biases"), got, want):
        assert same_bits(g, w), "G1 %s: %s differ (%d of %d)" % (what, name, int((raw(g) != raw(w)).sum()), np.size(g))


@pytest.mark.parametrize("dtype", [tb.F32, tb.F16], ids=["f32", "f16"])
@pytest.mark.parametrize("K,ags", G1_CASES, ids=["k%d_a%d" % c for c in G1_CASES])
def test_preprocessor_g1_full_precision(lib, oracle, K, ags, dtype):
    """Pins the LUT order of preprocessor_kernel: QLUT bytes, LUT scales and LUT biases equal oracle.preprocessor bit for bit, for
    one row of every kind and for 7 rows of mixed kinds, through device and host pointers.  The fp32 rows make the abs-sum, entry,
    addv8 and block sums round (tests/test_lut_order_cpu.py).  fp16 rows add exactly in nearly every abs-sum; of the F16 kinds,
    fp16_order is the one built so that a re-associated abs-sum changes the scale of every activation group, at every K and
    act group size here."""
    make, kinds = (rows, KINDS) if dtype == tb.F32 else (rows16, KINDS16)
    rng = np.random.default_rng(K * 3 + ags)
    for x in [make(rng, 1, K, ags, (k,)) for k in kinds] + [make(rng, 7, K, ags, kinds)]:
        want = oracle.preprocessor(x, ags)
        for device in (True, False):
            assert_g1(preprocess(x, ags, dtype, device), want, "N=%d %s" % (x.shape[0], "device" if device else "host"))


def test_ggml_task_init_writes_the_oracle_lut(lib, oracle):
    """ggml's task_init (the reference's preprocessor call shape, host workspace) on full-precision rows of every kind: the QLUT
    bytes, LUT scales and LUT biases it writes are the oracle's, bit for bit."""
    cfg = fp_cfg(640, 4096, 4, 128, 128, False)
    tb.check(lib.tmac_b200_register_kcfg(C.byref(kc(cfg))), "register")
    nag = cfg.K // cfg.act_group_size
    for kind in KINDS:
        x = np.ascontiguousarray(rows(np.random.default_rng(5), 1, cfg.K, cfg.act_group_size, (kind,)))
        q = np.full((1, cfg.K // 4, 16), 0x5a, np.int8)
        ls = np.full((1, nag), np.nan, np.float32); lb = ls.copy()
        lib.ggml_tmac_mul_mat_task_init(x.ctypes.data, q.ctypes.data, ls.ctypes.data, lb.ctypes.data, cfg.Mout, cfg.K, 1, cfg.bits)
        assert_g1((q, ls, lb), oracle.preprocessor(x, cfg.act_group_size), kind)


# ---- 2: the fused GEMV, every instantiation --------------------------------------------------------------------------------------
FP_PAIRS = [(128, 128), (128, 64), (128, 32), (64, 64), (64, 32), (32, 32)]     # (K per chunk, act group size)
FUSED_FP = [(ck, ags, b) for ck, ags in FP_PAIRS for b in (1, 2, 4)] + [(128, 64, 3)]
RUNS = [(1, ("mixed",)), (3, ("fp32", "zero", "outlier")), (3, ("ties", "mixed", "zero"))]   # (N, kinds of its rows)


def fused_and_two_call(t, dx, N):
    """tmac_b200_gemv (LUT built inside the GEMV) and preprocessor + qgemm_lut, on device rows dx; asserts the GEMV kernel ran."""
    fused = torch.zeros((N, t.cfg.Mout), device="cuda")
    tb.gemv(t.wt, N, dx, fused)
    ll = tb.last_launch()
    assert ll["batch"] >= 1, "expected the GEMV kernel, got %r" % ll
    q, ls, lb = lut_dev(t.cfg, dx)
    two = torch.zeros_like(fused)
    tb.qgemm_lut(t.wt, N, q, ls, lb, two)
    torch.cuda.synchronize()
    return fused.cpu().numpy(), two.cpu().numpy(), ll


@pytest.mark.parametrize("ck,ags,bits", FUSED_FP, ids=["c%d_a%d_w%d" % c for c in FUSED_FP])
def test_fused_gemv_fp_path(oracle, mk, ck, ags, bits):
    """Every fp-path instantiation of the fused GEMV (pick3_fused_qa: chunk 128 / 64 / 32 K, act group 128 / 64 / 32 K, 1, 2 and 4
    planes per word): with full-precision rows its output equals preprocessor + qgemm_lut bit for bit -- both build the LUT with the
    same device functions -- and the oracle within the fp tolerance."""
    t = mk(fp_cfg(384 if bits == 3 else 512, 2048, bits, ck, ags, bits in (2, 3)), seed=ck + ags + bits)
    rng = np.random.default_rng(ck * ags + bits)
    for N, kinds in RUNS:
        x = rows(rng, N, t.cfg.K, ags, kinds)
        fused, two, _ = fused_and_two_call(t, torch.from_numpy(x).cuda(), N)
        assert same_bits(fused, two), "fused != two-call, kinds %s" % (kinds,)
        assert_rows_close(fused, t.oracle(oracle, x), TIGHT_TOL, "kinds %s" % (kinds,))


@pytest.mark.parametrize("K", [3200, 8640, 96], ids=["k3200_whole_row_scan", "k8640_split_scan", "k96"])
def test_fused_gemv_integer_path(oracle, mk, K):
    """The fused GEMV's integer path (one act group = the row): the row-wide scale and the bias over K / 32 blocks are formed by a
    whole-row scan per CTA (K = 3200) or a scan split over the cluster (K = 8640).  On full-precision rows the output equals the
    oracle and the two-call path bit for bit; fp16 rows in / fp16 out equal the oracle's output rounded once to fp16."""
    t = mk(int_cfg(640, K), seed=K)
    rng = np.random.default_rng(K)
    for N, kinds in RUNS:
        x = rows(rng, N, K, K, kinds)
        fused, two, ll = fused_and_two_call(t, torch.from_numpy(x).cuda(), N)
        # the cluster splits the row scan when it has more than one CTA and the row is longer than one round of 4 loads per thread
        assert (ll["cluster"] > 1 and K // 4 > 4 * 32 * ll["warps_per_cta"]) == (K == 8640), ll
        Co = t.oracle(oracle, x)
        assert same_bits(fused, Co), "fused integer path, kinds %s" % (kinds,)
        assert same_bits(two, Co), "two-call integer path, kinds %s" % (kinds,)
    x = rows16(rng, len(KINDS16), K, K)
    h16 = torch.zeros((len(KINDS16), t.cfg.Mout), dtype=torch.float16, device="cuda")
    tb.gemv(t.wt, len(KINDS16), torch.from_numpy(x).cuda().half(), h16, dtype=tb.F16)
    assert tb.last_launch()["batch"] >= 1
    torch.cuda.synchronize()
    with np.errstate(over="ignore"):                        # fp16_edge rows overflow fp16 outputs to +-inf, on both sides
        assert same_bits(h16, t.oracle(oracle, x).astype(np.float16)), "fp16 in / out"


# ---- 3: the integer path against the oracle, bit for bit ---------------------------------------------------------------------------
def test_integer_path_grouped_gemv(oracle, mk):
    """tmac_b200_gemv_grouped over 3 BitNet tensors (one launch, LUT built inside) on full-precision rows: every output is the
    oracle's bit for bit."""
    ts = [mk(int_cfg(640, 3200), seed=200 + i) for i in range(3)]
    N = 5
    x = rows(np.random.default_rng(7), N, 3200, 3200)
    outs = [torch.zeros((N, 640), device="cuda") for _ in ts]
    tb.gemv_grouped([t.wt for t in ts], N, torch.from_numpy(x).cuda(), outs)
    assert tb.last_launch()["batch"] == 3, tb.last_launch()
    torch.cuda.synchronize()
    for i, (t, o) in enumerate(zip(ts, outs)):
        assert same_bits(o, t.oracle(oracle, x)), "tensor %d" % i


INT_TILES = [(3200, 3200, 128), (3200, 8640, 128), (8640, 3200, 64)]       # (Mout, K, N): each tensor's automatic threshold


def assert_int8_tile(N):
    ll = tb.last_launch()
    assert ll["batch"] == -N and ll["cluster"] == 1, "expected the int8 tile, got %r" % ll


@pytest.mark.parametrize("mout,K,N", INT_TILES, ids=["%dx%d_n%d" % c for c in INT_TILES])
def test_integer_path_int8_tile(oracle, mk, mout, K, N):
    """The int8 prefill tile on BitNet-3B shapes at the N where each starts taking it: full-precision rows through gemv and through
    preprocessor + qgemm_lut give the oracle's output bit for bit on 8 sampled tokens (one of every kind among them); on 8640 x 3200
    fp16 rows in / fp16 out equal the oracle's output rounded once to fp16."""
    t = mk(int_cfg(mout, K), seed=mout + K)
    rng = np.random.default_rng(N + K)
    x = rows(rng, N, K, K)
    dx = torch.from_numpy(x).cuda()
    one = torch.zeros((N, mout), device="cuda")
    tb.gemv(t.wt, N, dx, one)
    assert_int8_tile(N)
    q, ls, lb = lut_dev(t.cfg, dx)
    two = torch.zeros_like(one)
    tb.qgemm_lut(t.wt, N, q, ls, lb, two)
    assert_int8_tile(N)
    torch.cuda.synchronize()
    assert same_bits(one, two)
    assert same_bits(one, t.oracle(oracle, x))
    if mout == 8640:
        x16 = rows16(rng, N, K, K)
        h16 = torch.zeros((N, mout), dtype=torch.float16, device="cuda")
        tb.gemv(t.wt, N, torch.from_numpy(x16).cuda().half(), h16, dtype=tb.F16)
        assert_int8_tile(N)
        torch.cuda.synchronize()
        with np.errstate(over="ignore"):
            assert same_bits(h16, t.oracle(oracle, x16).astype(np.float16))


# ---- 4: fp-path prefill tiles ------------------------------------------------------------------------------------------------------
PF_CASES = [(256, 2048, 2, 128, 64, True, 130), (256, 2048, 4, 128, 128, False, 96), (256, 1024, 4, 32, 32, False, 70),
            (192, 1024, 3, 64, 32, True, 64)]        # (Mout, K, bits, K per chunk, act group, zero point, N)


@pytest.mark.parametrize("tile", ["int8", "fp16"])
@pytest.mark.parametrize("mout,K,bits,ck,ags,zp,N", PF_CASES, ids=["w%d_c%d_a%d_n%d" % (c[2], c[3], c[4], c[6]) for c in PF_CASES])
def test_fp_prefill_tiles(oracle, mk, mout, K, bits, ck, ags, zp, N, tile):
    """The fp-path prefill tiles on full-precision rows with zero rows and zero groups among the tokens and a ragged last token tile:
    the int8 tile matches the oracle per token at the fp tolerance, the fp16 tile at its own; both pass the dense NMSE check.  For
    the fp16 tile every row is clipped to |x| <= 2**8, which keeps its fp16 operands (fp16(LUT scale * T8), the hi / lo split of a
    chunk's activation sum) below 65504 (DESIGN.md section 1); the mixed rows still span magnitudes down to 2**-20."""
    t = mk(fp_cfg(mout, K, bits, ck, ags, zp), seed=N + bits)
    x = rows(np.random.default_rng(N * bits), N, K, ags)
    x[7] = 0.0
    x[N - 2] = -0.0
    if tile == "fp16":
        x = np.clip(x, -256.0, 256.0)
    tb.debug_set("prefill16", 1 if tile == "fp16" else 0)
    tb.debug_set("prefill_min_n", 32)
    q, ls, lb = lut_dev(t.cfg, torch.from_numpy(x).cuda())
    out = torch.zeros((N, mout), device="cuda")
    tb.qgemm_lut(t.wt, N, q, ls, lb, out)
    ll = tb.last_launch()
    assert ll["batch"] == -N and ll["cluster"] == (1 if tile == "int8" else 16), "expected the %s tile, got %r" % (tile, ll)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert_rows_close(got, t.oracle(oracle, x), TIGHT_TOL if tile == "int8" else P16_TOL, tile)
    assert T.nmse(T.dense_reference(t.w, t.sc, t.z, x, t.cfg), got) <= DENSE_NMSE


# ---- 5: caller-made tables with -128 -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 2, 3, 4])
def test_general_table_with_minus_128(lib, oracle, bits):
    """A caller-made, non-symmetric table with entries drawn from [-128, 127] (the int8 range a symmetric table never reaches):
    the integer plane sums (cbits) equal oracle.cbits and qgemm_lut matches the oracle, with the table in host memory and in device
    memory (lut_mode 1: a general table)."""
    cfg = T.Config(384 if bits == 3 else 512, 1024, bits, zero_point=(bits % 2 == 0)).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=50 + bits)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    rng = np.random.default_rng(60 + bits)
    nag = cfg.K // cfg.act_group_size
    N = 2
    q = rng.integers(-128, 128, size=(N, cfg.K // 4, 16)).astype(np.int8)
    q.reshape(-1)[::37] = -128
    ls = np.abs(rng.standard_normal((N, nag))).astype(np.float32); lb = rng.standard_normal((N, nag)).astype(np.float32)
    wt = tb.upload_reference_layout(kc(cfg), A, S)
    try:
        Co = oracle.qgemm(cfg, A, S, q, ls, lb)
        cbo = oracle.cbits(cfg, A, q)
        for dev in (False, True):
            tb.check(lib.tmac_b200_set_lut_mode(1 if dev else 0), "set_lut_mode")
            if dev:
                dq, dls, dlb = torch.from_numpy(q).cuda(), torch.from_numpy(ls).cuda(), torch.from_numpy(lb).cuda()
                dC = torch.zeros((N, cfg.Mout), device="cuda")
                dcb = torch.zeros((N, cfg.Mout * cfg.bits), dtype=torch.int32, device="cuda")
                tb.qgemm_lut(wt, N, dq, dls, dlb, dC)
                tb.cbits(wt, N, dq, dcb)
                torch.cuda.synchronize()
                Cout, cb = dC.cpu().numpy(), dcb.cpu().numpy()
            else:
                Cout = np.zeros((N, cfg.Mout), np.float32); cb = np.zeros((N, cfg.Mout * cfg.bits), np.int32)
                tb.qgemm_lut(wt, N, q, ls, lb, Cout)
                tb.cbits(wt, N, q, cb)
            where = "device" if dev else "host"
            assert np.array_equal(cb, cbo), "cbits (%s table)" % where
            assert_rows_close(Cout, Co, TIGHT_TOL, "%s table" % where)
    finally:
        wt.free()


# ---- 6: decode sequences -----------------------------------------------------------------------------------------------------------
# name -> (seq_impl, chain_flags, chain_ahead, LUT hand-over of the stream-K kernel)
SEQ_FORMS = {"flow": (1, 0, 1, True), "flow_no_ahead": (1, 0, 0, True), "barrier": (1, 1, 1, True), "streamk": (0, 0, 1, True),
             "streamk_no_handover": (0, 0, 1, False)}
SEQ_CASES = [(f, ags, off) for f in SEQ_FORMS for ags in (32, 64, 128) for off in ((0, 68) if f == "barrier" else (0, 2, 66))]


@contextlib.contextmanager
def seq_form(name):
    impl, flags, ahead, handover = SEQ_FORMS[name]
    tb.debug_set("seq_impl", impl); tb.debug_set("chain_flags", flags); tb.debug_set("chain_ahead", ahead)
    tb.debug_set("seq_handover", int(handover))
    try:
        yield
    finally:
        tb.debug_set("seq_impl", 2); tb.debug_set("chain_flags", 0); tb.debug_set("chain_ahead", 1); tb.debug_set("seq_handover", 1)


def run_seq(name, steps):
    """steps[i] = (tensor, src, offset): src a device vector (external input) or the index of an earlier step whose outputs
    [offset, offset + K) are the input.  Builds in form `name`, asserts the kernel the build chose, launches twice."""
    with seq_form(name):
        seq = tb.Sequence()
        try:
            outs = []
            for t, src, off in steps:
                out = torch.full((t.cfg.Mout,), float("nan"), device="cuda")
                if isinstance(src, int):
                    seq.add(t.wt, in_op=src, in_offset=off, out=out)
                else:
                    seq.add(t.wt, x=src, out=out)
                outs.append(out)
            seq.build()
            info = seq.info()
            if SEQ_FORMS[name][0] == 1:
                assert info["ring_slots"] == CHAIN_RING, "expected the resident chain, got %r" % info
            else:
                assert info["ring_slots"] > 0 and info["grid"] == torch.cuda.get_device_properties(0).multi_processor_count, info
            for _ in range(2):
                seq.launch()
            seq.status()
            torch.cuda.synchronize()
            return outs
        finally:
            seq.free()


@pytest.mark.parametrize("name,ags,off", SEQ_CASES, ids=["%s_a%d_off%d" % c for c in SEQ_CASES])
def test_sequence_external_equals_chained(oracle, mk, name, ags, off):
    """Decode sequences on full-precision inputs.  S1 = [A: x -> y, B: y[off:off + 768] -> z, C: z -> w] plus one op per kind of
    external input; S2 is the same ops with B and C reading fresh device copies of S1's y[off:...] and z as external inputs.  A
    chained op's LUT is built by the same lut_slice / lut_record as an external one's, so all outputs are bit for bit the same, and
    every op of S1 matches the oracle on the input it saw.  Offsets 2 and 66 make activation groups straddle A's 128-row super-blocks;
    A's rows 64-383 have scale 0 and zero point 0, so at every act group size and offset B sees whole activation groups of zeros
    (LUT scale 0) built from producer words, and groups that are only partly zero."""
    def cfg(M, K):
        return fp_cfg(M, K, 2, 128, ags, True)
    a = mk(cfg(1024, 512), seed=300 + ags, zero_rows=slice(64, 384))
    b, c = mk(cfg(512, 768), seed=301 + ags), mk(cfg(256, 512), seed=302 + ags)
    ext = [mk(cfg(256, 512), seed=310 + i) for i in range(len(KINDS))]
    rng = np.random.default_rng(ags + off)
    xs = [rows(rng, 1, 512, ags, (k,))[0] for k in ("mixed",) + KINDS]
    dxs = [torch.from_numpy(v).cuda() for v in xs]
    s1 = [(a, dxs[0], 0), (b, 0, off), (c, 1, 0)] + [(e, dxs[1 + i], 0) for i, e in enumerate(ext)]
    o1 = run_seq(name, s1)
    y = o1[0].cpu().numpy()
    assert not np.any(y[64:384]), "rows with scale 0 and zero point 0 must give 0"
    zero_groups = ~np.any(y[off:off + 768].reshape(-1, ags), axis=1)
    assert zero_groups.any() and not zero_groups.all(), "B must see whole zero activation groups and others"
    ins = [xs[0], y[off:off + 768], o1[1].cpu().numpy()] + xs[1:]
    for i, ((t, _, _), x) in enumerate(zip(s1, ins)):
        assert_rows_close(o1[i].cpu().numpy()[None], t.oracle(oracle, x[None]), TIGHT_TOL, "%s op %d" % (name, i))
    yb, zc = o1[0][off:off + 768].clone(), o1[1].clone()
    assert yb.data_ptr() % 16 == 0 and zc.data_ptr() % 16 == 0
    s2 = [(a, dxs[0], 0), (b, yb, 0), (c, zc, 0)] + s1[3:]
    o2 = run_seq(name, s2)
    for i, (u, v) in enumerate(zip(o1, o2)):
        assert same_bits(u, v), "%s: op %d differs between the chained and the external input" % (name, i)
