"""GPU suite (-m gpu): gemv3_kernel's fp path, every output bit against the model of its operation order (tests/gemv_order.py).

The other fp-path gates compare the GEMV with the oracle within TIGHT_TOL, and its call forms with each other bit for bit; a kernel
that summed its warps or cluster ranks in another order, or split an fma, passes them all.  Here every comparison is same_bits
against gemv_order.gemv at the decomposition the launch reports (tb.last_launch(): cluster size, warps per CTA, chunks per warp), so
the tests follow any tuning of choose_decomposition.  The rows are act_rows' full-precision kinds (fp16-rounded rows add exactly too
often to show an order), plus an all-zero row and weight rows with scale 0 and zero point 0, which must give +0.0.

Covered: every instantiation (bit widths, chunkings, symmetric table in the fused GEMV and in preprocessor + qgemm_lut, a caller's
general table with -128 entries, both register variants) at N = 1 and 3; the whole cs x wpc grid, with the stage double-buffered and
single-buffered, on 37-chunk tensors and on a 3-chunk one (idle warps and idle CTAs), and for the fused and two-call integer path
against the oracle; the grouped launches in their whole-super-block form, row ranges into a view between NaN canaries, a ragged
last super-block, fp16 output and input, fp32-stored scales, host pointers, the Llama-2-7B shapes, repeated launches, and the
residual and RMSNorm input forms.  N stays below every prefill threshold, and each launch is checked to be the GEMV kernel."""
import numpy as np
import pytest

import gemv_order as G
import tmac_b200 as tb
import tmac_oracle as T
from act_rows import KINDS16, rows, rows16
from seq_util import A_CASES, A_IDS, EPS, kc, norm_weight, rms_input, same_bits, stream  # noqa: F401 (stream: fixture)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

f32 = np.float32
KNOBS = {"cs": 0, "wpc": 0, "minb": 0, "nbuf": 0, "fused": 1, "prefill": 1, "lut_mode": 0}


@pytest.fixture(autouse=True)
def default_knobs(stream):
    for k, v in KNOBS.items():
        tb.debug_set(k, v)
    yield
    for k, v in KNOBS.items():
        tb.debug_set(k, v)


class Tensor:
    """One uploaded tensor, the problem it was made from and its model."""

    def __init__(self, cfg, w, sc, z):
        self.cfg, self.w, self.sc, self.z = cfg, w, sc, z
        self.A, self.S = T.pack_reference_layout(w, sc, z, cfg)
        self.wt = tb.upload_reference_layout(kc(cfg), self.A, self.S)
        self.prob = G.Problem.of(cfg, w, sc, z, self.A, self.S)

    def model(self, tables, ll, f16=False):
        q, ls, lb = tables
        return G.gemv_table(self.prob, q, ls, lb, ll["cluster"], ll["warps_per_cta"], ll["chunks_per_warp"], f16)


def fp_cfg(Mout, K, bits, g, ags, zp):
    return T.Config(Mout, K, bits, kfactor=ags // 4, group_size=g, act_group_size=ags, zero_point=zp).resolved()


@pytest.fixture
def mk(stream):
    """mk(cfg, seed, zero_rows=None, scale_mul=None) or mk(cfg, w=, sc=, z=) uploads a Tensor; all are freed after the test."""
    made = []

    def make(cfg, seed=0, zero_rows=None, scale_mul=None, w=None, sc=None, z=None):
        if w is None:
            w, sc, z, _ = T.make_problem(cfg, seed=seed)
        if scale_mul is not None:                  # not fp16-exact: the layout stores fp32 scales
            sc = (sc * f32(scale_mul)).astype(f32)
        if zero_rows is not None:                  # weight scale 0 and zero point 0: the row's outputs are +0.0
            sc = sc.copy(); sc[zero_rows] = 0.0
            if z is not None:
                z = z.copy(); z[zero_rows] = 0.0
        made.append(Tensor(cfg, w, sc, z))
        return made[-1]
    yield make
    for t in made:
        t.wt.free()


def gemv_launch():
    """The last launch's report; it must be the GEMV kernel (a prefill tile reports batch < 0)."""
    ll = tb.last_launch()
    assert ll["batch"] >= 1 and ll["cluster"] in (1, 2, 4, 8), "expected gemv3_kernel, got %r" % ll
    return ll


def out_like(N, Mout, f16=False):
    return torch.full((N, Mout), float("nan"), device="cuda", dtype=torch.float16 if f16 else torch.float32)


def fetch(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def fused(t, x, f16=False):
    """tmac_b200_gemv on device rows x (fp16 in and out with f16): (output, launch)."""
    N = x.shape[0]
    dx = torch.from_numpy(np.ascontiguousarray(x, f32)).cuda()
    out = out_like(N, t.cfg.Mout, f16)
    tb.gemv(t.wt, N, dx.half() if f16 else dx, out, dtype=tb.F16 if f16 else tb.F32)
    ll = gemv_launch()
    assert ll["sym_lut"] == 1, ll
    return fetch(out), ll


def device_tables(t, x, want):
    """The device preprocessor's table of rows x, checked to be the oracle's table `want` (the one the model is fed)."""
    N, K, ags = x.shape[0], t.cfg.K, t.cfg.act_group_size
    q = torch.zeros((N, K // 4, 16), dtype=torch.int8, device="cuda")
    ls = torch.zeros((N, K // ags), device="cuda"); lb = torch.zeros_like(ls)
    tb.preprocessor(K, N, ags, torch.from_numpy(np.ascontiguousarray(x, f32)).cuda(), ls, lb, q)
    for name, g, w in zip(("QLUT", "LUT scales", "LUT biases"), (q, ls, lb), want):
        assert same_bits(fetch(g), w), "device %s differ from the oracle's" % name
    return q, ls, lb


def two_call(t, dtab, sym=True, f16=False, **kw):
    """qgemm_lut on device tables dtab: (output, launch)."""
    N = dtab[0].shape[0]
    out = out_like(N, t.cfg.Mout, f16)
    tb.qgemm_lut(t.wt, N, *dtab, out, dtype=tb.F16 if f16 else tb.F32, **kw)
    ll = gemv_launch()
    assert ll["sym_lut"] == int(sym), ll
    return fetch(out), ll


def general_table(rng, N, cfg):
    """A caller's table: entries drawn from [-128, 127] with -128 planted, full-precision LUT scales and biases."""
    nag = cfg.K // cfg.act_group_size
    q = rng.integers(-128, 128, size=(N, cfg.K // 4, 16)).astype(np.int8)
    q.reshape(-1)[::37] = -128
    return q, np.abs(rng.standard_normal((N, nag), dtype=f32)), rng.standard_normal((N, nag), dtype=f32)


def to_dev(tables):
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in tables)


def assert_model(got, t, tables, ll, what, f16=False):
    want = t.model(tables, ll, f16)
    diff = int(np.sum(np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8)))
    assert same_bits(got, want), "%s at %r: %d bytes differ from the model" % (what, ll, diff)


# ---- every instantiation, natural decomposition --------------------------------------------------------------------------------
ZERO_ROWS = np.arange(5, 384, 37)


def instantiation_rows(rng, N, K, ags):
    if N == 1:
        return [rows(rng, 1, K, ags, ("mixed",))]
    z = rows(rng, 3, K, ags, ("zero", "mixed", "fp32"))
    z[2] = 0.0                                         # an all-zero row: LUT scale 0, every output +0.0
    return [rows(rng, 3, K, ags, ("fp32", "outlier", "ties")), z]


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_every_instantiation(oracle, mk, g, ags, bits, zp, N):
    """Every fp-path instantiation at the decomposition the library picks: the fused GEMV and preprocessor + qgemm_lut on the
    symmetric table (SYM), and qgemm_lut on a caller's general table with -128 entries (lut_mode 1, SYM = false), each with the
    register variant forced to MINB 3 and to 4, give the model's bits.  Weight rows with scale 0 and zero point 0 and the all-zero
    activation row give +0.0."""
    t = mk(fp_cfg(384 if bits == 3 else 512, 2048, bits, g, ags, zp), seed=g + ags + bits, zero_rows=ZERO_ROWS)
    rng = np.random.default_rng(g * ags + bits + N)
    for x in instantiation_rows(rng, N, t.cfg.K, ags):
        sym = oracle.preprocessor(x, ags)
        dsym = device_tables(t, x, sym)
        gen = general_table(rng, N, t.cfg)
        dgen = to_dev(gen)
        for minb in (3, 4):
            tb.debug_set("minb", minb)
            y, ll = fused(t, x)
            assert ll["min_blocks"] == minb, ll
            assert_model(y, t, sym, ll, "fused, MINB %d" % minb)
            assert not np.any(y[:, ZERO_ROWS].view(np.uint32)), "zero-scale rows must give +0.0"
            if N == 3 and not x[2].any():
                assert not np.any(y[2].view(np.uint32)), "the all-zero row must give +0.0"
            y, ll = two_call(t, dsym)
            assert_model(y, t, sym, ll, "two-call, MINB %d" % minb)
            tb.debug_set("lut_mode", 1)
            y, ll = two_call(t, dgen, sym=False)
            tb.debug_set("lut_mode", 0)
            assert_model(y, t, gen, ll, "general table, MINB %d" % minb)


# ---- every decomposition -------------------------------------------------------------------------------------------------------
def force(cs, wpc):
    tb.debug_set("cs", cs); tb.debug_set("wpc", wpc)


def assert_forced(ll, cs, wpc, nchunk):
    assert (ll["cluster"], ll["warps_per_cta"], ll["chunks_per_warp"]) == (cs, wpc, G.forced_bpw(nchunk, cs, wpc)), ll


@pytest.mark.parametrize("nbuf", [0, 1], ids=["nbuf_auto", "nbuf1"])
@pytest.mark.parametrize("name", sorted(G.GRID_TENSORS))
def test_every_decomposition(oracle, mk, name, nbuf):
    """The whole grid cs in {1, 2, 4, 8} x wpc in 1..8, forced, with the stage double-buffered when a warp has several chunks (the
    default) and single-buffered (nbuf 1): the fused GEMV and preprocessor + qgemm_lut give the model's bits at each reported
    decomposition.  37 chunks leave a ragged last warp at most grid points; the 3-chunk tensor has idle warps and idle CTAs."""
    cfg, w, sc, z, x = G.grid_problem(name)
    t = mk(cfg, w=w, sc=sc, z=z)
    sym = oracle.preprocessor(x, cfg.act_group_size)
    dsym = device_tables(t, x, sym)
    it = G.int_sums(w, cfg.bits, sym[0], cfg.act_group_size)
    tb.debug_set("nbuf", nbuf)
    for cs, wpc in G.GRID:
        force(cs, wpc)
        bpw = G.forced_bpw(t.prob.nchunk, cs, wpc)
        want = G.gemv(t.prob, it, sym[1], sym[2], cs, wpc, bpw)
        for form in ("fused", "two-call"):
            y, ll = fused(t, x) if form == "fused" else two_call(t, dsym)
            assert_forced(ll, cs, wpc, t.prob.nchunk)
            assert same_bits(y, want), "%s, cs %d wpc %d bpw %d: %d outputs differ from the model" % (
                form, cs, wpc, bpw, int(np.sum(y.view(np.uint32) != want.view(np.uint32))))


@pytest.mark.parametrize("nbuf", [0, 1], ids=["nbuf_auto", "nbuf1"])
@pytest.mark.parametrize("K", [3200, 8640])
def test_integer_path_every_decomposition(oracle, mk, K, nbuf):
    """The integer path (one act group = the row) over the same grid: the fused GEMV -- whose row scan is whole-row or split over
    the cluster, with the bias formed by the last rank's last warp -- and preprocessor + qgemm_lut equal the oracle bit for bit at
    every decomposition."""
    cfg = T.Config(640, K, 2, kfactor=8 if K % 64 else 16, one_scale=True).resolved()
    t = mk(cfg, seed=K)
    x = rows(np.random.default_rng(K), 3, K, K, ("fp32", "mixed", "outlier"))
    tabs = oracle.preprocessor(x, K)
    want = oracle.qgemm(cfg, t.A, t.S, *tabs)
    dtab = device_tables(t, x, tabs)
    tb.debug_set("nbuf", nbuf)
    split = set()
    for cs, wpc in G.GRID:
        force(cs, wpc)
        for form in ("fused", "two-call"):
            y, ll = fused(t, x) if form == "fused" else two_call(t, dtab)
            assert_forced(ll, cs, wpc, t.prob.nchunk)
            assert same_bits(y, want), "%s, cs %d wpc %d" % (form, cs, wpc)
        split.add(cs > 1 and K // 4 > 4 * 32 * wpc)
    assert split == {False, True}, split              # both row scans ran


# ---- call forms ------------------------------------------------------------------------------------------------------------------
def test_grouped_whole_super_blocks(oracle, mk):
    """qgemm_lut_grouped and gemv_grouped over 3 tensors at an N that fills the machine with whole super-blocks (cs = 1): every
    tensor's output is the model's."""
    cfg = fp_cfg(1024, 2048, 2, 128, 64, True)
    ts = [mk(cfg, seed=300 + i) for i in range(3)]
    nrsb = G.layout(cfg, ts[0].A, ts[0].S)[3]
    N = -(-4 * torch.cuda.get_device_properties(0).multi_processor_count // (nrsb * 3))
    assert N < 32
    x = rows(np.random.default_rng(3), N, cfg.K, cfg.act_group_size)
    sym = oracle.preprocessor(x, cfg.act_group_size)
    dq, dls, dlb = device_tables(ts[0], x, sym)
    outs = [out_like(N, cfg.Mout) for _ in ts]
    tb.qgemm_lut_grouped([t.wt for t in ts], N, [dq] * 3, [dls] * 3, [dlb] * 3, outs)
    ll = gemv_launch()
    assert ll["cluster"] == 1 and ll["batch"] == 3, ll
    for i, (t, o) in enumerate(zip(ts, outs)):
        assert_model(fetch(o), t, sym, ll, "qgemm_lut_grouped tensor %d" % i)
    outs = [out_like(N, cfg.Mout) for _ in ts]
    tb.gemv_grouped([t.wt for t in ts], N, torch.from_numpy(x).cuda(), outs)
    ll = gemv_launch()
    assert ll["cluster"] == 1 and ll["batch"] == 3, ll
    for i, (t, o) in enumerate(zip(ts, outs)):
        assert_model(fetch(o), t, sym, ll, "gemv_grouped tensor %d" % i)


def test_row_range_into_a_view_between_canaries(oracle, mk):
    """qgemm_lut over rows [37, 287) -- both ends off the super-block boundaries -- into a view of a larger buffer: the view gets the
    model's rows, the NaN canaries before and after it stay NaN."""
    cfg = fp_cfg(384, 2048, 3, 128, 64, True)
    t = mk(cfg, seed=7)
    x = rows(np.random.default_rng(7), 2, cfg.K, cfg.act_group_size, ("fp32", "mixed"))
    sym = oracle.preprocessor(x, cfg.act_group_size)
    dtab = device_tables(t, x, sym)
    row0, nrows, pad = 37, 250, 32
    buf = torch.full((2 * nrows + 2 * pad,), float("nan"), device="cuda")
    view = buf[pad:pad + 2 * nrows].view(2, nrows)
    tb.qgemm_lut(t.wt, 2, *dtab, view, row0=row0, rows=nrows)
    ll = gemv_launch()
    b = fetch(buf)
    assert np.isnan(b[:pad]).all() and np.isnan(b[pad + 2 * nrows:]).all(), "a canary was overwritten"
    want = t.model(sym, ll)[:, row0:row0 + nrows]
    assert same_bits(b[pad:pad + 2 * nrows].reshape(2, nrows), want)


@pytest.mark.parametrize("bits", [1, 2])
def test_ragged_last_super_block(oracle, mk, bits):
    """320 rows: the last row super-block is partly outside the tensor; fused and two-call give the model's bits on every row."""
    cfg = fp_cfg(320, 2048, bits, 128, 64, bits == 2)
    t = mk(cfg, seed=bits)
    lay = G.layout(cfg, t.A, t.S)
    assert cfg.Mout % lay[2], "the last super-block must be ragged"
    x = rows(np.random.default_rng(bits), 3, cfg.K, cfg.act_group_size, ("fp32", "mixed", "outlier"))
    sym = oracle.preprocessor(x, cfg.act_group_size)
    y, ll = fused(t, x)
    assert_model(y, t, sym, ll, "fused")
    y, ll = two_call(t, device_tables(t, x, sym))
    assert_model(y, t, sym, ll, "two-call")


def test_fp16_output_and_input(oracle, mk):
    """fp16 output is the model's fp32 result rounded once: qgemm_lut with an F16 output, and the fused GEMV with fp16 rows in and
    fp16 out (rows16: subnormals, values near +-2^15)."""
    cfg = fp_cfg(512, 2048, 4, 128, 32, False)
    t = mk(cfg, seed=16)
    rng = np.random.default_rng(16)
    x = rows(rng, 3, cfg.K, cfg.act_group_size, ("fp32", "mixed", "outlier"))
    sym = oracle.preprocessor(x, cfg.act_group_size)
    y, ll = two_call(t, device_tables(t, x, sym), f16=True)
    assert_model(y, t, sym, ll, "qgemm_lut F16 output", f16=True)
    x16 = rows16(rng, len(KINDS16), cfg.K, cfg.act_group_size)
    y, ll = fused(t, x16, f16=True)
    with np.errstate(over="ignore"):
        assert_model(y, t, oracle.preprocessor(x16, cfg.act_group_size), ll, "gemv fp16 in / out", f16=True)


def test_fp32_stored_scales(oracle, mk):
    """Scales that are not fp16-exact are stored as fp32 (layout sd = 4) and enter the model's fma unrounded."""
    cfg = fp_cfg(512, 2048, 2, 64, 32, True)
    t = mk(cfg, seed=32, scale_mul=1.0 + 2.0 ** -13)
    assert G.layout(cfg, t.A, t.S)[7] == 4
    x = rows(np.random.default_rng(32), 3, cfg.K, cfg.act_group_size, ("fp32", "mixed", "ties"))
    sym = oracle.preprocessor(x, cfg.act_group_size)
    y, ll = fused(t, x)
    assert_model(y, t, sym, ll, "fused")
    y, ll = two_call(t, device_tables(t, x, sym))
    assert_model(y, t, sym, ll, "two-call")


def test_host_pointers(oracle, mk):
    """qgemm_lut with the table and the output in host memory, and gemv with host rows and a host output, give the model's bits."""
    cfg = fp_cfg(512, 2048, 2, 128, 64, True)
    t = mk(cfg, seed=44)
    x = np.ascontiguousarray(rows(np.random.default_rng(44), 3, cfg.K, cfg.act_group_size, ("fp32", "mixed", "outlier")))
    sym = oracle.preprocessor(x, cfg.act_group_size)
    out = np.full((3, cfg.Mout), np.nan, f32)
    tb.qgemm_lut(t.wt, 3, *(np.ascontiguousarray(a) for a in sym), out)
    ll = gemv_launch()
    assert ll["sym_lut"] == 1, ll
    assert_model(out, t, sym, ll, "qgemm_lut, host table")
    out = np.full((3, cfg.Mout), np.nan, f32)
    tb.gemv(t.wt, 3, x, out)
    assert_model(out, t, sym, gemv_launch(), "gemv, host rows")


LLAMA = [(4096, 4096, 2, True), (11008, 4096, 2, True), (4096, 11008, 2, True), (4096, 4096, 4, False)]   # (Mout, K, bits, zp)


@pytest.mark.parametrize("mout,K,bits,zp", LLAMA, ids=["%dx%d_w%d" % c[:3] for c in LLAMA])
def test_llama2_7b_shapes_repeated_launches(oracle, mk, mout, K, bits, zp):
    """The Llama-2-7B projections at N = 1 (g128, act group 64; 11008 x 4096 W2 zero-point is bench.py's shape): three fused launches
    and a two-call launch each give the model's bits."""
    cfg = fp_cfg(mout, K, bits, 128, 64, zp)
    t = mk(cfg, seed=mout + K + bits)
    x = rows(np.random.default_rng(mout + K), 1, K, 64, ("mixed",))
    sym = oracle.preprocessor(x, 64)
    it = G.int_sums(t.w, bits, sym[0], 64)
    for i in range(3):
        y, ll = fused(t, x)
        want = G.gemv(t.prob, it, sym[1], sym[2], ll["cluster"], ll["warps_per_cta"], ll["chunks_per_warp"])
        assert same_bits(y, want), "fused launch %d at %r" % (i, ll)
    y, ll = two_call(t, device_tables(t, x, sym))
    assert same_bits(y, G.gemv(t.prob, it, sym[1], sym[2], ll["cluster"], ll["warps_per_cta"], ll["chunks_per_warp"])), ll


def test_residual_and_rmsnorm_inputs(oracle, mk):
    """gemv_residual is fadd(model, R); gemv_rmsnorm over 2 tensors is the model of the norm input seq_util.rms_input (its order is
    the one tmac_b200_gemv_rmsnorm documents)."""
    cfg = fp_cfg(512, 2048, 2, 128, 64, True)
    ts = [mk(cfg, seed=70 + i) for i in range(2)]
    rng = np.random.default_rng(70)
    N = 3
    x = rows(rng, N, cfg.K, cfg.act_group_size, ("fp32", "mixed", "outlier"))
    r = rng.standard_normal((N, cfg.Mout), dtype=f32)
    out = out_like(N, cfg.Mout)
    tb.gemv_residual(ts[0].wt, N, torch.from_numpy(x).cuda(), torch.from_numpy(r).cuda(), out)
    ll = gemv_launch()
    assert same_bits(fetch(out), (ts[0].model(oracle.preprocessor(x, 64), ll) + r).astype(f32)), ll
    nw = norm_weight(rng, cfg.K)
    a = rms_input(x, nw, EPS)
    outs = [out_like(N, cfg.Mout) for _ in ts]
    tb.gemv_rmsnorm([t.wt for t in ts], N, torch.from_numpy(x).cuda(), torch.from_numpy(nw).cuda(), EPS, outs)
    ll = gemv_launch()
    tabs = oracle.preprocessor(a, 64)
    for i, (t, o) in enumerate(zip(ts, outs)):
        assert_model(fetch(o), t, tabs, ll, "gemv_rmsnorm tensor %d" % i)
