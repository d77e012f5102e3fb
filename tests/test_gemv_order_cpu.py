"""CPU suite: the numpy model of gemv3_kernel's fp-path order (tests/gemv_order.py) -- its exact fma, its agreement with the oracle,
and the power of the GPU suite's rows and shapes (tests/test_gpu_gemv_order.py) to tell the kernel's order from a changed one.

The fp-path gates elsewhere compare the kernel with the oracle within 2e-5 of each row's largest output, and the GEMV's call forms
with each other bit for bit.  Neither pins the order DESIGN.md section 1 states: a kernel that reversed a reduction or split an fma
would still pass them.  The GPU suite compares every output bit with the model; the tests here keep that comparison meaningful."""
import itertools
from fractions import Fraction

import numpy as np
import pytest

import gemv_order as G
import tmac_oracle as T
from act_rows import rows
from seq_util import A_CASES, A_IDS, TIGHT_TOL

f32 = np.float32


def round32(q, a, b, c):
    """The float32 nearest to the rational q (ties to the even significand), with IEEE's sign for an exact zero of a*b + c."""
    if q == 0:
        neg = (np.signbit(a) != np.signbit(b)) and np.signbit(c)
        return f32(-0.0) if neg else f32(0.0)
    r = f32(float(q))
    cands = [np.nextafter(r, f32(-np.inf)), r, np.nextafter(r, f32(np.inf))]
    cands = [x for x in cands if np.isfinite(x)]
    best = min(cands, key=lambda x: (abs(Fraction(float(x)) - q), int(np.array(x, f32).view(np.uint32)) & 1))
    if best == 0:                                    # the rounded result keeps the sign of the exact one
        best = f32(-0.0) if q < 0 else f32(0.0)
    return f32(best)


def exact_fma(a, b, c):
    a, b, c = f32(a), f32(b), f32(c)
    return round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)), a, b, c)


def bits32(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def check_fma(a, b, c):
    got = G.fma32(a, b, c)
    want = np.array([exact_fma(x, y, z) for x, y, z in zip(a, b, c)], f32)
    bad = np.nonzero(bits32(got) != bits32(want))[0]
    assert bad.size == 0, "fma32(%r, %r, %r) = %r, exact %r" % (a[bad[0]], b[bad[0]], c[bad[0]], got[bad[0]], want[bad[0]])
    return got


def test_fma32_random_operands():
    """fma32 equals the correctly rounded exact a*b + c on operands of every relative magnitude, including cancellation and zeros."""
    rng = np.random.default_rng(0)
    n = 3000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n))).astype(f32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n))).astype(f32)
    c = (rng.standard_normal(n) * np.exp2(rng.integers(-60, 60, n))).astype(f32)
    c[::7] = (-(a[::7].astype(np.float64) * b[::7])).astype(f32)      # near-total cancellation
    c[::11] = 0.0
    c[1::11] = -0.0
    a[::13] = 0.0
    check_fma(a, b, c)


def test_fma32_float64_midpoints():
    """Operands whose float64 sum is exactly a float32 midpoint while the exact value is not: the tie must be resolved towards the
    exact value, not to even.  Built as c with an odd significand and a*b = +-2^-24 * (1 - k^2 2^-46) * 2^e, the exact value sits k^2 2^-70 * 2^e
    inside the midpoint on c's side; plain float64 rounding gives the even neighbour instead."""
    rng = np.random.default_rng(1)
    n = 400
    k = rng.integers(1, 256, n)                                     # k^2 2^-70 < 2^-53: lost in the float64 sum
    e1, e2 = rng.integers(-20, 20, n), rng.integers(-20, 20, n)
    sign = np.where(rng.integers(0, 2, n) == 1, 1.0, -1.0)
    side = np.where(rng.integers(0, 2, n) == 1, 1.0, -1.0)          # the product points away from zero or towards it
    a = ((1.0 + k * 2.0 ** -23) * np.exp2(e1)).astype(f32)
    b = (side * sign * 2.0 ** -24 * (1.0 - k * 2.0 ** -23) * np.exp2(e2)).astype(f32)
    odd = 2 * rng.integers(0, 2 ** 22, n) + 1
    c = (sign * (1.0 + odd * 2.0 ** -23) * np.exp2(e1 + e2)).astype(f32)
    got = check_fma(a, b, c)
    naive = (a.astype(np.float64) * b + c).astype(f32)
    assert np.all(bits32(naive) != bits32(got)), "every case must be a double-rounding case"


def test_fma32_subnormal_results():
    """Results in the float32 subnormal range, where the rounding step is 2^-149, and results that round to a signed zero."""
    rng = np.random.default_rng(2)
    n = 2000
    a = (rng.standard_normal(n) * 2.0 ** -70).astype(f32)
    b = (rng.standard_normal(n) * 2.0 ** -60).astype(f32)
    c = (rng.integers(-2 ** 23, 2 ** 23, n) * 2.0 ** -149).astype(f32)
    c[::5] = 0.0
    b[::9] *= f32(2.0 ** -30)
    got = check_fma(a, b, c)
    assert np.mean(np.abs(got) < np.finfo(f32).tiny) > 0.5


DECOMPS = [(1, 1), (1, 3), (2, 5), (4, 2), (8, 8)]       # (cs, wpc); bpw: the chunks spread over every warp


def oracle_case(g, ags, bits, zp):
    cfg = T.Config(384 if bits == 3 else 256, 2048, bits, kfactor=ags // 4, group_size=g, act_group_size=ags, zero_point=zp).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=g + ags + bits)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    return cfg, w, sc, z, A, S, G.Problem.of(cfg, w, sc, z, A, S)


def assert_rows_close(got, ref, what):
    for n in range(ref.shape[0]):
        err, bound = np.abs(got[n].astype(np.float64) - ref[n]).max(), TIGHT_TOL * np.abs(ref[n]).max()
        assert err <= bound, "%s: row %d: %.3g > %.3g" % (what, n, err, bound)


@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_model_matches_oracle(oracle, g, ags, bits, zp):
    """At every chunking and at several decompositions the model's output matches oracle.qgemm within TIGHT_TOL (it is the same sum
    in another order), on the preprocessor's symmetric table of full-precision rows and on a general table with -128 entries."""
    cfg, w, sc, z, A, S, P = oracle_case(g, ags, bits, zp)
    rng = np.random.default_rng(bits * 7 + ags)
    x = rows(rng, 3, cfg.K, ags, ("fp32", "mixed", "outlier"))
    sym = oracle.preprocessor(x, ags)
    nag = cfg.K // ags
    q = rng.integers(-128, 128, size=(2, cfg.K // 4, 16)).astype(np.int8)
    q.reshape(-1)[::37] = -128
    general = (q, np.abs(rng.standard_normal((2, nag))).astype(f32), rng.standard_normal((2, nag)).astype(f32))
    for name, (qt, ls, lb) in (("symmetric", sym), ("general", general)):
        Co = oracle.qgemm(cfg, A, S, qt, ls, lb)
        it = G.int_sums(w, bits, qt, ags)
        for cs, wpc in DECOMPS:
            y = G.gemv(P, it, ls, lb, cs, wpc, G.forced_bpw(P.nchunk, cs, wpc))
            assert_rows_close(y, Co, "%s table, cs %d wpc %d" % (name, cs, wpc))


def test_int_sums_match_oracle_plane_sums(oracle):
    """The model's integer sums are the oracle's plane sums weighted 2^b (the relation tests/test_layout_cpu.py checks through the
    stream layout), on a general table with -128 entries."""
    cfg = T.Config(256, 512, 3, kfactor=8, group_size=64, act_group_size=32).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=4)
    A, _ = T.pack_reference_layout(w, sc, z, cfg)
    q = np.random.default_rng(4).integers(-128, 128, size=(2, cfg.K // 4, 16)).astype(np.int8)
    cb = oracle.cbits(cfg, A, q).astype(np.int64)                   # [N][M*bits], reference plane rows
    r = np.arange(cfg.Mout)
    want = sum((1 << b) * cb[:, (r // 8) * 8 * cfg.bits + b * 8 + r % 8] for b in range(cfg.bits))
    assert np.array_equal(G.int_sums(w, cfg.bits, q, cfg.act_group_size).sum(axis=-1), want)


# ---- detection power: the GPU suite's grid tensors and rows ------------------------------------------------------------------------
def grid_model(oracle, name):
    cfg, w, sc, z, x = G.grid_problem(name)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    P = G.Problem.of(cfg, w, sc, z, A, S)
    q, ls, lb = oracle.preprocessor(x, cfg.act_group_size)
    return P, G.int_sums(w, cfg.bits, q, cfg.act_group_size), ls, lb


def share(a, b):
    return float(np.mean(bits32(a) != bits32(b)))


@pytest.mark.parametrize("name", sorted(G.GRID_TENSORS))
def test_grid_decompositions_give_distinct_bits(oracle, name):
    """Every pair of decompositions the GPU grid forces either has the same summation tree (gemv_order.order_tree) and the same
    model output, or differs in at least 10 % of the output bits on the grid's rows: a kernel that ran another decomposition than
    the one it reports, or split the chunks another way, fails the GPU comparison."""
    P, it, ls, lb = grid_model(oracle, name)
    outs, trees = {}, {}
    for cs, wpc in G.GRID:
        bpw = G.forced_bpw(P.nchunk, cs, wpc)
        outs[cs, wpc], trees[cs, wpc] = G.gemv(P, it, ls, lb, cs, wpc, bpw), G.order_tree(P.nchunk, cs, wpc, bpw)
    assert len(set(trees.values())) >= (3 if P.nchunk == 3 else 20)
    for a, b in itertools.combinations(G.GRID, 2):
        if trees[a] == trees[b]:
            assert share(outs[a], outs[b]) == 0, (a, b)
        else:
            assert share(outs[a], outs[b]) >= 0.10, (a, b, share(outs[a], outs[b]))


def applies(variant, P, cs, wpc, bpw):
    """Whether the variant changes the operations at this decomposition: a reversed reduction needs 3 non-zero terms (two commute),
    a split fold fma 2 act groups per chunk (the first fma adds +0), a split scale fma 2 chunks per warp or a zero point."""
    busy = lambda g: g * bpw < P.nchunk
    if variant == "rev_warps":
        return max(sum(busy(k * wpc + w) for w in range(wpc)) for k in range(cs)) >= 3
    if variant == "rev_ranks":
        return sum(busy(k * wpc) for k in range(cs)) >= 3
    if variant == "muladd_fold":
        return P.ck // P.cfg.act_group_size >= 2
    if variant == "muladd_scale":
        return bpw >= 2 or P.z is not None
    return True


@pytest.mark.parametrize("variant", G.VARIANTS)
def test_grid_rows_expose_every_variant(oracle, variant):
    """Each defect of gemv_order.VARIANTS -- reversed warp or rank order, mul+add in place of either fma, LUT biases carried in
    fp16 -- changes at least 10 % of the output bits at every grid decomposition where it changes the operations at all, and it
    does so on at least one grid tensor at 10 or more decompositions."""
    seen = 0
    for name in sorted(G.GRID_TENSORS):
        P, it, ls, lb = grid_model(oracle, name)
        for cs, wpc in G.GRID:
            bpw = G.forced_bpw(P.nchunk, cs, wpc)
            if not applies(variant, P, cs, wpc, bpw):
                continue
            s = share(G.gemv(P, it, ls, lb, cs, wpc, bpw, variant=variant), G.gemv(P, it, ls, lb, cs, wpc, bpw))
            assert s >= 0.10, (name, cs, wpc, s)
            seen += 1
    assert seen >= 10


def test_fp16_bias_sum_hides_inside_the_tolerance_gates(oracle):
    """The gap the bit comparison closes: carrying a chunk's LUT-bias sum in fp16 changes nearly every output bit of a W4 g128/a128
    tensor without a zero point (fp16-rounded inputs, as the rest of the suite draws them), yet stays within TIGHT_TOL of the oracle
    per row and within an NMSE of 1e-8 -- the gates the fp path had before the model."""
    cfg = T.Config(256, 4096, 4, kfactor=32, group_size=128, act_group_size=128).resolved()
    w, sc, z, x = T.make_problem(cfg, seed=1, N=2)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    P = G.Problem.of(cfg, w, sc, z, A, S)
    q, ls, lb = oracle.preprocessor(x, cfg.act_group_size)
    Co = oracle.qgemm(cfg, A, S, q, ls, lb)
    it = G.int_sums(w, cfg.bits, q, cfg.act_group_size)
    for cs, wpc in ((1, 8), (4, 8), (8, 4)):
        bpw = G.forced_bpw(P.nchunk, cs, wpc)
        bad = G.gemv(P, it, ls, lb, cs, wpc, bpw, variant="lb_f16")
        assert share(bad, G.gemv(P, it, ls, lb, cs, wpc, bpw)) >= 0.9
        assert_rows_close(bad, Co, "lb_f16, cs %d wpc %d" % (cs, wpc))
        assert T.nmse(Co, bad) <= 1e-8
