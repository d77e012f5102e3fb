"""CPU suite: the LUT builder's summation order, restated in numpy, against the oracle -- and the power of the activation rows of
tests/act_rows.py to tell that order from a re-associated one.

DESIGN.md section 1 promises the reference's order bit for bit: the abs-sum (|a0|+|a1|)+(|a2|+|a3|) whose maximum over the
activation group / 127 is the LUT scale, the odd entries ((b0+-b1)+-b2)+-b3, the _mm256_addv_ps tree over the LUT[0] of a
32-activation block, and the serial sum of those block sums from 0 that is the LUT bias.  The GPU gates on full-precision rows
(tests/test_gpu_full_precision.py) only catch a re-associated kernel if the rows make the sums round; the second test here keeps
them that way."""
import numpy as np
import pytest

from act_rows import KINDS, rows, rows16

f32 = np.float32


def abs_sum_ref(a):
    return (a[..., 0] + a[..., 1]) + (a[..., 2] + a[..., 3])


def abs_sum_serial(a):
    return ((a[..., 0] + a[..., 1]) + a[..., 2]) + a[..., 3]


def entries_ref(b, s1, s2, s3):
    return ((b[..., 0] + s1 * b[..., 1]) + s2 * b[..., 2]) + s3 * b[..., 3]


def entries_pairs(b, s1, s2, s3):
    return (b[..., 0] + s1 * b[..., 1]) + (s2 * b[..., 2] + s3 * b[..., 3])


def addv8_ref(v):
    r = [v[..., 4 + i] + v[..., i] for i in range(4)]
    return (r[0] + r[2]) + (r[1] + r[3])


def addv8_serial(v):
    acc = v[..., 0]
    for i in range(1, 8):
        acc = acc + v[..., i]
    return acc


def blocks_ref(blk):
    acc = np.zeros(blk.shape[:-1], f32)
    for j in range(blk.shape[-1]):
        acc = acc + blk[..., j]
    return acc


def blocks_pairwise(blk):
    while blk.shape[-1] > 1:
        n = blk.shape[-1]
        s = blk[..., 0:n - 1:2] + blk[..., 1:n:2]
        blk = np.concatenate([s, blk[..., n - 1:]], axis=-1) if n % 2 else s
    return blk[..., 0]


def lut(x, ags, abs_sum=abs_sum_ref, entries=entries_ref, addv8=addv8_ref, blocks=blocks_ref):
    """x [N][K] float32 -> (QLUT int8 [N][K/4][16], LUT scales [N][K/ags], LUT biases [N][K/ags]); every operation in float32."""
    N, K = x.shape
    nag = K // ags
    b = x.reshape(N, K // 4, 4).astype(f32)
    m = abs_sum(np.abs(b)).reshape(N, nag, ags // 4).max(axis=-1)
    scale = m / f32(127)
    ts = np.divide(f32(1), scale, out=np.zeros_like(scale), where=scale != 0)
    tab = np.zeros((N, K // 4, 16), f32)
    for i in range(8):
        idx = 2 * i + 1
        s = [f32(1) if idx & bit else f32(-1) for bit in (2, 4, 8)]
        od = entries(b, *s)
        tab[..., idx] = od
        tab[..., 14 - 2 * i] = -od
    q = np.clip(np.rint(tab * np.repeat(ts, ags // 4, axis=1)[..., None]), -128, 127).astype(np.int8)
    blk = addv8(tab[..., 0].reshape(N, K // 32, 8))
    bias = blocks(blk.reshape(N, nag, ags // 32))
    return q, scale.astype(f32), bias.astype(f32)


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


# (K, act group sizes): 8640 = 270 blocks of 32 takes no 128
SHAPES = [(4096, (32, 64, 128, 4096)), (3200, (32, 64, 128, 3200)), (8640, (32, 64, 8640))]


@pytest.mark.parametrize("K,agss", SHAPES, ids=["k%d" % s[0] for s in SHAPES])
@pytest.mark.parametrize("kind", KINDS + ("fp16_edge", "fp16_order"))
def test_restatement_equals_oracle_bit_for_bit(oracle, kind, K, agss):
    """The restatement above is the order the oracle (and, through the GPU gates, every kernel) computes: its QLUT bytes, LUT scales
    and LUT biases equal oracle.preprocessor's on every kind of row, at every act group size.  The rows make the sums round, so a
    restatement in another order would differ (the tests below); equality pins this one."""
    make = rows16 if kind.startswith("fp16") else rows
    for ags in agss:
        x = make(np.random.default_rng(K + ags), 4, K, ags, (kind,))
        q, ls, lb = lut(x, ags)
        qo, lso, lbo = oracle.preprocessor(x, ags)
        assert np.array_equal(q, qo), "QLUT bytes, ags %d" % ags
        assert np.array_equal(bits(ls), bits(lso)), "LUT scales, ags %d" % ags
        assert np.array_equal(bits(lb), bits(lbo)), "LUT biases, ags %d" % ags


REASSOCIATIONS = {
    "abs_sum_serial": (dict(abs_sum=abs_sum_serial), (32, 64, 128)),
    "entries_pairs": (dict(entries=entries_pairs), (32, 64, 128)),
    "addv8_serial": (dict(addv8=addv8_serial), (32, 64, 128)),
    "blocks_pairwise": (dict(blocks=blocks_pairwise), (128, 4096)),     # one or two blocks per act group have one order only
}


@pytest.mark.parametrize("kind", ["fp32", "mixed"])
@pytest.mark.parametrize("name", sorted(REASSOCIATIONS))
def test_rows_expose_every_reassociation(kind, name):
    """Each plausible re-association of the builder changes the LUT scale or bias of at least 10 % of the activation groups of
    the fp32 and mixed rows (8 rows of K = 4096, drawn by act_rows.rows as the GPU gates draw theirs).  On fp16-rounded rows most of
    these change nothing; if a later edit of act_rows made the rows that tame, the GPU gates would stop seeing a re-associated
    kernel, and this test fails instead."""
    kw, agss = REASSOCIATIONS[name]
    for ags in agss:
        x = rows(np.random.default_rng(1), 8, 4096, ags, (kind,))
        _, ls, lb = lut(x, ags)
        _, ls2, lb2 = lut(x, ags, **kw)
        changed = (bits(ls) != bits(ls2)) | (bits(lb) != bits(lb2))
        assert changed.mean() >= 0.10, "%s on %s rows, ags %d: %d of %d act groups changed" % (name, kind, ags, changed.sum(), changed.size)


G1_SHAPES = [(K, ags) for K in (256, 3200, 4096, 8640, 18944) for ags in (32, 64, 128, K) if K % ags == 0]


@pytest.mark.parametrize("K,ags", G1_SHAPES, ids=["k%d_a%d" % s for s in G1_SHAPES])
def test_fp16_order_rows_expose_the_abs_sum_order(K, ags):
    """The fp16 G1 gates (tests/test_gpu_full_precision.py, F16 inputs) see a re-associated abs-sum through the fp16_order rows:
    with ((|a0|+|a1|)+|a2|)+|a3| every activation group of such a row gets another LUT scale, at every K and act group size those
    gates run, including small K and ags = K, where the other fp16 kinds leave every scale unchanged."""
    x = rows16(np.random.default_rng(K + ags), 2, K, ags, ("fp16_order",))
    assert np.array_equal(x.astype(np.float16).astype(np.float32), x)
    _, ls, _ = lut(x, ags)
    _, ls2, _ = lut(x, ags, abs_sum=abs_sum_serial)
    assert np.all(bits(ls) != bits(ls2))
