"""gemv_order.py -- TEST INFRASTRUCTURE: numpy model of the fp32 operation order of gemv3_kernel's fp path (act_group_size < K),
t-mac_b200/csrc/tmac_kernels.cuh.  Given the plain problem (weight codes, scales, zero points), a table (QLUT, LUT scales, LUT biases)
and the launch's decomposition (cluster size cs, warps per CTA wpc, chunks per warp bpw), it returns the kernel's output bit for bit:

  integer sum per act group  iacc[n][r][a] = sum_b 2^b * sum_{K-group g in a} QLUT[n][g][idx_b(r, g)]   (all 16 entries as given)
  chunk c (TMAC_BLOCK_LOOKUPS, TMAC_GROUP_FOLD, TMAC_BLOCK_SCALES)
                             facc = +0;  facc = fma(ls[a], (float)iacc, facc)     over the chunk's act groups, ascending
                             lbsum = +0; lbsum = lbsum + lb[a]                    ascending
                             cacc = fma(0.5 * s[r][c], facc + lbsum, cacc);  with a zero point then cacc = fma(z[r][c], lbsum, cacc)
  warps                      warp w of cluster rank k owns chunks [(k*wpc + w)*bpw, +bpw) of [0, nchunk); its cacc starts at +0
  CTA reduction              t = +0; t += cacc_w for w = 0 .. wpc-1
  cluster reduction          y = +0; y += t_k for k = 0 .. cs-1 (the leader)
  output                     y, or y rounded once to fp16

s[r][c] is the scale of the weight group that holds chunk c (one_scale: the tensor's one scale).  The chunk's K extent comes from the
stream layout (tmac_b200_debug_encode, host only).  Every fp32 operation is emulated exactly: additions are numpy float32 additions
(IEEE round to nearest even), and fma32 rounds the exact a*b + c once.

`variant` restates the order with one plausible defect, for the CPU suite's detection-power tests (tests/test_gemv_order_cpu.py):
  rev_warps    the CTA reduction adds the warps from wpc-1 down to 0
  rev_ranks    the leader adds the cluster ranks from cs-1 down to 0
  muladd_fold  facc = ls * iacc + facc as a rounded multiply and a rounded add
  muladd_scale cacc = 0.5*s * (facc + lbsum) + cacc (and z * lbsum + cacc) as rounded multiplies and adds
  lb_f16       the chunk's LUT-bias sum carried in fp16"""
import ctypes as C

import numpy as np

import tmac_b200 as tb
import tmac_oracle as T

f32, f64 = np.float32, np.float64
VARIANTS = ("rev_warps", "rev_ranks", "muladd_fold", "muladd_scale", "lb_f16")


def fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays: a*b + c rounded once to float32 (round to nearest even).

    The float64 product of two float32 values is exact (24 + 24 <= 53 significand bits; products of float32 values stay far inside
    the float64 normal range), so s = fl64(p + c) with the TwoSum error e = (p + c) - s holds the exact sum s + e.  Rounding s to
    float32 rounds s + e the same way unless s lies exactly on a float32 midpoint: every float32 midpoint is a float64 number, so
    a midpoint strictly between s and s + e would be closer to s + e than s is.  On a midpoint with e != 0 the exact value lies on
    e's side of it, and that neighbour is the result."""
    a, b, c = (np.asarray(v, f32) for v in (a, b, c))
    p = a.astype(f64) * b.astype(f64)
    c64 = c.astype(f64)
    s = p + c64
    bv = s - p
    e = (p - (s - bv)) + (c64 - bv)
    r = s.astype(f32)
    r64 = r.astype(f64)
    other = np.nextafter(r, np.where(s > r64, f32(np.inf), f32(-np.inf)).astype(f32))
    mid = (s != r64) & (s == (r64 + other.astype(f64)) * 0.5)
    toward = (other.astype(f64) - r64) * e > 0
    return np.where(mid & toward, other, r).astype(f32)


def layout(cfg, A, S):
    """The stream layout's 12 fields of tmac_b200_debug_encode (host only): pb, rw, rsb, nrsb, ck, qch, nchunk, sd, zp, one_scale,
    blk, wbytes."""
    k = tb.make_kcfg(cfg.Mout, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale)
    lay = (C.c_int * 12)()
    n = tb.load().tmac_b200_debug_encode(C.byref(k), A.ctypes.data, S.ctypes.data, None, 0, lay)
    assert n > 0, tb.last_error()
    return [int(v) for v in lay]


def int_sums(w, bits, qlut, ags):
    """iacc int64 [N][Mout][K/ags]: each act group's integer sum of table entries, plane b weighted 2^b (T.plane_indices order)."""
    Mout, K = w.shape
    qlut = np.asarray(qlut, np.int8).reshape(-1, K // 4, 16)
    idx = T.plane_indices(w, bits).astype(np.int64)                 # [Mout][bits][K/4]
    base = np.arange(K // 4, dtype=np.int64) * 16
    out = np.zeros((qlut.shape[0], Mout, K // ags), np.int64)
    for n, tab in enumerate(qlut):
        flat = tab.reshape(-1).astype(np.int64)
        acc = np.zeros((Mout, K // 4), np.int64)
        for b in range(bits):
            acc += flat[base[None, :] + idx[:, b, :]] << b
        out[n] = acc.reshape(Mout, K // ags, ags // 4).sum(axis=-1)
    return out


class Problem:
    """The weight side of the model: codes w [Mout][K], scales and zero points [Mout][K/group_size] (as uploaded), and the chunk
    size ck of the tensor's stream layout."""

    def __init__(self, cfg, w, sc, z, ck):
        self.cfg, self.w, self.ck = cfg, w, ck
        self.nchunk = cfg.K // ck
        if cfg.one_scale:
            s = np.full((cfg.Mout, self.nchunk), np.asarray(sc, f32).reshape(-1)[0], f32)
        else:
            per = cfg.group_size // ck                               # chunks per weight group (the layout keeps ck <= group_size)
            assert per >= 1 and cfg.group_size % ck == 0
            s = np.repeat(np.asarray(sc, f32), per, axis=1)
        self.half_s = (f32(0.5) * s).astype(f32)                     # 0.5f * s: exact
        self.z = np.repeat(np.asarray(z, f32), cfg.group_size // ck, axis=1) if cfg.zero_point else None

    @classmethod
    def of(cls, cfg, w, sc, z, A, S):
        return cls(cfg, w, sc, z, layout(cfg, A, S)[4])


def chunk_terms(prob, iacc, ls, lb, variant=None):
    """Per chunk: facc [N][Mout][nchunk] and lbsum [N][1][nchunk]."""
    cfg = prob.cfg
    ags, nchunk = cfg.act_group_size, prob.nchunk
    napc = prob.ck // ags                                            # act groups per chunk
    N, Mout = iacc.shape[0], cfg.Mout
    it = iacc.reshape(N, Mout, nchunk, napc).astype(f32)             # |iacc| < 2^24: exact
    lsc = np.asarray(ls, f32).reshape(N, 1, nchunk, napc)
    lbc = np.asarray(lb, f32).reshape(N, 1, nchunk, napc)
    facc = np.zeros((N, Mout, nchunk), f32)
    lbsum = np.zeros((N, 1, nchunk), np.float16 if variant == "lb_f16" else f32)
    for j in range(napc):
        if variant == "muladd_fold":
            facc = (lsc[..., j] * it[..., j]).astype(f32) + facc
        else:
            facc = fma32(lsc[..., j], it[..., j], facc)
        lbsum = lbsum + lbc[..., j].astype(lbsum.dtype)
    return facc, lbsum.astype(f32)


def gemv(prob, iacc, ls, lb, cs, wpc, bpw, f16=False, variant=None):
    """The kernel's output [N][Mout] (float32, or float16 with f16) for integer sums iacc = int_sums(...), LUT scales ls and biases
    lb [N][K/ags] and the decomposition (cs, wpc, bpw)."""
    assert variant in (None,) + VARIANTS, variant
    nchunk = prob.nchunk
    nw = cs * wpc
    assert nw * bpw >= nchunk, (cs, wpc, bpw, nchunk)
    facc, lbsum = chunk_terms(prob, iacc, ls, lb, variant)
    N, Mout = facc.shape[:2]
    cacc = np.zeros((N, Mout, nw), f32)
    for i in range(bpw):
        c = np.arange(nw) * bpw + i
        live = c < nchunk
        cc = np.minimum(c, nchunk - 1)
        t = (facc[..., cc] + lbsum[..., cc]).astype(f32)
        hs = prob.half_s[None, :, cc]
        if variant == "muladd_scale":
            v = (hs * t).astype(f32) + cacc
            if prob.z is not None:
                v = (prob.z[None, :, cc] * lbsum[..., cc]).astype(f32) + v
        else:
            v = fma32(hs, t, cacc)
            if prob.z is not None:
                v = fma32(prob.z[None, :, cc], np.broadcast_to(lbsum[..., cc], v.shape), v)
        cacc = np.where(live, v, cacc).astype(f32)
    ranks = []
    for k in range(cs):
        t = np.zeros((N, Mout), f32)
        for w in (reversed(range(wpc)) if variant == "rev_warps" else range(wpc)):
            t = t + cacc[..., k * wpc + w]
        ranks.append(t)
    y = np.zeros((N, Mout), f32)
    for k in (reversed(range(cs)) if variant == "rev_ranks" else range(cs)):
        y = y + ranks[k]
    return y.astype(np.float16) if f16 else y


def gemv_table(prob, qlut, ls, lb, cs, wpc, bpw, f16=False, variant=None):
    """gemv() from a table (QLUT [N][K/4][16], LUT scales, LUT biases)."""
    return gemv(prob, int_sums(prob.w, prob.cfg.bits, qlut, prob.cfg.act_group_size), ls, lb, cs, wpc, bpw, f16, variant)


def order_tree(nchunk, cs, wpc, bpw):
    """The summation tree of a decomposition, normalised so that two decompositions have equal trees exactly when the model gives
    them the same operations: a warp is the tuple of its chunks; a sum node ('+', x0, x1, ...) is ((+0 + x0) + x1) + ...  A warp
    without chunks contributes +0 and drops out, a sum of one term is that term (+0 + x = x: no term is -0), and a sum whose first
    term is itself a sum continues it."""
    def fold(items):
        items = [x for x in items if x != ()]
        if not items:
            return ()
        if len(items) == 1:
            return items[0]
        if items[0][0] == "+":
            return items[0] + tuple(items[1:])
        return ("+",) + tuple(items)

    def warp(g):
        return tuple(range(g * bpw, min(nchunk, (g + 1) * bpw)))
    return fold([fold([warp(k * wpc + w) for w in range(wpc)]) for k in range(cs)])


# ---- the problems of the GPU suite's decomposition grid (tests/test_gpu_gemv_order.py), shared with the CPU suite's detection tests
# name -> (Mout, K, bits, group_size, act_group_size, zero_point).  37 chunks, so that no cs * wpc divides the work evenly; K = 96 is
# 3 chunks, so that most of the grid has idle warps and idle CTAs.
GRID_TENSORS = {"w2_g128_a64_zp": (256, 4736, 2, 128, 64, True), "w4_g128_a128": (256, 4736, 4, 128, 128, False),
                "w1_g32_a32": (256, 1184, 1, 32, 32, False), "w1_g32_a32_k96": (256, 96, 1, 32, 32, False),
                "w3_g64_a32_zp": (384, 2368, 3, 64, 32, True)}
GRID = [(cs, wpc) for cs in (1, 2, 4, 8) for wpc in range(1, 9)]
GRID_KINDS = ("fp32", "mixed", "outlier")


def grid_cfg(name):
    Mout, K, bits, g, ags, zp = GRID_TENSORS[name]
    return T.Config(Mout, K, bits, kfactor=ags // 4, group_size=g, act_group_size=ags, zero_point=zp).resolved()


def grid_problem(name):
    """(cfg, w, scales, zeros, rows x [3][K]) of a grid tensor, seeded by its name."""
    import act_rows
    cfg = grid_cfg(name)
    seed = sum(map(ord, name))
    w, sc, z, _ = T.make_problem(cfg, seed=seed)
    return cfg, w, sc, z, act_rows.rows(np.random.default_rng(seed), len(GRID_KINDS), cfg.K, cfg.act_group_size, GRID_KINDS)


def forced_bpw(nchunk, cs, wpc):
    """Chunks per warp of a launch whose cs and wpc are forced: the chunks spread over every warp of the cluster."""
    return -(-nchunk // (cs * wpc))
