"""Activation rows that expose the summation order of the LUT builder (tests/test_lut_order_cpu.py, tests/test_gpu_full_precision.py).

The rest of the suite draws activations as fp16-rounded standard normals.  Almost every fp32 sum of a dozen such values is exact, so
the order in which the LUT builder adds them (DESIGN.md section 1: the abs-sum (|a0|+|a1|)+(|a2|+|a3|), the entries ((b0+-b1)+-b2)+-b3,
the _mm256_addv_ps tree, the serial sum over 32-activation blocks) does not show in its LUT scales and biases.  None of the kinds
here rounds to fp16, so those sums round and a re-associated sum gives other bits.

Kinds (one per row):
  fp32     standard normal drawn in float32
  mixed    fp32 standard normal times 2**e per K-group of 4 activations, e uniform in [-20, 12]: every add across K-groups rounds
  zero     fp32 standard normal with a +0.0 unit at the start and at the end and a -0.0 unit in the middle; the unit is an activation
           group when the row has at least 3 of them, else a 32-activation block
  outlier  fp32 standard normal with one activation per activation group multiplied by 2**12
  ties     every activation group has LUT scale exactly 1.0: its first K-group is (+-127, 0, 0, 0), every other K-group holds one
           odd multiple of 0.5 and three integers, so each of their table entries is a half-integer and the int8 rounding (round half
           to even) decides every byte
The fp16 variant (rows16) rounds the same kinds to fp16 and adds
  fp16_edge   fp16 subnormals, values within 2**9 of +-2**15 and ordinary values, mixed inside every K-group
  fp16_order  standard normal, except that one K-group per activation group is (+-2**15, 0, +-2**-9, +-2**-9): its abs-sum is the
              group's largest, and (2**15 + 0) + (2**-9 + 2**-9) = 2**15 + 2**-8 while ((2**15 + 0) + 2**-9) + 2**-9 rounds (half to
              even, twice) to 2**15, so the serial abs-sum changes the LUT scale of every activation group.  fp16 rows of the other
              kinds add exactly in nearly every abs-sum; at small K and at ags = K none of their scales sees that re-association."""
import numpy as np

KINDS = ("fp32", "mixed", "zero", "outlier", "ties")
KINDS16 = KINDS + ("fp16_edge", "fp16_order")


def _row(rng, K, ags, kind):
    nag = K // ags
    if kind == "fp32":
        return rng.standard_normal(K, dtype=np.float32)
    if kind == "mixed":
        e = rng.integers(-20, 13, size=K // 4)
        return (rng.standard_normal((K // 4, 4), dtype=np.float32) * np.exp2(e).astype(np.float32)[:, None]).reshape(K)
    if kind == "zero":
        x = rng.standard_normal(K, dtype=np.float32)
        unit = ags if nag >= 3 else 32
        n = K // unit
        x[:unit] = 0.0
        x[(n - 1) * unit:] = 0.0
        x[(n // 2) * unit:(n // 2 + 1) * unit] = -0.0
        return x
    if kind == "outlier":
        x = rng.standard_normal(K, dtype=np.float32)
        pos = np.arange(nag) * ags + rng.integers(0, ags, size=nag)
        x[pos] *= np.float32(4096.0)
        return x
    if kind == "ties":
        g = rng.integers(-8, 9, size=(K // 4, 4)).astype(np.float32)
        half = rng.integers(0, 4, size=K // 4)                                     # which activation of the K-group is the half-integer
        g[np.arange(K // 4), half] = (2 * rng.integers(-8, 8, size=K // 4) + 1) * np.float32(0.5)   # odd multiples of 0.5, |v| <= 7.5
        first = np.arange(nag) * (ags // 4)
        g[first] = 0.0
        g[first, 0] = np.where(rng.integers(0, 2, size=nag) == 1, 127.0, -127.0)   # abs-sum 127 -> scale 1.0; the others' is <= 31.5
        return g.reshape(K)
    if kind == "fp16_edge":
        sub = rng.integers(-1023, 1024, size=K).astype(np.float32) * np.float32(2.0 ** -24)      # fp16 subnormals (and zeros)
        big = np.where(rng.integers(0, 2, size=K) == 1, 1.0, -1.0).astype(np.float32) * (32768.0 + 32.0 * rng.integers(-16, 17, size=K)).astype(np.float32)
        pick = rng.integers(0, 3, size=K)
        return np.where(pick == 0, sub, np.where(pick == 1, big, rng.standard_normal(K, dtype=np.float32))).astype(np.float32)
    if kind == "fp16_order":
        x = rng.standard_normal(K, dtype=np.float32)
        k0 = np.arange(nag) * ags + 4 * rng.integers(0, ags // 4, size=nag)     # first activation of the chosen K-group
        sign = np.where(rng.integers(0, 2, size=(nag, 3)) == 1, 1.0, -1.0).astype(np.float32)
        x[k0] = sign[:, 0] * np.float32(2.0 ** 15)
        x[k0 + 1] = 0.0
        x[k0 + 2] = sign[:, 1] * np.float32(2.0 ** -9)
        x[k0 + 3] = sign[:, 2] * np.float32(2.0 ** -9)
        return x
    raise ValueError("unknown kind %r" % kind)


def rows(rng, N, K, ags, kinds=KINDS):
    """[N][K] float32 activation rows, row n of kind kinds[n % len(kinds)]; ags = the activation group size they are laid out for."""
    assert K % ags == 0 and ags % 32 == 0
    return np.stack([_row(rng, K, ags, kinds[n % len(kinds)]) for n in range(N)]).astype(np.float32)


def rows16(rng, N, K, ags, kinds=KINDS16):
    """The fp16 variant: float32 rows whose values are fp16-representable (pass .astype(np.float16) to an F16 call)."""
    return rows(rng, N, K, ags, kinds).astype(np.float16).astype(np.float32)
