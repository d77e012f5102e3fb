"""Helpers of the fused-input GPU suites (the transformed-input calls in both forms and the routed experts at prefill sizes): library
knobs for a block, the call dtype of a torch dtype, a tensor's block rows, the tile check, the dense tile call the prefill forms are
compared against, and an order of the sum of squares that the calls do not use."""
import contextlib

import numpy as np
import pytest

import tmac_b200 as tb

torch = pytest.importorskip("torch")

KNOB_DEFAULTS = {"prefill16": 1, "prefill_min_n": 0, "cs": 0, "wpc": 0}


@contextlib.contextmanager
def knobs(**kv):
    """Set library knobs for the block, then put back their defaults."""
    for k, v in kv.items():
        tb.debug_set(k, v)
    try:
        yield
    finally:
        for k in kv:
            tb.debug_set(k, KNOB_DEFAULTS[k])


def tdt(dtype):
    return tb.F16 if dtype == torch.float16 else tb.F32


def bm_of(M, bits):
    return next(b for b in ((192, 384, 576, 768) if bits == 3 else (256, 128, 512, 1024, 320, 640)) if (M * bits) % b == 0)


def launched(t16, N):
    launch = tb.last_launch()
    assert launch["cluster"] == (16 if t16 else 1) and launch["batch"] == -N, launch


def dense_tile(wt, X, t16, dtype=torch.float32):
    """tmac_b200_gemv of the rows X (device [n][K]) passed as dtype on the fp16 (t16) or the int8 tile: numpy [n][Mout].  Fewer than 64
    rows on the fp16 tile are padded to 64 with copies of the first."""
    n = X.shape[0]
    pad = max(0, 64 - n) if t16 else 0
    if pad:
        X = torch.cat([X, X[:1].expand(pad, -1)])
    out = torch.full((n + pad, wt.cfg.M), float("nan"), device="cuda", dtype=dtype)
    with knobs(prefill_min_n=1, prefill16=int(t16)):
        tb.gemv(wt, n + pad, X.to(dtype).contiguous(), out, dtype=tdt(dtype))
        launched(t16, n + pad)
    torch.cuda.synchronize()
    return out[:n].cpu().numpy()


def serial_input(x, w, eps):
    """rmsnorm(x) * w with the sum of squares of the 4-groups taken serially: an order the calls do not use."""
    g = x.reshape(-1, 4)
    q = (g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + (g[:, 2] * g[:, 2] + g[:, 3] * g[:, 3])
    s = np.float32(0.0)
    for v in q:
        s = np.float32(s + v)
    return (x * (np.float32(1.0) / np.sqrt(s / np.float32(x.size) + np.float32(eps)))) * w
