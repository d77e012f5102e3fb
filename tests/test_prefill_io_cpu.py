"""CPU suite: the prefill forms of the transformed-input calls (tmac_b200_prefill_rmsnorm / _glu / _residual) refuse to run without
a CUDA device -- there is no CPU fallback."""
import ctypes as C

import numpy as np
import pytest

import tmac_b200 as tb


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_prefill_io_fail_with_a_message_without_a_device():
    lib = tb.load()
    handles = (C.c_int64 * 3)(1, 2, 3)
    H, w, R = np.zeros((2, 128), np.float32), np.ones(128, np.float32), np.zeros((2, 64), np.float32)
    out = np.zeros((2, 64), np.float32)
    outs = (C.c_void_p * 3)(*([out.ctypes.data] * 3))
    assert lib.tmac_b200_prefill_rmsnorm(handles, 3, 2, tb.F32, H.ctypes.data, w.ctypes.data, 1e-5, outs) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
    assert lib.tmac_b200_prefill_glu(1, 2, tb.F32, H.ctypes.data, H.ctypes.data, R.ctypes.data, out.ctypes.data) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
    assert lib.tmac_b200_prefill_residual(1, 2, tb.F32, H.ctypes.data, R.ctypes.data, out.ctypes.data) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
