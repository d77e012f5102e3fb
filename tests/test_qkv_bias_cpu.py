"""CPU suite: tmac_b200_gemv_rmsnorm_bias and tmac_b200_prefill_rmsnorm_bias refuse to run without a CUDA device -- there is no CPU
fallback -- and leave the outputs untouched."""
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
@pytest.mark.parametrize("name", ["tmac_b200_gemv_rmsnorm_bias", "tmac_b200_prefill_rmsnorm_bias"])
@pytest.mark.parametrize("count", [1, 3])
def test_fails_with_a_message_without_a_device(name, count):
    lib = tb.load()
    handles = (C.c_int64 * count)(*range(1, count + 1))
    H, w = np.zeros((2, 128), np.float32), np.ones(128, np.float32)
    bias = [np.ones(64, np.float32) for _ in range(count)]
    outs_np = [np.full((2, 64), 7.0, np.float32) for _ in range(count)]
    outs = (C.c_void_p * count)(*[o.ctypes.data for o in outs_np])
    biases = (C.c_void_p * count)(*[b.ctypes.data for b in bias])
    assert getattr(lib, name)(handles, count, 2, tb.F32, H.ctypes.data, w.ctypes.data, C.c_float(1e-5), biases, outs) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
    assert all((o == 7.0).all() for o in outs_np)
