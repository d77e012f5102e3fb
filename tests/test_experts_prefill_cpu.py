"""CPU suite: the routed-expert prefill entry points refuse to run without a CUDA device -- there is no CPU fallback."""
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
def test_prefill_experts_fail_with_a_message_without_a_device():
    lib = tb.load()
    handles = (C.c_int64 * 2)(1, 2)
    B, G = np.zeros((1, 128), np.float32), np.zeros((1, 2, 128), np.float32)
    ids, w, out = np.zeros((1, 2), np.int32), np.full((1, 2), 0.5, np.float32), np.zeros((1, 2, 64), np.float32)
    outs = (C.c_void_p * 1)(out.ctypes.data)
    assert lib.tmac_b200_prefill_experts(handles, 1, 2, 1, tb.F32, B.ctypes.data, ids.ctypes.data, 2, outs) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
    assert lib.tmac_b200_prefill_experts_glu(handles, 2, 1, tb.F32, G.ctypes.data, G.ctypes.data, ids.ctypes.data, w.ctypes.data, 2,
                                             None, out.ctypes.data) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
