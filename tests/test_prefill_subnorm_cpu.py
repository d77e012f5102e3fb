"""CPU suite: tmac_b200_prefill_subnorm, the prompt-sized form of gemv_subnorm, refuses to run without a CUDA device -- there is no
CPU fallback."""
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
def test_prefill_subnorm_fails_with_a_message_without_a_device():
    lib = tb.load()
    G, w, R = np.zeros((2, 128), np.float32), np.ones(128, np.float32), np.zeros((2, 64), np.float32)
    out = np.zeros((2, 64), np.float32)
    assert lib.tmac_b200_prefill_subnorm(1, 2, tb.F32, G.ctypes.data, G.ctypes.data, w.ctypes.data, 1e-5, R.ctypes.data,
                                         out.ctypes.data) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
