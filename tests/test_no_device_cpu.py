"""CPU suite: every transformed-input and routed-expert entry point, both forms (tmac_b200_gemv_* and tmac_b200_prefill_*), refuses
to run without a CUDA device -- there is no CPU fallback -- and leaves its outputs untouched."""
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


K, M, N, TOPK = 128, 64, 2, 2
H, W, R = np.zeros((N, K), np.float32), np.ones(K, np.float32), np.zeros((N, M), np.float32)
G = np.zeros((N, TOPK, K), np.float32)
IDS, WTS = np.zeros((N, TOPK), np.int32), np.full((N, TOPK), 0.5, np.float32)
BIAS = [np.ones(M, np.float32) for _ in range(3)]


def args(call, count, outs):
    """The arguments of tmac_b200_<form>_<call> on host arrays, count tensors (experts: count tensors of 2 experts), into outs."""
    p = lambda a: a.ctypes.data
    handles = (C.c_int64 * (2 * count))(*range(1, 2 * count + 1))
    O = (C.c_void_p * count)(*[p(o) for o in outs])
    B = (C.c_void_p * count)(*[p(b) for b in BIAS[:count]])
    return {"rmsnorm": (handles, count, N, tb.F32, p(H), p(W), 1e-5, O),
            "rmsnorm_bias": (handles, count, N, tb.F32, p(H), p(W), 1e-5, B, O),
            "glu": (1, N, tb.F32, p(H), p(H), p(R), p(outs[0])),
            "residual": (1, N, tb.F32, p(H), p(R), p(outs[0])),
            "subnorm": (1, N, tb.F32, p(H), p(H), p(W), 1e-5, p(R), p(outs[0])),
            "subnorm_relu2": (1, N, tb.F32, p(H), p(H), p(W), 1e-5, p(R), p(outs[0])),
            "experts": (handles, count, 2, N, tb.F32, p(H), p(IDS), TOPK, O),
            "experts_glu": (handles, 2, N, tb.F32, p(G), p(G), p(IDS), p(WTS), TOPK, None, p(outs[0]))}[call]


CALLS = [("rmsnorm", 1), ("rmsnorm", 3), ("rmsnorm_bias", 1), ("rmsnorm_bias", 3), ("glu", 1), ("residual", 1), ("subnorm", 1),
         ("subnorm_relu2", 1), ("experts", 1), ("experts_glu", 1)]


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
@pytest.mark.parametrize("form", ["gemv", "prefill"])
@pytest.mark.parametrize("call,count", CALLS, ids=["%s-%d" % c for c in CALLS])
def test_fails_without_a_device(form, call, count):
    lib = tb.load()
    outs = [np.full((N, TOPK, M) if call == "experts" else (N, M), 7.0, np.float32) for _ in range(count)]
    assert getattr(lib, "tmac_b200_%s_%s" % (form, call))(*args(call, count, outs)) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()
    assert all((o == 7.0).all() for o in outs)
