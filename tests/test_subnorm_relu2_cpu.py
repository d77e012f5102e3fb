"""CPU suite: tmac_b200_gemv_subnorm_relu2 and tmac_b200_prefill_subnorm_relu2 refuse to run without a CUDA device -- there is no CPU
fallback -- and the decode harness rejects the option combinations it does not build (before anything touches a device)."""
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
@pytest.mark.parametrize("name", ["tmac_b200_gemv_subnorm_relu2", "tmac_b200_prefill_subnorm_relu2"])
def test_fails_with_a_message_without_a_device(name):
    lib = tb.load()
    G, w, R = np.zeros((2, 128), np.float32), np.ones(128, np.float32), np.zeros((2, 64), np.float32)
    out = np.zeros((2, 64), np.float32)
    assert getattr(lib, name)(1, 2, tb.F32, G.ctypes.data, G.ctypes.data, w.ctypes.data, 1e-5, R.ctypes.data, out.ctypes.data) == -1
    assert b"no CUDA device" in lib.tmac_b200_last_error()


@pytest.mark.parametrize("kw", [dict(ffn_act="relu2"), dict(ffn_act="relu2", fused_ops=True), dict(ffn_act="gelu", sub_norms=True),
                                dict(kv_heads=3), dict(kv_heads=0), dict(kv_heads=8)],
                         ids=["relu2-without-sub-norms", "relu2-fused-without-sub-norms", "unknown-act", "kv-heads-3-of-4",
                              "kv-heads-0", "kv-heads-8-of-4"])
def test_harness_rejects(kw):
    pytest.importorskip("torch")
    from decode_harness import DecodeLayer, DecodeModel
    with pytest.raises(ValueError):
        DecodeLayer(512, 1408, 4, 2, False, seed=0, **kw)
    with pytest.raises(ValueError):
        DecodeModel(1, 512, 1408, 4, 2, False, ctx=8, **kw)
