"""CPU suite: the decode harness rejects the option combinations it does not build (squared-ReLU layers without sub-norms, an
unknown activation, KV head counts that do not divide the heads), before anything touches a device."""
import pytest


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
