"""GPU suite (-m gpu): the decode harness (t-mac_b200/decode_harness.py, SURVEY 8 f1).  One decoder layer whose seven linears go
through the library must match the same layer with dense dequantised fp32 weights (torch matmul) within the reference's own
gate for this path, NMSE <= 5e-4 (python/t_mac/ops/qgemm.py:277-282) -- the remaining difference is the int8 LUT quantisation
noise the CPU kernel has too.  Also: the CUDA-graphed token step of a small model replays to the same output as the eager step."""
import pytest

from seq_util import stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_layer_matches_dense_dequant_layer(stream, bits, zp):
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx = 1024, 2816, 8, 64
    layer = DecodeLayer(hidden, ffn, heads, bits, zp, seed=3)
    try:
        hd = hidden // heads
        kc = torch.randn((heads, ctx, hd), device="cuda") * 0.3; vc = torch.randn((heads, ctx, hd), device="cuda") * 0.3
        kc2, vc2 = kc.clone(), vc.clone()
        pos = ctx - 1
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
        x = torch.randn((1, hidden), device="cuda")
        got = layer.forward(x, kc, vc, pos, cos, sin).clone()
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.forward(x, kc2, vc2, pos, cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T)).clone()
        torch.cuda.synchronize()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= 5e-4, nmse
    finally:
        layer.free()


def test_graphed_token_step_replays(stream):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=3, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=32)
    try:
        with torch.cuda.stream(stream):
            m.step()
        torch.cuda.synchronize()
        eager = m.y.clone()
        m.capture(stream)
        m.y.zero_()
        m.graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.y, eager)
        assert m.tokens_per_s(stream, n=3) > 0
    finally:
        m.free()
