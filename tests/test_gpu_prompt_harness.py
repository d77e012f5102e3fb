"""GPU suite (-m gpu): the decode harness's prompt step (DecodeLayer.prompt, DecodeModel.prompt).  A fused_ops layer (its linears in
the prefill_* forms) and a MoE layer (prefill_experts) run a prompt of P tokens and must match the same layer with dense dequantised
fp32 weights (torch matmul) within the gate of test_gpu_decode_harness.py, NMSE <= 5e-4; so must the decode step at position P that
follows the prompt.  The CUDA-graphed prompt step of a small model replays to the eager step's bits."""
import pytest

from seq_util import DENSE_NMSE, stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def nmse(got, ref):
    return float(((got - ref) ** 2).mean() / (ref ** 2).mean())


@pytest.mark.parametrize("P", [64, 77])
@pytest.mark.parametrize("experts", [0, 4], ids=["dense", "moe"])
def test_prompt_then_token_match_dense_layer(stream, experts, P):
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx = 1024, 2816, 8, 128
    layer = DecodeLayer(hidden, ffn, heads, 2, True, seed=5, fused_ops=True, experts=experts, topk=2)
    try:
        hd = hidden // heads
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref_lin = lambda n, inp, out: out.copy_(inp @ dense[n].T)
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        ang = torch.arange(P + 1, device="cuda").float()[:, None] * inv[None, :]
        cos, sin = torch.cos(ang), torch.sin(ang)
        x = torch.randn((P, hidden), device="cuda")
        kc, vc = torch.zeros((heads, ctx, hd), device="cuda"), torch.zeros((heads, ctx, hd), device="cuda")
        kc2, vc2 = kc.clone(), vc.clone()
        got = layer.prompt(x, kc, vc, cos[:P], sin[:P]).clone()
        routed = (layer.pbuf["ids"].clone(), layer.pbuf["wts"].clone()) if experts else None
        ref = layer.prompt(x, kc2, vc2, cos[:P], sin[:P], linear=ref_lin, routed=routed).clone()
        torch.cuda.synchronize()
        assert nmse(got, ref) <= DENSE_NMSE, nmse(got, ref)
        # the token at position P attends over the prompt's cache entries
        xt = torch.randn((1, hidden), device="cuda")
        tok = layer.forward(xt, kc, vc, P, cos[P:P + 1], sin[P:P + 1]).clone()
        routed = (layer.buf["ids"].clone(), layer.buf["wts"].clone()) if experts else None
        tref = layer.forward(xt, kc2, vc2, P, cos[P:P + 1], sin[P:P + 1], linear=ref_lin, routed=routed).clone()
        torch.cuda.synchronize()
        assert nmse(tok, tref) <= DENSE_NMSE, nmse(tok, tref)
    finally:
        layer.free()


@pytest.mark.parametrize("experts", [0, 4], ids=["dense", "moe"])
def test_graphed_prompt_step_replays(stream, experts):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=2, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=128, fused_ops=True, experts=experts,
                    prompt_len=96)
    try:
        with torch.cuda.stream(stream):
            m.prompt()
        torch.cuda.synchronize()
        eager = m.py.clone()
        m.capture_prompt(stream)
        m.py.zero_()
        m.prompt_graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.py, eager)
        assert m.prompt_tokens_per_s(stream, n=3) > 0
    finally:
        m.free()
