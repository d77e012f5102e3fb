"""The prompt step of the decode harness (DecodeLayer.prompt): P tokens through a stack of decoder layers with causal attention over
cache positions [0, P), Llama-2-7B (hidden 4096, FFN 11008, 32 heads, `--layers` 32) in W2 g128 zp and W4 g128, P = 16 .. 512, in
three forms of the linears:

  prefill    the fused_ops layer's prompt step: prefill_rmsnorm([q, k, v]), prefill_residual(o), prefill_rmsnorm([gate, up]),
             prefill_glu(down, + h) -- the wgmma tiles, one launch for q/k/v and one for gate/up;
  per_linear the norm, SiLU * mul and residuals as torch ops and one tmac_b200_gemv per tensor (the dense call, which takes a tile
             from its own threshold);
  gemv_io    the same four calls in their gemv_* forms (gemv_rmsnorm, gemv_residual, gemv_glu: the GEMV kernel, whose time grows
             with P), only up to P = --gemv-max.

Each form is captured in one CUDA graph per P and replayed `--reps` times between CUDA events; the forms alternate, best of
`--rounds`.  Reported per P: ms per prompt step, prompt tokens/s, and for the prefill form the linears' share of the step's kernel
time (the library's kernels over all kernels, from a torch.profiler run made after the timed runs).  grouped_qkv: prefill_rmsnorm
of q/k/v in one launch against three single-tensor launches, over all layers, graphed.  Then a Mixtral-8x7B MoE layer stack
(`--moe-layers`, 8 experts, top-2) at P = 64 and 512: the prefill form (prefill_experts, prefill_experts_glu) against the gemv_* forms
(gemv_experts, gemv_experts_glu).  The card's name, power limit and SM clocks are read in the same run, before and after.

--bitnet: BitNet-3B instead (hidden 3200, FFN 8640, 32 heads, `--layers` 26; ternary one-scale W2 tensors with activation groups of
64, and the attention and FFN sub-norms) in the same three forms, where prefill is prefill_rmsnorm([q, k, v]), prefill_subnorm(o, + x),
prefill_rmsnorm([gate, up]), prefill_subnorm(down, + h), and gemv_io their gemv_* forms (gemv_subnorm for prefill_subnorm).

    python tools/prompt_bench.py [--layers 32] [--moe-layers 8] [--ps 16,32,64,128,512] [--formats w2zp,w4] [--gemv-max 128]
--bitnet2b: BitNet b1.58 2B4T instead (hidden 2560, FFN 6912, 20 query heads and 5 KV heads of 128, `--layers` 30, the squared-ReLU
FFN), in the same three forms: q/k/v are one stacked tensor, and the down projection is prefill_subnorm_relu2 (gemv_subnorm_relu2).

--qwen2: Qwen2-7B instead (hidden 3584, FFN 18944, 28 query heads and 4 KV heads of 128, W4 g128 with zero points, `--layers` 28,
a bias on q/k/v), in the same three forms: q/k/v are one stacked tensor (4608 rows) run by prefill_rmsnorm_bias (gemv_rmsnorm_bias).
Then one line timing that tensor of every layer at N = 256 as prefill_rmsnorm followed by a torch add of the bias against
prefill_rmsnorm_bias (graphed, alternated).

    python tools/prompt_bench.py --bitnet [--layers 26] [--ps 16,32,64,128,512] [--gemv-max 128]
    python tools/prompt_bench.py --bitnet2b [--layers 30] [--ps 16,32,64,128,512] [--gemv-max 128]
    python tools/prompt_bench.py --qwen2 [--layers 28] [--ps 16,32,64,128,512] [--gemv-max 128]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "t-mac_b200"))
import torch                                    # noqa: E402
import tmac_b200 as tb                          # noqa: E402
import decode_harness                           # noqa: E402
from decode_harness import DecodeModel          # noqa: E402

FORMATS = {"w2zp": (2, True), "w4": (4, False)}
LLAMA = dict(hidden=4096, ffn=11008, heads=32)
MIXTRAL = dict(hidden=4096, ffn=14336, heads=32, experts=8, topk=2)
BITNET = dict(hidden=3200, ffn=8640, heads=32, bits=2, zero_point=False, sub_norms=True)
BITNET2B = dict(hidden=2560, ffn=6912, heads=20, kv_heads=5, bits=2, zero_point=False, sub_norms=True, ffn_act="relu2")
QWEN2 = dict(hidden=3584, ffn=18944, heads=28, kv_heads=4, bits=4, zero_point=True, qkv_bias=True)

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=None, help="decoder layers (default 32, BitNet-3B 26, BitNet b1.58 2B4T 30, Qwen2-7B 28)")
ap.add_argument("--bitnet", action="store_true", help="BitNet-3B's prompt step instead of Llama-2-7B and Mixtral-8x7B")
ap.add_argument("--bitnet2b", action="store_true", help="BitNet b1.58 2B4T's prompt step instead of Llama-2-7B and Mixtral-8x7B")
ap.add_argument("--qwen2", action="store_true", help="Qwen2-7B's prompt step instead of Llama-2-7B and Mixtral-8x7B")
ap.add_argument("--moe-layers", type=int, default=8)
ap.add_argument("--ps", default="16,32,64,128,512")
ap.add_argument("--moe-ps", default="64,512")
ap.add_argument("--formats", default="w2zp,w4")
ap.add_argument("--gemv-max", type=int, default=128)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()
if args.layers is None:
    args.layers = 28 if args.qwen2 else 30 if args.bitnet2b else 26 if args.bitnet else 32

if not torch.cuda.is_available():
    sys.exit("prompt_bench.py needs a CUDA device")
lib = tb.load(); tb.check(lib.tmac_b200_init(0), "init")
st = torch.cuda.Stream(); torch.cuda.set_stream(st); tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                     # the timing stands without it, but says so
        q = "nvidia-smi unavailable: %s" % ex
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q}


@contextlib.contextmanager
def gemv_forms():
    """The harness's prefill_* calls swapped for their gemv_* forms, which take the same arguments."""
    names = {"prefill_rmsnorm": tb.gemv_rmsnorm, "prefill_rmsnorm_bias": tb.gemv_rmsnorm_bias, "prefill_residual": tb.gemv_residual, "prefill_glu": tb.gemv_glu,
             "prefill_subnorm": tb.gemv_subnorm, "prefill_subnorm_relu2": tb.gemv_subnorm_relu2, "prefill_experts": tb.gemv_experts, "prefill_experts_glu": tb.gemv_experts_glu}
    saved = {n: getattr(decode_harness.tb, n) for n in names}
    for n, f in names.items():
        setattr(decode_harness.tb, n, f)
    try:
        yield
    finally:
        for n, f in saved.items():
            setattr(decode_harness.tb, n, f)


def graph(fn):
    """A CUDA graph of fn after one eager call (workspaces, pointer tables, the allocator)."""
    with torch.cuda.stream(st):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        fn()
    return g


def timed(g, n):
    """ms per replay of g, n replays between CUDA events."""
    with torch.cuda.stream(st):
        g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(n):
            g.replay()
        e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def best(graphs):
    """{name: best ms per replay} over the rounds, the graphs alternating."""
    out = {k: float("inf") for k in graphs}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            out[k] = min(out[k], timed(g, args.reps))
    return out


def library_share(fn):
    """The library's kernels' share of fn's kernel time, from one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with torch.cuda.stream(st):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(st):
            fn()
        torch.cuda.synchronize()
    lib_us = all_us = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        all_us += t
        if "tmac_b200" in e.key:
            lib_us += t
    return lib_us / all_us if all_us else float("nan")


def prompt_fn(m, P, x, linear=None):
    def run():
        h = x
        for i, layer in enumerate(m.layers):
            lin = None if linear is None else (lambda n, inp, out, layer=layer: layer.lin[n](inp, out))
            h = layer.prompt(h, m.kc[i], m.vc[i], m.pcos[:P], m.psin[:P], linear=lin)
    return run


def qkv_bias_pair(m, P):
    """Every layer's stacked q/k/v tensor at N = P: prefill_rmsnorm then a torch add of the bias, against prefill_rmsnorm_bias, graphed
    and alternated.  The two outputs of the last layer must be equal bit for bit (F32, the same tile)."""
    lays = m.layers
    x = torch.randn((P, m.hidden), device="cuda")
    outs = {k: torch.zeros((P, lays[0].lin["qkv"].mout), device="cuda") for k in ("add", "bias")}

    def add():
        for l in lays:
            tb.prefill_rmsnorm([l.lin["qkv"].wt], P, x, l.norm1, l.EPS, [outs["add"]])
            outs["add"].add_(l.qkv_b["qkv"])

    def bias():
        for l in lays:
            tb.prefill_rmsnorm_bias([l.lin["qkv"].wt], P, x, l.norm1, l.EPS, [l.qkv_b["qkv"]], [outs["bias"]])
    ms = best({"prefill_rmsnorm_plus_add": graph(add), "prefill_rmsnorm_bias": graph(bias)})
    print(json.dumps({"model": "qwen2_7b", "qkv_bias_P": P, "rows": lays[0].lin["qkv"].mout, "K": m.hidden,
                      "us_per_layer": {k: round(v * 1e3 / len(lays), 2) for k, v in ms.items()},
                      "bit_equal": bool(torch.equal(outs["add"], outs["bias"]))}), flush=True)


def dense_model(fmt, ps):
    if fmt == "qwen2":
        m = DecodeModel(args.layers, ctx=512, fused_ops=True, prompt_len=max(ps), **QWEN2)
    elif fmt in ("bitnet", "bitnet2b"):
        m = DecodeModel(args.layers, ctx=512, fused_ops=True, prompt_len=max(ps), **(BITNET2B if fmt == "bitnet2b" else BITNET))
    else:
        bits, zp = FORMATS[fmt]
        m = DecodeModel(args.layers, bits=bits, zero_point=zp, ctx=512, fused_ops=True, prompt_len=max(ps), **LLAMA)
    try:
        for P in ps:
            x = m.px[:P].contiguous()
            forms = {"prefill": prompt_fn(m, P, x), "per_linear": prompt_fn(m, P, x, linear=True)}
            graphs = {k: graph(f) for k, f in forms.items()}
            if P <= args.gemv_max:
                with gemv_forms():
                    graphs["gemv_io"] = graph(forms["prefill"])
            ms = best(graphs)
            if fmt in ("bitnet", "bitnet2b", "qwen2"):
                share = library_share(forms["prefill"])
                model = {"bitnet2b": "bitnet_b1_58_2b4t", "bitnet": "bitnet_b1_58_3b", "qwen2": "qwen2_7b"}[fmt]
                print(json.dumps({"model": model, "format": "w4_g128_zp" if fmt == "qwen2" else "w2_one_scale_a64", "layers": args.layers, "P": P,
                                  "ms_per_prompt": {k: round(v, 3) for k, v in ms.items()},
                                  "prompt_tokens_per_s": {k: round(P * 1e3 / v, 1) for k, v in ms.items()},
                                  "prefill_linears_share": round(share, 3)}), flush=True)
                del graphs
                torch.cuda.synchronize()
                continue
            # q/k/v of every layer: one grouped launch against three single-tensor launches
            lays = m.layers
            h1 = torch.randn((P, LLAMA["hidden"]), device="cuda")
            qkv = [[l.lin[n].wt for n in ("q", "k", "v")] for l in lays]
            outs = [[l.pbuf[n] for n in ("q", "k", "v")] for l in lays]
            grouped = graph(lambda: [tb.prefill_rmsnorm(w, P, h1, l.norm1, l.EPS, o) for w, o, l in zip(qkv, outs, lays)])
            single = graph(lambda: [tb.prefill_rmsnorm([w[i]], P, h1, l.norm1, l.EPS, [o[i]])
                                    for w, o, l in zip(qkv, outs, lays) for i in range(3)])
            q = best({"grouped": grouped, "three_launches": single})
            share = library_share(forms["prefill"])
            res = {"model": "llama2_7b", "format": fmt, "layers": args.layers, "P": P,
                   "ms_per_prompt": {k: round(v, 3) for k, v in ms.items()},
                   "prompt_tokens_per_s": {k: round(P * 1e3 / v, 1) for k, v in ms.items()},
                   "prefill_linears_share": round(share, 3),
                   "qkv_us_per_layer": {k: round(v * 1e3 / args.layers, 1) for k, v in q.items()}}
            print(json.dumps(res), flush=True)
            del graphs, grouped, single
            torch.cuda.synchronize()
        if fmt == "qwen2":
            qkv_bias_pair(m, 256)
    finally:
        m.free()


def moe_model(fmt, ps):
    bits, zp = FORMATS[fmt]
    m = DecodeModel(args.moe_layers, bits=bits, zero_point=zp, ctx=512, fused_ops=True, prompt_len=max(ps), **MIXTRAL)
    try:
        for P in ps:
            x = m.px[:P].contiguous()
            graphs = {"prefill": graph(prompt_fn(m, P, x))}
            with gemv_forms():
                graphs["gemv_io"] = graph(prompt_fn(m, P, x))
            ms = best(graphs)
            print(json.dumps({"model": "mixtral_8x7b", "format": fmt, "layers": args.moe_layers, "P": P,
                              "ms_per_prompt": {k: round(v, 3) for k, v in ms.items()},
                              "prompt_tokens_per_s": {k: round(P * 1e3 / v, 1) for k, v in ms.items()}}), flush=True)
            del graphs
            torch.cuda.synchronize()
    finally:
        m.free()


print(json.dumps({"card": card()}), flush=True)
if args.qwen2 or args.bitnet or args.bitnet2b:
    dense_model("qwen2" if args.qwen2 else "bitnet2b" if args.bitnet2b else "bitnet", [int(p) for p in args.ps.split(",")])
else:
    for fmt in args.formats.split(","):
        dense_model(fmt, [int(p) for p in args.ps.split(",")])
    for fmt in args.formats.split(","):
        if args.moe_layers:
            moe_model(fmt, [int(p) for p in args.moe_ps.split(",")])
print(json.dumps({"card_after": card()}), flush=True)
