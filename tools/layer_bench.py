"""Time the decode harness's token step (DecodeModel: 32 Llama-2-7B layers, hidden 4096, FFN 11008, ctx 512, CUDA-graphed) four
ways: every linear its own launch ("off"), each FFN one decode sequence ("ffn_sequence"), each layer's half after attention --
o-projection, residual add, RMSNorm, FFN, second residual add -- one decode sequence ("post_attn_sequence"), and the linears as
four launches that take the RMSNorms, the SiLU*mul and the residual adds into their inputs and outputs ("fused_ops").  The models are
resident together and timed alternately, best of `--rounds`; the kernel serving each layer's sequence is recorded beside the time,
and so are the card's name, power limit and max SM clock.  With `--bitnet` the layers are BitNet-3B's (26 layers, hidden 3200,
FFN 8640, 32 heads; ternary one-scale tensors with activation groups of 64, and the attn / ffn sub-norms), timed in the modes
"off" and "fused_ops".  With `--bitnet2b` they are BitNet b1.58 2B4T's (30 layers, hidden 2560, FFN 6912, 20 query heads and 5 KV
heads of 128, the squared-ReLU FFN: ffn_act="relu2", kv_heads=5), in the same two modes.  With `--qwen2` they are Qwen2-7B's (28
layers, hidden 3584, FFN 18944, 28 query heads and 4 KV heads of 128, W4 g128 with zero points, a bias on q/k/v: kv_heads=4,
qkv_bias=True), in the same two modes, plus one line that times the stacked q/k/v tensor (4608 x 3584) of every layer at N = 1 as
gemv_rmsnorm followed by a torch add of the bias against gemv_rmsnorm_bias (CUDA-graphed, alternated, us per layer).

    python tools/layer_bench.py [--layers 32] [--reps 20] [--rounds 3] [--formats w2zp,w4]
    python tools/layer_bench.py --bitnet [--layers 26] [...]
    python tools/layer_bench.py --bitnet2b [--layers 30] [...]
    python tools/layer_bench.py --qwen2 [--layers 28] [...]
    python tools/layer_bench.py --profile [...]     # kernels per token of each mode (torch.profiler, one eager step; no timing)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "t-mac_b200")); sys.path.insert(0, ROOT)
import torch                                    # noqa: E402
import tmac_b200 as tb                          # noqa: E402
from decode_harness import DecodeModel          # noqa: E402

HIDDEN, FFN, HEADS, CTX = 4096, 11008, 32, 512
FORMATS = {"w2zp": (2, True), "w4": (4, False)}
MODES = {"off": {}, "ffn_sequence": {"ffn_sequence": True}, "post_attn_sequence": {"post_attn_sequence": True},
         "fused_ops": {"fused_ops": True}}

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=None, help="default 32, 26 with --bitnet, 30 with --bitnet2b, 28 with --qwen2")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--formats", default="w2zp,w4")
ap.add_argument("--profile", action="store_true", help="count the kernels of one token step per mode instead of timing")
ap.add_argument("--bitnet", action="store_true", help="BitNet-3B layers with sub-norms, modes off and fused_ops")
ap.add_argument("--bitnet2b", action="store_true", help="BitNet b1.58 2B4T layers (relu2 FFN, 5 KV heads), modes off and fused_ops")
ap.add_argument("--qwen2", action="store_true", help="Qwen2-7B layers (W4 g128 zp, 4 KV heads, q/k/v biases), modes off and fused_ops")
args = ap.parse_args()
if args.qwen2:
    qwen = dict(kv_heads=4, qkv_bias=True)
    HIDDEN, FFN, HEADS = 3584, 18944, 28
    args.formats = "qwen2_w4g128zp"
    FORMATS = {args.formats: (4, True)}
    MODES = {"off": qwen, "fused_ops": dict(qwen, fused_ops=True)}
elif args.bitnet or args.bitnet2b:
    sub = dict(sub_norms=True, ffn_act="relu2", kv_heads=5) if args.bitnet2b else dict(sub_norms=True)
    HIDDEN, FFN, HEADS = (2560, 6912, 20) if args.bitnet2b else (3200, 8640, 32)
    args.formats = "bitnet2b" if args.bitnet2b else "bitnet"
    FORMATS = {args.formats: (2, False)}
    MODES = {"off": sub, "fused_ops": dict(sub, fused_ops=True)}
if args.layers is None:
    args.layers = 28 if args.qwen2 else 30 if args.bitnet2b else 26 if args.bitnet else 32

if not torch.cuda.is_available():
    sys.exit("layer_bench.py needs a CUDA device")
lib = tb.load(); tb.check(lib.tmac_b200_init(0), "init")
st = torch.cuda.Stream(); torch.cuda.set_stream(st); tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                     # the timing stands without it, but says so
        q = "nvidia-smi unavailable: %s" % ex
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q}


def kernel_of(m):
    seq = m.layers[0].ffn_seq or m.layers[0].post_seq
    if seq is None:
        return None
    return "resident chain" if seq.info()["ring_slots"] < 0 else "stream-K"


def kernels_per_token(m):
    from torch.profiler import ProfilerActivity, profile
    with torch.cuda.stream(st):
        m.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(st):
            m.step()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kern = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
    return {"kernels": len(kern), "library_kernels": sum("tmac_b200::" in n for n in kern), "memcpy_memset": len(names) - len(kern)}


def qkv_bias_pair(m):
    """Every layer's stacked q/k/v tensor at N = 1: gemv_rmsnorm then a torch add of the bias, against gemv_rmsnorm_bias; each a CUDA
    graph over the layers, alternated, best of --rounds.  The two outputs of the last layer must be equal bit for bit (F32)."""
    lays = m.layers
    x = torch.randn((1, HIDDEN), device="cuda")
    outs = {k: torch.zeros((1, lays[0].lin["qkv"].mout), device="cuda") for k in ("add", "bias")}

    def add():
        for l in lays:
            tb.gemv_rmsnorm([l.lin["qkv"].wt], 1, x, l.norm1, l.EPS, [outs["add"]])
            outs["add"].add_(l.qkv_b["qkv"])

    def bias():
        for l in lays:
            tb.gemv_rmsnorm_bias([l.lin["qkv"].wt], 1, x, l.norm1, l.EPS, [l.qkv_b["qkv"]], [outs["bias"]])
    graphs = {"gemv_rmsnorm_plus_add": m._graph(add, st), "gemv_rmsnorm_bias": m._graph(bias, st)}
    us = {k: float("inf") for k in graphs}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            us[k] = min(us[k], 1e6 / m._per_s(g.replay, st, args.reps) / len(lays))
    return {"qkv_bias_N1": {"rows": lays[0].lin["qkv"].mout, "K": HIDDEN, "us_per_layer": {k: round(v, 2) for k, v in us.items()},
                            "bit_equal": bool(torch.equal(outs["add"], outs["bias"]))}}


def case(fmt):
    bits, zp = FORMATS[fmt]
    res = {"format": fmt, "layers": args.layers, "ctx": CTX}
    models = {}
    try:
        for mode, kw in MODES.items():
            torch.manual_seed(0)                # the same input and KV cache in every model
            models[mode] = DecodeModel(args.layers, HIDDEN, FFN, HEADS, bits, zp, ctx=CTX, **kw)
            res.setdefault("sequence_kernel", {})[mode] = kernel_of(models[mode])
        if args.profile:
            res["per_token"] = {mode: kernels_per_token(m) for mode, m in models.items()}
            return res
        if args.qwen2:
            res.update(qkv_bias_pair(models["fused_ops"]))
        for m in models.values():
            m.capture(st)
        runs = {mode: [] for mode in models}
        for _ in range(args.rounds):            # alternated
            for mode, m in models.items():
                runs[mode].append(1e3 / m.tokens_per_s(st, n=args.reps))
        # the models share weights and inputs (same seeds): the modes differ by the K split of the fp32 sums and the rounding of
        # the torch ops they replace -- a sanity bound, not a test
        y0 = models["off"].y
        for mode, m in models.items():
            res[mode] = {"ms_per_token": round(min(runs[mode]), 3), "runs_ms": [round(t, 3) for t in runs[mode]],
                         "max_rel_diff_vs_off": float(((m.y - y0).abs().max() / y0.abs().max()).item())}
        return res
    finally:
        for m in models.values():
            m.free()


print(json.dumps({"card": card()}), flush=True)
for fmt in args.formats.split(","):
    print(json.dumps(case(fmt)), flush=True)
print(json.dumps({"card_after": card()}), flush=True)
