"""Routed MoE experts at prefill sizes: Mixtral-8x7B's FFN (hidden 4096, FFN 14336, 8 experts, top-2), W2 g128 zp and W4 g128,
N = 16 .. 2048 tokens, with a uniform seeded routing (each token's two experts drawn without replacement) and a skewed one (expert e
drawn with weight 1 / (e + 1)^2, so expert 0 takes about half the slots).  The router's ids and weights are fixed and already on the
device; only the expert part is timed, in three forms:

  prefill  (a) prefill_experts([gate, up]) + prefill_experts_glu(down, + h): each expert's tokens grouped on the device, the tiles,
               on the tile the library's rule picks (`tile`); prefill_int8 is the same with the int8 tile forced (prefill16 = 0), to
               tune that rule;
  gemv     (b) gemv_experts([gate, up]) + gemv_experts_glu(down, + h): one GEMV per (token, slot) -- the switch-over N is where (a)
               overtakes (b);
  host     (c) ids copied to the host, each expert's rows gathered in torch, tmac_b200_gemv per expert and tensor (the dense call,
               which takes a tile at these N), SiLU * mul and the weighted combine in torch (eager: one device-to-host sync per FFN).

(a) and (b) are captured in one CUDA graph per form over `--layers` distinct resident layers (clones: the expert bytes come from HBM),
replayed `--reps` times between CUDA events; (c) runs eagerly between events.  Best of `--rounds` alternated runs, us per MoE FFN.
route_us: the time of the routing kernel (pf_route_kernel, both calls of one FFN) from a torch.profiler run of (a), made after the
timed runs.  The card's name, power limit and SM clocks are read in the same run, before and after.

    python tools/moe_prefill_bench.py [--layers 2] [--reps 3] [--rounds 2] [--formats w2zp,w4] [--ns 16,32,...,2048]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "t-mac_b200"))
import torch                                    # noqa: E402
import tmac_b200 as tb                          # noqa: E402
from decode_harness import QLinear              # noqa: E402

HIDDEN, FFN, EXPERTS, TOPK = 4096, 14336, 8, 2
FORMATS = {"w2zp": (2, True), "w4": (4, False)}

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=2)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--rounds", type=int, default=2)
ap.add_argument("--formats", default="w2zp,w4")
ap.add_argument("--ns", default="16,32,64,128,256,512,1024,2048")
ap.add_argument("--routings", default="uniform,skewed")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("moe_prefill_bench.py needs a CUDA device")
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


def timed(fn, n):
    """ms of n calls of fn on the stream, between CUDA events."""
    with torch.cuda.stream(st):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(n):
            fn()
        e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def graphed(body):
    """A CUDA graph of body(l) for every layer, after one eager pass (workspaces, pointer tables)."""
    with torch.cuda.stream(st):
        for l in range(args.layers):
            body(l)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for l in range(args.layers):
            body(l)
    return g


def routing(kind, N, rng):
    if kind == "uniform":
        return np.stack([rng.choice(EXPERTS, TOPK, replace=False) for _ in range(N)]).astype(np.int32)
    p = 1.0 / (np.arange(EXPERTS) + 1.0) ** 2
    return np.stack([rng.choice(EXPERTS, TOPK, replace=False, p=p / p.sum()) for _ in range(N)]).astype(np.int32)


def route_us(g):
    """us of pf_route_kernel per replay of g, over the layers: from a torch.profiler run of one replay."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.replay()
        torch.cuda.synchronize()
    t = sum(e.device_time_total for e in prof.key_averages() if "pf_route_kernel" in e.key)
    return t / args.layers


def case(fmt, layers, kind, N, rng):
    ids_h = routing(kind, N, rng)
    ids = torch.from_numpy(ids_h).cuda()
    w = torch.softmax(torch.randn((N, TOPK), device="cuda"), dim=-1)
    h2, h = torch.randn((N, HIDDEN), device="cuda"), torch.randn((N, HIDDEN), device="cuda")
    G, U, y = torch.zeros((N, TOPK, FFN), device="cuda"), torch.zeros((N, TOPK, FFN), device="cuda"), torch.zeros((N, HIDDEN), device="cuda")

    def prefill(l):
        L = layers[l]
        tb.prefill_experts([[x.wt for x in L["gate"]], [x.wt for x in L["up"]]], N, h2, ids, [G, U])
        tb.prefill_experts_glu([x.wt for x in L["down"]], N, G, U, ids, w, y, R=h)

    def gemv(l):
        L = layers[l]
        tb.gemv_experts([[x.wt for x in L["gate"]], [x.wt for x in L["up"]]], N, h2, ids, [G, U])
        tb.gemv_experts_glu([x.wt for x in L["down"]], N, G, U, ids, w, y, R=h)

    def host(l):
        L = layers[l]
        hid = ids.cpu().numpy()                 # the device-to-host sync of a host-routed step
        acc = h.clone()
        for e in range(EXPERTS):
            n, j = np.nonzero(hid == e)
            if len(n) == 0:
                continue
            tn, tj = torch.from_numpy(n).cuda(), torch.from_numpy(j).cuda()
            x = h2[tn].contiguous()
            g, u = torch.empty((len(n), FFN), device="cuda"), torch.empty((len(n), FFN), device="cuda")
            tb.gemv(L["gate"][e].wt, len(n), x, g)
            tb.gemv(L["up"][e].wt, len(n), x, u)
            a = torch.nn.functional.silu(g) * u
            d = torch.empty((len(n), HIDDEN), device="cuda")
            tb.gemv(L["down"][e].wt, len(n), a, d)
            acc.index_add_(0, tn, w[tn, tj][:, None] * d)
        y.copy_(acc)

    def int8(body):                             # body under prefill16 = 0
        def run(l):
            tb.debug_set("prefill16", 0)
            try:
                body(l)
            finally:
                tb.debug_set("prefill16", 1)
        return run

    # both tiles' eager calls first: the library workspaces reach their final size before any graph holds their addresses
    with torch.cuda.stream(st):
        for l in range(args.layers):
            prefill(l); int8(prefill)(l)
    torch.cuda.synchronize()
    graphs = {"prefill": graphed(prefill), "prefill_int8": graphed(int8(prefill)), "gemv": graphed(gemv)}
    for l in range(args.layers):                # warm-up of the eager form
        host(l)
    torch.cuda.synchronize()
    best = {k: float("inf") for k in ("prefill", "prefill_int8", "gemv", "host")}
    for _ in range(args.rounds):                # alternated
        for k, g in graphs.items():
            g.replay(); torch.cuda.synchronize()
            best[k] = min(best[k], timed(g.replay, args.reps) * 1e3 / (args.reps * args.layers))
        best["host"] = min(best["host"], timed(lambda: [host(l) for l in range(args.layers)], args.reps) * 1e3 / (args.reps * args.layers))
    tb.prefill_experts([[x.wt for x in layers[0]["gate"]], [x.wt for x in layers[0]["up"]]], N, h2, ids, [G, U])
    tile = "fp16" if tb.last_launch()["cluster"] == 16 else "int8"
    counts = np.bincount(ids_h.ravel(), minlength=EXPERTS).tolist()
    return {"format": fmt, "routing": kind, "N": N, "tile": tile, "rows_per_expert": counts,
            **{"us_" + k: round(v, 1) for k, v in best.items()},
            "route_us": round(route_us(graphs["prefill"]), 1),
            "prefill_speedup_vs_gemv": round(best["gemv"] / best["prefill"], 2),
            "prefill_speedup_vs_host": round(best["host"] / best["prefill"], 2)}


print(json.dumps({"card": card()}), flush=True)
for fmt in args.formats.split(","):
    bits, zp = FORMATS[fmt]
    first = {n: [QLinear(m, k, bits, 128, zp, seed=10 * e + i) for e in range(EXPERTS)]
             for i, (n, m, k) in enumerate((("gate", FFN, HIDDEN), ("up", FFN, HIDDEN), ("down", HIDDEN, FFN)))}
    layers = [first] + [{n: [QLinear(0, 0, bits, 128, zp, 0, share=x) for x in v] for n, v in first.items()}
                        for _ in range(args.layers - 1)]
    try:
        rng = np.random.default_rng(0)
        for kind in args.routings.split(","):
            for N in (int(v) for v in args.ns.split(",")):
                print(json.dumps(case(fmt, layers, kind, N, rng)), flush=True)
    finally:
        for L in layers:
            for v in L.values():
                for x in v:
                    x.free()
print(json.dumps({"card_after": card()}), flush=True)
