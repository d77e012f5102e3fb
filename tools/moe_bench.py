"""Routed MoE experts at Mixtral-8x7B's FFN shape (hidden 4096, FFN 14336, 8 experts, top-2), W2 g128 zp and W4 g128, N = 1, 2, 4.
The router's ids and weights are fixed and already on the device, so only the expert part is timed, in four forms:

  routed     (a) gemv_experts([gate, up]) + gemv_experts_glu(down, + h): the two launches that pick the experts on the device;
  host       (b) ids copied to the host, then gemv_grouped over each token's selected gate/up, gemv_glu per slot, combine in torch
                 (eager: the copy is a device-to-host sync per FFN);
  all        (c) every expert: gemv_grouped over all gate/up at N rows, gemv_glu per expert, a masked combine in torch;
  known      (d) gemv_grouped over the selected gate/up, then over the selected down on a precomputed GLU input, with the handles
                 known on the host -- no usable step, but (a) - (d) is the cost of routing on the device.

(a), (c) and (d) are captured in one CUDA graph per form over `--layers` distinct resident layers (clones: every layer's expert
bytes come from HBM, far beyond the 50 MB L2), replayed `--reps` times between CUDA events; (b) runs eagerly between events.
Best of `--rounds` alternated runs.  us per MoE FFN, and GB/s over the bytes of the experts the tokens selected (each distinct
expert's gate, up and down once).  The card's name, power limit and SM clocks are read in the same run.

    python tools/moe_bench.py [--layers 4] [--reps 20] [--rounds 3] [--formats w2zp,w4] [--ns 1,2,4]
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
ap.add_argument("--layers", type=int, default=4)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--formats", default="w2zp,w4")
ap.add_argument("--ns", default="1,2,4")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("moe_bench.py needs a CUDA device")
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


def case(fmt, layers, N, rng):
    ids_h = np.stack([rng.choice(EXPERTS, TOPK, replace=False) for _ in range(N)]).astype(np.int32)
    ids = torch.from_numpy(ids_h).cuda()
    w = torch.softmax(torch.randn((N, TOPK), device="cuda"), dim=-1)
    mask = torch.zeros((N, EXPERTS), device="cuda").scatter_(1, ids.long(), w)       # (c): the dense routing weights
    h2, h = torch.randn((N, HIDDEN), device="cuda"), torch.randn((N, HIDDEN), device="cuda")
    G, U, y = torch.zeros((N, TOPK, FFN), device="cuda"), torch.zeros((N, TOPK, FFN), device="cuda"), torch.zeros((N, HIDDEN), device="cuda")
    Gall, Uall = [torch.zeros((N, FFN), device="cuda") for _ in range(EXPERTS)], [torch.zeros((N, FFN), device="cuda") for _ in range(EXPERTS)]
    Yall = torch.zeros((EXPERTS, N, HIDDEN), device="cuda")
    S = N * TOPK
    dG, dU = [torch.zeros((1, FFN), device="cuda") for _ in range(2 * S)], [torch.zeros((1, FFN), device="cuda") for _ in range(S)]
    act, dY = torch.randn((1, FFN), device="cuda"), [torch.zeros((1, HIDDEN), device="cuda") for _ in range(S)]
    sel = [(n, int(ids_h[n, j])) for n in range(N) for j in range(TOPK)]

    def routed(l):
        L = layers[l]
        tb.gemv_experts([[x.wt for x in L["gate"]], [x.wt for x in L["up"]]], N, h2, ids, [G, U])
        tb.gemv_experts_glu([x.wt for x in L["down"]], N, G, U, ids, w, y, R=h)

    def everything(l):
        L = layers[l]
        tb.gemv_grouped([x.wt for x in L["gate"]] + [x.wt for x in L["up"]], N, h2, Gall + Uall)
        for e in range(EXPERTS):
            tb.gemv_glu(L["down"][e].wt, N, Gall[e], Uall[e], Yall[e])
        y.copy_(h + torch.einsum("ne,enh->nh", mask, Yall))

    def known(l):
        L = layers[l]
        tb.gemv_grouped([L["gate"][e].wt for _, e in sel] + [L["up"][e].wt for _, e in sel], 1, h2[:1], dG)
        tb.gemv_grouped([L["down"][e].wt for _, e in sel], 1, act, dY)

    def host(l):
        L = layers[l]
        hid = ids.cpu().numpy()                 # the device-to-host sync of a host-routed step
        ys = []
        for n in range(N):
            es = [int(e) for e in hid[n]]
            gu = [torch.empty((1, FFN), device="cuda") for _ in range(2 * TOPK)]
            tb.gemv_grouped([L["gate"][e].wt for e in es] + [L["up"][e].wt for e in es], 1, h2[n:n + 1], gu)
            yn = torch.empty((TOPK, HIDDEN), device="cuda")
            for j, e in enumerate(es):
                tb.gemv_glu(L["down"][e].wt, 1, gu[j], gu[TOPK + j], yn[j:j + 1])
            ys.append(h[n] + (w[n, :, None] * yn).sum(dim=0))
        y.copy_(torch.stack(ys))

    graphs = {"routed": graphed(routed), "all": graphed(everything), "known": graphed(known)}
    for l in range(args.layers):                # warm-up of the eager form
        host(l)
    torch.cuda.synchronize()
    best = {k: float("inf") for k in ("routed", "host", "all", "known")}
    for _ in range(args.rounds):                # alternated
        for k, g in graphs.items():
            g.replay(); torch.cuda.synchronize()
            best[k] = min(best[k], timed(g.replay, args.reps) * 1e3 / (args.reps * args.layers))
        best["host"] = min(best["host"], timed(lambda: [host(l) for l in range(args.layers)], args.reps) * 1e3 / (args.reps * args.layers))
    L0 = layers[0]
    nbytes = sum(L0[n][e].wt.nbytes for e in set(ids_h.ravel().tolist()) for n in ("gate", "up", "down"))
    return {"format": fmt, "N": N, "ids": ids_h.tolist(), "selected_MB": round(nbytes / 1e6, 1),
            **{"us_" + k: round(v, 1) for k, v in best.items()},
            **{"GBs_" + k: round(nbytes / (v * 1e-6) / 1e9, 1) for k, v in best.items()},
            "us_routing_cost": round(best["routed"] - best["known"], 1)}


print(json.dumps({"card": card()}), flush=True)
for fmt in args.formats.split(","):
    bits, zp = FORMATS[fmt]
    first = {n: [QLinear(m, k, bits, 128, zp, seed=10 * e + i) for e in range(EXPERTS)]
             for i, (n, m, k) in enumerate((("gate", FFN, HIDDEN), ("up", FFN, HIDDEN), ("down", HIDDEN, FFN)))}
    layers = [first] + [{n: [QLinear(0, 0, bits, 128, zp, 0, share=x) for x in v] for n, v in first.items()}
                        for _ in range(args.layers - 1)]
    try:
        rng = np.random.default_rng(0)
        for N in (int(v) for v in args.ns.split(",")):
            print(json.dumps(case(fmt, layers, N, rng)), flush=True)
    finally:
        for L in layers:
            for v in L.values():
                for x in v:
                    x.free()
print(json.dumps({"card_after": card()}), flush=True)
