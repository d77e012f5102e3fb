"""Time the decode sequence kernel on the bench workload (32 distinct 11008x4096 W2 g128 zp tensors):
independent inputs vs a true dependency chain (x_{i+1} = first K outputs of op i); optional per-op timeline.

    python tools/seq_bench.py [--trace] [--layers 32] [--reps 20] [--distinct N]

--distinct N: the ops cycle over N distinct resident tensors (op i runs tensor i % N).  At N = 2 the chain's weights (25 MB)
stay in the H100's 50 MB L2, so the chain runs without the HBM weight stream: the bound that the stream sets on the op period.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "t-mac_b200")); sys.path.insert(0, ROOT)
import torch                      # noqa: E402
import tmac_b200 as tb            # noqa: E402
import bench                      # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--trace", action="store_true")
ap.add_argument("--layers", type=int, default=32)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--distinct", type=int, default=0, help="distinct tensors the ops cycle over (0 = one per op)")
ap.add_argument("--bits", type=int, default=2)
ap.add_argument("--mout", type=int, default=bench.MOUT)
ap.add_argument("--k", type=int, default=bench.K)
ap.add_argument("--smem", type=int, default=0)
ap.add_argument("--impl", type=int, default=2, help="0 stream-K sequence kernel, 1 resident gemv3 chain, 2 auto")
ap.add_argument("--dump", type=str, default="", help="save the raw chain trace [ops][grid][16] (ns) to this .npy")
ap.add_argument("--flags", type=str, default="", help="comma list of chain_flags values to time (resident chain only): 0 data flow, 1 grid-barrier form")
args = ap.parse_args()

lib = tb.load(); tb.check(lib.tmac_b200_init(0), "init")
st = torch.cuda.Stream(); torch.cuda.set_stream(st); tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")
if args.trace:
    tb.debug_set("trace", 1)
if args.smem:
    tb.debug_set("seq_smem_kb", args.smem)
tb.debug_set("seq_impl", args.impl)
L = args.layers
w, sc, z = bench.synth(100, args.mout, args.k, args.bits, 128, True, False)
bm = 256 if (args.mout * args.bits) % 256 == 0 else 128
cfg = tb.make_kcfg(args.mout, args.k, args.bits, bm, 16, 128, 64, True, False)
base = tb.upload_plain(cfg, w, sc, z)
nd = args.distinct if args.distinct > 0 else L
tensors = [base] + [tb.clone(base) for _ in range(min(nd, L) - 1)]
layers = [tensors[i % len(tensors)] for i in range(L)]
x = torch.randn((L, args.k), device="cuda").half().float()
out = torch.zeros((L, args.mout), device="cuda")
abytes = bench.algorithmic_bytes(args.mout, args.k, args.bits, 128, True)


def timed(seq, reps):
    for _ in range(3):
        seq.launch()
    seq.status()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        seq.launch()
    e1.record(st); torch.cuda.synchronize()
    seq.status()
    return e0.elapsed_time(e1) / reps * 1e3


def chain_trace(seq):
    """Resident chain: globaltimer stamps of warp 0 of every CTA, [ops][grid][16] (tmac_chain.cuh)."""
    seq.launch(); seq.status()
    raw = seq.trace()
    if args.dump:
        np.save(args.dump, raw)
    t = raw.astype(np.float64) / 1e3
    ops = slice(2, None)
    def fmt(a):
        return "%.2f/%.2f/%.2f" % (np.median(a), np.percentile(a, 90), a.max())
    flow = bool(t[ops, :, 1].max() == 0)          # data-flow mode: no barrier stamps
    phases = [(2, 3, "input wait + LUT slice"), (3, 4, "block wait"), (4, 5, "lookups"),
              (5, 6, "buffer guard + red sync" if flow else "red sync"),
              (6, 7, "CTA sums + send" if flow else "CTA sums + cluster sync"),
              (7, 8, "leader: partials landed, sum, publish" if flow else "leader: sum, publish")]
    if not flow:
        phases = [(0, 1, "top->barrier seen"), (1, 2, "syncthreads")] + phases
    leaders = t[:, ::4, 8] > 0                    # (op, cluster) with published rows: stamp 8 is the leader's
    for k0, k1, nme in phases:
        a = t[ops, :, k1] - t[ops, :, k0]
        if k1 == 8:
            a = a[:, ::4][leaders[ops]]
        print("    %-30s median/p90/max us: %s" % (nme, fmt(a)))
    # stamp 6 follows the CTA barrier after its 4 warps' lookups: the cluster's latest one starts the tail of the reduction
    last = t[:, :, 6].reshape(t.shape[0], -1, 4).max(axis=2)
    print("    last CTA barrier of the cluster -> rows published median/p90/max us: %s" % fmt((t[:, ::4, 8] - last)[ops][leaders[ops]]))
    end = np.where(t[:, :, 8] > 0, t[:, :, 8], t[:, :, 7])
    per = np.diff(end.max(axis=1))
    if flow:
        print("    op period median %.2f us (data-flow mode: CTAs are not aligned per op)" % np.median(per))
        return
    print("    op period median %.2f us; last leader arrive -> CTAs see barrier: median %.2f max %.2f us; spread of 'lookups done' across CTAs %.2f us" % (
        np.median(per), np.median(t[3:, :, 1] - end[2:-1].max(axis=1)[:, None]), (t[3:, :, 1] - end[2:-1].max(axis=1)[:, None]).max(),
        np.median(t[ops, :, 5].max(axis=1) - t[ops, :, 5].min(axis=1))))


for fl in [int(v) for v in args.flags.split(",") if v != ""]:
    tb.debug_set("chain_flags", fl); tb.debug_set("seq_impl", 1)
    seq = tb.Sequence()
    for i, wt in enumerate(layers):
        if i > 0:
            seq.add(wt, in_op=i - 1, in_offset=0, out=out[i])
        else:
            seq.add(wt, x=x[i], out=out[i])
    seq.build()
    us = timed(seq, args.reps)
    print("chain_flags %d dependent: %.2f us per GEMV  %s" % (fl, us / L, seq.info()), flush=True)
    if args.trace:
        chain_trace(seq)
    seq.free()
if args.flags:
    sys.exit(0)

for name, chained in (("independent inputs", False), ("dependent chain", True)):
    if chained and args.k > args.mout:
        continue
    seq = tb.Sequence()
    for i, wt in enumerate(layers):
        if chained and i > 0:
            seq.add(wt, in_op=i - 1, in_offset=0, out=out[i])
        else:
            seq.add(wt, x=x[i], out=out[i])
    seq.build()
    us = timed(seq, args.reps)
    print("%-20s: %.1f us per launch of %d GEMVs = %.2f us per GEMV = %.0f GB/s (%.3f of 3350, H100 SXM data sheet)  %s" %
          (name, us, L, us / L, abytes * L / us / 1e3, abytes * L / us / 1e3 / 3350, seq.info()), flush=True)
    if args.trace:
        seq.launch(); seq.status()
        t = seq.trace().astype(np.float64) / 1e3    # [ops][grid][16] us
        t0 = t[0, :, 0].min()
        ent, lut, res, m0, mL, mM, sums, pub, pr0, pr1 = (t[:, :, k] - t0 for k in range(10))
        mlast = np.maximum(np.maximum(m0, mL), mM)
        print("  cycles waiting for weights per op: warp 0 median %.0f max %.0f | last warp median %.0f max %.0f" % (np.median(t[:, :, 10]) * 1e3, t[:, :, 10].max() * 1e3, np.median(t[:, :, 11]) * 1e3, t[:, :, 11].max() * 1e3))

        def fmt(a):
            return "%.2f/%.2f/%.2f" % (np.median(a), np.percentile(a, 90), a.max())
        print("  per (op, CTA) us, median/p90/max:  enter->own LUT done %s | ->first block resident (bar A + weights) %s | lookups warp0 %s, last of 3 sampled warps %s | bar B + sums %s | publish/finish %s" % (
            fmt(lut - ent), fmt(res - lut), fmt(m0 - res), fmt(mlast - res), fmt(sums - mlast), fmt(pub - sums)))
        print("  producer lead (consumers enter op - producer finished requesting it): median %.2f min %.2f us" % (np.median((ent - pr1)[1:]), (ent - pr1)[1:].min()))
        per_op = np.diff(pub.max(axis=1))
        print("  op period: median %.2f us (min %.2f, max %.2f); spread of 'enter' across CTAs: median %.2f us; of 'lookups done': %.2f us" % (
            np.median(per_op), per_op.min(), per_op.max(), np.median(ent.max(axis=1) - ent.min(axis=1)), np.median(mlast.max(axis=1) - mlast.min(axis=1))))
        mid = min(L - 1, 10)
        wt_ = seq.warp_trace.astype(np.float64)
        names = ["enter", "LUT own", "barA rel", "pre-wait", "blk res", "lookups", "sums", "xchg", "y pub", "barLUT", "LUT built", "end"]
        for c in (np.argsort(ent[mid])[len(ent[mid]) // 2], np.argsort(pub[mid])[-1]):
            base = wt_[mid, c, :, 0].min()
            print("  op %d cta %d per warp, SM cycles since the first warp entered the op (0 = not stamped):" % (mid, c))
            print("        " + " ".join("%9s" % n for n in names) + "   | next op enter")
            for w in range(wt_.shape[2]):
                nxt = wt_[mid + 1, c, w, 0] - base if mid + 1 < L else 0
                print("    w%02d " % w + " ".join("%9d" % (v - base if v else 0) for v in wt_[mid, c, w, :12]) + "   | %9d" % nxt)
        order = np.argsort(ent[mid])
        print("  op %d timeline (us after launch), 6 CTAs:" % mid)
        for c in order[:: max(1, len(order) // 6)][:6]:
            print("    cta %3d: enter %.2f  lut %.2f  resident %.2f  lookups(w0/mid/last) %.2f/%.2f/%.2f  sums %.2f  published %.2f" % (
                c, ent[mid, c], lut[mid, c], res[mid, c], m0[mid, c], mM[mid, c], mL[mid, c], sums[mid, c], pub[mid, c]))
    seq.free()
