"""Prefill tile timing: for each shape and N, CUDA events over repeated calls after a warm-up, of
    pre+tile   tb.gemv (LUT build + the tile, the one-call form)
    tile only  tb.qgemm_lut on a prepared LUT
    gemv       the same qgemm_lut call with the tiles disabled (debug knob prefill = 0): the GEMV kernel per activation row
    gemv 1-call  tb.gemv with the tiles disabled: the GEMV per activation row, with the LUT built inside it where the grouping
                 allows (the integer path's one-call form before it took the tile)
The tile's minimum N is set to the smallest N of the run, so that the tile is timed below the library's threshold too.

    python tools/pf_bench.py                          # W2 g128 zp 11008 x 4096, N = 32 .. 512 (as before)
    python tools/pf_bench.py --bits 4                 # W4 g128 zp: 4096x4096, 11008x4096, 4096x11008, 18944x3584, N = 16 .. 512
    python tools/pf_bench.py --bits 3 --shapes 11008x4096
    python tools/pf_bench.py --bitnet                 # W2 integer path (one scale, act group = K): BitNet-3B 3200x3200, 8640x3200,
                                                      # 3200x8640, N = 16 .. 512
    python tools/pf_bench.py --bits 4 --group 32 --act-group 32 --sym   # ggml Q4_0's grouping (W4 g32, act group 32)

Rates: dense-equivalent = 2*N*M*K / time; MMA = the tile's tensor-core work (padded to whole 128-row x token tiles, contraction
2K entries + the fp16 tile's bias columns) / time, against the H100 SXM data-sheet peaks (dense): 989 TFLOP/s fp16, 1979 TOP/s int8.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "t-mac_b200")); sys.path.insert(0, os.path.join(ROOT, "oracle")); sys.path.insert(0, ROOT)
import torch  # noqa: E402
import tmac_b200 as tb, bench  # noqa: E402
import tmac_oracle as T  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--bits", type=int, default=2)
ap.add_argument("--shapes", default=None, help="comma-separated MxK (rows x K); default: 11008x4096 for W2, the Llama-2 / Qwen2 W4 shapes otherwise")
ap.add_argument("--ns", default=None, help="comma-separated N; default: 32..512 for W2, 16..512 otherwise")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--sym", action="store_true", help="no zero points")
ap.add_argument("--bitnet", action="store_true", help="W2 integer path: one weight scale, one activation group per row (BitNet)")
ap.add_argument("--group", type=int, default=128, help="weight group size (the stream layout's chunk is min(group, 128))")
ap.add_argument("--act-group", type=int, default=64, help="activation group size (<= the chunk)")
a = ap.parse_args()
if a.bitnet:
    a.bits, a.sym = 2, True
shapes = a.shapes or ("3200x3200,8640x3200,3200x8640" if a.bitnet else
                      "%dx%d" % (bench.MOUT, bench.K) if a.bits == 2 else "4096x4096,11008x4096,4096x11008,18944x3584")
shapes = [tuple(int(v) for v in s.split("x")) for s in shapes.split(",")]
ns = [int(v) for v in a.ns.split(",")] if a.ns else ([32, 64, 128, 256, 512] if a.bits == 2 and not a.bitnet else [16, 32, 64, 128, 256, 512])

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip())
lib = tb.load(); tb.check(lib.tmac_b200_init(0), "init")
st = torch.cuda.Stream(); torch.cuda.set_stream(st); tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "ss")
tb.debug_set("prefill_min_n", min(ns))


def time_us(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(a.reps):
        fn()
    e1.record(st); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.reps * 1e3


try:
    for M, K in shapes:
        w, sc, z = bench.synth(9, mout=M, k=K, bits=a.bits, zp=not a.sym, one_scale=a.bitnet)
        ags = K if a.bitnet else a.act_group
        kfactor = 16 if a.bitnet else ags // 4                   # the reference's tile: kfactor * 4 K positions per activation group
        cfg = tb.make_kcfg(M, K, a.bits, T.default_bm(M * a.bits, a.bits), kfactor, a.group, ags, not a.sym, a.bitnet)
        wt = tb.upload_plain(cfg, w, sc, z)
        nag = K // ags
        print("W%d %s %d x %d" % (a.bits, "bitnet (one scale, act group K)" if a.bitnet else
                                  "g%d a%d %s" % (a.group, ags, "sym" if a.sym else "zp"), M, K))
        for N in ns:
            x = torch.randn((N, K), device="cuda"); o = torch.zeros((N, M), device="cuda")
            q = torch.zeros((N, K // 4, 16), dtype=torch.int8, device="cuda"); ls = torch.zeros((N, nag), device="cuda"); lb = torch.zeros_like(ls)
            tb.preprocessor(K, N, ags, x, ls, lb, q)
            row = {}
            for name, fn in (("pre+tile", lambda: tb.gemv(wt, N, x, o)), ("tile only", lambda: tb.qgemm_lut(wt, N, q, ls, lb, o)),
                             ("gemv", lambda: tb.qgemm_lut(wt, N, q, ls, lb, o)), ("gemv 1-call", lambda: tb.gemv(wt, N, x, o))):
                tb.debug_set("prefill", 0 if name.startswith("gemv") else 1)
                us = time_us(fn)
                ll = tb.last_launch()
                row[name] = us
                dense = 2.0 * N * M * K / us / 1e6
                if ll["batch"] >= 0:
                    kind, mma = "GEMV", ""
                elif ll["cluster"] == 16:    # fp16 tile: 256-token tiles, K/64 + ceil(chunks/32) steps of 128 entries
                    work = 2.0 * ((N + 255) // 256 * 256) * ((M + 127) // 128 * 128) * 128 * (K // 64 + (K // min(a.group, 128) + 31) // 32)
                    kind, mma = "fp16 tile", "  MMA %6.1f TFLOP/s (%4.1f%% of 989)" % (work / us / 1e6, 100.0 * work / us / 1e6 / 989)
                else:                        # int8 tile: 128-token tiles, contraction 2K bytes
                    work = 2.0 * ((N + 127) // 128 * 128) * ((M + 127) // 128 * 128) * (2 * K)
                    kind, mma = "int8 tile", "  MMA %6.1f TOP/s (%4.1f%% of 1979)" % (work / us / 1e6, 100.0 * work / us / 1e6 / 1979)
                print("  N=%4d %-10s %9.1f us   dense-equivalent %6.1f TFLOP/s  [%s]%s" % (N, name, us, dense, kind, mma))
            print("  N=%4d tile/gemv = %.2f  (tile %s)   pre+tile/gemv 1-call = %.2f" % (N, row["tile only"] / row["gemv"],
                  "faster" if row["tile only"] < row["gemv"] else "SLOWER", row["pre+tile"] / row["gemv 1-call"]))
        wt.free()
finally:
    tb.debug_set("prefill", 1); tb.debug_set("prefill_min_n", 0)
