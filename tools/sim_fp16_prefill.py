"""CPU study of the fp16 prefill tile (tmac_prefill16.cuh): how far from the reference kernel is the formulation that folds both
scales into fp16 operands -- A = 0.5*scale[m][wg]*S[m][g][e], B = lut_scale[n][ag]*T8[n][g][e] -- and accumulates the whole K in
fp32, with the LUT-bias / zero-point terms kept exact?  W2 and the 4-plane layouts (W3, W4) that the tile serves, at 512 x 4096
and at the Llama-2 / Qwen2 K of 11008 and 18944.  Uses the oracle (TEST INFRASTRUCTURE) as the truth.

    python tools/sim_fp16_prefill.py         # 8 tokens, seed 3: max|dC|/max|C| 1.4e-4 (W2) .. 2.7e-4 (W4 512 x 4096 sym); bar 1e-3
                                             # the other groupings: 1.3e-4 .. 3.1e-4
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import tmac_oracle as T   # noqa: E402

o = T.load_oracle()
# (Mout, K, bits, zero points, group size, act group size): g128 / a64, then the other groupings the tiles take
CASES = [(512, 4096, 2, True, 128, 64), (512, 4096, 4, True, 128, 64), (512, 4096, 4, False, 128, 64), (384, 4096, 3, True, 128, 64),
         (256, 11008, 4, False, 128, 64), (256, 18944, 4, True, 128, 64), (384, 11008, 3, True, 128, 64),
         (512, 4096, 4, False, 32, 32), (256, 11008, 4, False, 32, 32), (384, 4096, 3, True, 32, 32), (512, 4096, 2, True, 64, 64),
         (512, 4096, 2, True, 64, 32), (512, 4096, 4, True, 128, 32), (512, 4096, 4, True, 128, 128), (512, 4096, 2, True, 128, 128),
         (256, 11008, 4, True, 128, 128)]
for Mout, Kc, bits, zp, gs_, ags_ in CASES:
    # the reference's kfactor is ags / 4 (16 for ags 64); with kfactor 16 at ags 128 its packing describes another problem
    cfg = T.Config(Mout, Kc, bits, kfactor=ags_ // 4, group_size=gs_, act_group_size=ags_, zero_point=zp).resolved()
    N = 8
    w, sc, z, x = T.make_problem(cfg, seed=3, N=N)
    A, S_ = T.pack_reference_layout(w, sc, z, cfg)
    q, ls, lb = o.preprocessor(x, cfg.act_group_size)
    Cref = o.qgemm(cfg, A, S_, q, ls, lb)
    M, K = cfg.Mout, cfg.K
    G = K // 4
    wb = np.stack([(w >> b) & 1 for b in range(bits)], axis=0).astype(np.int32)
    idx = (wb.reshape(bits, M, G, 4) * np.array([1, 2, 4, 8])).sum(-1)
    e, sg = np.where(idx < 8, idx, 15 - idx), np.where(idx < 8, 1, -1)
    S = np.zeros((M, G, 8), np.float32)                       # one-hot-signed expansion: sum_b 2*alpha_b * sign * [j == e]
    for b in range(bits):
        np.add.at(S, (np.arange(M)[:, None], np.arange(G)[None, :], e[b]), (sg[b] * (1 << b)).astype(np.float32))
    T8 = q[:, :, :8].astype(np.float32)
    gs, ags = cfg.group_size, cfg.act_group_size
    s_g, ls_g = np.repeat(sc, gs // 4, axis=1), np.repeat(ls, ags // 4, axis=1)
    Aop = (0.5 * s_g[:, :, None] * S).astype(np.float16).astype(np.float32).reshape(M, -1)
    Bop = (ls_g[:, :, None] * T8).astype(np.float16).astype(np.float32).reshape(N, -1)
    LB = lb.reshape(N, K // gs, gs // ags).sum(-1)
    rest = LB.astype(np.float64) @ (0.5 * sc + (z if zp else 0.0)).astype(np.float64).T
    C = (Bop @ Aop.T).astype(np.float64) + rest
    print("W%d g%-3d a%-3d %4d x %5d %-3s fp16 operands, fp32 accumulate: max|dC|/max|C| = %.2e   nmse %.2e"
          % (bits, gs, ags, M, K, "zp" if zp else "sym", np.abs(C - Cref).max() / np.abs(Cref).max(), T.nmse(Cref, C.astype(np.float32))))
