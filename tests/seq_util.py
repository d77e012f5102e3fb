"""Helpers shared by the decode-sequence GPU tests (test_gpu_sequence.py, test_gpu_chain.py): upload a chain of tensors in the
reference layout and run the oracle on one op."""
import tmac_b200 as tb
import tmac_oracle as T


def kc(cfg):
    return tb.make_kcfg(cfg.Mout, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale)


def oracle_gemv(oracle, cfg, A, S, x):
    q, ls, lb = oracle.preprocessor(x.reshape(1, -1), cfg.act_group_size)
    return oracle.qgemm(cfg, A, S, q, ls, lb)[0]


def build_chain(cfgs, seed):
    """[(cfg, A, S, weights handle)] for a chain of shapes; consecutive K <= previous Mout."""
    out = []
    for i, cfg in enumerate(cfgs):
        w, sc, z, _ = T.make_problem(cfg, seed=seed + i)
        A, S = T.pack_reference_layout(w, sc, z, cfg)
        out.append((cfg, A, S, tb.upload_reference_layout(kc(cfg), A, S)))
    return out
