"""GPU suite (-m gpu): the decode SEQUENCE kernel (tmac_b200_seq_*, t-mac_b200/csrc/tmac_seq.cuh) against the oracle.

A sequence is a chain of GEMVs in one persistent launch; op i+1 may read its input from op i's output (true data
dependency carried through HBM {value, epoch} words).  Every op's plain output C is compared with the oracle run on the
SAME input the GPU op saw (the GPU's own previous output), at the fp-path tolerance; the CTA-boundary placements (row
super-blocks cut in 2, 3, many pieces; CTAs without work) are swept through the `seq_grid` knob.
No test here reads /root/reference."""
import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from seq_util import build_chain, kc, oracle_gemv

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
TIGHT_TOL = 2e-5


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; libtmac_b200 has no CPU fallback")
    lib = tb.load()
    tb.check(lib.tmac_b200_init(0), "init")
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")
    yield lib
    torch.cuda.synchronize()
    tb.debug_set("seq_grid", 0)
    tb.check(lib.tmac_b200_set_stream(None), "set_stream")


@pytest.fixture(scope="module")
def oracle():
    return T.load_oracle()


def run_chain(lib, oracle, chain, x0, offsets, launches=2):
    seq = tb.Sequence()
    outs = []
    try:
        dx = torch.from_numpy(x0).cuda()
        for i, (cfg, A, S, wt) in enumerate(chain):
            o = torch.full((cfg.Mout,), float(i + 1), device="cuda")
            outs.append(o)
            if i == 0:
                seq.add(wt, x=dx, out=o)
            else:
                seq.add(wt, in_op=i - 1, in_offset=offsets[i], out=o)
        seq.build()
        for _ in range(launches):       # relaunch: epochs advance, every slot is reused
            seq.launch()
        seq.status()
        torch.cuda.synchronize()
        x = x0
        for i, (cfg, A, S, wt) in enumerate(chain):
            got = outs[i].cpu().numpy()
            ref = oracle_gemv(oracle, cfg, A, S, x)
            err = np.abs(got - ref).max() / np.abs(ref).max()
            assert err <= TIGHT_TOL, "op %d (%dx%d): rel err %.3g" % (i, cfg.Mout, cfg.K, err)
            if i + 1 < len(chain):
                nk = chain[i + 1][0].K
                x = got[offsets[i + 1]:offsets[i + 1] + nk].copy()     # the GPU's own output is the next op's input
        return seq.info()
    finally:
        seq.free()


CHAINS = {
    "w2zp": [T.Config(1024, 1024, 2, zero_point=True), T.Config(640, 1024, 2, zero_point=True), T.Config(512, 512, 2, zero_point=True),
             T.Config(1280, 512, 2, zero_point=True)],
    "w4": [T.Config(512, 1024, 4), T.Config(256, 512, 4), T.Config(768, 256, 4)],
    "w4zp_k11008": [T.Config(11008, 512, 4, zero_point=True), T.Config(320, 11008, 4, zero_point=True)],
    "w1": [T.Config(512, 2048, 1), T.Config(512, 512, 1)],
    "w3zp": [T.Config(384, 1024, 3, zero_point=True), T.Config(192, 384, 3, zero_point=True)],
    "partial": [T.Config(1024, 512, 2, zero_point=True), T.Config(640, 512, 2, zero_point=True), T.Config(512, 256, 2, zero_point=True),
                T.Config(256, 256, 2, zero_point=True)],      # later ops read only the leading rows of their producer
    "ragged": [T.Config(192, 512, 2, bm=128, zero_point=True), T.Config(320, 128, 2, bm=128, zero_point=True)],
}


CHAIN_FLAGS = (0, 1)           # resident chain (tmac_chain.cuh): data flow (default), grid-barrier form
CHAIN_DEFAULT = 0

# the per-CTA reduction buffer grows with the number of row super-blocks one CTA touches: the 11008-row chain needs >= 7 CTAs
CASES = [(n, g) for n in CHAINS for g in (0, 1, 2, 3, 7, 37) if not (n == "w4zp_k11008" and 0 < g < 7)]


@pytest.mark.parametrize("name,grid", CASES, ids=["%s-grid%d" % c for c in CASES])
def test_sequence_chain_matches_oracle(lib, oracle, name, grid):
    cfgs = [c.resolved() for c in CHAINS[name]]
    tb.debug_set("seq_grid", grid)
    chain = build_chain(cfgs, seed=31)
    try:
        x0 = np.random.default_rng(5).standard_normal(cfgs[0].K).astype(np.float16).astype(np.float32)
        offsets = [0] + [2 * (i % 3) if cfgs[i].K + 4 <= cfgs[i - 1].Mout else 0 for i in range(1, len(cfgs))]
        tb.debug_set("seq_impl", 0)                     # the stream-K sequence kernel
        info = run_chain(lib, oracle, chain, x0, offsets)
        assert info["grid"] == (grid if grid else torch.cuda.get_device_properties(0).multi_processor_count) and info["ring_slots"] > 0
        if grid == 0:                                   # the resident gemv3 chain, where the sequence qualifies (else it falls back)
            tb.debug_set("seq_impl", 2)
            for flags in CHAIN_FLAGS:                   # grid-barrier form and data-flow form
                tb.debug_set("chain_flags", flags)
                info = run_chain(lib, oracle, chain, x0, offsets)
                # every cluster must be resident (11008 W4 rows = 172 clusters are too many); the grid-barrier form reads its
                # chained inputs as float4, so it also needs offsets that are multiples of 4
                chained = name != "w4zp_k11008" and all(o % (4 if flags & 1 else 2) == 0 for o in offsets)
                assert (info["ring_slots"] == -4) if chained else (info["ring_slots"] > 0), (flags, info)
    finally:
        for c in chain:
            c[3].free()
        tb.debug_set("seq_grid", 0); tb.debug_set("seq_impl", 2); tb.debug_set("chain_flags", CHAIN_DEFAULT)


def test_sequence_equals_single_launch_path_within_reassociation(lib, oracle):
    """Same tensor through tmac_b200_gemv (gemv3, fused LUT) and through a one-op sequence (whichever kernel serves it): identical
    LUT bytes, so the outputs differ at most by fp32 re-association of the K split."""
    cfg = T.Config(2048, 4096, 2, zero_point=True).resolved()
    w, sc, z, x = T.make_problem(cfg, seed=41)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_reference_layout(kc(cfg), A, S)
    seq = tb.Sequence()
    try:
        dx = torch.from_numpy(x).cuda()
        a = torch.zeros((1, cfg.Mout), device="cuda"); b = torch.zeros((cfg.Mout,), device="cuda")
        tb.gemv(wt, 1, dx, a)
        seq.add(wt, x=dx[0], out=b)
        seq.build(); seq.launch(); seq.status()
        torch.cuda.synchronize()
        ref = oracle_gemv(oracle, cfg, A, S, x[0])
        for got in (a[0].cpu().numpy(), b.cpu().numpy()):
            assert np.abs(got - ref).max() <= TIGHT_TOL * np.abs(ref).max()
    finally:
        seq.free(); wt.free()


def test_sequence_independent_inputs_and_long_chain(lib, oracle):
    """32 ops on clones of one tensor, alternating external inputs and chained inputs, ring reuse across ops."""
    cfg = T.Config(1024, 1024, 2, zero_point=True).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=51)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    base = tb.upload_reference_layout(kc(cfg), A, S)
    wts = [base] + [tb.clone(base) for _ in range(7)]
    seq = tb.Sequence()
    try:
        rng = np.random.default_rng(6)
        xs = rng.standard_normal((32, cfg.K)).astype(np.float16).astype(np.float32)
        dxs = torch.from_numpy(xs).cuda()
        outs = torch.zeros((32, cfg.Mout), device="cuda")
        for i in range(32):
            if i % 3 == 0:
                seq.add(wts[i % 8], x=dxs[i], out=outs[i])
            else:
                seq.add(wts[i % 8], in_op=i - 1, in_offset=0, out=outs[i])
        seq.build()
        for _ in range(3):
            seq.launch()
        seq.status()
        got = outs.cpu().numpy()
        for i in range(32):
            x = xs[i] if i % 3 == 0 else got[i - 1][:cfg.K]
            ref = oracle_gemv(oracle, cfg, A, S, x)
            assert np.abs(got[i] - ref).max() <= TIGHT_TOL * np.abs(ref).max(), "op %d" % i
    finally:
        seq.free()
        for wt in wts:
            wt.free()


@pytest.mark.parametrize("impl,flags", [(0, 0), (1, 0), (1, 1)], ids=["streamk", "resident_chain", "resident_chain_grid_barrier"])
def test_sequence_full_size_llama_shape(lib, oracle, impl, flags):
    """BASELINE shape 11008x4096 W2 g128 zp at full size, two chained ops (down-projection shape second)."""
    cfgs = [T.Config(11008, 4096, 2, zero_point=True).resolved(), T.Config(4096, 11008, 2, zero_point=True).resolved()]
    chain = build_chain(cfgs, seed=61)
    tb.debug_set("seq_impl", impl); tb.debug_set("chain_flags", flags)
    try:
        x0 = np.random.default_rng(7).standard_normal(4096).astype(np.float16).astype(np.float32)
        info = run_chain(lib, oracle, chain, x0, [0, 0], launches=3)
        assert (info["ring_slots"] < 0) == (impl == 1)
    finally:
        tb.debug_set("seq_impl", 2); tb.debug_set("chain_flags", CHAIN_DEFAULT)
        for c in chain:
            c[3].free()


def test_sequence_rejects_bad_arguments(lib):
    cfg = T.Config(256, 512, 2, zero_point=True).resolved()
    w, sc, z, _ = T.make_problem(cfg, seed=1)
    A, S = T.pack_reference_layout(w, sc, z, cfg)
    wt = tb.upload_reference_layout(kc(cfg), A, S)
    cfg4 = T.Config(256, 512, 4).resolved()
    w4, sc4, z4, _ = T.make_problem(cfg4, seed=2)
    A4, S4 = T.pack_reference_layout(w4, sc4, z4, cfg4)
    wt4 = tb.upload_reference_layout(kc(cfg4), A4, S4)
    seq = tb.Sequence()
    try:
        with pytest.raises(tb.TMACError):
            seq.add(wt, in_op=0)                       # no earlier op
        x = torch.zeros(512, device="cuda")
        seq.add(wt, x=x)
        with pytest.raises(tb.TMACError):
            seq.add(wt, in_op=0, in_offset=0)          # K = 512 > producer's 256 rows
        seq.add(wt4, x=x)
        with pytest.raises(tb.TMACError):
            seq.build()                                # mixed bit widths
    finally:
        seq.free(); wt.free(); wt4.free()
