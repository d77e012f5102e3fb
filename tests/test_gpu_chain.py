"""GPU suite (-m gpu): the decode sequence kernels -- the resident chain (tmac_chain.cuh, both forms) and the stream-K sequence
kernel (tmac_seq.cuh) -- at every chunking they are instantiated for, with inputs that change between launches, fan-out and skip
reads, internal and fp16 outputs, fp32 scales, peer outputs, and pinned per-warp ring depths.

Every op is compared with the oracle run on the input the GPU op saw (an external input, or the GPU's own output of its
producer), and where cheap with the float64 dense dequantised GEMV (W = (w - 2^(bits-1)) * s - z) at the reference's NMSE gate.
kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
from types import SimpleNamespace

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from seq_util import (A_CASES, A_IDS, CHAIN_RING, DENSE_NMSE, FORMS, TIGHT_TOL, expect_kernel, fetch, form, host, inputs, mk,
                      oracle_gemv, run_form, same_bits, sequence, step, stream, kc)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def check(oracle, steps, xs, got, dense=True):
    """Every op against the oracle, on the input the GPU op saw, and against the float64 dense dequantised GEMV."""
    for i, (o, src, off, *_) in enumerate(steps):
        x = xs[src] if isinstance(src, str) else got[src][off:off + o.cfg.K].astype(np.float32)
        ref = oracle_gemv(oracle, o.cfg, o.A, o.S, x)
        err = np.abs(got[i] - ref).max() / np.abs(ref).max()
        assert err <= TIGHT_TOL, "op %d (%dx%d W%d): rel err %.3g" % (i, o.cfg.Mout, o.cfg.K, o.cfg.bits, err)
        if dense:
            e = T.nmse(T.dense_reference(o.w, o.sc, o.z, x, o.cfg)[0], got[i])
            assert e <= DENSE_NMSE, "op %d: NMSE %.3g against the dense dequantised GEMV" % (i, e)


def f16_at(steps, i):
    """The same steps with op i storing fp16."""
    return [s._replace(f16=True) if k == i else s for k, s in enumerate(steps)]


def ring_stages(info):
    """Stages per warp of a resident-chain sequence, from its shared-memory size.  Mirrors the size seq_build_chain (tmac_b200.cu)
    gives chain_kernel: (kChainCS + kChainWarps) * rsb * 4 + kChainWarps * (S * slot + qch * 32) + kChainWarps * S * 8 + 32,
    with rsb = 32 * 8 / planes per word and slot = the largest block rounded up to 128 bytes."""
    rsb = 32 * 8 // info["planes_per_word"]
    s, rem = divmod(info["smem_bytes"] - 32 - 8 * rsb * 4 - 4 * info["quads_per_chunk"] * 32, 4 * info["slot_bytes"] + 32)
    assert rem == 0 and s >= 2, info
    return s


def bpw(K, ck=128):
    return -(-(K // ck) // 16)          # blocks per warp: chunks over the 16 warps of a cluster


# ---- A: every instantiation (qch, agq) x planes per word, in every form ----------------------------------------------------------
def chunking_chain(mk, g, ags, bits, zp):
    ck = min(g, 128)
    kw = dict(g=g, ags=ags, zp=zp)
    return [
        step(mk(768, 20 * ck, bits, seed=1, **kw), "x0"),     # 20 chunks: some warps hold 2 blocks, some 1
        step(mk(640, 512, bits, seed=2, **kw), 0),            # fewer rows than op 0: idle clusters
        step(mk(512, 512, bits, seed=3, **kw), 1, 128),       # offset on an activation group boundary (stream-K LUT hand-over)
        step(mk(384 // bits, 256, bits, seed=4, **kw), 2, 4), # ragged (not a whole row super-block, except W3); 256/ck < 16 chunks
    ]


@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_every_chunking_in_every_form(oracle, mk, g, ags, bits, zp):
    steps = chunking_chain(mk, g, ags, bits, zp)
    xs, ext = inputs(np.random.default_rng(g + ags + bits), x0=steps[0].op.cfg.K)
    got = {}
    for name in ("flow", "barrier", "streamk", "streamk_g7"):
        info, got[name] = run_form(name, steps, ext)
        assert (info["quads_per_chunk"], info["quads_per_act_group"]) == (min(g, 128) // 16, ags // 16), info
        check(oracle, steps, xs, got[name], dense=name == "flow")
    # both chain forms: same inputs, same summation order
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), "op %d: the chain forms differ" % i
    # stream-K without the LUT hand-over: the consumers build the LUT bytes the producers would have handed over
    tb.debug_set("seq_handover", 0)
    try:
        _, own = run_form("streamk", steps, ext)
    finally:
        tb.debug_set("seq_handover", 1)
    check(oracle, steps, xs, own, dense=False)
    for i, (a, b) in enumerate(zip(got["streamk"], own)):
        assert same_bits(a, b), "op %d: stream-K with and without the LUT hand-over differ" % i


# ---- B: inputs that change between launches (the {value, epoch} protocol) ----------------------------------------------------------
def epoch_chain(mk):
    kw = dict(zp=True)
    return [
        step(mk(1024, 1024, 2, seed=11, **kw), "x0"),
        step(mk(768, 1024, 2, seed=12, **kw), 0),
        step(mk(128, 11008, 2, seed=13, **kw), "xm"),         # external input in the middle of the chain; one cluster, 6 blocks
        step(mk(1024, 128, 2, seed=14, **kw), 2),             # clusters 1..7 have no work in op 2: they wait for its rows at once
        step(mk(768, 768, 2, seed=15, **kw), 1),              # reads the producer three ops back
        step(mk(640, 512, 2, seed=16, **kw), 4, 4),
    ]


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["flow", "barrier", "streamk"])
def test_inputs_change_between_launches(stream, oracle, mk, name, graph):
    """A consumer that accepted a word from the previous launch would read the previous launch's value: every launch gets new
    inputs, written in place on the library stream, and every op is checked against that launch's inputs.  With `graph`, one
    capture of seq.launch() is replayed instead."""
    steps = epoch_chain(mk)
    rng = np.random.default_rng(17)
    ext = {"x0": torch.zeros(1024, device="cuda"), "xm": torch.zeros(11008, device="cuda")}
    impl = FORMS[name][0]
    with form(name), sequence(steps, ext) as (seq, outs):
        expect_kernel(seq.info(), impl == 1)
        g = None
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                seq.launch()
        try:
            for _ in range(3):
                xs = host(rng, **{k: v.numel() for k, v in ext.items()})
                for k, v in ext.items():
                    v.copy_(torch.from_numpy(xs[k]))           # current stream = the library stream: ordered before the launch
                if graph:
                    g.replay()
                else:
                    seq.launch()
                seq.status()
                check(oracle, steps, xs, fetch(outs), dense=False)
        finally:
            if g is not None:
                torch.cuda.synchronize()
                g.reset()


# ---- C: fan-out and skips, internal outputs, fp16 outputs, fp32 scales, peer outputs ---------------------------------------------
def fanout_chain(mk):
    kw = dict(zp=True)
    return [
        step(mk(1024, 1024, 2, seed=31, **kw), "x0"),
        step(mk(768, 512, 2, seed=32, **kw), 0),              # op 0 feeds ops 1, 2, 3
        step(mk(512, 512, 2, seed=33, **kw), 0, 4),
        step(mk(640, 512, 2, seed=34, **kw), 0, 2),           # offset 2: float4 loads of the barrier form do not allow it
        step(mk(256, 768, 2, seed=35, **kw), 1),              # skip: reads op 1
    ]


def test_fanout_and_skips(oracle, mk):
    steps = fanout_chain(mk)
    xs, ext = inputs(np.random.default_rng(3), x0=1024)
    with pytest.raises(tb.TMACError):
        with form("barrier"), sequence(steps, ext):
            pass
    full = {}
    for name, chained in (("flow", True), ("auto_barrier", False), ("streamk", False)):
        _, full[name] = run_form(name, steps, ext, chained=chained)
        check(oracle, steps, xs, full[name], dense=name == "flow")
    # internal outputs: every intermediate op writes the library's buffer, only the last op is observed
    for name in ("flow", "streamk"):
        _, got = run_form(name, steps, ext, observe={len(steps) - 1})
        assert got[:-1] == [None] * (len(steps) - 1)
        assert same_bits(got[-1], full[name][-1]), name


@pytest.mark.parametrize("name", ["flow", "streamk"])
def test_fp16_final_output(mk, name):
    steps = fanout_chain(mk)
    _, ext = inputs(np.random.default_rng(4), x0=1024)
    _, f32 = run_form(name, steps, ext)
    _, f16 = run_form(name, f16_at(steps, len(steps) - 1), ext)
    assert f16[-1].dtype == np.float16 and same_bits(f16[-1], f32[-1].astype(np.float16))
    for i in range(len(steps) - 1):
        assert same_bits(f16[i], f32[i]), i


def test_fp16_producer_falls_back(oracle, mk):
    """An fp16 output that a later op reads cannot feed the chain's float4 loads: the chain refuses it, stream-K serves it (its
    consumers read the fp32 words) and computes what the fp32 sequence computes."""
    steps = fanout_chain(mk)
    xs, ext = inputs(np.random.default_rng(5), x0=1024)
    with pytest.raises(tb.TMACError):
        with form("flow"), sequence(f16_at(steps, 1), ext):
            pass
    _, ref = run_form("streamk", steps, ext)
    check(oracle, steps, xs, ref, dense=False)
    _, got = run_form("auto", f16_at(steps, 1), ext, chained=False)
    assert same_bits(got[1], ref[1].astype(np.float16))
    for i in (0, 2, 3, 4):
        assert same_bits(got[i], ref[i]), i


def test_fp32_scales_mixed_with_fp16_scales(oracle, mk):
    """Tensors whose scales are not fp16-exact keep fp32 scales (larger blocks) in the same ring as fp16-scale tensors."""
    f32s = 1 + 2 ** -13
    steps = [
        step(mk(1024, 1024, 2, zp=True, seed=41), "x0"),
        step(mk(768, 1024, 2, zp=True, seed=42, scale_mul=f32s), 0),
        step(mk(1024, 512, 2, zp=True, seed=43), 1, 4),
        step(mk(640, 512, 2, zp=True, seed=44, scale_mul=f32s), 2, 8),
    ]
    xs, ext = inputs(np.random.default_rng(6), x0=1024)
    got = {}
    for name in ("flow", "barrier", "streamk"):
        info, got[name] = run_form(name, steps, ext)
        assert info["slot_bytes"] == 8 * 512 + 128 * 4 * 2, info           # W2 zp g128 block with fp32 scales and zeros
        check(oracle, steps, xs, got[name], dense=name == "flow")
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), i


@pytest.mark.parametrize("npeer", [1, 7])
@pytest.mark.parametrize("name", ["flow", "barrier"])
def test_peer_outputs_on_one_gpu(oracle, mk, name, npeer):
    """seq_peer_outputs with peer addresses that are ordinary local buffers: each holds exactly what C holds."""
    steps = [step(mk(1024, 1024, 2, zp=True, seed=51), "x0"), step(mk(768, 1024, 2, zp=True, seed=52), 0, f16=True)]
    xs, ext = inputs(np.random.default_rng(7), x0=1024)
    bufs = {0: [torch.full((1024,), float("nan"), device="cuda") for _ in range(npeer)],
            1: [torch.full((768,), float("nan"), dtype=torch.float16, device="cuda") for _ in range(npeer)]}
    peers = {i: [b.data_ptr() for b in bl] for i, bl in bufs.items()}
    _, got = run_form(name, steps, ext, peers=peers)
    check(oracle, steps[:1], xs, got[:1])
    for i, bl in bufs.items():
        for q, b in enumerate(bl):
            assert same_bits(b, got[i]), (i, q)
    with pytest.raises(tb.TMACError):                       # stream-K has no peer stores: the build must refuse them
        with form("streamk_g7"), sequence(steps, ext, peers=peers):
            pass


# ---- D: the per-warp ring depth ----------------------------------------------------------------------------------------------------
def test_ring_depth_of_the_bench_chain(stream):
    """The bench chain (11008x4096 W2 zp g128, bpw 2) gets a 3-stage ring: 60544 bytes of shared memory per CTA."""
    cfg = T.Config(11008, 4096, 2, zero_point=True).resolved()
    w, sc, z, x = T.make_problem(cfg, seed=8)
    wt = tb.upload_plain(kc(cfg), w, sc, z)
    wt2 = tb.clone(wt)
    try:
        ext = {"x0": torch.from_numpy(x[0]).cuda()}
        steps = [step(SimpleNamespace(wt=wt, cfg=cfg), "x0"), step(SimpleNamespace(wt=wt2, cfg=cfg), 0)]
        with form("flow"), sequence(steps, ext) as (seq, outs):
            info = seq.info()
            seq.launch()
            seq.status()
        assert info["ring_slots"] == CHAIN_RING and info["smem_bytes"] == 60544 and ring_stages(info) == 3, info
    finally:
        wt.free(); wt2.free()


@pytest.mark.parametrize("K", [2048, 4096, 6144, 11008])
def test_ring_depth_is_one_op_ahead_when_it_fits(oracle, mk, K):
    """Few rows (2 clusters): the deepest ring, max bpw + 1 stages (bpw 1, 2, 3, 6), fits in 227 KB and is chosen."""
    steps = [step(mk(256, K, 2, zp=True, seed=61), "x0"), step(mk(256, 256, 2, zp=True, seed=62), 0)]
    xs, ext = inputs(np.random.default_rng(K), x0=K)
    info, got = run_form("flow", steps, ext)
    s = ring_stages(info)
    assert s == bpw(K) + 1, (s, info)
    check(oracle, steps, xs, got)


def test_ring_carries_blocks_across_op_boundaries(oracle, mk):
    """Per-op block counts 6, 1, 1, 3, 1, 6 for warp 0 through a 7-stage ring: stages are reused across several ops and the
    mbarrier phase flips in the middle of an op."""
    kw = dict(zp=True)
    steps = [
        step(mk(512, 11008, 2, seed=71, **kw), "xa"),
        step(mk(512, 256, 2, seed=72, **kw), 0),
        step(mk(384, 512, 2, seed=73, **kw), 1),
        step(mk(640, 6144, 2, seed=74, **kw), "xd"),
        step(mk(256, 512, 2, seed=75, **kw), 3, 4),
        step(mk(256, 11008, 2, seed=76, **kw), "xf"),
    ]
    xs, ext = inputs(np.random.default_rng(9), xa=11008, xd=6144, xf=11008)
    got = {}
    for name in ("flow", "barrier"):
        info, got[name] = run_form(name, steps, ext, launches=2)
        assert ring_stages(info) == 7, info
        check(oracle, steps, xs, got[name], dense=False)
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), i


def depth_chains(mk):
    kw = dict(zp=True)
    shallow = [                                                # max bpw 1, 8 row super-blocks
        step(mk(1024, 1024, 2, seed=81, **kw), "x0"),
        step(mk(640, 1024, 2, seed=82, **kw), 0),
        step(mk(1024, 512, 2, seed=83, **kw), 1, 4),
    ]
    deep = shallow + [step(mk(256, 11008, 2, seed=84, **kw), "xk")]   # bpw 6, few rows: 7 stages
    return shallow, deep


@pytest.mark.parametrize("name", ["flow", "barrier"])
def test_outputs_do_not_depend_on_ring_depth(oracle, mk, name):
    shallow, deep = depth_chains(mk)
    xs, ext = inputs(np.random.default_rng(10), x0=1024, xk=11008)
    si, s_got = run_form(name, shallow, ext)
    di, d_got = run_form(name, deep, ext)
    assert (ring_stages(si), ring_stages(di)) == (2, 7), (si, di)
    check(oracle, deep, xs, d_got, dense=False)
    for i in range(len(shallow)):
        assert same_bits(s_got[i], d_got[i]), i


def test_interleaved_ring_depths_keep_launching(oracle, mk):
    """A deep sequence built before a shallow one on the same kernel still launches after the shallow one was built and run."""
    shallow, deep = depth_chains(mk)
    xs, ext = inputs(np.random.default_rng(11), x0=1024, xk=11008)
    with form("flow"), sequence(deep, ext) as (dseq, douts), sequence(shallow, ext) as (sseq, souts):
        assert (ring_stages(dseq.info()), ring_stages(sseq.info())) == (7, 2)
        for seq, outs, steps in ((dseq, douts, deep), (sseq, souts, shallow), (dseq, douts, deep)):
            for o in outs:
                o.fill_(float("nan"))
            seq.launch()
            seq.status()
            check(oracle, steps, xs, fetch(outs), dense=False)


def test_sequence_rejects_integer_path_and_odd_offset(mk):
    xs, ext = inputs(np.random.default_rng(12), x=512)
    bitnet = mk(256, 512, 2, one_scale=True, seed=91)          # act group = K: the integer path, which no sequence kernel runs
    for name in ("auto", "streamk"):
        with pytest.raises(tb.TMACError):
            with form(name), sequence([step(bitnet, "x")], ext):
                pass
    op = mk(1024, 512, 2, zp=True, seed=92)
    seq = tb.Sequence()
    try:
        seq.add(op.wt, x=ext["x"])
        with pytest.raises(tb.TMACError):
            seq.add(op.wt, in_op=0, in_offset=1)               # inputs start on an even element
    finally:
        seq.free()
