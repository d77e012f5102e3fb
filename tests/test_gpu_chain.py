"""GPU suite (-m gpu): the decode sequence kernels -- the resident chain (tmac_chain.cuh, both forms) and the stream-K sequence
kernel (tmac_seq.cuh) -- at every chunking they are instantiated for, with inputs that change between launches, fan-out and skip
reads, internal and fp16 outputs, fp32 scales, peer outputs, and pinned per-warp ring depths.

Every op is compared with the oracle run on the input the GPU op saw (an external input, or the GPU's own output of its
producer), and where cheap with the float64 dense dequantised GEMV (W = (w - 2^(bits-1)) * s - z) at the reference's NMSE gate.
kfactor = act_group_size / 4 everywhere: the oracle (like the reference) is only right then."""
import contextlib
from types import SimpleNamespace

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T
from seq_util import kc, oracle_gemv

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TIGHT_TOL = 2e-5        # max |got - oracle| / max |oracle|
DENSE_NMSE = 5e-4       # against the dense dequantised GEMV (python/t_mac/ops/qgemm.py:277-282 of the reference)
CHAIN_RING = -4         # info()["ring_slots"] of a sequence served by the resident chain kernel (-kChainCS)

# (seq_impl, chain_flags, seq_grid) of the ways a sequence can be run; "auto*" let the build pick the chain when it qualifies
FORMS = {"flow": (1, 0, 0), "barrier": (1, 1, 0), "streamk": (0, 0, 0), "streamk_g7": (0, 0, 7), "auto": (2, 0, 0),
         "auto_barrier": (2, 1, 0)}


@pytest.fixture(scope="module")
def stream():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; libtmac_b200 has no CPU fallback")
    lib = tb.load()
    tb.check(lib.tmac_b200_init(0), "init")
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    tb.check(lib.tmac_b200_set_stream(st.cuda_stream), "set_stream")
    yield st
    torch.cuda.synchronize()
    tb.check(lib.tmac_b200_set_stream(None), "set_stream")
    torch.cuda.set_stream(torch.cuda.default_stream())


class Op:
    """One uploaded tensor and the problem it was made from (for the oracle and the dense reference)."""

    def __init__(self, Mout, K, bits, g=128, ags=64, zp=False, bm=0, seed=0, scale_mul=1.0, one_scale=False):
        self.cfg = cfg = T.Config(Mout, K, bits, bm=bm, kfactor=16 if one_scale else ags // 4, group_size=g, act_group_size=ags,
                                  zero_point=zp, one_scale=one_scale).resolved()
        self.w, sc, self.z, _ = T.make_problem(cfg, seed=seed)
        self.sc = (sc * np.float32(scale_mul)).astype(np.float32)      # scale_mul = 1 + 2^-13: not fp16-exact, stored as fp32
        self.A, self.S = T.pack_reference_layout(self.w, self.sc, self.z, cfg)
        self.wt = tb.upload_reference_layout(kc(cfg), self.A, self.S)


@pytest.fixture
def mk(stream):
    made = []

    def make(*a, **k):
        made.append(Op(*a, **k))
        return made[-1]
    yield make
    for o in made:
        o.wt.free()


@contextlib.contextmanager
def form(name):
    impl, flags, grid = FORMS[name]
    try:
        tb.debug_set("seq_impl", impl); tb.debug_set("chain_flags", flags); tb.debug_set("seq_grid", grid)
        yield
    finally:
        tb.debug_set("seq_impl", 2); tb.debug_set("chain_flags", 0); tb.debug_set("seq_grid", 0)


@contextlib.contextmanager
def sequence(steps, ext, dtypes=None, observe=None, peers=None):
    """Builds steps[i] = (op, src, offset): src names an external input in `ext` (device vectors) or is the index of an earlier
    step, whose outputs [offset, offset + K) are the input.  Yields (seq, outs); outs[i] is None where the step is unobserved
    (its output goes to the library's internal buffer).  Knobs must be set before: they are read at build time."""
    dtypes, peers = dtypes or {}, peers or {}
    seq = tb.Sequence()
    try:
        outs = []
        for i, (o, src, off) in enumerate(steps):
            dt = dtypes.get(i, tb.F32)
            out = None
            if observe is None or i in observe:
                out = torch.full((o.cfg.Mout,), float("nan"), dtype=torch.float16 if dt == tb.F16 else torch.float32, device="cuda")
            if isinstance(src, str):
                seq.add(o.wt, x=ext[src], out=out, dtype=dt)
            else:
                seq.add(o.wt, in_op=src, in_offset=off, out=out, dtype=dt)
            outs.append(out)
        for i, ptrs in peers.items():
            seq.peer_outputs(i, ptrs)
        seq.build()
        yield seq, outs
    finally:
        seq.free()


def fetch(outs):
    return [None if o is None else o.cpu().numpy() for o in outs]


def expect_kernel(info, chained, grid=0):
    if chained:
        assert info["ring_slots"] == CHAIN_RING, info
    else:
        assert info["ring_slots"] > 0, info
        assert info["grid"] == (grid or torch.cuda.get_device_properties(0).multi_processor_count), info


def run_form(name, steps, ext, chained=None, launches=1, **kw):
    """Builds and launches the sequence in form `name`; asserts which kernel serves it. Returns (info, outputs)."""
    impl, _, grid = FORMS[name]
    with form(name), sequence(steps, ext, **kw) as (seq, outs):
        info = seq.info()
        expect_kernel(info, impl == 1 if chained is None else chained, grid)
        for _ in range(launches):
            seq.launch()
        seq.status()
        return info, fetch(outs)


def check(oracle, steps, xs, got, dense=True):
    """Every op against the oracle, on the input the GPU op saw, and against the float64 dense dequantised GEMV."""
    for i, (o, src, off) in enumerate(steps):
        x = xs[src] if isinstance(src, str) else got[src][off:off + o.cfg.K].astype(np.float32)
        ref = oracle_gemv(oracle, o.cfg, o.A, o.S, x)
        err = np.abs(got[i] - ref).max() / np.abs(ref).max()
        assert err <= TIGHT_TOL, "op %d (%dx%d W%d): rel err %.3g" % (i, o.cfg.Mout, o.cfg.K, o.cfg.bits, err)
        if dense:
            e = T.nmse(T.dense_reference(o.w, o.sc, o.z, x, o.cfg)[0], got[i])
            assert e <= DENSE_NMSE, "op %d: NMSE %.3g against the dense dequantised GEMV" % (i, e)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def inputs(rng, **sizes):
    """fp16-representable activations: host copies and device vectors."""
    xs = {k: rng.standard_normal(n).astype(np.float16).astype(np.float32) for k, n in sizes.items()}
    return xs, {k: torch.from_numpy(v).cuda() for k, v in xs.items()}


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
CHUNKINGS = [(128, 128), (128, 64), (128, 32), (64, 64), (64, 32), (32, 32), (256, 64)]    # (group_size, act_group_size)
A_CASES = [(g, a, b, b == 2) for g, a in CHUNKINGS for b in (1, 2, 4)] + [(128, 64, 3, True)]


def chunking_chain(mk, g, ags, bits, zp):
    ck = min(g, 128)
    kw = dict(g=g, ags=ags, zp=zp)
    return [
        (mk(768, 20 * ck, bits, seed=1, **kw), "x0", 0),      # 20 chunks: some warps hold 2 blocks, some 1
        (mk(640, 512, bits, seed=2, **kw), 0, 0),             # fewer rows than op 0: idle clusters
        (mk(512, 512, bits, seed=3, **kw), 1, 128),           # offset on an activation group boundary (stream-K LUT hand-over)
        (mk(384 // bits, 256, bits, seed=4, **kw), 2, 4),     # ragged (not a whole row super-block, except W3); 256/ck < 16 chunks
    ]


@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=["g%d-ags%d-w%d%s" % (g, a, b, "zp" if z else "") for g, a, b, z in A_CASES])
def test_every_chunking_in_every_form(oracle, mk, monkeypatch, g, ags, bits, zp):
    steps = chunking_chain(mk, g, ags, bits, zp)
    xs, ext = inputs(np.random.default_rng(g + ags + bits), x0=steps[0][0].cfg.K)
    got = {}
    for name in ("flow", "barrier", "streamk", "streamk_g7"):
        info, got[name] = run_form(name, steps, ext)
        assert (info["quads_per_chunk"], info["quads_per_act_group"]) == (min(g, 128) // 16, ags // 16), info
        check(oracle, steps, xs, got[name], dense=name == "flow")
    # both chain forms: same inputs, same summation order
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), "op %d: the chain forms differ" % i
    # stream-K without the LUT hand-over: the consumers build the LUT bytes the producers would have handed over
    monkeypatch.setenv("TMAC_B200_SEQ_HANDOVER", "0")
    _, own = run_form("streamk", steps, ext)
    check(oracle, steps, xs, own, dense=False)
    for i, (a, b) in enumerate(zip(got["streamk"], own)):
        assert same_bits(a, b), "op %d: stream-K with and without the LUT hand-over differ" % i


# ---- B: inputs that change between launches (the {value, epoch} protocol) ----------------------------------------------------------
def epoch_chain(mk):
    kw = dict(zp=True)
    return [
        (mk(1024, 1024, 2, seed=11, **kw), "x0", 0),
        (mk(768, 1024, 2, seed=12, **kw), 0, 0),
        (mk(128, 11008, 2, seed=13, **kw), "xm", 0),          # external input in the middle of the chain; one cluster, 6 blocks
        (mk(1024, 128, 2, seed=14, **kw), 2, 0),              # clusters 1..7 have no work in op 2: they wait for its rows at once
        (mk(768, 768, 2, seed=15, **kw), 1, 0),               # reads the producer three ops back
        (mk(640, 512, 2, seed=16, **kw), 4, 4),
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
                xs = {k: rng.standard_normal(v.numel()).astype(np.float16).astype(np.float32) for k, v in ext.items()}
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
        (mk(1024, 1024, 2, seed=31, **kw), "x0", 0),
        (mk(768, 512, 2, seed=32, **kw), 0, 0),               # op 0 feeds ops 1, 2, 3
        (mk(512, 512, 2, seed=33, **kw), 0, 4),
        (mk(640, 512, 2, seed=34, **kw), 0, 2),               # offset 2: float4 loads of the barrier form do not allow it
        (mk(256, 768, 2, seed=35, **kw), 1, 0),               # skip: reads op 1
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
    _, f16 = run_form(name, steps, ext, dtypes={len(steps) - 1: tb.F16})
    assert f16[-1].dtype == np.float16 and same_bits(f16[-1], f32[-1].astype(np.float16))
    for i in range(len(steps) - 1):
        assert same_bits(f16[i], f32[i]), i


def test_fp16_producer_falls_back(oracle, mk):
    """An fp16 output that a later op reads cannot feed the chain's float4 loads: the chain refuses it, stream-K serves it (its
    consumers read the fp32 words) and computes what the fp32 sequence computes."""
    steps = fanout_chain(mk)
    xs, ext = inputs(np.random.default_rng(5), x0=1024)
    with pytest.raises(tb.TMACError):
        with form("flow"), sequence(steps, ext, dtypes={1: tb.F16}):
            pass
    _, ref = run_form("streamk", steps, ext)
    check(oracle, steps, xs, ref, dense=False)
    _, got = run_form("auto", steps, ext, chained=False, dtypes={1: tb.F16})
    assert same_bits(got[1], ref[1].astype(np.float16))
    for i in (0, 2, 3, 4):
        assert same_bits(got[i], ref[i]), i


def test_fp32_scales_mixed_with_fp16_scales(oracle, mk):
    """Tensors whose scales are not fp16-exact keep fp32 scales (larger blocks) in the same ring as fp16-scale tensors."""
    f32s = 1 + 2 ** -13
    steps = [
        (mk(1024, 1024, 2, zp=True, seed=41), "x0", 0),
        (mk(768, 1024, 2, zp=True, seed=42, scale_mul=f32s), 0, 0),
        (mk(1024, 512, 2, zp=True, seed=43), 1, 4),
        (mk(640, 512, 2, zp=True, seed=44, scale_mul=f32s), 2, 8),
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
    steps = [(mk(1024, 1024, 2, zp=True, seed=51), "x0", 0), (mk(768, 1024, 2, zp=True, seed=52), 0, 0)]
    xs, ext = inputs(np.random.default_rng(7), x0=1024)
    bufs = {0: [torch.full((1024,), float("nan"), device="cuda") for _ in range(npeer)],
            1: [torch.full((768,), float("nan"), dtype=torch.float16, device="cuda") for _ in range(npeer)]}
    peers = {i: [b.data_ptr() for b in bl] for i, bl in bufs.items()}
    _, got = run_form(name, steps, ext, dtypes={1: tb.F16}, peers=peers)
    check(oracle, steps[:1], xs, got[:1])
    for i, bl in bufs.items():
        for q, b in enumerate(bl):
            assert same_bits(b.cpu().numpy(), got[i]), (i, q)
    with pytest.raises(tb.TMACError):                       # stream-K has no peer stores: the build must refuse them
        with form("streamk_g7"), sequence(steps, ext, dtypes={1: tb.F16}, peers=peers):
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
        steps = [(SimpleNamespace(wt=wt, cfg=cfg), "x0", 0), (SimpleNamespace(wt=wt2, cfg=cfg), 0, 0)]
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
    steps = [(mk(256, K, 2, zp=True, seed=61), "x0", 0), (mk(256, 256, 2, zp=True, seed=62), 0, 0)]
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
        (mk(512, 11008, 2, seed=71, **kw), "xa", 0),
        (mk(512, 256, 2, seed=72, **kw), 0, 0),
        (mk(384, 512, 2, seed=73, **kw), 1, 0),
        (mk(640, 6144, 2, seed=74, **kw), "xd", 0),
        (mk(256, 512, 2, seed=75, **kw), 3, 4),
        (mk(256, 11008, 2, seed=76, **kw), "xf", 0),
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
        (mk(1024, 1024, 2, seed=81, **kw), "x0", 0),
        (mk(640, 1024, 2, seed=82, **kw), 0, 0),
        (mk(1024, 512, 2, seed=83, **kw), 1, 4),
    ]
    deep = shallow + [(mk(256, 11008, 2, seed=84, **kw), "xk", 0)]    # bpw 6, few rows: 7 stages
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
            with form(name), sequence([(bitnet, "x", 0)], ext):
                pass
    op = mk(1024, 512, 2, zp=True, seed=92)
    seq = tb.Sequence()
    try:
        seq.add(op.wt, x=ext["x"])
        with pytest.raises(tb.TMACError):
            seq.add(op.wt, in_op=0, in_offset=1)               # inputs start on an even element
    finally:
        seq.free()
