"""Harness shared by the decode-sequence and fused-input GPU suites: the library stream, tensors uploaded in the reference layout,
the ways a sequence can be run, a sequence built from step tuples, and the oracle, bit and norm helpers their checks use.
Fixtures are imported by name (from seq_util import stream, mk).  kfactor = act_group_size / 4 everywhere on the fp path: the
oracle (like the reference) is only right then."""
import collections
import contextlib

import numpy as np
import pytest

import tmac_b200 as tb
import tmac_oracle as T

torch = pytest.importorskip("torch")

TIGHT_TOL = 2e-5        # max |got - oracle| / max |oracle|
DENSE_NMSE = 5e-4       # against the dense dequantised GEMV (python/t_mac/ops/qgemm.py:277-282 of the reference)
CHAIN_RING = -4         # info()["ring_slots"] of a sequence served by the resident chain kernel (-kChainCS)
EPS = 1e-5

# (seq_impl, chain_flags, seq_grid) of the ways a sequence can be run; "auto*" let the build pick the chain when it qualifies
FORMS = {"flow": (1, 0, 0), "barrier": (1, 1, 0), "streamk": (0, 0, 0), "streamk_g7": (0, 0, 7), "auto": (2, 0, 0),
         "auto_barrier": (2, 1, 0), "auto_g7": (2, 0, 7)}

CHUNKINGS = [(128, 128), (128, 64), (128, 32), (64, 64), (64, 32), (32, 32), (256, 64)]    # (group_size, act_group_size)
A_CASES = [(g, a, b, b == 2) for g, a in CHUNKINGS for b in (1, 2, 4)] + [(128, 64, 3, True)]
A_IDS = ["g%d-ags%d-w%d%s" % (g, a, b, "zp" if z else "") for g, a, b, z in A_CASES]


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


@pytest.fixture(scope="module")
def stream():
    """A private stream for torch and the library, so torch's fills and copies are ordered with the library's launches."""
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
    """mk(*Op arguments) uploads an Op; every Op made in the test is freed after it."""
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


# One op of a sequence.  src: the name of an external input | the index of an earlier op, whose outputs [off, off + K) are the
# input | glu(...) | norm(...).  res: None | the name of an external residual | the index of an earlier op whose output is added.
# f16: the op stores fp16.
step = collections.namedtuple("step", "op src off res f16", defaults=(0, None, False))


def glu(gate_op, gate_off, up_op, up_off):
    """Source silu(g) * u, g and u the outputs [off, off + K) of the earlier ops gate_op and up_op."""
    return ("glu", gate_op, gate_off, up_op, up_off)


def norm(in_op, w, eps=EPS):
    """Source rmsnorm(h) * w: h the whole output of the earlier op in_op, w the name of an external [K] weight."""
    return ("norm", in_op, w, eps)


@contextlib.contextmanager
def sequence(steps, ext, n=1, observe=None, peers=None, explicit_batch=False):
    """Builds the sequence of `steps` over n activation rows; ext maps names to device tensors ([n][len] per-row vectors when
    n > 1, [K] norm weights).  Yields (seq, outs): outs[i] is op i's NaN-filled output, [Mout] or [n][Mout] for n > 1, or None
    where i is not in `observe` (the op writes the library's internal buffer).  peers: {op: peer addresses}.  explicit_batch:
    tmac_b200_seq_set_batch is called even for n = 1.  Knobs must be set before: they are read at build time."""
    seq = tb.Sequence(n)
    try:
        if explicit_batch:
            tb.check(tb.load().tmac_b200_seq_set_batch(seq.h, n), "tmac_b200_seq_set_batch")
        outs = []
        for i, (o, src, off, res, f16) in enumerate(steps):
            d = tb.F16 if f16 else tb.F32
            out = None
            if observe is None or i in observe:
                out = torch.full((o.cfg.Mout,) if n == 1 else (n, o.cfg.Mout), float("nan"), device="cuda",
                                 dtype=torch.float16 if f16 else torch.float32)
            if isinstance(src, str):
                seq.add(o.wt, x=ext[src], out=out, dtype=d)
            elif isinstance(src, int):
                seq.add(o.wt, in_op=src, in_offset=off, out=out, dtype=d)
            elif src[0] == "glu":
                seq.add_glu(o.wt, *src[1:], out=out, dtype=d)
            else:
                seq.add_rmsnorm(o.wt, src[1], ext[src[2]], src[3], out=out, dtype=d)
            if isinstance(res, str):
                seq.residual(i, r=ext[res])
            elif res is not None:
                seq.residual(i, r_op=res)
            outs.append(out)
        for i, ptrs in (peers or {}).items():
            seq.peer_outputs(i, ptrs)
        seq.build()
        yield seq, outs
    finally:
        seq.free()


def fetch(outs):
    return [None if o is None else o.cpu().numpy() for o in outs]


def expect_kernel(info, chained, grid=0):
    """The resident chain serves the sequence, or else the stream-K kernel on `grid` CTAs (0: one per SM)."""
    if chained:
        assert info["ring_slots"] == CHAIN_RING, info
    else:
        assert info["ring_slots"] > 0, info
        assert info["grid"] == (grid or torch.cuda.get_device_properties(0).multi_processor_count), info


def run_form(name, steps, ext, chained=None, launches=1, **kw):
    """Builds and launches the sequence in form `name`; asserts which kernel serves it (chained: the resident chain; by default
    when the form forces it).  kw goes to sequence().  Returns (info, outputs as numpy arrays, None where unobserved)."""
    impl, _, grid = FORMS[name]
    with form(name), sequence(steps, ext, **kw) as (seq, outs):
        info = seq.info()
        expect_kernel(info, impl == 1 if chained is None else chained, grid)
        for _ in range(launches):
            seq.launch()
        seq.status()
        return info, fetch(outs)


def host(rng, **sizes):
    """fp16-representable activations {name: array of that size}; a size is a length or a shape ([n][len] for a batch)."""
    return {k: rng.standard_normal(n).astype(np.float16).astype(np.float32) for k, n in sizes.items()}


def device(xs):
    return {k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda() for k, v in xs.items()}


def inputs(rng, **sizes):
    """host() activations and their device copies."""
    xs = host(rng, **sizes)
    return xs, device(xs)


def same_bits(a, b):
    """Same dtype, shape and bytes; numpy arrays or tensors."""
    a, b = (np.ascontiguousarray(t.cpu().numpy() if hasattr(t, "cpu") else t) for t in (a, b))
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def norm_weight(rng, K):
    """Norm weights around 1 with zeros and negative values."""
    w = (1.0 + 0.2 * rng.standard_normal(K)).astype(np.float32)
    w[rng.integers(0, K, size=K // 16)] = 0.0
    w[rng.integers(0, K, size=K // 16)] *= -1.0
    return w


def rms_input(h, w, eps):
    """The norm input a of each row of h ([N][K] or [K]; returns [N][K]), in numpy float32 in the documented order: lane l sums the
    4-element groups l, l + 32, ... in ascending order as (h0*h0 + h1*h1) + (h2*h2 + h3*h3), the 32 lane sums meet in the shfl_xor
    butterfly 16, 8, 4, 2, 1."""
    out = []
    for row in np.asarray(h, np.float32).reshape(-1, np.shape(h)[-1]):
        K = row.size
        g = row.reshape(-1, 4)
        q = (g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + (g[:, 2] * g[:, 2] + g[:, 3] * g[:, 3])
        q = np.concatenate([q, np.zeros(-len(q) % 32, np.float32)]).reshape(-1, 32)
        s = np.zeros(32, np.float32)
        for part in q:
            s = s + part
        for m in (16, 8, 4, 2, 1):
            s = s + s[np.arange(32) ^ m]
        inv = np.float32(1.0) / np.sqrt(s[0] / np.float32(K) + np.float32(eps))
        out.append((row * inv) * np.asarray(w, np.float32))
    return np.stack(out)
