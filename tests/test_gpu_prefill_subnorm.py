"""GPU suite (-m gpu): one-scale fp-path tensors (one weight scale, activation groups < K: BitNet b1.58's grouping) on the routed
wgmma tiles, and tmac_b200_prefill_subnorm, the prompt-sized form of gemv_subnorm.

A one-scale tensor's row on either tile is checked bit for bit against the same row of its twin on the same tile: the same codes
uploaded with per-row scales all equal to the one scale, no zero points, the same group and activation group.  At K % 128 == 64 (chunk
64 K, the int8 tile only) the twin is not a tile tensor, so the rows are checked against the float oracle on the twin's config.
prefill_subnorm on per-row-scale tensors is checked bit for bit against tmac_b200_gemv on the same tile fed the input materialised in
fp32 (the GLU on the GPU, the norm in numpy float32 in the documented order), plus a numpy float32 add of the residual."""
import types

import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
import tmac_oracle as T
from fused_util import bm_of, dense_tile, knobs, launched, serial_input, tdt
from seq_util import DENSE_NMSE, EPS, TIGHT_TOL, mk, norm_weight, rms_input, same_bits, stream
from test_gpu_gemv_fused_io import dev, expect, glu_ref, nan_out, normal

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TILES = [True, False]
TILE_IDS = ["fp16", "int8"]
SCALE0 = float(np.float32(np.float16(0.037)))


@pytest.fixture
def pair(stream):
    """pair(M, K, bits, ags, seed) uploads a one-scale tensor and its twin with make_kcfg + upload_plain, as QLinear does.  The
    group is the chunk the layout picks for the one-scale tensor: 128 K, or 64 K when K % 128 == 64.  Both are freed after the test."""
    made = []

    def make(M, K, bits, ags, seed):
        rng = np.random.default_rng(seed)
        w = rng.integers(0, 1 << bits, size=(M, K), dtype=np.uint8)
        g, bm = (128 if K % 128 == 0 else 64), bm_of(M, bits)
        one = tb.upload_plain(tb.make_kcfg(M, K, bits, bm, ags // 4, g, ags, False, True), w, np.array([SCALE0], np.float32))
        made.append(one)
        sc = np.full((M, K // g), SCALE0, np.float32)
        twin = tb.upload_plain(tb.make_kcfg(M, K, bits, bm, ags // 4, g, ags, False, False), w, sc)
        made.append(twin)
        cfg = T.Config(M, K, bits, bm=bm, kfactor=ags // 4, group_size=g, act_group_size=ags).resolved()
        return types.SimpleNamespace(one=one, twin=twin, w=w, sc=sc, cfg=cfg, M=M, K=K)
    yield make
    for wt in made:
        wt.free()


def twin_forms(p, N, rng, t16, ags):
    """Every prefill_* form on the one-scale tensor and on its twin, on the same inputs: the outputs as numpy arrays."""
    M, K = p.M, p.K
    H, G, U = dev(act_rows.rows(rng, N, K, ags)), dev(act_rows.rows(rng, N, K, ags)), dev(normal(rng, N, K))   # U normal: no overflow
    R, w = dev(normal(rng, N, M)), dev(norm_weight(rng, K))
    out = {}
    for name, wt in (("one", p.one), ("twin", p.twin)):
        res = []
        with knobs(prefill16=int(t16)):
            o = [nan_out(N, M), nan_out(N, M)]
            tb.prefill_rmsnorm([wt, wt], N, H, w, EPS, o); launched(t16, N); res += o
            o = nan_out(N, M); tb.prefill_glu(wt, N, G, U, o, R=R); launched(t16, N); res.append(o)
            o = nan_out(N, M); tb.prefill_residual(wt, N, H, R, o); launched(t16, N); res.append(o)
            for dtype in (torch.float32, torch.float16):
                for u in (None, U):
                    for r in (None, R):
                        o = nan_out(N, M, dtype)
                        tb.prefill_subnorm(wt, N, G.to(dtype), w, EPS, o, U=None if u is None else u.to(dtype),
                                           R=None if r is None else r.to(dtype), dtype=tdt(dtype))
                        launched(t16, N)
                        res.append(o)
        torch.cuda.synchronize()
        out[name] = [x.cpu().numpy() for x in res]
    return out


# ---- 1: twin equality at K % 128 == 0 ---------------------------------------------------------------------------------------------
TWIN_CASES = [(2, 128), (2, 64), (2, 32), (4, 128), (4, 64), (4, 32), (3, 64)]


@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("bits,ags", TWIN_CASES, ids=["w%d-a%d" % c for c in TWIN_CASES])
def test_one_scale_equals_its_twin(pair, bits, ags, t16):
    """M = 384, K = 1024, N = 257 (a ragged last token tile on either tile): every call form, F32 and F16."""
    p = pair(384, 1024, bits, ags, seed=bits * 1000 + ags)
    got = twin_forms(p, 257, np.random.default_rng(bits + ags), t16, ags)
    for i, (a, b) in enumerate(zip(got["one"], got["twin"])):
        assert not np.isnan(a.astype(np.float32)).any(), "call %d left rows unwritten" % i
        assert same_bits(a, b), "call %d: the one-scale tensor differs from its twin" % i


@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_one_scale_experts_equal_their_twins(pair, t16):
    """prefill_experts over [gate, up] of 4 one-scale experts and prefill_experts_glu over their downs, against the twins."""
    E, topk, N, H, F = 4, 2, 520, 512, 1024       # N * topk >= 256 * E: prefill16 on picks the fp16 tile
    gate, up = [pair(F, H, 2, 64, seed=100 + e) for e in range(E)], [pair(F, H, 2, 64, seed=200 + e) for e in range(E)]
    down = [pair(H, F, 2, 64, seed=300 + e) for e in range(E)]
    rng = np.random.default_rng(5)
    ids = torch.from_numpy(rng.integers(0, E, size=(N, topk)).astype(np.int32)).cuda()
    wts = torch.from_numpy(rng.random((N, topk)).astype(np.float32)).cuda()
    B, R = dev(normal(rng, N, H)), dev(normal(rng, N, H))
    G, U = dev(normal(rng, N * topk, F)).view(N, topk, F), dev(normal(rng, N * topk, F)).view(N, topk, F)
    got = {}
    for kind in ("one", "twin"):
        pick = lambda ps: [getattr(x, kind) for x in ps]
        outs = [nan_out(N, topk * F).view(N, topk, F) for _ in range(2)]
        y = nan_out(N, H)
        with knobs(prefill16=int(t16)):
            tb.prefill_experts([pick(gate), pick(up)], N, B, ids, outs)
            launch = tb.last_launch()
            assert launch["cluster"] == (16 if t16 else 1) and launch["batch"] == -N * topk, launch
            tb.prefill_experts_glu(pick(down), N, G, U, ids, wts, y, R=R)
        torch.cuda.synchronize()
        got[kind] = [o.cpu().numpy() for o in outs + [y]]
    for a, b in zip(got["one"], got["twin"]):
        assert not np.isnan(a).any() and same_bits(a, b)


# ---- 2: K % 128 == 64 ---------------------------------------------------------------------------------------------------------------
def oracle_rows(oracle, p, a):
    """The float oracle on the twin's config (per-row scales all SCALE0): [N][M] for the fp32 rows a."""
    A, S = T.pack_reference_layout(p.w, p.sc, None, p.cfg)
    q, ls, lb = oracle.preprocessor(a, p.cfg.act_group_size)
    return oracle.qgemm(p.cfg, A, S, q, ls, lb)


@pytest.mark.parametrize("M,K,ags,N", [(384, 1088, 64, 257), (384, 1088, 32, 257), (3200, 8640, 64, 130)],
                         ids=["k1088-a64", "k1088-a32", "bitnet3b-down"])
def test_chunk64_on_the_int8_tile(pair, oracle, M, K, ags, N):
    """The int8 tile serves them with prefill16 on; every row within 2e-5 of the oracle; a row's bits do not depend on its
    neighbours or its token position; the result agrees with gemv_subnorm within 2e-5."""
    p = pair(M, K, 2, ags, seed=K + ags)
    rng = np.random.default_rng(K + ags)
    G, U = normal(rng, N, K), normal(rng, N, K)
    w = norm_weight(rng, K)

    def run(G_, U_):
        out = nan_out(N, M)
        with knobs(prefill16=1):
            tb.prefill_subnorm(p.one, N, dev(G_), dev(w), EPS, out, U=dev(U_))
            launched(False, N)
        torch.cuda.synchronize()
        return out.cpu().numpy()
    got = run(G, U)
    a = rms_input(glu_ref(dev(G), dev(U)).cpu().numpy(), w, EPS)
    ref = oracle_rows(oracle, p, a)
    for n in range(N):
        assert np.abs(got[n] - ref[n]).max() <= TIGHT_TOL * np.abs(ref[n]).max(), "row %d" % n
    gem = nan_out(N, M)
    tb.gemv_subnorm(p.one, N, dev(G), dev(w), EPS, gem, U=dev(U))
    torch.cuda.synchronize()
    assert np.abs(got - gem.cpu().numpy()).max() <= TIGHT_TOL * np.abs(ref).max()
    # row 0 at five token positions among other rows (both token tiles when N > 128)
    for pos in sorted({1, 63, 127 % N, 128 % N, N - 1}):
        G2, U2 = normal(rng, N, K), normal(rng, N, K)
        G2[pos], U2[pos] = G[0], U[0]
        assert same_bits(run(G2, U2)[pos], got[0]), "row 0 moved to position %d changed" % pos


# ---- 3: prefill_subnorm on per-row-scale tensors -------------------------------------------------------------------------------------
def check_subnorm(wt, N, G, w, t16, U=None, R=None, eps=EPS, dtype=torch.float32, out=None):
    """prefill_subnorm of host rows G (U, R) passed as dtype against dense_tile on the materialised input; returns a."""
    f16 = dtype == torch.float16
    dG, dU, dR = dev(G, dtype), None if U is None else dev(U, dtype), None if R is None else dev(R, dtype)
    out = nan_out(N, wt.cfg.M, dtype) if out is None else out
    with knobs(prefill16=int(t16)):
        tb.prefill_subnorm(wt, N, dG, dev(w), eps, out, U=dU, R=dR, dtype=tdt(dtype))
        launched(t16 and N >= 64, N)
    torch.cuda.synchronize()
    x = dG.float() if dU is None else glu_ref(dG, dU)
    a = rms_input(x.cpu().numpy(), w, eps)
    expect(out, dense_tile(wt, dev(a), t16 and N >= 64), None if dR is None else dR.float().cpu().numpy(), f16,
           "prefill_subnorm (U %s, R %s, %s)" % (U is not None, R is not None, "F16" if f16 else "F32"))
    return a


SUB_CASES = [("w2zp-g128-a64", 2, 128, 64, True), ("w4-g32-a32", 4, 32, 32, False)]


@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("name,bits,g,ags,zp", SUB_CASES, ids=[c[0] for c in SUB_CASES])
def test_subnorm_per_row_scales(mk, name, bits, g, ags, zp, t16):
    K, M, N = 2560, 512, 96
    op = mk(M, K, bits, g=g, ags=ags, zp=zp, seed=bits + g)
    rng = np.random.default_rng(g + ags)
    w = norm_weight(rng, K)
    for with_u in (False, True):
        for with_r in (False, True):
            check_subnorm(op.wt, N, act_rows.rows(rng, N, K, ags), w, t16, U=normal(rng, N, K) if with_u else None,
                          R=normal(rng, N, M) if with_r else None)
    # the two-magnitude SwiGLU row (the documented sum-of-squares order, not a serial one) and the all-zero row among normal rows
    g_two, u_two = np.abs(normal(rng, K)) + np.float32(4.0), np.float32(0.1) * normal(rng, K)
    u_two[:4] = 4096.0
    G, U = normal(rng, N, K), normal(rng, N, K)
    G[0], U[0], G[1] = g_two, u_two, 0.0
    R = normal(rng, N, M)
    a = check_subnorm(op.wt, N, G, w, t16, U=U)
    s = glu_ref(dev(G), dev(U)).cpu().numpy()
    assert not np.array_equal(a[0], serial_input(s[0], w, EPS)), "the two-magnitude row no longer tells the orders apart"
    assert not np.any(a[1])
    out = nan_out(N, M)
    check_subnorm(op.wt, N, G, w, t16, U=U, R=R, out=out)
    assert same_bits(out.cpu().numpy()[1], R[1]), "the zero row's output is R"
    for eps in (0.0, 0.5):
        check_subnorm(op.wt, N - 1, G[[0] + list(range(2, N))], w, t16, U=U[[0] + list(range(2, N))], eps=eps)
    # fp16 inputs and outputs
    h16 = lambda *s: act_rows.rows16(rng, s[0], s[1], ags)
    check_subnorm(op.wt, N, h16(N, K), w, t16, U=h16(N, K), R=normal(rng, N, M).astype(np.float16).astype(np.float32),
                  dtype=torch.float16)
    # R == C in place
    for dtype in (torch.float32, torch.float16):
        dG, dU, dR = dev(G, dtype), dev(U, dtype), dev(R, dtype)
        sep, inplace = nan_out(N, M, dtype), dR.clone()
        with knobs(prefill16=int(t16)):
            tb.prefill_subnorm(op.wt, N, dG, dev(w), EPS, sep, U=dU, R=dR, dtype=tdt(dtype))
            tb.prefill_subnorm(op.wt, N, dG, dev(w), EPS, inplace, U=dU, R=inplace, dtype=tdt(dtype))
        torch.cuda.synchronize()
        assert same_bits(inplace.cpu().numpy(), sep.cpu().numpy())


# ---- 4: graphs ------------------------------------------------------------------------------------------------------------------------
def test_graph_replays_follow_the_inputs(stream, pair):
    """A captured (o, down) pair of prefill_subnorm calls on buffers rewritten before every replay equals eager calls."""
    H, F, N = 1024, 1088, 130
    o, down = pair(H, H, 2, 64, seed=1), pair(H, F, 2, 64, seed=2)
    rng = np.random.default_rng(3)
    w_as, w_fs = dev(norm_weight(rng, H)), dev(norm_weight(rng, F))
    x, att, g, u = nan_out(N, H), nan_out(N, H), nan_out(N, F), nan_out(N, F)
    h, y = nan_out(N, H), nan_out(N, H)
    gen = torch.Generator(device="cuda").manual_seed(4)

    def calls():
        tb.prefill_subnorm(o.one, N, att, w_as, EPS, h, R=x)
        tb.prefill_subnorm(down.one, N, g, w_fs, EPS, y, U=u, R=h)

    def fill():
        for t in (x, att, g, u):
            t.copy_(torch.randn(t.shape, device="cuda", generator=gen))

    fill(); calls(); torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    seen = []
    for _ in range(3):
        fill()
        cg.replay()
        torch.cuda.synchronize()
        replayed = [h.clone(), y.clone()]
        seen.append(att.clone())
        calls()
        torch.cuda.synchronize()
        for a, b in zip(replayed, (h, y)):
            assert same_bits(a.cpu().numpy(), b.cpu().numpy())
    assert not torch.equal(seen[0], seen[1])


# ---- 5: rejections ----------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    from decode_harness import QLinear
    K, M, N = 1024, 512, 64
    op = mk(M, K, 2, zp=True, seed=80)
    w1 = mk(M, K, 1, seed=82)
    k64 = mk(M, 1088, 2, g=64, ags=64, zp=True, seed=83)          # per-row scales, K % 128 == 64: the GEMV only
    ip = QLinear(M, K, 2, 128, False, seed=84, one_scale=True)   # the integer path
    try:
        rng = np.random.default_rng(85)
        H, R, w = dev(normal(rng, N, K)), dev(normal(rng, N, M)), dev(norm_weight(rng, K))
        H64, w64 = dev(normal(rng, N, 1088)), dev(norm_weight(rng, 1088))
        out = nan_out(N, M)
        wbuf = torch.zeros(K + 4, device="cuda")
        lib = tb.load()
        huge = 1 << 25                                            # more than 65535 token tiles; nothing is read
        sub = lambda wt=op.wt, n=N, G=H, w_=w, eps=EPS, C=out, U=None, R_=R: tb.prefill_subnorm(wt, n, G, w_, eps, C, U=U, R=R_)
        bad = {
            "integer path": lambda: sub(wt=ip.wt),
            "w1": lambda: sub(wt=w1.wt, U=H),
            "K % 128 per-row": lambda: sub(wt=k64.wt, G=H64, w_=w64, U=H64),
            "host G": lambda: sub(G=H.cpu()),
            "host U": lambda: sub(U=H.cpu()),
            "host w": lambda: sub(w_=w.cpu()),
            "host R": lambda: sub(R_=R.cpu()),
            "host C": lambda: sub(C=out.cpu()),
            "null G": lambda: tb.check(lib.tmac_b200_prefill_subnorm(op.wt.handle, N, tb.F32, None, None, tb.ptr(w), EPS, None,
                                                                     tb.ptr(out)), "null G"),
            "null w": lambda: sub(w_=None),
            "unaligned w": lambda: sub(w_=wbuf[1:]),
            "negative eps": lambda: sub(eps=-1e-5),
            "nan eps": lambda: sub(eps=float("nan")),
            "inf eps": lambda: sub(eps=float("inf")),
            "N 0": lambda: sub(n=0),
            "token tiles": lambda: sub(n=huge),
        }
        msgs = {}
        for name, call in bad.items():
            out.fill_(float("nan"))
            torch.cuda.synchronize()
            try:
                call()
            except tb.TMACError as ex:
                msgs[name] = str(ex)
            else:
                pytest.fail("'%s' was not rejected" % name)
            torch.cuda.synchronize()
            assert torch.isnan(out).all(), "rejected call '%s' launched" % name
        for name in ("integer path", "w1", "K % 128 per-row"):
            assert "use gemv_subnorm" in msgs[name], msgs[name]
        assert "too large" in msgs["token tiles"]
        peer = nan_out(1, M)
        out.fill_(float("nan"))
        tb.peer_outputs([peer.data_ptr()])
        with pytest.raises(tb.TMACError):
            sub()
        torch.cuda.synchronize()
        assert torch.isnan(out).all()
        tb.gemv(op.wt, 1, torch.zeros((1, K), device="cuda"), torch.zeros((1, M), device="cuda"))
        torch.cuda.synchronize()
        assert torch.isnan(peer).all(), "the peer output stayed armed"
    finally:
        ip.free()


# ---- 6: the BitNet layer of the decode harness ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [16, 130])
def test_harness_bitnet_prompt(stream, P):
    """A sub_norms + fused_ops layer's prompt step (four tile launches) against the dense fp32 reference layer."""
    from decode_harness import DecodeLayer
    H, F = 1024, 1088
    layer = DecodeLayer(H, F, 8, 2, False, seed=11, fused_ops=True, sub_norms=True)
    try:
        torch.manual_seed(12)
        x = torch.randn((P, H), device="cuda")
        hd = H // 8
        ang = torch.arange(P, device="cuda").float()[:, None] / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(ang), torch.sin(ang)
        kc, vc = torch.zeros((8, P, hd), device="cuda"), torch.zeros((8, P, hd), device="cuda")
        got = layer.prompt(x, kc, vc, cos, sin).clone()
        assert tb.last_launch()["batch"] == -P, "the down projection did not run a tile"
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        want = layer.prompt(x, kc.clone(), vc.clone(), cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T)).clone()
        nmse = float(((got - want) ** 2).mean() / (want ** 2).mean())
        assert nmse < DENSE_NMSE, nmse
    finally:
        layer.free()


def test_harness_bitnet3b_graphed_prompt(stream):
    """Two BitNet-3B-shaped layers (hidden 3200, FFN 8640): the captured prompt step replays to the eager step's bits."""
    from decode_harness import DecodeModel
    m = DecodeModel(2, 3200, 8640, 32, 2, False, ctx=160, fused_ops=True, sub_norms=True, prompt_len=130)
    try:
        m.prompt()
        torch.cuda.synchronize()
        eager = m.py.clone()
        m.capture_prompt(stream)
        m.py.fill_(float("nan"))
        m.prompt_graph.replay()
        torch.cuda.synchronize()
        assert same_bits(m.py.cpu().numpy(), eager.cpu().numpy())
    finally:
        m.free()
