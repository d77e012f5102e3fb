"""GPU suite (-m gpu): routed MoE experts -- tmac_b200_gemv_experts (gate and up of every selected expert in one launch) and
tmac_b200_gemv_experts_glu (down behind SiLU*mul, with the weighted combine), both picking each token's experts from device ids.

Every slot is checked bit for bit against the equivalence the header documents: tmac_b200_gemv_grouped over the N * count * topk
selected tensors at N = 1 (the same decomposition), fed the slot's row -- the GLU input materialised on the GPU as
g / (1 + exp(-g)) * u.  The combine is restated in numpy float32 from those rows: w_0 * y_0, then + w_j * y_j in ascending j, then
+ R, rounded once to fp16 for an F16 call.  kfactor = act_group_size / 4 everywhere, as in the sequence tests."""
import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
from seq_util import A_CASES, A_IDS, DENSE_NMSE, TIGHT_TOL, mk, oracle_gemv, same_bits, stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def dev(x, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda().to(dtype)


def nan_out(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def normal(rng, *shape):
    return rng.standard_normal(shape).astype(np.float32)


def glu_ref(G, U):
    g, u = G.float(), U.float()
    return g / (1 + torch.exp(-g)) * u


def mout(obj):
    return obj.wt.cfg.M


def slot_rows(tab, ids, rows_of, key_of=lambda n, i, j: n, dtype=torch.float32):
    """The rows every slot must give.  tab(i, e) is tensor i of expert e, ids host int [N][topk], rows_of(n, i, j) the slot's input
    row (device [K]); slots with equal key_of take the same row.  As the header states: gemv_grouped at N = 1 over all
    N * count * topk selected tensors, fed the slot's row (one call per distinct row).  Returns {(n, i, j): numpy [Mout]}."""
    N, topk = ids.shape
    slots = [(n, i, j) for n in range(N) for i in range(tab.count) for j in range(topk)]
    sel = [tab(i, int(ids[n, j])) for n, i, j in slots]
    f16 = dtype == torch.float16
    out = {}
    for key in dict.fromkeys(key_of(*s) for s in slots):
        mine = [k for k, s in enumerate(slots) if key_of(*s) == key]
        outs = [nan_out(1, sel[0].cfg.M, dtype=dtype) for _ in sel]
        tb.gemv_grouped(sel, 1, rows_of(*slots[mine[0]])[None, :].contiguous(), outs, dtype=tb.F16 if f16 else tb.F32)
        torch.cuda.synchronize()
        for k in mine:
            out[slots[k]] = outs[k][0].cpu().numpy()
    return out


class Table:
    """tables[i][e] (objects with a .wt): tab(i, e) is its Weights."""

    def __init__(self, ops):
        self.ops, self.count = ops, len(ops)

    def __call__(self, i, e):
        return self.ops[i][e].wt

    def tables(self):
        return [[o.wt for o in row] for row in self.ops]


def combine(ys, w, R=None, f16=False):
    """ys [topk] numpy float32 rows, w [topk] float32: the documented combine in numpy float32."""
    acc = np.float32(w[0]) * ys[0]
    for j in range(1, len(ys)):
        acc = (acc + np.float32(w[j]) * ys[j]).astype(np.float32)
    if R is not None:
        acc = (acc + np.asarray(R, np.float32)).astype(np.float32)
    return acc.astype(np.float16) if f16 else acc


def run_experts(tab, N, B, ids, dtype=torch.float32):
    topk = ids.shape[1]
    outs = [nan_out(N, topk, mout(tab.ops[0][0]), dtype=dtype) for _ in range(tab.count)]
    tb.gemv_experts(tab.tables(), N, B.to(dtype), ids, outs, dtype=tb.F16 if dtype == torch.float16 else tb.F32)
    launch = tb.last_launch()
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs], launch


def check_experts(tab, N, B, hids, oracle=None, dtype=torch.float32):
    """gemv_experts of tab on B (device [N][K]) with host ids [N][topk]: every slot bit-identical to gemv_grouped."""
    ids = torch.from_numpy(hids.astype(np.int32)).cuda()
    got, launch = run_experts(tab, N, B, ids, dtype)
    assert launch["batch"] == tab.count * hids.shape[1], launch
    ref = slot_rows(tab, hids, lambda n, i, j: B[n].to(dtype), dtype=dtype)
    hB = B.float().cpu().numpy()
    for (n, i, j), r in ref.items():
        assert same_bits(got[i][n, j], r), "slot (n=%d, i=%d, j=%d) differs from gemv_grouped" % (n, i, j)
        if oracle is not None:
            op = tab.ops[i][int(hids[n, j])]
            o = oracle_gemv(oracle, op.cfg, op.A, op.S, hB[n])
            assert np.max(np.abs(got[i][n, j] - o)) <= TIGHT_TOL * np.max(np.abs(o))
    return got


def glu_expect(downs, hids, G, U, w, R=None, f16=False):
    """The C gemv_experts_glu must give: the slots' rows from gemv_grouped on the materialised GLU inputs, combined in numpy."""
    N, topk = hids.shape
    a = glu_ref(G, U)                                       # [N][topk][K] fp32
    ys = slot_rows(Table([downs]), hids, lambda n, i, j: a[n, j], key_of=lambda n, i, j: (n, j))
    hw = w.cpu().numpy()
    hR = None if R is None else R.float().cpu().numpy()
    return np.stack([combine([ys[(n, 0, j)] for j in range(topk)], hw[n], None if hR is None else hR[n], f16) for n in range(N)])


def run_glu(downs, N, G, U, ids, w, R=None, out=None, dtype=torch.float32):
    out = nan_out(N, mout(downs[0]), dtype=dtype) if out is None else out
    tb.gemv_experts_glu([o.wt for o in downs], N, G, U, ids, w, out, R=R, dtype=tb.F16 if dtype == torch.float16 else tb.F32)
    torch.cuda.synchronize()
    return out


def rand_ids(rng, N, topk, E):
    """ids in [0, E) with repeats inside a token (when topk > 1) and across tokens."""
    ids = rng.integers(0, E, size=(N, topk))
    if topk > 1:
        ids[0, 1] = ids[0, 0]
    if N > 1:
        ids[N - 1] = ids[0]
    return ids


def softmax_weights(rng, N, topk):
    v = normal(rng, N, topk)
    e = np.exp(v - v.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)


# ---- 1: every chunking -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g,ags,bits,zp", A_CASES, ids=A_IDS)
def test_every_chunking(mk, oracle, g, ags, bits, zp):
    """N in {1, 3}, topk in {1, 2, 4}, n_experts in {1, 8}, count in {1, 2}, with repeated ids; the GLU form on the same tensors."""
    K, M = 20 * min(g, 128), 256                  # 20 chunks: some warps hold 2 blocks, some 1
    ops = [[mk(M, K, bits, g=g, ags=ags, zp=zp, seed=100 * i + e) for e in range(8)] for i in range(2)]
    rng = np.random.default_rng(g + ags + bits)
    for N in (1, 3):
        B = dev(act_rows.rows(rng, N, K, ags))
        for topk in (1, 2, 4):
            for E in (1, 8):
                hids = rand_ids(rng, N, topk, E)
                for count in (1, 2):
                    full = topk == 2 and E == 8 and count == 2
                    check_experts(Table([row[:E] for row in ops[:count]]), N, B, hids, oracle if full else None)
                downs = ops[0][:E]
                G, U = dev(normal(rng, N, topk, K)), dev(act_rows.rows(rng, N * topk, K, ags).reshape(N, topk, K))
                ids, w = torch.from_numpy(hids.astype(np.int32)).cuda(), dev(softmax_weights(rng, N, topk))
                R = dev(normal(rng, N, M)) if topk != 1 else None
                got = run_glu(downs, N, G, U, ids, w, R=R)
                assert same_bits(got.cpu().numpy(), glu_expect(downs, hids, G, U, w, R)), (N, topk, E)


# ---- 2: the GLU form -------------------------------------------------------------------------------------------------------------
def test_glu_residual_forms(mk):
    """Without R, with R, with R == C, and fp16 G, U, R and C."""
    K, M, N, topk, E = 1024, 768, 3, 2, 4
    downs = [mk(M, K, 2, zp=True, seed=200 + e) for e in range(E)]
    rng = np.random.default_rng(201)
    hids = rand_ids(rng, N, topk, E)
    ids = torch.from_numpy(hids.astype(np.int32)).cuda()
    w = dev(softmax_weights(rng, N, topk))
    G, U, R = dev(normal(rng, N, topk, K)), dev(normal(rng, N, topk, K)), dev(normal(rng, N, M))
    got = run_glu(downs, N, G, U, ids, w)
    assert same_bits(got.cpu().numpy(), glu_expect(downs, hids, G, U, w))
    sep = run_glu(downs, N, G, U, ids, w, R=R)
    assert same_bits(sep.cpu().numpy(), glu_expect(downs, hids, G, U, w, R))
    inplace = R.clone()
    run_glu(downs, N, G, U, ids, w, R=inplace, out=inplace)
    assert same_bits(inplace.cpu().numpy(), sep.cpu().numpy())
    h16 = lambda *s: torch.from_numpy(act_rows.rows16(rng, int(np.prod(s[:-1])), s[-1], 64).reshape(s)).cuda().half()
    G16, U16, R16 = h16(N, topk, K), h16(N, topk, K), h16(N, M)
    got16 = run_glu(downs, N, G16, U16, ids, w, R=R16, dtype=torch.float16)
    assert same_bits(got16.cpu().numpy(), glu_expect(downs, hids, G16, U16, w, R16, f16=True))


def test_experts_fp16(mk):
    """fp16 B and C: each slot is gemv_grouped's fp16 output on the same row."""
    K, M, N, topk, E = 1024, 512, 2, 2, 3
    ops = [[mk(M, K, 4, seed=300 + 10 * i + e) for e in range(E)] for i in range(2)]
    rng = np.random.default_rng(301)
    hids = rand_ids(rng, N, topk, E)
    B16 = torch.from_numpy(act_rows.rows16(rng, N, K, 64)).cuda().half()
    check_experts(Table(ops), N, B16, hids, dtype=torch.float16)


# ---- 3: inputs that change, graphs -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_inputs_change_between_launches(stream, mk, graph):
    """ids, weights and inputs rewritten on the device before every launch (or CUDA-graph replay): both calls follow them, and the
    host never reads the ids."""
    K, F, N, topk, E = 1024, 2048, 2, 2, 4
    gu = Table([[mk(F, K, 2, zp=True, seed=400 + 10 * i + e) for e in range(E)] for i in range(2)])
    downs = [mk(K, F, 2, zp=True, seed=420 + e) for e in range(E)]
    rng = np.random.default_rng(430)
    x, ids, w = nan_out(N, K), torch.zeros((N, topk), dtype=torch.int32, device="cuda"), nan_out(N, topk)
    G, U, y = nan_out(N, topk, F), nan_out(N, topk, F), nan_out(N, K)
    gen = torch.Generator(device="cuda").manual_seed(431)

    def calls():
        tb.gemv_experts(gu.tables(), N, x, ids, [G, U])
        tb.gemv_experts_glu([o.wt for o in downs], N, G, U, ids, w, y, R=x)

    def fill():                                   # on the device only
        x.copy_(torch.randn((N, K), device="cuda", generator=gen))
        ids.copy_(torch.randint(0, E, (N, topk), device="cuda", generator=gen, dtype=torch.int32))
        w.copy_(torch.softmax(torch.randn((N, topk), device="cuda", generator=gen), dim=-1))

    fill(); calls(); torch.cuda.synchronize()     # warm-up: pointer tables, workspace, module load
    cg = None
    if graph:
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=stream):
            calls()
    seen = set()
    for _ in range(4):
        fill()
        if cg is not None:
            cg.replay()
        else:
            calls()
        torch.cuda.synchronize()
        hids = ids.cpu().numpy()
        seen.add(hids.tobytes())
        ref = slot_rows(gu, hids, lambda n, i, j: x[n])
        hG, hU = G.cpu().numpy(), U.cpu().numpy()
        for (n, i, j), r in ref.items():
            assert same_bits((hG, hU)[i][n, j], r)
        assert same_bits(y.cpu().numpy(), glu_expect(downs, hids, G, U, w, x))
    assert len(seen) > 1


# ---- 4: out-of-range ids ---------------------------------------------------------------------------------------------------------
def test_out_of_range_ids(mk):
    """A bad id gives NaN in exactly that slot (gemv_experts) or that token (gemv_experts_glu); the rest is unaffected, and the next
    call with valid ids is right (the combine's counters are back at zero)."""
    K, M, N, topk, E = 1024, 512, 3, 2, 4
    tab = Table([[mk(M, K, 2, zp=True, seed=500 + 10 * i + e) for e in range(E)] for i in range(2)])
    downs = [mk(M, K, 2, zp=True, seed=520 + e) for e in range(E)]
    rng = np.random.default_rng(530)
    B = dev(normal(rng, N, K))
    good = rand_ids(rng, N, topk, E)
    bad = good.copy()
    bad[0, 1], bad[2, 0] = E, -1                   # token 1 keeps valid ids
    got, _ = run_experts(tab, N, B, torch.from_numpy(bad.astype(np.int32)).cuda())
    ref = slot_rows(tab, good, lambda n, i, j: B[n])
    for (n, i, j), r in ref.items():
        if (n, j) in ((0, 1), (2, 0)):
            assert np.isnan(got[i][n, j]).all()
        else:
            assert same_bits(got[i][n, j], r)
    G, U = dev(normal(rng, N, topk, K)), dev(normal(rng, N, topk, K))
    w, R = dev(softmax_weights(rng, N, topk)), dev(normal(rng, N, M))
    y = run_glu(downs, N, G, U, torch.from_numpy(bad.astype(np.int32)).cuda(), w, R=R).cpu().numpy()
    want = glu_expect(downs, good, G, U, w, R)
    assert np.isnan(y[0]).all() and np.isnan(y[2]).all()
    assert same_bits(y[1], want[1])
    for ids in (np.full((N, topk), 2 ** 31 - 1), good):
        got, _ = run_experts(tab, N, B, torch.from_numpy(ids.astype(np.int32)).cuda())
        y = run_glu(downs, N, G, U, torch.from_numpy(ids.astype(np.int32)).cuda(), w, R=R).cpu().numpy()
    for (n, i, j), r in ref.items():
        assert same_bits(got[i][n, j], r)
    assert same_bits(y, want)


# ---- 5: a Mixtral-8x7B FFN ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_mixtral_ffn(stream, bits, zp):
    """hidden 4096, FFN 14336, 8 experts, top-2 at N = 1 and 4: against the gemv_grouped reference, and NMSE against dense
    dequantised experts."""
    from decode_harness import QLinear
    H, F, E, topk = 4096, 14336, 8, 2
    lin = {(n, e): QLinear(m, k, bits, 128, zp, seed=600 + 3 * e + t) for e in range(E)
           for t, (n, m, k) in enumerate((("gate", F, H), ("up", F, H), ("down", H, F)))}
    try:
        ex = lambda n: [lin[(n, e)] for e in range(E)]
        tab = Table([ex("gate"), ex("up")])
        rng = np.random.default_rng(601)
        deq = {}                                  # dense dequantised experts, made once
        for N in (1, 4):
            hids = np.stack([rng.choice(E, topk, replace=False) for _ in range(N)])
            ids = torch.from_numpy(hids.astype(np.int32)).cuda()
            h2, R = dev(normal(rng, N, H)), dev(normal(rng, N, H))
            w = dev(softmax_weights(rng, N, topk))
            G, U = nan_out(N, topk, F), nan_out(N, topk, F)
            tb.gemv_experts(tab.tables(), N, h2, ids, [G, U])
            y = nan_out(N, H)
            tb.gemv_experts_glu([l.wt for l in ex("down")], N, G, U, ids, w, y, R=R)
            torch.cuda.synchronize()
            hG, hU = G.cpu().numpy(), U.cpu().numpy()
            for (n, i, j), r in slot_rows(tab, hids, lambda n, i, j: h2[n]).items():
                assert same_bits((hG, hU)[i][n, j], r)
            assert same_bits(y.cpu().numpy(), glu_expect(ex("down"), hids, G, U, w, R))
            dense = torch.zeros_like(y)
            for n in range(N):
                for j in range(topk):
                    d = lambda name: deq.setdefault((name, int(hids[n, j])), lin[(name, int(hids[n, j]))].dense(torch))
                    g, u = h2[n] @ d("gate").T, h2[n] @ d("up").T
                    dense[n] += w[n, j] * ((torch.nn.functional.silu(g) * u) @ d("down").T)
            dense += R
            nmse = float(((y - dense) ** 2).mean() / (dense ** 2).mean())
            assert nmse <= DENSE_NMSE, (N, nmse)
    finally:
        for l in lin.values():
            l.free()


# ---- 6: rejections ---------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    K, M, N, topk, E = 1024, 512, 1, 2, 2
    tab = Table([[mk(M, K, 2, zp=True, seed=700 + e) for e in range(E)]])
    other = mk(2 * M, K, 2, zp=True, seed=710)
    downs = [mk(M, K, 2, zp=True, seed=720 + e) for e in range(E)]
    dw = [o.wt for o in downs]
    B, ids, w = torch.zeros((N, K), device="cuda"), torch.zeros((N, topk), dtype=torch.int32, device="cuda"), torch.full((N, topk), 0.5, device="cuda")
    G, U, R = torch.zeros((N, topk, K), device="cuda"), torch.zeros((N, topk, K), device="cuda"), torch.zeros((N, M), device="cuda")
    out, y = nan_out(N, topk, M), nan_out(N, M)
    ids9 = torch.zeros((N, 9), dtype=torch.int32, device="cuda")
    ids0 = torch.zeros((N, 0), dtype=torch.int32, device="cuda")
    hB, hids = np.zeros((N, K), np.float32), np.zeros((N, topk), np.int32)
    lib = tb.load()
    H = lambda ws: (tb.C.c_int64 * len(ws))(*[x.handle for x in ws])
    bad = [
        lambda: tb.gemv_experts(tab.tables(), N, B, ids9, [out]),                     # topk > 8, topk < 1
        lambda: tb.gemv_experts(tab.tables(), N, B, ids0, [out]),
        lambda: tb.gemv_experts_glu(dw, N, G, U, ids9, w, y),
        lambda: tb.gemv_experts_glu(dw, N, G, U, ids0, w, y),
        lambda: tb.gemv_experts(tab.tables(), 0, B, ids, [out]),                      # N < 1
        lambda: tb.gemv_experts_glu(dw, 0, G, U, ids, w, y),
        lambda: tb.check(lib.tmac_b200_gemv_experts(H(tab.tables()[0]), 1, 0, N, tb.F32, tb.ptr(B), tb.ptr(ids), topk,
                                                    (tb.C.c_void_p * 1)(tb.ptr(out))), "n_experts 0"),
        lambda: tb.check(lib.tmac_b200_gemv_experts_glu(H(dw), 0, N, tb.F32, tb.ptr(G), tb.ptr(U), tb.ptr(ids), tb.ptr(w), topk, 0,
                                                        tb.ptr(y)), "n_experts 0"),
        lambda: tb.check(lib.tmac_b200_gemv_experts(H(tab.tables()[0]), 1, E, N, 7, tb.ptr(B), tb.ptr(ids), topk,
                                                    (tb.C.c_void_p * 1)(tb.ptr(out))), "dtype"),
        lambda: tb.gemv_experts(tab.tables(), N, hB, ids, [out]),                     # host pointers
        lambda: tb.gemv_experts(tab.tables(), N, B, hids, [out]),
        lambda: tb.gemv_experts_glu(dw, N, G, U, hids, w, y),
        lambda: tb.gemv_experts_glu(dw, N, G, U, ids, w.cpu(), y),
        lambda: tb.gemv_experts_glu(dw, N, G.cpu(), U, ids, w, y),
        lambda: tb.gemv_experts_glu(dw, N, G, U.cpu(), ids, w, y),
        lambda: tb.gemv_experts_glu(dw, N, G, U, ids, w, y, R=R.cpu()),
        lambda: tb.gemv_experts(tab.tables(), N, B, None, [out]),                     # null ids, weights, U
        lambda: tb.gemv_experts_glu(dw, N, G, U, None, w, y),
        lambda: tb.gemv_experts_glu(dw, N, G, U, ids, None, y),
        lambda: tb.gemv_experts_glu(dw, N, G, None, ids, w, y),
        lambda: tb.gemv_experts([[tab.ops[0][0].wt, other.wt]], N, B, ids, [out]),    # different geometry
        lambda: tb.gemv_experts_glu([dw[0], other.wt], N, G, U, ids, w, y),
    ]
    torch.cuda.synchronize()
    for i, call in enumerate(bad):
        out.fill_(float("nan")); y.fill_(float("nan"))
        with pytest.raises(tb.TMACError):
            call()
        torch.cuda.synchronize()
        assert torch.isnan(out).all() and torch.isnan(y).all(), "rejected call %d launched" % i
    # an armed peer output makes the call fail, launch nothing and be disarmed, as for gemv_grouped
    for call in (lambda: tb.gemv_experts(tab.tables(), N, B, ids, [out]), lambda: tb.gemv_experts_glu(dw, N, G, U, ids, w, y)):
        peer = nan_out(1, M)
        out.fill_(float("nan")); y.fill_(float("nan"))
        tb.peer_outputs([peer.data_ptr()])
        with pytest.raises(tb.TMACError):
            call()
        torch.cuda.synchronize()
        assert torch.isnan(out).all() and torch.isnan(y).all()
        tb.gemv(dw[0], 1, torch.zeros((1, K), device="cuda"), torch.zeros((1, M), device="cuda"))   # would store into peer if armed
        torch.cuda.synchronize()
        assert torch.isnan(peer).all(), "the peer output stayed armed"
        call()


# ---- 7: the decode harness ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,zp", [(2, True), (4, False)], ids=["w2zp", "w4"])
def test_harness_moe_layer(stream, bits, zp):
    """A MoE layer against the same layer with dense dequantised fp32 weights and the same router choice, NMSE <= 5e-4."""
    from decode_harness import DecodeLayer
    hidden, ffn, heads, ctx, E = 1024, 2816, 8, 64, 4
    layer = DecodeLayer(hidden, ffn, heads, bits, zp, seed=5, fused_ops=True, experts=E, topk=2)
    try:
        hd = hidden // heads
        kc_, vc = torch.randn((heads, ctx, hd), device="cuda") * 0.3, torch.randn((heads, ctx, hd), device="cuda") * 0.3
        kc2, vc2 = kc_.clone(), vc.clone()
        pos = ctx - 1
        inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
        cos, sin = torch.cos(pos * inv)[None, :], torch.sin(pos * inv)[None, :]
        x = torch.randn((1, hidden), device="cuda")
        got = layer.forward(x, kc_, vc, pos, cos, sin).clone()
        routed = (layer.buf["ids"].clone(), layer.buf["wts"].clone())
        dense = {n: l.dense(torch) for n, l in layer.lin.items()}
        ref = layer.forward(x, kc2, vc2, pos, cos, sin, linear=lambda n, inp, out: out.copy_(inp @ dense[n].T), routed=routed).clone()
        torch.cuda.synchronize()
        nmse = float(((got - ref) ** 2).mean() / (ref ** 2).mean())
        assert nmse <= DENSE_NMSE, nmse
    finally:
        layer.free()


def test_harness_graphed_moe_token_step(stream):
    from decode_harness import DecodeModel
    m = DecodeModel(layers=3, hidden=1024, ffn=2816, heads=8, bits=2, zero_point=True, ctx=32, fused_ops=True, experts=4, topk=2)
    try:
        with torch.cuda.stream(stream):
            m.step()
        torch.cuda.synchronize()
        eager = m.y.clone()
        m.capture(stream)
        m.y.zero_()
        m.graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(m.y, eager)
    finally:
        m.free()


@pytest.mark.parametrize("kw", [dict(), dict(fused_ops=True, ffn_sequence=True), dict(fused_ops=True, post_attn_sequence=True)],
                         ids=["no_fused_ops", "ffn_sequence", "post_attn_sequence"])
def test_harness_rejects_experts_without_fused_ops(stream, kw):
    from decode_harness import DecodeLayer, DecodeModel
    with pytest.raises(ValueError):
        DecodeLayer(256, 512, 2, 2, True, seed=0, experts=4, **kw)
    with pytest.raises(ValueError):
        DecodeModel(1, 256, 512, 2, 2, True, ctx=8, experts=4, **kw)
