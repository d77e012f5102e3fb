"""GPU suite (-m gpu): routed MoE experts at prefill sizes -- tmac_b200_prefill_experts and tmac_b200_prefill_experts_glu, which
group each expert's slots on the device and run them on the wgmma tiles.

Every slot is checked bit for bit against the equality the header documents: the dense tile call tmac_b200_gemv on the expert's
rows in ascending slot order, forced onto the same tile (prefill_min_n = 1; prefill16 = 0 for the int8 tile; rows padded past the
expert's own to 64 when the fp16 tile needs them -- the padding comes after the real rows, so it moves none of them).  The GLU
form's rows are the GLU input materialised on the GPU as g / (1 + exp(-g)) * u, and its combine is the numpy restatement of the
GEMV form's suite.  kfactor = act_group_size / 4 everywhere, as in the sequence tests."""

import numpy as np
import pytest

import act_rows
import tmac_b200 as tb
from fused_util import dense_tile, knobs, tdt
from seq_util import DENSE_NMSE, TIGHT_TOL, mk, oracle_gemv, same_bits, stream
from test_gpu_experts import Table, combine, dev, glu_ref, nan_out, normal, rand_ids, softmax_weights

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

PF16_TOL = 5e-4                  # the fp16 tile against the oracle, max |got - oracle| / max |oracle| (DESIGN 3.3)
TILES = [True, False]
TILE_IDS = ["fp16", "int8"]
GROUPINGS = [(128, 128), (128, 64), (128, 32), (64, 64), (64, 32), (32, 32)]    # every fp grouping the tiles take
G_CASES = [(g, a, b) for g, a in GROUPINGS for b in (2, 4)] + [(128, 64, 3)]
G_IDS = ["g%d-ags%d-w%d" % c for c in G_CASES]


def expert_slots(hids, E):
    """{e: the slots s = n * topk + j of expert e, ascending} for the valid ids."""
    flat = hids.reshape(-1)
    return {e: np.nonzero(flat == e)[0] for e in range(E) if (flat == e).any()}


def slot_refs(tab, hids, rows, t16, dtype=torch.float32):
    """[count] numpy [N * topk][Mout]: each slot's row from the dense tile on its expert's rows (rows(slots) -> device rows); NaN
    where the id is out of range."""
    N, topk = hids.shape
    E = len(tab.ops[0])
    refs = []
    for i in range(tab.count):
        ref = np.full((N * topk, tab(i, 0).cfg.M), np.nan, np.float16 if dtype == torch.float16 else np.float32)
        for e, sl in expert_slots(hids, E).items():
            ref[sl] = dense_tile(tab(i, e), rows(sl), t16, dtype)
        refs.append(ref)
    return refs


def run_plain(tab, N, B, hids, dtype=torch.float32):
    topk = hids.shape[1]
    ids = torch.from_numpy(hids.astype(np.int32)).cuda()
    outs = [nan_out(N, topk, tab(i, 0).cfg.M, dtype=dtype) for i in range(tab.count)]
    tb.prefill_experts(tab.tables(), N, B.to(dtype), ids, outs, dtype=tdt(dtype))
    launch = tb.last_launch()
    torch.cuda.synchronize()
    return [o.cpu().numpy().reshape(N * topk, -1) for o in outs], launch


def check_plain(tab, N, B, hids, t16, dtype=torch.float32, oracle=None):
    """prefill_experts on the tile the rule picks (prefill16 on or off): each slot bit-identical to the dense tile, NaN rows for
    the slots of out-of-range ids; with `oracle`, a few slots within the tile's bound of the float oracle."""
    topk = hids.shape[1]
    with knobs(prefill16=int(t16)):
        got, launch = run_plain(tab, N, B, hids, dtype)
    assert launch["cluster"] == (16 if t16 else 1) and launch["batch"] == -N * topk, launch
    refs = slot_refs(tab, hids, lambda sl: B[sl // topk], t16, dtype)
    ok = ((hids >= 0) & (hids < len(tab.ops[0]))).reshape(-1)
    for i in range(tab.count):
        assert same_bits(got[i][ok], refs[i][ok]), "tensor %d differs from the dense tile" % i
        assert np.isnan(got[i][~ok]).all()
    if oracle is not None:                   # the tiles' bounds: max |got - oracle| over the checked slots <= tol * max |oracle|
        hB = B.float().cpu().numpy()
        sl = [s for s in np.linspace(0, N * topk - 1, 32).astype(int) if ok[s]]
        o = np.stack([oracle_gemv(oracle, tab.ops[0][e].cfg, tab.ops[0][e].A, tab.ops[0][e].S, hB[s // topk])
                      for s, e in ((s, int(hids.reshape(-1)[s])) for s in sl)])
        assert np.abs(got[0][sl] - o).max() <= (PF16_TOL if t16 else TIGHT_TOL) * np.abs(o).max()
    return got


def skewed_ids(rng, N, topk, E, big, big_count):
    """ids [N][topk] with exactly big_count slots of expert `big`, the rest spread over the experts other than big and E - 1 (which
    gets none); repeats inside a token allowed."""
    flat = rng.permutation(np.concatenate([np.full(big_count, big), rng.choice([e for e in range(E - 1) if e != big] or [big],
                                                                                N * topk - big_count)]))
    return flat.reshape(N, topk)


def same_glu(y, want):
    """y equals glu_refs' want bit for bit, NaN rows (tokens with an out-of-range id) as NaN."""
    y = y.cpu().numpy() if hasattr(y, "cpu") else y
    nan = np.isnan(want).all(axis=1)
    return same_bits(y[~nan], want[~nan]) and np.isnan(y[nan]).all()


def glu_refs(downs, hids, G, U, w, t16, R=None, f16=False):
    """The C prefill_experts_glu must give: the slots' rows from the dense tile on the materialised GLU inputs, combined in numpy
    (NaN rows for the tokens with an out-of-range id)."""
    N, topk = hids.shape
    a = glu_ref(G, U).reshape(N * topk, -1)
    ys = slot_refs(Table([downs]), hids, lambda sl: a[sl], t16)[0]
    hw = w.cpu().numpy()
    hR = None if R is None else R.float().cpu().numpy()
    bad = ((hids < 0) | (hids >= len(downs))).any(axis=1)
    out = []
    for n in range(N):
        if bad[n]:
            out.append(np.full(ys.shape[1], np.nan, np.float16 if f16 else np.float32))
        else:
            out.append(combine([ys[n * topk + j] for j in range(topk)], hw[n], None if hR is None else hR[n], f16))
    return np.stack(out)


def run_glu(downs, N, G, U, ids, w, R=None, out=None, dtype=torch.float32):
    out = nan_out(N, downs[0].wt.cfg.M, dtype=dtype) if out is None else out
    tb.prefill_experts_glu([o.wt for o in downs], N, G, U, ids, w, out, R=R, dtype=tdt(dtype))
    torch.cuda.synchronize()
    return out


# ---- 1: every fp grouping, both tiles ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("g,ags,bits", G_CASES, ids=G_IDS)
def test_groupings(mk, oracle, g, ags, bits, t16):
    """E = 4, N = 512, top-2: expert 0 has 260 rows (past a token-tile boundary of either tile), expert 3 none."""
    K, M, N, topk, E = 1024, 256, 512, 2, 4
    tab = Table([[mk(M, K, bits, g=g, ags=ags, zp=bits == 2, seed=10 * bits + e) for e in range(E)]])
    rng = np.random.default_rng(g + ags + bits)
    hids = skewed_ids(rng, N, topk, E, 0, 260)
    B = dev(act_rows.rows(rng, N, K, ags))
    check_plain(tab, N, B, hids, t16, oracle=oracle)


# ---- 2: grouping edges -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_grouping_edges(mk, t16):
    """All slots to one expert; experts of exactly T and T + 1 rows; top-1 and top-8 with repeated ids; one expert and 64 experts."""
    K, M = 512, 256
    T = 256 if t16 else 128
    rng = np.random.default_rng(40)
    tab = Table([[mk(M, K, 2, zp=True, seed=400 + e) for e in range(4)]])
    N = 520
    B = dev(normal(rng, N, K))
    check_plain(Table([tab.ops[0][:2]]), N, B, np.ones((N, 1), int), t16)                 # all slots to expert 1
    N = 2 * T + 1
    B = dev(normal(rng, N, K))
    check_plain(Table([tab.ops[0][:2]]), N, B, rng.permutation(np.r_[np.zeros(T, int), np.ones(T + 1, int)])[:, None], t16)
    N = 128
    B = dev(normal(rng, N, K))
    check_plain(tab, N, B, rand_ids(rng, N, 8, 4), t16)                                   # top-8, repeats inside tokens
    one = Table([[mk(M, K, 4, seed=410)]])
    N = 256
    check_plain(one, N, dev(normal(rng, N, K)), np.zeros((N, 1), int), t16)
    E, Ms, Ks = 64, 128, 256
    many = Table([[mk(Ms, Ks, 2, zp=True, seed=500 + e) for e in range(E)]])
    N = 8192 if t16 else 300                                                              # the fp16 tile needs N * topk >= 256 * E
    check_plain(many, N, dev(normal(rng, N, Ks)), rand_ids(rng, N, 2, E), t16)


@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_fp16_inputs_and_outputs(mk, t16):
    K, M, N, topk, E = 1024, 512, 384, 2, 3
    tab = Table([[mk(M, K, 4, seed=600 + e) for e in range(E)]])
    rng = np.random.default_rng(601)
    B16 = torch.from_numpy(act_rows.rows16(rng, N, K, 64)).cuda().half()
    check_plain(tab, N, B16, rand_ids(rng, N, topk, E), t16, dtype=torch.float16)


@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_count_two(mk, t16):
    """Gate and up of every selected expert in one launch."""
    K, M, N, topk, E = 1024, 384, 512, 2, 4
    tab = Table([[mk(M, K, 2, zp=True, seed=700 + 10 * i + e) for e in range(E)] for i in range(2)])
    rng = np.random.default_rng(701)
    check_plain(tab, N, dev(normal(rng, N, K)), rand_ids(rng, N, topk, E), t16)


# ---- 3: column independence ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_column_independence(mk, t16):
    """The same token row at different tile positions and among different neighbours gives the same bits: the property the
    per-slot equality rests on."""
    K, M, N = 1024, 512, 300
    tab = Table([[mk(M, K, 4, seed=800)]])
    rng = np.random.default_rng(801)
    x = dev(normal(rng, 1, K))
    got = []
    for pos in (0, 5, 137, 255, 299):
        B = dev(normal(rng, N, K))
        B[pos] = x[0]
        with knobs(prefill16=int(t16)):
            out, _ = run_plain(tab, N, B, np.zeros((N, 1), int))
        got.append(out[0][pos])
    for r in got[1:]:
        assert same_bits(r, got[0])


# ---- 4: the GLU form -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_glu_forms(mk, t16):
    """Without R, with R, with R == C, and fp16 G, U, R and C."""
    K, M, N, topk, E = 1024, 768, 512, 2, 4
    downs = [mk(M, K, 2, zp=True, seed=900 + e) for e in range(E)]
    rng = np.random.default_rng(901)
    hids = skewed_ids(rng, N, topk, E, 1, 270)
    ids = torch.from_numpy(hids.astype(np.int32)).cuda()
    w = dev(softmax_weights(rng, N, topk))
    G, U, R = dev(normal(rng, N, topk, K)), dev(normal(rng, N, topk, K)), dev(normal(rng, N, M))
    with knobs(prefill16=int(t16)):
        got = run_glu(downs, N, G, U, ids, w)
        assert tb.last_launch()["cluster"] == (16 if t16 else 1)
        sep = run_glu(downs, N, G, U, ids, w, R=R)
        inplace = R.clone()
        run_glu(downs, N, G, U, ids, w, R=inplace, out=inplace)
    assert same_glu(got, glu_refs(downs, hids, G, U, w, t16))
    assert same_glu(sep, glu_refs(downs, hids, G, U, w, t16, R))
    assert same_bits(inplace.cpu().numpy(), sep.cpu().numpy())
    h16 = lambda *s: torch.from_numpy(act_rows.rows16(rng, int(np.prod(s[:-1])), s[-1], 64).reshape(s)).cuda().half()
    G16, U16, R16 = h16(N, topk, K), h16(N, topk, K), h16(N, M)
    with knobs(prefill16=int(t16)):
        got16 = run_glu(downs, N, G16, U16, ids, w, R=R16, dtype=torch.float16)
    assert same_glu(got16, glu_refs(downs, hids, G16, U16, w, t16, R16, f16=True))


def test_moe_ffn_against_dense(stream):
    """prefill_experts (gate, up) -> prefill_experts_glu (down) against a float64 dequantised FFN with the same routing."""
    from decode_harness import QLinear
    H, F, E, topk, N = 1024, 2816, 4, 2, 512
    lin = {(n, e): QLinear(m, k, 2, 128, True, seed=1000 + 3 * e + t) for e in range(E)
           for t, (n, m, k) in enumerate((("gate", F, H), ("up", F, H), ("down", H, F)))}
    try:
        ex = lambda n: [lin[(n, e)] for e in range(E)]
        rng = np.random.default_rng(1001)
        hids = np.stack([rng.choice(E, topk, replace=False) for _ in range(N)])
        ids = torch.from_numpy(hids.astype(np.int32)).cuda()
        x, R, w = dev(normal(rng, N, H)), dev(normal(rng, N, H)), dev(softmax_weights(rng, N, topk))
        G, U, y = nan_out(N, topk, F), nan_out(N, topk, F), nan_out(N, H)
        tb.prefill_experts(Table([ex("gate"), ex("up")]).tables(), N, x, ids, [G, U])
        assert tb.last_launch()["cluster"] == 16
        tb.prefill_experts_glu([l.wt for l in ex("down")], N, G, U, ids, w, y, R=R)
        torch.cuda.synchronize()
        x64, y64 = x.double(), R.double().clone()
        for e in range(E):
            d = {n: lin[(n, e)].dense(torch).double() for n in ("gate", "up", "down")}
            for j in range(topk):
                rows = np.nonzero(hids[:, j] == e)[0]
                if len(rows) == 0:
                    continue
                r = torch.from_numpy(rows).cuda()
                h = torch.nn.functional.silu(x64[r] @ d["gate"].T) * (x64[r] @ d["up"].T)
                y64[r] += w[r, j].double()[:, None] * (h @ d["down"].T)
        nmse = float(((y.double() - y64) ** 2).mean() / (y64 ** 2).mean())
        assert nmse <= DENSE_NMSE, nmse
    finally:
        for l in lin.values():
            l.free()


# ---- 5: out-of-range ids ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t16", TILES, ids=TILE_IDS)
def test_out_of_range_ids(mk, t16):
    """-1 and n_experts: NaN in exactly those slots (plain) or tokens (GLU); every other slot as the dense tile on the valid
    grouping, and a following call with valid ids is right."""
    K, M, N, topk, E = 1024, 256, 512, 2, 4
    tab = Table([[mk(M, K, 2, zp=True, seed=1100 + 10 * i + e) for e in range(E)] for i in range(2)])
    downs = [mk(M, K, 2, zp=True, seed=1120 + e) for e in range(E)]
    rng = np.random.default_rng(1130)
    B = dev(normal(rng, N, K))
    good = rand_ids(rng, N, topk, E)
    bad = good.copy()
    bad[0, 1], bad[7, 0], bad[100, 1] = E, -1, E
    got = check_plain(tab, N, B, bad, t16)
    for s in (1, 14, 201):
        assert all(np.isnan(got[i][s]).all() for i in range(2))
    G, U = dev(normal(rng, N, topk, K)), dev(normal(rng, N, topk, K))
    w, R = dev(softmax_weights(rng, N, topk)), dev(normal(rng, N, M))
    with knobs(prefill16=int(t16)):
        y = run_glu(downs, N, G, U, torch.from_numpy(bad.astype(np.int32)).cuda(), w, R=R).cpu().numpy()
    want = glu_refs(downs, bad, G, U, w, t16, R)
    assert np.isnan(y[[0, 7, 100]]).all() and np.isnan(want[[0, 7, 100]]).all()
    assert same_glu(y, want)
    check_plain(tab, N, B, good, t16)
    with knobs(prefill16=int(t16)):
        y = run_glu(downs, N, G, U, torch.from_numpy(good.astype(np.int32)).cuda(), w, R=R).cpu().numpy()
    assert same_glu(y, glu_refs(downs, good, G, U, w, t16, R))


# ---- 6: graph replays ------------------------------------------------------------------------------------------------------------
def test_graph_replays(stream, mk):
    """B, ids and weights rewritten on the device before every replay: the outputs equal eager calls on the same inputs, bit for
    bit, and the host never reads the ids."""
    K, F, N, topk, E = 1024, 1024, 192, 2, 4
    gu = Table([[mk(F, K, 2, zp=True, seed=1200 + 10 * i + e) for e in range(E)] for i in range(2)])
    downs = [mk(K, F, 2, zp=True, seed=1220 + e) for e in range(E)]
    x, ids, w = nan_out(N, K), torch.zeros((N, topk), dtype=torch.int32, device="cuda"), nan_out(N, topk)
    G, U, y = nan_out(N, topk, F), nan_out(N, topk, F), nan_out(N, K)
    gen = torch.Generator(device="cuda").manual_seed(1231)

    def calls():
        tb.prefill_experts(gu.tables(), N, x, ids, [G, U])
        tb.prefill_experts_glu([o.wt for o in downs], N, G, U, ids, w, y, R=x)

    def fill():
        x.copy_(torch.randn((N, K), device="cuda", generator=gen))
        ids.copy_(torch.randint(0, E, (N, topk), device="cuda", generator=gen, dtype=torch.int32))
        w.copy_(torch.softmax(torch.randn((N, topk), device="cuda", generator=gen), dim=-1))

    fill(); calls(); torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg, stream=stream):
        calls()
    seen = set()
    for _ in range(3):
        fill()
        cg.replay()
        torch.cuda.synchronize()
        replayed = [t.clone() for t in (G, U, y)]
        seen.add(ids.cpu().numpy().tobytes())
        calls()
        torch.cuda.synchronize()
        for a, b in zip(replayed, (G, U, y)):
            assert same_bits(a.cpu().numpy(), b.cpu().numpy())
    assert len(seen) > 1


# ---- 7: reporting ----------------------------------------------------------------------------------------------------------------
def test_reports_the_tile_the_rule_picks(mk):
    K, M, topk, E = 512, 256, 2, 4
    tab = Table([[mk(M, K, 2, zp=True, seed=1300 + e) for e in range(E)]])
    rng = np.random.default_rng(1301)
    for N, want in ((512, 16), (511, 1)):                 # N * topk >= 256 * n_experts: the fp16 tile
        _, launch = run_plain(tab, N, dev(normal(rng, N, K)), rand_ids(rng, N, topk, E))
        assert launch["cluster"] == want and launch["batch"] == -N * topk, (N, launch)
    with knobs(prefill16=0):
        _, launch = run_plain(tab, 512, dev(normal(rng, 512, K)), rand_ids(rng, 512, topk, E))
    assert launch["cluster"] == 1 and launch["warps_per_cta"] == 12, launch


# ---- 8: the Mixtral shape --------------------------------------------------------------------------------------------------------
def test_mixtral_w2_against_gemv_experts(stream):
    """Mixtral-8x7B's FFN (4096 / 14336, 8 experts, top-2) at N = 512, W2 g128 zp: both calls within the fp16 tile's bound of the
    GEMV forms on the same inputs (the tile the rule picks here is the int8 one, whose bound is tighter)."""
    from decode_harness import QLinear
    H, F, E, topk, N = 4096, 14336, 8, 2, 512
    lin = {(n, e): QLinear(m, k, 2, 128, True, seed=1400 + 3 * e + t) for e in range(E)
           for t, (n, m, k) in enumerate((("gate", F, H), ("up", F, H), ("down", H, F)))}
    try:
        ex = lambda n: [lin[(n, e)].wt for e in range(E)]
        rng = np.random.default_rng(1401)
        hids = np.stack([rng.choice(E, topk, replace=False) for _ in range(N)])
        ids = torch.from_numpy(hids.astype(np.int32)).cuda()
        x, R, w = dev(normal(rng, N, H)), dev(normal(rng, N, H)), dev(softmax_weights(rng, N, topk))
        outs = {k: nan_out(N, topk, F) for k in ("pG", "pU", "gG", "gU")}
        tb.prefill_experts([ex("gate"), ex("up")], N, x, ids, [outs["pG"], outs["pU"]])
        tb.gemv_experts([ex("gate"), ex("up")], N, x, ids, [outs["gG"], outs["gU"]])
        yp, yg = nan_out(N, H), nan_out(N, H)
        tb.prefill_experts_glu(ex("down"), N, outs["gG"], outs["gU"], ids, w, yp, R=R)
        tb.gemv_experts_glu(ex("down"), N, outs["gG"], outs["gU"], ids, w, yg, R=R)
        torch.cuda.synchronize()
        for a, b in ((outs["pG"], outs["gG"]), (outs["pU"], outs["gU"]), (yp - R, yg - R)):
            assert float((a - b).abs().max()) <= (PF16_TOL + TIGHT_TOL) * float(b.abs().max())
    finally:
        for l in lin.values():
            l.free()


# ---- 9: rejections ---------------------------------------------------------------------------------------------------------------
def test_rejections(mk):
    from decode_harness import QLinear
    K, M, N, topk, E = 1024, 512, 64, 2, 2
    tab = Table([[mk(M, K, 2, zp=True, seed=1500 + e) for e in range(E)]])
    other = mk(2 * M, K, 2, zp=True, seed=1510)
    w1 = [QLinear(M, K, 1, 128, False, seed=1520 + e) for e in range(E)]
    ip = [QLinear(M, K, 2, 128, False, seed=1530 + e, one_scale=True) for e in range(E)]
    dw = [o.wt for o in tab.ops[0]]
    try:
        B, ids, w = torch.zeros((N, K), device="cuda"), torch.zeros((N, topk), dtype=torch.int32, device="cuda"), torch.full((N, topk), 0.5, device="cuda")
        G, U, R = torch.zeros((N, topk, K), device="cuda"), torch.zeros((N, topk, K), device="cuda"), torch.zeros((N, M), device="cuda")
        out, y = nan_out(N, topk, M), nan_out(N, M)
        ids9 = torch.zeros((N, 9), dtype=torch.int32, device="cuda")
        ids0 = torch.zeros((N, 0), dtype=torch.int32, device="cuda")
        hB, hids = np.zeros((N, K), np.float32), np.zeros((N, topk), np.int32)
        lib = tb.load()
        H = lambda ws: (tb.C.c_int64 * len(ws))(*[x.handle for x in ws])
        big = (tb.C.c_int64 * (257 * 256))(*([dw[0].handle] * (257 * 256)))
        outs257 = (tb.C.c_void_p * 257)(*([tb.ptr(out)] * 257))
        msgs = {}
        bad = [
            ("w1", lambda: tb.prefill_experts([[l.wt for l in w1]], N, B, ids, [out])),
            ("w1 glu", lambda: tb.prefill_experts_glu([l.wt for l in w1], N, G, U, ids, w, y)),
            ("integer path", lambda: tb.prefill_experts([[l.wt for l in ip]], N, B, ids, [out])),
            ("integer path glu", lambda: tb.prefill_experts_glu([l.wt for l in ip], N, G, U, ids, w, y)),
            ("host B", lambda: tb.prefill_experts(tab.tables(), N, hB, ids, [out])),
            ("host ids", lambda: tb.prefill_experts(tab.tables(), N, B, hids, [out])),
            ("host ids glu", lambda: tb.prefill_experts_glu(dw, N, G, U, hids, w, y)),
            ("host weights", lambda: tb.prefill_experts_glu(dw, N, G, U, ids, w.cpu(), y)),
            ("host G", lambda: tb.prefill_experts_glu(dw, N, G.cpu(), U, ids, w, y)),
            ("host R", lambda: tb.prefill_experts_glu(dw, N, G, U, ids, w, y, R=R.cpu())),
            ("topk 9", lambda: tb.prefill_experts(tab.tables(), N, B, ids9, [out])),
            ("topk 0", lambda: tb.prefill_experts(tab.tables(), N, B, ids0, [out])),
            ("topk 9 glu", lambda: tb.prefill_experts_glu(dw, N, G, U, ids9, w, y)),
            ("n_experts 0", lambda: tb.check(lib.tmac_b200_prefill_experts(H(dw), 1, 0, N, tb.F32, tb.ptr(B), tb.ptr(ids), topk,
                                                                           (tb.C.c_void_p * 1)(tb.ptr(out))), "n_experts 0")),
            ("n_experts 257", lambda: tb.check(lib.tmac_b200_prefill_experts_glu(big, 257, N, tb.F32, tb.ptr(G), tb.ptr(U), tb.ptr(ids),
                                                                                 tb.ptr(w), topk, 0, tb.ptr(y)), "n_experts 257")),
            ("count * n_experts", lambda: tb.check(lib.tmac_b200_prefill_experts(big, 257, 256, N, tb.F32, tb.ptr(B), tb.ptr(ids), topk,
                                                                                 outs257), "count * n_experts")),
            ("geometry", lambda: tb.prefill_experts([[dw[0], other.wt]], N, B, ids, [out])),
            ("geometry glu", lambda: tb.prefill_experts_glu([dw[0], other.wt], N, G, U, ids, w, y)),
        ]
        torch.cuda.synchronize()
        for name, call in bad:
            out.fill_(float("nan")); y.fill_(float("nan"))
            with pytest.raises(tb.TMACError) as err:
                call()
            msgs[name] = str(err.value)
            torch.cuda.synchronize()
            assert torch.isnan(out).all() and torch.isnan(y).all(), "rejected call '%s' launched" % name
        for name in ("w1", "integer path"):
            assert "gemv_experts" in msgs[name], msgs[name]
        assert "gemv_experts_glu" in msgs["w1 glu"], msgs["w1 glu"]
        # an armed peer output makes the call fail, launch nothing and be disarmed
        for call in (lambda: tb.prefill_experts(tab.tables(), N, B, ids, [out]), lambda: tb.prefill_experts_glu(dw, N, G, U, ids, w, y)):
            peer = nan_out(1, M)
            out.fill_(float("nan")); y.fill_(float("nan"))
            tb.peer_outputs([peer.data_ptr()])
            with pytest.raises(tb.TMACError):
                call()
            torch.cuda.synchronize()
            assert torch.isnan(out).all() and torch.isnan(y).all()
            tb.gemv(dw[0], 1, torch.zeros((1, K), device="cuda"), torch.zeros((1, M), device="cuda"))
            torch.cuda.synchronize()
            assert torch.isnan(peer).all(), "the peer output stayed armed"
            call()
    finally:
        for l in w1 + ip:
            l.free()
