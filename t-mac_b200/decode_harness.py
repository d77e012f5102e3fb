"""decode_harness.py -- stand-in for the reference's end-to-end measurement (`llama-bench` through tools/bench_e2e.py:19-29 and
tools/run_pipeline.py:279-331): a Llama-style decoder whose quantised linears (attn q/k/v/o, ffn gate/up/down -- the set the
reference's converter quantises, 3rdparty/llama.cpp/convert_hf_to_gguf.py:353-362,1897-1905) go through the C ABI of
libtmac_b200 and whose other operators (RMSNorm, RoPE, attention over a KV cache, SiLU*mul, residuals) are plain fp16/fp32
torch ops, in the real per-layer order, with synthetic weights at the real shapes.  The token step is captured in one CUDA
graph; `tokens_per_s()` reports the full step, bench.py reports the matmul-only chain next to it.  With `ffn_sequence=True` each
layer's FFN (gate, up, SiLU*mul, down) is one decode sequence launch instead (tools/ffn_bench.py times both); with
`post_attn_sequence=True` everything after attention -- o-projection, residual add, RMSNorm, FFN and the second residual add -- is
one; with `fused_ops=True` the seven linears run as four library launches whose inputs and outputs take the RMSNorms, the
SiLU*mul and the residual adds (tools/layer_bench.py times the four); adding `experts=E` makes the FFN a routed MoE of E experts with
top-k routing, run as two library launches that pick the experts on the device (tools/moe_bench.py times them); `sub_norms=True`
makes the layer BitNet b1.58's, with an RMSNorm before o and one before down (tools/layer_bench.py --bitnet; with `ffn_act="relu2"`
and `kv_heads` < heads, BitNet b1.58 2B4T's, tools/layer_bench.py --bitnet2b); `qkv_bias=True` gives q/k/v a bias, as Qwen2's
(tools/layer_bench.py --qwen2).  `prompt()` is the
prompt step: P tokens through every layer, with causal attention over cache positions [0, P) and the linears on the prefill tiles
(tmac_b200_prefill_*; tools/prompt_bench.py times it).

Not a model implementation: no tokenizer, no sampling, no checkpoint loading (SURVEY 8 f1 scope).  torch is used for device
memory, streams and the non-matmul ops only; every linear is a library launch.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

import tmac_b200 as tb


class QLinear:
    """One quantised linear resident in HBM: y = gemv(W, x) through tmac_b200_gemv (LUT build fused for the fp path)."""

    def __init__(self, mout: int, k: int, bits: int, group_size: int, zero_point: bool, seed: int, one_scale: bool = False, share: Optional["QLinear"] = None,
                 act_group_size: Optional[int] = None):
        """act_group_size: K positions per LUT scale; by default the whole row (the integer path) for one_scale tensors, else 64."""
        self.mout, self.k, self.bits, self.gs, self.zp, self.one_scale = mout, k, bits, group_size, zero_point, one_scale
        if share is not None:                       # another layer with the same synthetic tensor: its own HBM copy, one host encode
            self.w, self.sc, self.z, self.wt = share.w, share.sc, share.z, tb.clone(share.wt)
            return
        rng = np.random.default_rng(seed)
        if one_scale:
            self.w = (rng.integers(-1, 2, size=(mout, k)) + 2).astype(np.uint8)
            self.sc = np.array([0.037], np.float16).astype(np.float32); self.z = None
        else:
            self.w = rng.integers(0, 1 << bits, size=(mout, k), dtype=np.uint8)
            self.sc = (np.abs(rng.standard_normal((mout, k // group_size))) * 0.01 + 1e-4).astype(np.float16).astype(np.float32)
            self.z = (rng.standard_normal((mout, k // group_size)) * 0.01).astype(np.float16).astype(np.float32) if zero_point else None
        bm = next(b for b in ((192, 384, 576, 768) if bits == 3 else (256, 128, 512, 1024, 320, 640)) if (mout * bits) % b == 0)
        if act_group_size is None:
            act_group_size = k if one_scale else 64
        cfg = tb.make_kcfg(mout, k, bits, bm, 16, group_size, act_group_size, zero_point, one_scale)
        self.wt = tb.upload_plain(cfg, self.w, self.sc, self.z)

    def __call__(self, x, out):
        tb.gemv(self.wt, x.shape[0], x, out)      # one row per token: 1 in the token step, P in the prompt step
        return out

    def dense(self, torch):
        """Dense dequantised fp32 weight W_real = (w - 2^(bits-1)) * s - z (tests/test_e2e.py:69-77 of the reference)."""
        w = torch.from_numpy(self.w.astype(np.float32)) - float(1 << (self.bits - 1))
        if self.one_scale:
            return (w * float(self.sc[0])).cuda()
        s = torch.from_numpy(np.repeat(self.sc, self.gs, axis=1))
        d = w * s
        if self.z is not None:
            d = d - torch.from_numpy(np.repeat(self.z, self.gs, axis=1))
        return d.cuda()

    def free(self):
        self.wt.free()


class DecodeLayer:
    def __init__(self, hidden: int, ffn: int, heads: int, bits: int, zero_point: bool, seed: int, share: Optional["DecodeLayer"] = None, group_size: int = 128,
                 ffn_sequence: bool = False, post_attn_sequence: bool = False, fused_ops: bool = False, experts: int = 0, topk: int = 2,
                 sub_norms: bool = False, ffn_act: str = "silu", kv_heads: Optional[int] = None, qkv_bias: bool = False):
        """ffn_sequence: the FFN (gate, up, SiLU*mul, down) runs as ONE decode sequence whose down op reads the gated activation of
        the gate and up ops (tmac_b200_seq_add_gemv_glu) instead of three launches and a torch op.
        post_attn_sequence: the layer after attention runs as ONE decode sequence [o(att) + x, gate(rmsnorm(h) * w2),
        up(rmsnorm(h) * w2), down(silu(gate) * up) + h] (tmac_b200_seq_residual, tmac_b200_seq_add_gemv_rmsnorm); the layer keeps
        its input x in a buffer of its own, because the sequence's external vectors are fixed when it is built.
        fused_ops: the linears run as four launches and no torch op around them: gemv_rmsnorm([q, k, v], x, norm1),
        gemv_residual(o, att, x) -> h, gemv_rmsnorm([gate, up], h, norm2), gemv_glu(down, gate, up, h).
        experts > 0 (with fused_ops): the FFN is a MoE with Mixtral's structure -- `experts` gate/up/down triples, a dense fp32 router
        Wr [experts][hidden] on h2 = rmsnorm(h) * norm2, the top `topk` logits and a softmax over them -- run as
        gemv_experts([gate, up], h2, ids) and gemv_experts_glu(down, gate, up, ids, weights, h), with no host sync.
        sub_norms: a BitNet b1.58 layer -- ternary one-scale tensors (bits = 2) with activation groups of 64, and two more RMSNorms,
        o(rmsnorm(att) * w_as) and down(rmsnorm(silu(gate) * up) * w_fs) (HF attn inner_attn_ln and mlp ffn_layernorm).  With
        fused_ops the linears still run as four launches: gemv_rmsnorm([q, k, v], x, norm1), gemv_subnorm(o, att, w_as, R=x) -> h,
        gemv_rmsnorm([gate, up], h, norm2), gemv_subnorm(down, gate, w_fs, U=up, R=h).
        ffn_act: the FFN gate's activation, "silu" (silu(gate) * up) or, with sub_norms only, "relu2" (relu(gate)^2 * up, BitNet b1.58
        2B4T's), whose fused down projection is gemv_subnorm_relu2 / prefill_subnorm_relu2.
        kv_heads (default heads): kv_heads < heads is grouped-query attention -- each KV head serves heads / kv_heads consecutive
        query heads and the KV cache holds kv_heads heads.  q, k and v are then one stacked tensor "qkv" of hidden + 2 * kv_heads * hd
        rows (one launch, whose output q / k / v are views of), the usual way to group GQA projections.
        qkv_bias: q, k and v (or the stacked qkv) carry a seeded fp32 bias, as Qwen2's (HF Qwen2Attention, bias=True on q_proj,
        k_proj and v_proj only).  fused_ops layers run gemv_rmsnorm_bias / prefill_rmsnorm_bias for them; the other layers and the
        dense reference (`linear`) add the bias with torch after each projection.
        The prompt step (`prompt`) runs the fused_ops launches in their prefill forms (prefill_rmsnorm, prefill_residual,
        prefill_glu, prefill_subnorm, prefill_experts, prefill_experts_glu); the sequences are decode-only, so sequence layers run
        per-linear calls."""
        import torch
        if ffn_sequence and post_attn_sequence:
            raise ValueError("ffn_sequence and post_attn_sequence are alternatives: the second one contains the FFN")
        if fused_ops and (ffn_sequence or post_attn_sequence):
            raise ValueError("fused_ops runs the layer's linears as single launches; it cannot be combined with a sequence")
        if experts and (not fused_ops or ffn_sequence or post_attn_sequence):
            raise ValueError("experts > 0 runs the routed FFN with the fused_ops launches; it needs fused_ops and no sequence")
        if experts and not 1 <= topk <= min(experts, 8):
            raise ValueError("topk must lie in [1, min(experts, 8)]")
        if sub_norms and (ffn_sequence or post_attn_sequence or experts):
            raise ValueError("sub_norms has no sequence op and no routed FFN: it cannot be combined with a sequence or experts")
        if sub_norms and bits != 2:
            raise ValueError("sub_norms layers have ternary weights: bits must be 2")
        if ffn_act not in ("silu", "relu2"):
            raise ValueError("ffn_act must be 'silu' or 'relu2'")
        if ffn_act == "relu2" and not sub_norms:
            raise ValueError("ffn_act='relu2' is BitNet b1.58 2B4T's FFN: it needs sub_norms")
        kv_heads = heads if kv_heads is None else kv_heads
        if not 1 <= kv_heads <= heads or heads % kv_heads:
            raise ValueError("kv_heads must divide heads")
        self.fused_ops, self.experts, self.topk, self.sub_norms, self.ffn_act_name = fused_ops, experts, topk, sub_norms, ffn_act
        self.torch, self.hidden, self.ffn, self.heads, self.hd = torch, hidden, ffn, heads, hidden // heads
        self.kv_heads, kvd = kv_heads, kv_heads * (hidden // heads)
        self.qkv_names = ("q", "k", "v") if kv_heads == heads else ("qkv",)
        names = [("q", hidden, hidden), ("k", hidden, hidden), ("v", hidden, hidden)] if kv_heads == heads else [("qkv", hidden + 2 * kvd, hidden)]
        names += [("o", hidden, hidden)]
        ffn_names = [("gate", ffn, hidden), ("up", ffn, hidden), ("down", hidden, ffn)]
        names += ffn_names if not experts else [("%s.%d" % (n, e), m, k) for e in range(experts) for n, m, k in ffn_names]
        qkw = dict(zero_point=False, one_scale=True, act_group_size=64) if sub_norms else dict(zero_point=zero_point)
        self.lin = {n: QLinear(m, k, bits, group_size, seed=seed + i, share=share.lin[n] if share else None, **qkw)
                    for i, (n, m, k) in enumerate(names)}
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.norm1 = (1.0 + 0.1 * torch.randn(hidden, generator=g)).cuda()
        self.norm2 = (1.0 + 0.1 * torch.randn(hidden, generator=g)).cuda()
        f = lambda n: torch.zeros((1, n), device="cuda")
        self.buf = {"h1": f(hidden), "q": f(hidden), "k": f(hidden), "v": f(hidden), "att": f(hidden), "o": f(hidden), "h2": f(hidden),
                    "gate": f(ffn), "up": f(ffn), "act": f(ffn), "down": f(hidden), "x": f(hidden), "out": f(hidden), "h": f(hidden)}
        self.qkv_views(self.buf, 1)
        if experts:
            self.router = (0.05 * torch.randn((experts, hidden), generator=g)).cuda()
            self.buf.update(gate=torch.zeros((1, topk, ffn), device="cuda"), up=torch.zeros((1, topk, ffn), device="cuda"),
                            ids=torch.zeros((1, topk), dtype=torch.int32, device="cuda"), wts=torch.zeros((1, topk), device="cuda"))
        if sub_norms:
            self.w_as = (1.0 + 0.1 * torch.randn(hidden, generator=g)).cuda()
            self.w_fs = (1.0 + 0.1 * torch.randn(ffn, generator=g)).cuda()
            self.buf["att_n"] = f(hidden)
        # drawn last, so that every other tensor of the layer is the one it has without biases
        self.qkv_b = {n: (0.5 * torch.randn(self.lin[n].mout, generator=g)).cuda() for n in self.qkv_names} if qkv_bias else None
        self.pbuf = {}                              # the prompt step's buffers, [P][...], made by its first call
        self.ffn_seq = self.post_seq = None
        if ffn_sequence:
            seq = tb.Sequence()
            try:
                seq.add(self.lin["gate"].wt, x=self.buf["h2"])
                seq.add(self.lin["up"].wt, x=self.buf["h2"])
                seq.add_glu(self.lin["down"].wt, 0, 0, 1, 0, out=self.buf["down"])
                self.ffn_seq = seq.build()
            except Exception:
                seq.free()
                self.free()
                raise
        if post_attn_sequence:
            seq = tb.Sequence()
            try:
                seq.add(self.lin["o"].wt, x=self.buf["att"])                       # 0: h = o(att) + x
                seq.residual(0, r=self.buf["x"])
                seq.add_rmsnorm(self.lin["gate"].wt, 0, self.norm2, self.EPS)      # 1, 2: gate / up of rmsnorm(h) * w2
                seq.add_rmsnorm(self.lin["up"].wt, 0, self.norm2, self.EPS)
                seq.add_glu(self.lin["down"].wt, 1, 0, 2, 0, out=self.buf["out"])  # 3: down(silu(gate) * up) + h
                seq.residual(3, r_op=0)
                self.post_seq = seq.build()
            except Exception:
                seq.free()
                self.free()
                raise

    EPS = 1e-5

    def qkv_views(self, b, n):
        """A GQA layer's buffers of n rows: the stacked output qkv [n][hidden + 2 * kv_dim], and q, k and v as views of it."""
        if self.qkv_names == ("qkv",):
            H, kvd = self.hidden, self.kv_heads * self.hd
            qkv = self.torch.zeros((n, H + 2 * kvd), device="cuda")
            b.update(qkv=qkv, q=qkv[:, :H], k=qkv[:, H:H + kvd], v=qkv[:, H + kvd:])

    def kv(self, c):
        """The cache positions c [kv_heads, L, hd] repeated over each KV head's query group: [heads, L, hd]."""
        return c if self.kv_heads == self.heads else c.repeat_interleave(self.heads // self.kv_heads, dim=0)

    @staticmethod
    def rmsnorm(torch, x, w, eps=EPS):
        return x * torch.rsqrt((x * x).mean(dim=-1, keepdim=True) + eps) * w

    def rope(self, x, pos_cos, pos_sin):
        """x [n, heads * hd] (q) or [n, kv_heads * hd] (k), pos_cos / pos_sin [n, hd / 2]: row i rotated by the angles of its position."""
        t = x.view(x.shape[0], -1, self.hd // 2, 2)
        a, b = t[..., 0], t[..., 1]
        c, s = pos_cos[:, None, :], pos_sin[:, None, :]
        return self.torch.stack((a * c - b * s, a * s + b * c), dim=-1).reshape(x.shape[0], -1)

    def route(self, h2, b=None):
        """The MoE router on h2 [n, hidden]: the ids (int32) and softmax weights of the top `topk` logits, in the buffers b."""
        b = self.buf if b is None else b
        vals, idx = self.torch.topk(h2 @ self.router.T, self.topk, dim=-1)
        b["ids"].copy_(idx.to(self.torch.int32))
        b["wts"].copy_(self.torch.softmax(vals, dim=-1))

    def forward(self, x, kcache, vcache, pos: int, pos_cos, pos_sin, linear=None, routed=None):
        """x [1, hidden] fp32 -> [1, hidden].  kcache / vcache [kv_heads, ctx, hd]; `linear(name, inp, out)` overrides the library call
        (the dense fp32 reference layer in the tests).  MoE layers: `routed` = (ids, weights) replaces the router's choice, so that a
        reference can follow the choice of the library path; with `linear` every expert runs densely and the chosen ones are combined."""
        torch, b = self.torch, self.buf
        lin = linear or (lambda n, inp, out: self.lin[n](inp, out))
        fused = self.fused_ops and linear is None
        self.qkv(x, b, 1, fused, lin)
        q = self.rope(b["q"], pos_cos, pos_sin).view(self.heads, 1, self.hd)
        kcache[:, pos] = self.rope(b["k"], pos_cos, pos_sin).view(self.kv_heads, self.hd)
        vcache[:, pos] = b["v"].view(self.kv_heads, self.hd)
        att = torch.softmax((q @ self.kv(kcache[:, :pos + 1]).transpose(1, 2)) / math.sqrt(self.hd), dim=-1) @ self.kv(vcache[:, :pos + 1])
        b["att"].copy_(att.reshape(1, -1))
        if self.post_seq is not None and linear is None:
            b["x"].copy_(x)
            self.post_seq.launch()                  # o(att) + x, rmsnorm, gate, up, down(silu(gate) * up) + h -> b["out"]
            return b["out"]
        if self.experts:
            return self.moe(x, linear, routed, b, 1)
        if fused:
            return self.post_attn(x, b, 1)
        lin("o", self.attn_sub_norm(b), b["o"])
        h = x + b["o"]
        b["h2"].copy_(self.rmsnorm(torch, h, self.norm2))
        if self.ffn_seq is not None and linear is None:
            self.ffn_seq.launch()                   # gate(h2), up(h2), down(silu(gate) * up) -> b["down"]
        else:
            lin("gate", b["h2"], b["gate"]); lin("up", b["h2"], b["up"])
            self.ffn_act(b)
            lin("down", b["act"], b["down"])
        return h + b["down"]

    def qkv(self, x, b, n, fused, lin):
        """The q/k/v projections of rmsnorm(x) * norm1 into the buffers b (n rows: the token step's GEMV forms at n = 1, else the
        prompt step's prefill forms), plus their biases in a qkv_bias layer."""
        wts, outs = [self.lin[m].wt for m in self.qkv_names], [b[m] for m in self.qkv_names]
        decode = b is self.buf
        if fused and self.qkv_b is not None:
            bias = [self.qkv_b[m] for m in self.qkv_names]
            (tb.gemv_rmsnorm_bias if decode else tb.prefill_rmsnorm_bias)(wts, n, x, self.norm1, self.EPS, bias, outs)
        elif fused:
            (tb.gemv_rmsnorm if decode else tb.prefill_rmsnorm)(wts, n, x, self.norm1, self.EPS, outs)
        else:
            b["h1"].copy_(self.rmsnorm(self.torch, x, self.norm1))
            for m in self.qkv_names:
                lin(m, b["h1"], b[m])
                if self.qkv_b is not None:
                    b[m].add_(self.qkv_b[m])

    def post_attn(self, x, b, n):
        """The layer after attention of a fused_ops layer over the n rows of the buffers b (n = 1: the token step's GEMV forms, else
        the prompt step's prefill forms), three launches into b["out"]: h = o(att) + x (sub_norms: o(rmsnorm(att) * w_as) + x), gate
        and up of rmsnorm(h) * norm2, out = down(silu(gate) * up) + h (sub_norms: down(rmsnorm(act(gate, up)) * w_fs) + h)."""
        decode, (o, gate, up, down) = b is self.buf, (self.lin[m].wt for m in ("o", "gate", "up", "down"))
        subnorm = tb.gemv_subnorm if decode else tb.prefill_subnorm
        if self.sub_norms:
            subnorm(o, n, b["att"], self.w_as, self.EPS, b["h"], R=x)
        else:
            (tb.gemv_residual if decode else tb.prefill_residual)(o, n, b["att"], x, b["h"])
        (tb.gemv_rmsnorm if decode else tb.prefill_rmsnorm)([gate, up], n, b["h"], self.norm2, self.EPS, [b["gate"], b["up"]])
        if not self.sub_norms:
            (tb.gemv_glu if decode else tb.prefill_glu)(down, n, b["gate"], b["up"], b["out"], R=b["h"])
        else:
            if self.ffn_act_name == "relu2":
                subnorm = tb.gemv_subnorm_relu2 if decode else tb.prefill_subnorm_relu2
            subnorm(down, n, b["gate"], self.w_fs, self.EPS, b["out"], U=b["up"], R=b["h"])
        return b["out"]

    def attn_sub_norm(self, b):
        """The o projection's input from the buffers b: att, or rmsnorm(att) * w_as in a sub_norms layer (torch ops)."""
        if not self.sub_norms:
            return b["att"]
        b["att_n"].copy_(self.rmsnorm(self.torch, b["att"], self.w_as))
        return b["att_n"]

    def ffn_act(self, b):
        """b["act"] = silu(gate) * up (relu2 layers: relu(gate)^2 * up), then rmsnorm(.) * w_fs in a sub_norms layer (torch ops)."""
        if self.ffn_act_name == "relu2":
            act = self.torch.square(self.torch.relu(b["gate"])) * b["up"]
        else:
            act = self.torch.nn.functional.silu(b["gate"]) * b["up"]
        b["act"].copy_(self.rmsnorm(self.torch, act, self.w_fs) if self.sub_norms else act)

    def moe(self, x, linear, routed, b, n):
        """The layer after attention with the routed FFN over the n rows of the buffers b (n = 1: the token step's GEMV forms, else
        the prompt step's prefill forms): h = o(att) + x, h2 = rmsnorm(h) * norm2, out = h + sum_j w_j expert_j(h2)."""
        torch, E = self.torch, self.experts
        if linear is None:
            (tb.gemv_residual if b is self.buf else tb.prefill_residual)(self.lin["o"].wt, n, b["att"], x, b["h"])
        else:
            linear("o", b["att"], b["o"])
            b["h"].copy_(x + b["o"])
        b["h2"].copy_(self.rmsnorm(torch, b["h"], self.norm2))
        if routed is None:
            self.route(b["h2"], b)
        else:
            b["ids"].copy_(routed[0]); b["wts"].copy_(routed[1])
        if linear is None:
            ex = lambda name: [self.lin["%s.%d" % (name, e)].wt for e in range(E)]
            decode = b is self.buf
            (tb.gemv_experts if decode else tb.prefill_experts)([ex("gate"), ex("up")], n, b["h2"], b["ids"], [b["gate"], b["up"]])
            (tb.gemv_experts_glu if decode else tb.prefill_experts_glu)(ex("down"), n, b["gate"], b["up"], b["ids"], b["wts"], b["out"], R=b["h"])
            return b["out"]
        ys = torch.zeros((E, n, self.hidden), device="cuda")                # every expert, then the chosen ones: no host sync
        g, u = torch.zeros((n, self.ffn), device="cuda"), torch.zeros((n, self.ffn), device="cuda")
        for e in range(E):
            linear("gate.%d" % e, b["h2"], g); linear("up.%d" % e, b["h2"], u)
            linear("down.%d" % e, torch.nn.functional.silu(g) * u, ys[e])
        sel = ys[b["ids"].long(), torch.arange(n, device="cuda")[:, None]]  # [n][topk][hidden]
        y = (b["wts"][:, :, None] * sel).sum(dim=1)
        return b["h"] + y

    def prompt_buffers(self, P: int) -> dict:
        """The prompt step's buffers for P tokens, kept for later calls (and CUDA graphs) at the same P."""
        if self.pbuf.get("P") != P:
            torch = self.torch
            f = lambda *s: torch.zeros(s, device="cuda")
            H, F = self.hidden, self.ffn
            self.pbuf = {"P": P, "h1": f(P, H), "q": f(P, H), "k": f(P, H), "v": f(P, H), "att": f(P, H), "o": f(P, H), "h2": f(P, H),
                         "gate": f(P, F), "up": f(P, F), "act": f(P, F), "down": f(P, H), "out": f(P, H), "h": f(P, H), "att_n": f(P, H)}
            self.qkv_views(self.pbuf, P)
            if self.experts:
                self.pbuf.update(gate=f(P, self.topk, F), up=f(P, self.topk, F), wts=f(P, self.topk),
                                 ids=torch.zeros((P, self.topk), dtype=torch.int32, device="cuda"))
        return self.pbuf

    def prompt(self, x, kcache, vcache, cos, sin, linear=None, routed=None):
        """The prompt step: x [P, hidden] fp32 -> [P, hidden] (a buffer of the layer).  Writes cache positions [0, P) and runs causal
        attention over them; cos / sin [P, hd / 2] are the positions' RoPE angles.  fused_ops layers run their linears as
        prefill_rmsnorm([q, k, v]), prefill_residual(o), prefill_rmsnorm([gate, up]) and prefill_glu(down, R=h); MoE layers as
        prefill_rmsnorm([q, k, v]), prefill_residual(o), the torch router over the P tokens, prefill_experts([gate, up]) and
        prefill_experts_glu(down, R=h); sub_norms + fused_ops layers as prefill_rmsnorm([q, k, v]), prefill_subnorm(o, att, w_as,
        R=x), prefill_rmsnorm([gate, up]) and prefill_subnorm(down, gate, w_fs, U=up, R=h) (relu2 layers: prefill_subnorm_relu2);
        GQA layers run [qkv] in place of [q, k, v], qkv_bias layers prefill_rmsnorm_bias in place of prefill_rmsnorm for them; the
        other layers as one call per linear.
        `linear` and `routed` as for forward."""
        torch, P = self.torch, x.shape[0]
        b = self.prompt_buffers(P)
        lin = linear or (lambda n, inp, out: self.lin[n](inp, out))
        fused = self.fused_ops and linear is None
        self.qkv(x, b, P, fused, lin)
        q = self.rope(b["q"], cos, sin).view(P, self.heads, self.hd).transpose(0, 1)
        kcache[:, :P] = self.rope(b["k"], cos, sin).view(P, self.kv_heads, self.hd).transpose(0, 1)
        vcache[:, :P] = b["v"].view(P, self.kv_heads, self.hd).transpose(0, 1)
        s = (q @ self.kv(kcache[:, :P]).transpose(1, 2)) / math.sqrt(self.hd)
        s = s.masked_fill(torch.ones((P, P), dtype=torch.bool, device="cuda").triu(1), float("-inf"))
        att = torch.softmax(s, dim=-1) @ self.kv(vcache[:, :P])             # [heads][P][hd]
        b["att"].copy_(att.transpose(0, 1).reshape(P, -1))
        if self.experts:
            return self.moe(x, linear, routed, b, P)
        if fused:
            return self.post_attn(x, b, P)
        lin("o", self.attn_sub_norm(b), b["o"])
        b["h"].copy_(x + b["o"])
        b["h2"].copy_(self.rmsnorm(torch, b["h"], self.norm2))
        lin("gate", b["h2"], b["gate"]); lin("up", b["h2"], b["up"])
        self.ffn_act(b)
        lin("down", b["act"], b["down"])
        b["out"].copy_(b["h"] + b["down"])
        return b["out"]

    def free(self):
        for s in (self.ffn_seq, self.post_seq):
            if s is not None:
                s.free()
        self.ffn_seq = self.post_seq = None
        for l in self.lin.values():
            l.free()


class DecodeModel:
    """`layers` decoder layers of one shape (synthetic; layers > 0 share one host tensor set but own their HBM copies, so every
    weight byte of a token streams from HBM), a KV cache of `ctx` positions, one token step per call.  prompt_len = P > 0: also a
    prompt step of P tokens (`prompt()`) that fills cache positions [0, P)."""

    def __init__(self, layers: int, hidden: int, ffn: int, heads: int, bits: int, zero_point: bool, ctx: int = 512, seed: int = 0,
                 ffn_sequence: bool = False, post_attn_sequence: bool = False, fused_ops: bool = False, experts: int = 0, topk: int = 2,
                 prompt_len: int = 0, sub_norms: bool = False, ffn_act: str = "silu", kv_heads: Optional[int] = None,
                 qkv_bias: bool = False):
        import torch
        self.torch, self.hidden, self.ctx, self.heads, self.hd = torch, hidden, ctx, heads, hidden // heads
        kw = dict(ffn_sequence=ffn_sequence, post_attn_sequence=post_attn_sequence, fused_ops=fused_ops, experts=experts, topk=topk,
                  sub_norms=sub_norms, ffn_act=ffn_act, kv_heads=kv_heads, qkv_bias=qkv_bias)
        first = DecodeLayer(hidden, ffn, heads, bits, zero_point, seed, **kw)
        self.layers: List[DecodeLayer] = [first] + [DecodeLayer(hidden, ffn, heads, bits, zero_point, seed, share=first, **kw)
                                                    for _ in range(layers - 1)]
        kvh = first.kv_heads
        self.kc = [torch.randn((kvh, ctx, self.hd), device="cuda") * 0.1 for _ in range(layers)]
        self.vc = [torch.randn((kvh, ctx, self.hd), device="cuda") * 0.1 for _ in range(layers)]
        inv = 1.0 / (10000.0 ** (torch.arange(0, self.hd, 2, device="cuda").float() / self.hd))
        self.pos = ctx - 1                          # decode at the last cache position: attention over the whole context
        ang = self.pos * inv
        self.cos, self.sin = torch.cos(ang)[None, :], torch.sin(ang)[None, :]
        self.x = torch.randn((1, hidden), device="cuda")
        self.y = torch.zeros((1, hidden), device="cuda")
        self.graph = self.prompt_graph = None
        if not 0 <= prompt_len <= ctx:
            raise ValueError("prompt_len must lie in [0, ctx]")
        self.P = prompt_len
        if prompt_len:
            ang = torch.arange(prompt_len, device="cuda").float()[:, None] * inv[None, :]
            self.pcos, self.psin = torch.cos(ang), torch.sin(ang)
            self.px = torch.randn((prompt_len, hidden), device="cuda")
            self.py = torch.zeros((prompt_len, hidden), device="cuda")

    def step(self):
        h = self.x
        for i, layer in enumerate(self.layers):
            h = layer.forward(h, self.kc[i], self.vc[i], self.pos, self.cos, self.sin)
        self.y.copy_(h)

    def prompt(self):
        """The prompt step: the P rows px through every layer into py, cache positions [0, P) written."""
        h = self.px
        for i, layer in enumerate(self.layers):
            h = layer.prompt(h, self.kc[i], self.vc[i], self.pcos, self.psin)
        self.py.copy_(h)

    def _graph(self, fn, stream):
        torch = self.torch
        with torch.cuda.stream(stream):
            fn()                                    # eager warm-up: library workspaces, torch allocator
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            fn()
        return graph

    def capture(self, stream):
        self.graph = self._graph(self.step, stream)
        return self

    def capture_prompt(self, stream):
        self.prompt_graph = self._graph(self.prompt, stream)
        return self

    def _per_s(self, run, stream, n):
        torch = self.torch
        with torch.cuda.stream(stream):
            for _ in range(2):
                run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(n):
                run()
            e1.record(stream)
        torch.cuda.synchronize()
        return n / (e0.elapsed_time(e1) * 1e-3)

    def tokens_per_s(self, stream, n: int = 10) -> float:
        return self._per_s(self.graph.replay if self.graph is not None else self.step, stream, n)

    def prompt_tokens_per_s(self, stream, n: int = 10) -> float:
        """Prompt tokens per second: P over the time of one prompt step (graphed when capture_prompt was called)."""
        return self.P * self._per_s(self.prompt_graph.replay if self.prompt_graph is not None else self.prompt, stream, n)

    def free(self):
        self.graph = self.prompt_graph = None
        for l in self.layers:
            l.free()
