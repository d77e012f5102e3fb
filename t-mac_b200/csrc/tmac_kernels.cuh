// tmac_kernels.cuh -- hand-written sm_90a kernels of the T-MAC hot path.
//
//   preprocessor_kernel : activation row -> per-act-group LUT scale, LUT bias, int8 LUT
//                         (python/t_mac/intrins/lut_ctor.cc:38-260; loop nest
//                          deploy/tuned/kernels.cc:1002-1040).  Bit-exact with the x86 reference.
//   gemv3_kernel        : table-lookup GEMV over the stream layout (tmac_layout.h)
//                         (python/t_mac/intrins/tbl.cc:323-630 + generated recombine
//                          deploy/tuned/aarch64-llama-2-7b-2bit/kernels.cc:1059-1075).
//
// Lookup primitive.  The reference does 16 (NEON) / 32 (AVX2) byte lookups per `tbl`/`pshufb`
// in a 16-entry int8 table.  On the GPU the register-file analogue is PRMT: 4 byte lookups in an
// 8-byte table held in two registers.  The LUT is odd-symmetric (LUT[15-i] = -LUT[i],
// lut_ctor.cc:153-155), so 8 entries + a sign bit are enough; the sign is applied by DP4A, whose
// second operand (+-plane weights 2*alpha_b = 1,2,4,8) is itself fetched with one PRMT from an
// 8-byte constant table indexed by the sign bits.  One DP4A therefore does "negate, scale by
// the bit-plane weight, add the 4 lookups" = the int16 adder tree + alpha recombination of the
// reference, exactly, in int32.
//
// Shared by every kernel of the project (all headers include this one):
//   the activation LUT   : lut_abs_sum, lut_scale, lut_ts, lut_odd_entries, lut_q8, lut_stored, lut_addv8, lut_group, lut_bias,
//                          lut_slice (one chunk's slice in a warp); swiglu (the gated input of a sequence op); rms_sumsq,
//                          rms_warp_sum, rms_inv, rms_scale (its RMS-norm input);
//   the block step       : TMAC_QUAD_LOOKUP, TMAC_GROUP_FOLD (gemv3_kernel, chain_kernel, seq_kernel), TMAC_BLOCK_LOOKUPS
//                          (written with those two), TMAC_BLOCK_SCALES (gemv3_kernel and chain_kernel); the quad step split in
//                          its weight part (QuadWord, quad_decode -> QuadCodes) and table part (Quad<PB, SYM>::lookup,
//                          TMAC_QUAD_TABLE), which chain_kernel runs apart (TMAC_BLOCK_LOOKUPS_AHEAD);
//   PTX wrappers         : smem_u32, mbar_init, mbar_fence_init, fence_proxy_async, mbar_arrive, expect_tx, bulk_load,
//                          bulk_load_hint, mbar_wait_parity, mbar_wait_bounded<LIMIT>, cluster_arrive_relaxed / cluster_wait, globaltimer_ns;
//   the output store     : store_out (fp16 or fp32).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "tmac_layout.h"

namespace tmac_b200 {

// (a & b) | c in ONE LOP3 (the compiler splits it in two when b and c are immediates)
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(s));
    return r;
}
// x >> 16 on the FMA pipe (IMAD.HI) instead of the ALU pipe (SHF): the PRMT/LOP3 work of the lookup
// loop saturates the ALU pipe, the FMA pipe only carries the DP4As.
#ifdef TMAC_HI16_SHF
__device__ __forceinline__ uint32_t hi16(uint32_t x) { return x >> 16; }
#else
__device__ __forceinline__ uint32_t hi16(uint32_t x) { return __umulhi(x, 65536u); }
#endif
__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// ------------------------------------------------------------------------------------------
// The quad step: 4 K-groups x the lane's RW rows.  acc[r] += sum_{k<4} sum_b 2*alpha_b * sgn * T_k[j]
// In two parts.  The weight part reads only the lane's code word (a uint4, words w0..w3).  For each word, with h = 0 for its
// low half and h = 1 for hi16 of it, it gives two table selectors t = w & 0x77777777 (the PRMT selectors into the quad's
// table entries) and two sign words, from sel = sign_sel(w) -- SYM: the signed plane-weight word prmt(2w, 2w, sel) that dp4a_sw
// multiplies by; !SYM: the selector itself, which picks between two looked-up candidates.  The table part,
// Quad<PB, SYM>::lookup, takes those and the quad's table entries and does the table PRMTs, the transposes and the DP4As.
// It reads the weight part through a C, one of two classes with the same interface (i = 2 * word + h):
//   t(i)               the table selector;
//   sel(i)             the word's sign selectors (i even);
//   sw(half(sel, h))   the sign word of half h.
// QuadWord<SYM> computes these where lookup uses them, so TMAC_QUAD_LOOKUP is the step as one piece.  QuadCodes holds them in
// registers, computed by quad_decode, so that a kernel can decode a quad while it waits for its activations: about half of the
// step's ALU-pipe instructions read only the code word.
// ------------------------------------------------------------------------------------------
template <int PB, bool SYM> struct Quad;

// Sign handling of the symmetric (8 stored entries) path without a shift: the selector nibble of the sign PRMT is
// neg << 3 | byte position, i.e. the weight word ANDed in place.  PRMT's replicate mode (selector bit 3) turns the
// selected byte 2*w (msb clear) into 0x00, so prmt(2w, sel) = 2*w*(1 - neg); with the constant vector -w,
//   dp4a(v, 2w(1-neg)) + dp4a(v, -w) = sum v*w*(1 - 2*neg)
// exactly.  One LOP3 per word instead of SHF + LOP3 on the saturated ALU pipe; the extra DP4A rides the FMA pipe.
// The general (16 stored entries) path keeps neg << 2 | position: it selects between two looked-up candidates.
template <bool SYM> __device__ __forceinline__ uint32_t sign_sel(uint32_t w) {
    return SYM ? and_or(w, 0x88888888u, 0x32103210u) : and_or(w >> 1, 0x44444444u, 0x32103210u);
}
// sum v * w * (1 - 2*neg) with sw = prmt(2w, 2w, sel) and the constant vector wneg = -w
__device__ __forceinline__ int dp4a_sw(uint32_t v, uint32_t sw, uint32_t wneg, int acc) {
    return __dp4a((int)v, (int)sw, __dp4a((int)v, (int)wneg, acc));
}

// The weight part computed where it is used.
template <bool SYM> struct QuadWord {
    uint4 q;
    uint32_t wtx;
    __device__ __forceinline__ QuadWord(const uint4 q_, uint32_t wtx_) : q(q_), wtx(wtx_) {}
    __device__ __forceinline__ uint32_t word(int i) const { return (i >> 1) == 0 ? q.x : (i >> 1) == 1 ? q.y : (i >> 1) == 2 ? q.z : q.w; }
    __device__ __forceinline__ uint32_t t(int i) const {
        const uint32_t j = word(i) & 0x77777777u;
        return (i & 1) ? hi16(j) : j;
    }
    __device__ __forceinline__ uint32_t sel(int i) const { return sign_sel<SYM>(word(i)); }
    __device__ __forceinline__ uint32_t half(uint32_t sl, int h) const { return h ? hi16(sl) : sl; }
    __device__ __forceinline__ uint32_t sw(uint32_t sl) const { return SYM ? prmt(wtx << 1, wtx << 1, sl) : sl; }
};
// The weight part in registers: tv[i] = t(i), sv[i] = the sign word of lookup i.
struct QuadCodes {
    uint32_t tv[8], sv[8];
    __device__ __forceinline__ uint32_t t(int i) const { return tv[i]; }
    __device__ __forceinline__ uint2 sel(int i) const { return make_uint2(sv[i], sv[i + 1]); }
    __device__ __forceinline__ uint32_t half(uint2 sl, int h) const { return h ? sl.y : sl.x; }
    __device__ __forceinline__ uint32_t sw(uint32_t s) const { return s; }
};
template <bool SYM> __device__ __forceinline__ QuadCodes quad_decode(const uint4 w, uint32_t wtx) {
    const QuadWord<SYM> q(w, wtx);
    QuadCodes c;
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
        const uint32_t sl = q.sel(i);
        c.tv[i] = q.t(i); c.tv[i + 1] = q.t(i + 1);
        c.sv[i] = q.sw(q.half(sl, 0)); c.sv[i + 1] = q.sw(q.half(sl, 1));
    }
    return c;
}

// sign/plane-weight tables (bytes): index = plane-position | neg << 2
//   PB 4: {1,2,4,8 | -1,-2,-4,-8}   (bits 3: plane 3 weight 0)
//   PB 2: {1,2,1,2 | -1,-2,-1,-2}
//   PB 1: {1,1,1,1 | -1,-1,-1,-1}
// With a QuadWord, the order in which lookup reads the weight part is the order in which its instructions reach the compiler,
// and the kernels' register allocation depends on it: per word pair (or word) the selectors first, then the sign selectors, then
// each lookup with its halves.  In this order every kernel compiles to the instructions it had with the step as one function.
template <bool SYM> struct Quad<4, SYM> {
    template <class C>
    static __device__ __forceinline__ void lookup(const C &c, const uint32_t *tab /* 4 tables */, int *acc, uint32_t wtx, uint32_t wty) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t wj = c.t(2 * k);
            const auto ws = c.sel(2 * k);
            uint32_t v0, v1;
            if (SYM) {
                v0 = prmt(tab[2 * k], tab[2 * k + 1], wj);
                v1 = prmt(tab[2 * k], tab[2 * k + 1], c.t(2 * k + 1));
                acc[0] = dp4a_sw(v0, c.sw(c.half(ws, 0)), wty, acc[0]);
                acc[1] = dp4a_sw(v1, c.sw(c.half(ws, 1)), wty, acc[1]);
            } else {
                const uint32_t *g = tab + 4 * k;
                v0 = prmt(prmt(g[0], g[1], wj), prmt(g[2], g[3], wj), c.sw(c.half(ws, 0)));
                v1 = prmt(prmt(g[0], g[1], c.t(2 * k + 1)), prmt(g[2], g[3], c.t(2 * k + 1)), c.sw(c.half(ws, 1)));
                acc[0] = __dp4a((int)v0, (int)wtx, acc[0]);
                acc[1] = __dp4a((int)v1, (int)wtx, acc[1]);
            }
        }
    }
};

template <bool SYM> struct Quad<2, SYM> {
    template <class C>
    static __device__ __forceinline__ void lookup(const C &c, const uint32_t *tab, int *acc, uint32_t wtx, uint32_t wty) {
#pragma unroll
        for (int pr = 0; pr < 2; ++pr) {
            const int e = 4 * pr, o = 4 * pr + 2;                   // words 2pr and 2pr + 1
            const uint32_t je = c.t(e), jo = c.t(o);
            const auto se = c.sel(e), so = c.sel(o);
            if (SYM) {
                const uint32_t *te = tab + 4 * pr, *to = tab + 4 * pr + 2;
                const uint32_t v0a = prmt(te[0], te[1], je), v0b = prmt(te[0], te[1], c.t(e + 1));
                const uint32_t v1a = prmt(to[0], to[1], jo), v1b = prmt(to[0], to[1], c.t(o + 1));
                acc[0] = dp4a_sw(prmt(v0a, v1a, 0x5410), c.sw(c.half(se, 0)), wty, acc[0]);
                acc[1] = dp4a_sw(prmt(v0a, v1a, 0x7632), c.sw(c.half(se, 1)), wty, acc[1]);
                acc[2] = dp4a_sw(prmt(v0b, v1b, 0x5410), c.sw(c.half(so, 0)), wty, acc[2]);
                acc[3] = dp4a_sw(prmt(v0b, v1b, 0x7632), c.sw(c.half(so, 1)), wty, acc[3]);
            } else {
                const uint32_t *ge = tab + 8 * pr, *go = tab + 8 * pr + 4;
                const uint32_t l0a = prmt(ge[0], ge[1], je), l0b = prmt(ge[0], ge[1], c.t(e + 1));
                const uint32_t h0a = prmt(ge[2], ge[3], je), h0b = prmt(ge[2], ge[3], c.t(e + 1));
                const uint32_t l1a = prmt(go[0], go[1], jo), l1b = prmt(go[0], go[1], c.t(o + 1));
                const uint32_t h1a = prmt(go[2], go[3], jo), h1b = prmt(go[2], go[3], c.t(o + 1));
                // transpose lo and hi candidates, then pick by the (row-ordered) sign bits
                acc[0] = __dp4a((int)prmt(prmt(l0a, l1a, 0x5410), prmt(h0a, h1a, 0x5410), c.sw(c.half(se, 0))), (int)wtx, acc[0]);
                acc[1] = __dp4a((int)prmt(prmt(l0a, l1a, 0x7632), prmt(h0a, h1a, 0x7632), c.sw(c.half(se, 1))), (int)wtx, acc[1]);
                acc[2] = __dp4a((int)prmt(prmt(l0b, l1b, 0x5410), prmt(h0b, h1b, 0x5410), c.sw(c.half(so, 0))), (int)wtx, acc[2]);
                acc[3] = __dp4a((int)prmt(prmt(l0b, l1b, 0x7632), prmt(h0b, h1b, 0x7632), c.sw(c.half(so, 1))), (int)wtx, acc[3]);
            }
        }
    }
};

__device__ __forceinline__ void transpose4(uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, uint32_t *x) {
    const uint32_t t01 = prmt(v0, v1, 0x5140), t23 = prmt(v2, v3, 0x5140);
    const uint32_t u01 = prmt(v0, v1, 0x7362), u23 = prmt(v2, v3, 0x7362);
    x[0] = prmt(t01, t23, 0x5410);
    x[1] = prmt(t01, t23, 0x7632);
    x[2] = prmt(u01, u23, 0x5410);
    x[3] = prmt(u01, u23, 0x7632);
}

template <bool SYM> struct Quad<1, SYM> {
    template <class C>
    static __device__ __forceinline__ void lookup(const C &c, const uint32_t *tab, int *acc, uint32_t wtx, uint32_t wty) {
        using Sel = decltype(c.sel(0));
        Sel s[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) s[k] = c.sel(2 * k);
        uint32_t xa[4], xb[4];
        if (SYM) {
            uint32_t va[4], vb[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                va[k] = prmt(tab[2 * k], tab[2 * k + 1], c.t(2 * k));
                vb[k] = prmt(tab[2 * k], tab[2 * k + 1], c.t(2 * k + 1));
            }
            transpose4(va[0], va[1], va[2], va[3], xa);
            transpose4(vb[0], vb[1], vb[2], vb[3], xb);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const uint32_t sa = c.half(s[r >> 1], r & 1);           // rows 0..3: words 0,0,1,1
                const uint32_t sb = c.half(s[2 + (r >> 1)], r & 1);     // rows 4..7: words 2,2,3,3
                acc[r] = dp4a_sw(xa[r], c.sw(sa), wty, acc[r]);
                acc[4 + r] = dp4a_sw(xb[r], c.sw(sb), wty, acc[4 + r]);
            }
        } else {
            uint32_t la[4], lb[4], ha[4], hb[4], xla[4], xlb[4], xha[4], xhb[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t *g = tab + 4 * k;
                la[k] = prmt(g[0], g[1], c.t(2 * k)); lb[k] = prmt(g[0], g[1], c.t(2 * k + 1));
                ha[k] = prmt(g[2], g[3], c.t(2 * k)); hb[k] = prmt(g[2], g[3], c.t(2 * k + 1));
            }
            transpose4(la[0], la[1], la[2], la[3], xla);
            transpose4(ha[0], ha[1], ha[2], ha[3], xha);
            transpose4(lb[0], lb[1], lb[2], lb[3], xlb);
            transpose4(hb[0], hb[1], hb[2], hb[3], xhb);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const uint32_t sa = c.half(s[r >> 1], r & 1);
                const uint32_t sb = c.half(s[2 + (r >> 1)], r & 1);
                acc[r] = __dp4a((int)prmt(xla[r], xha[r], c.sw(sa)), (int)wtx, acc[r]);
                acc[4 + r] = __dp4a((int)prmt(xlb[r], xhb[r], c.sw(sb)), (int)wtx, acc[4 + r]);
            }
        }
        (void)xa; (void)xb;
    }
};

// Host helper: the two constant registers handed to Quad<>::decode / lookup.
//  SYM : (wtx, wty) = byte table {+w0,+w1,+w2,+w3 | -w0,-w1,-w2,-w3}
//  !SYM: wtx = constant plane weights (w0..w3), wty unused
__host__ __device__ inline void plane_weight_regs(int bits, bool sym, uint32_t *wtx, uint32_t *wty) {
    int w[4];
    if (bits >= 3) { w[0] = 1; w[1] = 2; w[2] = 4; w[3] = (bits == 4) ? 8 : 0; }
    else if (bits == 2) { w[0] = 1; w[1] = 2; w[2] = 1; w[3] = 2; }
    else { w[0] = w[1] = w[2] = w[3] = 1; }
    uint32_t p = 0, n = 0;
    for (int i = 0; i < 4; ++i) { p |= (uint32_t)(w[i] & 0xff) << (8 * i); n |= (uint32_t)((-w[i]) & 0xff) << (8 * i); }
    *wtx = p; *wty = n;
    (void)sym;
}

__device__ __forceinline__ float load_scale(const unsigned char *p, int sd, int i) {
    return sd == 2 ? __half2float(reinterpret_cast<const __half *>(p)[i]) : reinterpret_cast<const float *>(p)[i];
}

// The plane codes of lane-row i, K-group k of a lane's quad w4 (its four words, the stream layout of tmac_layout.h): nibble b of
// the result is the code (j | neg << 3) of plane b; 16 bits for PB 4, 8 for PB 2, 4 for PB 1.  PB 4 keeps each code whole in
// word k; PB 2 and PB 1 keep the j bits there and the neg bits of a group pair (PB 2) / quad (PB 1) together in one word.
template <int PB>
__device__ __forceinline__ uint32_t row_codes(const uint32_t *w4, int k, int i) {
    static_assert(PB == 1 || PB == 2 || PB == 4, "planes per word");
    if constexpr (PB == 4) return (w4[k] >> (16 * i)) & 0xffffu;
    else if constexpr (PB == 2) return ((w4[k] >> (8 * i)) & 0x77u) | (((w4[2 * (k >> 1) + (i >> 1)] >> (16 * (i & 1) + 8 * (k & 1) + 3)) & 0x11u) << 3);
    else return ((w4[k] >> (4 * i)) & 7u) | (((w4[i >> 1] >> (16 * (i & 1) + 4 * k + 3)) & 1u) << 3);
}

// ------------------------------------------------------------------------------------------
// The activation LUT: the operation order of the AVX2 branch of lut_ctor.cc, with explicit round-to-nearest operations so
// that no FMA contraction can change a rounding.  Every kernel that builds LUT bytes, LUT scales or LUT biases
// (preprocessor_kernel, gemv3_kernel's row inputs, chain_kernel, seq_kernel) builds them with these functions.
// ------------------------------------------------------------------------------------------
// abs-sum of one K-group, whose maximum over the activation group gives the LUT scale (lut_ctor.cc:242-256; association :251)
__device__ __forceinline__ float lut_abs_sum(float x0, float x1, float x2, float x3) {
    return __fadd_rn(__fadd_rn(fabsf(x0), fabsf(x1)), __fadd_rn(fabsf(x2), fabsf(x3)));
}
__device__ __forceinline__ float lut_scale(float abs_sum_max) { return __fdiv_rn(abs_sum_max, 127.0f); }              // :256
__device__ __forceinline__ float lut_ts(float scale) { return (scale != 0.0f) ? __fdiv_rn(1.0f, scale) : 0.0f; }     // :124
// odd entries od[i] = LUT[2i + 1] = ((x0 +- x1) +- x2) +- x3 (:133-151); LUT[14 - 2i] = -od[i] (:153-155), so LUT[0] = -od[7]
__device__ __forceinline__ void lut_odd_entries(float x0, float x1, float x2, float x3, float *od) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = 2 * i + 1;
        float v = x0;
        v = (idx & 2) ? __fadd_rn(v, x1) : __fsub_rn(v, x1);
        v = (idx & 4) ? __fadd_rn(v, x2) : __fsub_rn(v, x2);
        v = (idx & 8) ? __fadd_rn(v, x3) : __fsub_rn(v, x3);
        od[i] = v;
    }
}
// int8 table entry: round half-even (:160-171), saturate as the packs (:173-176)
__device__ __forceinline__ int lut_q8(float v, float ts) { return max(-128, min(127, __float2int_rn(__fmul_rn(v, ts)))); }
// The 8 stored entries LUT[0..7] of the odd-symmetric table as int8 bytes lo | hi; returns LUT[0].
__device__ __forceinline__ float lut_stored(float x0, float x1, float x2, float x3, float ts, uint32_t &lo, uint32_t &hi) {
    float od[8];
    lut_odd_entries(x0, x1, x2, x3, od);
    lo = 0; hi = 0;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const uint32_t q = (uint32_t)(lut_q8((e & 1) ? od[e >> 1] : -od[(15 - e) >> 1], ts) & 0xff);
        if (e < 4) lo |= q << (8 * e); else hi |= q << (8 * (e - 4));
    }
    return -od[7];
}
// _mm256_addv_ps of 8 consecutive lanes' values (lut_ctor.cc:24-31), the result in all 8 lanes.  All 32 lanes must call it.
__device__ __forceinline__ float lut_addv8(float v) {
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 2));
    return __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, 1));
}
// Warp form, lane = K-group, WL lanes per activation group: the group's LUT scale and the lane's stored entries lo | hi; returns
// the lane's LUT[0], whose lut_addv8 lut_bias sums into the group's bias.  All 32 lanes must call it.  (The kernels store lo | hi
// before the addv8 shuffles: issued after them, the store costs the hot kernels extra instructions.)
template <int WL>
__device__ __forceinline__ float lut_group(float x0, float x1, float x2, float x3, uint32_t &lo, uint32_t &hi, float &scale) {
    float m = lut_abs_sum(x0, x1, x2, x3);
#pragma unroll
    for (int s = WL / 2; s >= 1; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
    scale = lut_scale(m);
    return lut_stored(x0, x1, x2, x3, lut_ts(scale), lo, hi);
}
// LUT bias of the activation group whose first lane is `first`, from blk = lut_addv8(LUT[0]): the serial sum over the group's
// 8-lane blocks from 0 (:157), in every lane.
template <int WL>
__device__ __forceinline__ float lut_bias(float blk, int first) {
    float bias = 0.f;
#pragma unroll
    for (int k = 0; k < WL / 8; ++k) bias = __fadd_rn(bias, __shfl_sync(0xffffffffu, blk, first + 8 * k));
    return bias;
}
// LUT slice of one chunk of NAG activation groups, lane = K-group (x0..x3 = its four activations, zero in lanes >= NAG * WL):
// the lane's stored entries to the warp's table (lanes < NAG * WL), the groups' LUT scales to lsv; returns the sum of their LUT
// biases.  All 32 lanes must call it.
template <int WL, int NAG>
__device__ __forceinline__ float lut_slice(float x0, float x1, float x2, float x3, int lane, unsigned char *tab, float *lsv) {
    uint32_t lo, hi;
    float scale, lbsum = 0.f;
    const float l0 = lut_group<WL>(x0, x1, x2, x3, lo, hi, scale);
    if (lane < NAG * WL) reinterpret_cast<uint2 *>(tab)[lane] = make_uint2(lo, hi);
    const float blk = lut_addv8(l0);
#pragma unroll
    for (int a = 0; a < NAG; ++a) {
        lsv[a] = __shfl_sync(0xffffffffu, scale, a * WL);
        lbsum += lut_bias<WL>(blk, a * WL);
    }
    return lbsum;
}
// The gated activation of a SwiGLU FFN, silu(g) * u, as the input of a sequence op that reads two producers (the gate and up
// projections): fp32 with exactly this rounding -- expf, not __expf (the build has no fast-math) -- so that the op equals a plain
// op fed with the vector of these values.  Its LUT is then built with lut_slice / lut_record like any input.
__device__ __forceinline__ float swiglu(float g, float u) { return __fmul_rn(__fdiv_rn(g, __fadd_rn(1.0f, expf(-g))), u); }
// The gated activation of a squared-ReLU FFN (BitNet b1.58 2B4T, HF hidden_act "relu2"), relu(g)^2 * u, in fp32 with exactly this
// rounding: r = g when g > 0 or g is NaN (torch's relu propagates NaN), else +0; then (r * r) * u.  The GEMV's kInRelu2Norm and the
// prompt form's pf_swiglu_kernel<T, true> both call it, so the two forms build the same input.
__device__ __forceinline__ float relu2(float g, float u) {
    const float r = (g > 0.f || isnan(g)) ? g : 0.f;
    return __fmul_rn(__fmul_rn(r, r), u);
}

// The RMS norm of a producer's whole output row h[0, K) as the input of a sequence op: a[k] = (h[k] * inv) * w[k] with
// inv = 1 / sqrt(ss / K + eps).  The sum of squares ss has one order, so that every consumer (a warp of chain_kernel, a CTA of
// seq_kernel) computes the same bits without an exchange: lane l of a warp owns the 4-element groups g = l, l + 32, l + 64, ...
// and adds them in ascending order with rms_sumsq to a sum that starts at +0; rms_warp_sum then combines the 32 lane sums with
// the shfl_xor butterfly over 16, 8, 4, 2, 1 (IEEE addition is commutative, so every lane ends with the same bits).  Every
// operation is rounded on its own (no contraction into fma).
__device__ __forceinline__ float rms_sumsq(float s, float x0, float x1, float x2, float x3) {
    return __fadd_rn(s, __fadd_rn(__fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1)), __fadd_rn(__fmul_rn(x2, x2), __fmul_rn(x3, x3))));
}
__device__ __forceinline__ float rms_warp_sum(float s) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, m));
    return s;
}
__device__ __forceinline__ float rms_inv(float ss, int K, float eps) { return __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, (float)K), eps))); }
__device__ __forceinline__ float rms_scale(float h, float inv, float w) { return __fmul_rn(__fmul_rn(h, inv), w); }

// ------------------------------------------------------------------------------------------
// The arithmetic of one (row super-block, K chunk) block, shared by gemv3_kernel and chain_kernel, whose lookups seq_kernel runs
// too: the fp32 operation order decides the result, so they run this one code.  The block is the stream layout (tmac_layout.h):
// QCH quads of 32 lanes x 16 code bytes, then RSB weight scales and (zp) RSB zero points of sd bytes each; tab is the warp's LUT
// slice of the chunk.  These are macros, not functions: the compiler simplifies a callee before it inlines it, and as
// __forceinline__ functions the step changed the kernels' SASS (the row-input gemv3_kernel<2,true,8,4,3> 1752 -> 1768 instructions,
// chain_kernel<2,8,4> another shared-memory load mix).  Expanded in place they compile to the instructions of the code they
// replaced.
// ------------------------------------------------------------------------------------------
// TMAC_QUAD_TABLE: quad q of the block from its QuadCodes (Quad<PB, SYM>::decode of the lane's code word) and the quad's table
// entries, through Quad<PB, SYM>::lookup into iacc.
#define TMAC_QUAD_TABLE(PB, SYM, codes, tab, q, wtx, wty, iacc)                                                                   \
    do {                                                                                                                          \
        uint32_t t_[(SYM) ? 8 : 16];                                                                                              \
        if (SYM) {                                                                                                                \
            const uint4 a_ = reinterpret_cast<const uint4 *>(tab)[2 * (q)], b_ = reinterpret_cast<const uint4 *>(tab)[2 * (q) + 1]; \
            t_[0] = a_.x; t_[1] = a_.y; t_[2] = a_.z; t_[3] = a_.w; t_[4] = b_.x; t_[5] = b_.y; t_[6] = b_.z; t_[7] = b_.w;        \
        } else {                                                                                                                  \
            _Pragma("unroll") for (int k_ = 0; k_ < 4; ++k_) {                                                                    \
                const uint4 a_ = reinterpret_cast<const uint4 *>(tab)[4 * (q) + k_];                                              \
                t_[4 * k_] = a_.x; t_[4 * k_ + 1] = a_.y; t_[4 * k_ + 2] = a_.z; t_[4 * k_ + 3] = a_.w;                           \
            }                                                                                                                     \
        }                                                                                                                         \
        Quad<PB, SYM>::lookup((codes), t_, (iacc), (wtx), (wty));                                                                 \
    } while (0)
// TMAC_QUAD_LOOKUP: quad q of the block -- the lane's code word at wp[q * 32] (wp = the block's first uint4 + lane), decoded in
// place -- through TMAC_QUAD_TABLE into iacc.
#define TMAC_QUAD_LOOKUP(PB, SYM, wp, tab, q, wtx, wty, iacc)                                                                     \
    do {                                                                                                                          \
        const uint4 wq_ = (wp)[(q) * 32];                                                                                         \
        TMAC_QUAD_TABLE(PB, SYM, (QuadWord<SYM>(wq_, (wtx))), tab, q, wtx, wty, iacc);                                               \
    } while (0)
// TMAC_GROUP_FOLD: the end of an activation group, facc[i] += ls * iacc[i] with the group's LUT scale ls; iacc is left at zero.
#define TMAC_GROUP_FOLD(PB, ls, iacc, facc)                                                                                       \
    do {                                                                                                                          \
        _Pragma("unroll") for (int i_ = 0; i_ < 8 / (PB); ++i_) {                                                                 \
            (facc)[i_] = fmaf((ls), (float)(iacc)[i_], (facc)[i_]);                                                               \
            (iacc)[i_] = 0;                                                                                                       \
        }                                                                                                                         \
    } while (0)
// TMAC_BLOCK_LOOKUPS: facc[i] = sum over the chunk's activation groups a of lsv[a] * (lane's row i lookups of a's AGQ quads),
// Quad<PB, SYM> into iacc, which is left at zero.  AGQ == 0 (integer path, one activation group = the whole row): only iacc
// accumulates.  Arguments are evaluated more than once.
#define TMAC_BLOCK_LOOKUPS(PB, SYM, QCH, AGQ, stage, tab, lane, wtx, wty, lsv, iacc, facc)                                        \
    TMAC_BLOCK_LOOKUPS_AHEAD(PB, SYM, QCH, AGQ, 0, (const QuadCodes *)nullptr, stage, tab, lane, wtx, wty, lsv, iacc, facc)
// TMAC_BLOCK_LOOKUPS_AHEAD: TMAC_BLOCK_LOOKUPS with quads 0 .. QD - 1 already decoded into codes[0 .. QD - 1] (decoded ahead,
// while the kernel waited for the chunk's input); the other quads are decoded in place.
#define TMAC_BLOCK_LOOKUPS_AHEAD(PB, SYM, QCH, AGQ, QD, codes, stage, tab, lane, wtx, wty, lsv, iacc, facc)                       \
    do {                                                                                                                          \
        constexpr int AQ_ = (AGQ) ? (AGQ) : 1;                                                                                    \
        const uint4 *wp_ = reinterpret_cast<const uint4 *>(stage) + (lane);                                                       \
        _Pragma("unroll") for (int i_ = 0; i_ < 8 / (PB); ++i_) (facc)[i_] = 0.f;                                                 \
        _Pragma("unroll") for (int q_ = 0; q_ < (QCH); ++q_) {                                                                    \
            if (q_ < (QD)) TMAC_QUAD_TABLE(PB, SYM, (codes)[q_], tab, q_, wtx, wty, iacc);                                        \
            else TMAC_QUAD_LOOKUP(PB, SYM, wp_, tab, q_, wtx, wty, iacc);                                                         \
            if ((AGQ) && ((q_ + 1) % AQ_) == 0) TMAC_GROUP_FOLD(PB, (lsv)[q_ / AQ_], iacc, facc);                                 \
        }                                                                                                                         \
    } while (0)
// TMAC_BLOCK_SCALES: cacc[i] += 0.5*s * (facc[i] + lbsum) (+ z * lbsum) with the weight scale s (scale0 for one_scale tensors)
// and zero point z of the lane's row i: tbl.cc:435-529 re-associated, lbsum = the LUT biases of the chunk's activation groups.
#define TMAC_BLOCK_SCALES(PB, QCH, stage, lane, one_scale, scale0, sd, zp, facc, lbsum, cacc)                                     \
    do {                                                                                                                          \
        constexpr int RW_ = 8 / (PB), RSB_ = 32 * RW_;                                                                            \
        const unsigned char *sp_ = (stage) + (size_t)(QCH) * 512;                                                                 \
        _Pragma("unroll") for (int i_ = 0; i_ < RW_; ++i_) {                                                                      \
            const float s_ = (one_scale) ? (scale0) : load_scale(sp_, (sd), (lane) * RW_ + i_);                                   \
            float v_ = fmaf(0.5f * s_, (facc)[i_] + (lbsum), (cacc)[i_]);                                                         \
            if (zp) v_ = fmaf(load_scale(sp_ + (size_t)RSB_ * (sd), (sd), (lane) * RW_ + i_), (lbsum), v_);                       \
            (cacc)[i_] = v_;                                                                                                      \
        }                                                                                                                         \
    } while (0)

// ==========================================================================================
// gemv3_kernel -- the production GEMV.
//
//   decomposition : CTA = (row super-block, K slice); the K slices of one super-block form a
//                   thread-block CLUSTER (size CS <= 8) and are summed through distributed shared
//                   memory in rank order -- deterministic, no global scratch, no atomics.
//   warps         : warp-autonomous.  Warp w of CTA rank r owns the `bpw` consecutive K chunks
//                   starting at (r*WPC + w)*bpw.  Every lane owns RW rows (no cross-lane reduce).
//   memory        : each warp copies its (contiguous, 16-byte aligned) block HBM -> its private
//                   shared-memory stage with cp.async (LDGSTS, L2 evict-first) BEFORE
//                   griddepcontrol.wait: weights are static, so under programmatic dependent launch
//                   the stream of launch i+1 overlaps the math of launch i, and because the bytes
//                   wait in shared memory (not registers) both launches fit on an SM together.
//                   The activation LUT slice of the chunk (QCH*4 groups x 16 B) is fetched after the
//                   wait into a warp-private table and read back as broadcast LDS.128.
//                   One lane per warp can also issue cp.async.bulk.prefetch.L2 for the same block of
//                   the NEXT tensor (optional hint).
//   arithmetic    : Quad<PB,SYM> (PRMT lookups + DP4A), per-act-group fp32 scale, per-chunk weight
//                   scale / zero point, exactly the algebra of tbl.cc:435-529 re-associated.
//   template AGQ  : quads per activation group inside a chunk (2, 4, 8); 0 = integer path
//                   (one LUT scale for the whole row, python/t_mac/ops/qgemm.py:93-96).
// ==========================================================================================
struct Gemv3Params {
    const unsigned char *W;        // first block of the launch's first row super-block
    const unsigned char *Wnext;    // same, for the tensor that will be used next (L2 prefetch) or null
    const int8_t *qlut;            // [N][K/4][16]
    const float *lut_scales, *lut_biases;  // [N][K/ags]
    void *C;                       // [N][ldc]
    int K, ldc, row_begin, row_end, c_row0, bits;
    int nrsb, rsb0, nchunk;
    int ags;
    int zp, one_scale, sd, out_f16;
    int blk_bytes;                 // bytes per block (weights + scales)
    int cs, wpc, bpw;              // cluster size, warps per CTA, chunks per warp
    int nbuf;                      // stage buffers per warp (1 or 2)
    int pdl_late;                  // trigger dependents after the math instead of at entry
    // grouped launch: blockIdx.z selects one of `nbatch` problems with identical geometry
    int nbatch;
    const unsigned char *const *Wv;
    const int8_t *const *qlutv;
    const float *const *lsv, *const *lbv;
    void *const *Cv;
    // LUT built inside the kernel (IN != kInTable): activations [N][K] f32 or f16 instead of qlut / lut_scales / lut_biases
    const void *act;
    int act_f16;
    int ioff;                      // byte offset in shared memory of the integer path's row-scan scratch / kInNorm's row
    size_t rsb_stride;
    float scale0;
    long long *trace;
    // multi-GPU row sharding: the finished rows are also stored straight into the peers' output vectors (P2P over NVLink),
    // Cpeer[q] already offset to this shard's first row; N = 1 only
    int npeer;
    void *Cpeer[7];
};
// The input of a gemv3_kernel instantiation, its template parameter IN: kInTable reads QLUT / LUT_Scales / LUT_Biases; every other
// kind builds the LUT from activation rows p.act (the plain row, the norm's h, the GLU's g) with a symmetric table.
// The routed-expert kinds (kInExperts, kInExpertsGlu) pick each slot's tensor on the device: slot z = i * topk + j of token n
// (blockIdx.z, blockIdx.y) runs pointer-table entry i * n_experts + ids[n * topk + j].
// kInGluNorm is the RMS norm of the SwiGLU row (BitNet's ffn_sub_norm before the down projection); kInRelu2Norm the RMS norm of
// the squared-ReLU row (the same sub-norm in BitNet b1.58 2B4T, whose FFN gate is relu2).  kInNormBias is kInNorm whose outputs
// take a per-tensor bias (Qwen2's q/k/v projections).
enum : int { kInTable = 0, kInRow = 1, kInNorm = 2, kInGlu = 3, kInExperts = 4, kInExpertsGlu = 5, kInGluNorm = 6, kInRelu2Norm = 7,
             kInNormBias = 8 };
// What each kind does.  The kernel, its launch and the host's choice of kind for a call (io_kind) test these, never a list of kinds.
enum : int { kGateNone = 0, kGateSilu = 1, kGateRelu2 = 2 };
// kGateNone: the row of p.act; else the row gate(g, u) of p.act and the second input io.act2, swiglu or relu2.
__host__ __device__ constexpr int in_gate(int in) {
    return in == kInRelu2Norm ? kGateRelu2 : in == kInGlu || in == kInGluNorm || in == kInExpertsGlu ? kGateSilu : kGateNone;
}
// The RMS norm of that row with io.nw and io.eps.
__host__ __device__ constexpr bool in_norm(int in) { return in == kInNorm || in == kInGluNorm || in == kInRelu2Norm || in == kInNormBias; }
// The outputs take the tensor's bias from io.biasv.
__host__ __device__ constexpr bool in_bias(int in) { return in == kInNormBias; }
// Routed experts: each slot picks its tensor by the id it reads.
__host__ __device__ constexpr bool in_experts(int in) { return in == kInExperts || in == kInExpertsGlu; }
// The input transform and residual of the row kinds: the kernel's last parameter, so that Gemv3Params, wtx and wty keep their
// parameter offsets.
struct Gemv3Io {
    const void *act2;              // kInGlu, kInGluNorm, kInRelu2Norm, kInExpertsGlu: u [N][K] / [N][topk][K], dtype of p.act
    const float *nw;               // kInNorm, kInGluNorm, kInRelu2Norm, kInNormBias: the norm weight w [K] (16-byte aligned)
    float eps;                     // kInNorm, kInGluNorm, kInRelu2Norm, kInNormBias
    const void *res;               // fp path, kInRow / kInNorm / kInGlu / kInGluNorm / kInRelu2Norm / kInExpertsGlu: residual r [N][ldc] of the output's dtype,
                                   // or null; may equal C
    const int32_t *ids;            // experts: [N][topk], written by earlier work in the stream (read after the dependency wait)
    const float *wts;              // kInExpertsGlu: combine weights [N][topk]
    float *ws;                     // kInExpertsGlu: the slots' fp32 rows [N][topk][ldc]
    unsigned *cnt;                 // kInExpertsGlu: arrivals per (token, row super-block) [N][nrsb], 0 between launches
    int topk, n_experts;           // experts
    const float *const *biasv;     // kInNormBias: bias[z] fp32 [Mout] of the grouped launch's tensor z (device pointer table)
};
__device__ __forceinline__ long long globaltimer_ns() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#ifdef TMAC_ENABLE_TRACE
// slots 0..6: clock64 (SM cycles) since entry; slot 7: globaltimer (ns) at entry.
#define TMAC_TRACE(slot) do { if (p.trace) p.trace[(size_t)blockIdx.x * 8 + (slot)] = globaltimer_ns(); } while (0)
#else
#define TMAC_TRACE(slot) do { } while (0)
#endif

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void l2_prefetch_bulk(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async16_plain(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Split cluster barrier.  gemv3 uses it to establish "every CTA of the cluster is running" before the first distributed-shared-
// memory access (required by the programming model) without stalling at entry; chain_kernel to guard only the RE-USE of shared-
// memory buffers, whose readers have consumed their values before they arrive.  Neither carries data, so the arrive needs no
// release -- which ptxas turns into MEMBAR.ALL.GPU per thread.  (barrier.cluster.wait has only the acquire form.)
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ void st_cluster_f32(float *local_ptr, uint32_t rank, float v) {
    uint32_t raddr;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(local_ptr)), "r"(rank));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(raddr), "f"(v) : "memory");
}

// mbarriers and bulk (TMA) copies.  One bulk copy per block instead of a per-lane cp.async loop: 1 instruction from one lane
// instead of ~4 per 16 bytes on the ALU pipe that the lookup loop saturates; completion on an mbarrier.
__device__ __forceinline__ void mbar_init(uint64_t *b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy shared-memory accesses before this point are ordered before later bulk copies / wgmma reads (async proxy)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_load(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    expect_tx(bar, bytes);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// bulk_load with an L2 eviction policy for the copied lines (policy_evict_first: data read once)
__device__ __forceinline__ void bulk_load_hint(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar, uint64_t pol) {
    expect_tx(bar, bytes);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void mbar_wait_parity(uint64_t *b, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}\n"
        ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
// Bounded form of the persistent kernels: false if the phase has not completed after LIMIT polls.
template <int LIMIT> __device__ __forceinline__ bool mbar_wait_bounded(uint64_t *b, uint32_t parity) {
    uint32_t ok = 0;
    for (int spins = 0; spins < LIMIT && !ok; ++spins)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
    return ok != 0;
}

// One output element C[i], fp16 or fp32.  C by reference and i of the caller's type: the pointer is then read inside the branch
// and the index widened as at the call site, as in the stores this replaced, and every epilogue compiles as before.
template <typename I> __device__ __forceinline__ void store_out(void *const &C, I i, float v, int f16) {
    if (f16) reinterpret_cast<__half *>(C)[i] = __float2half_rn(v);
    else reinterpret_cast<float *>(C)[i] = v;
}

// Integer-path (BitNet) output of one row and token from its exact integer sum isum = sum_b 2*alpha_b*CBits_b, the token's LUT
// scale ls and bias lb and the tensor's one weight scale:
// C = ((sum_b alpha_b*CBits_b) * LUT_Scales[0] + LUT_Biases[0]*alpha_0) * Scales[0] (python/t_mac/ops/qgemm.py:160,171-174),
// every operation rounded on its own (no contraction into an fma), in the reference's order.
__device__ __forceinline__ float int_path_out(int isum, float ls, float lb, float scale0) {
    const float cb = __fmul_rn((float)isum, 0.5f);
    const float t1 = __fmul_rn(cb, ls);
    const float t2 = __fmul_rn(lb, 0.5f);
    return __fmul_rn(__fadd_rn(t1, t2), scale0);
}

constexpr int kG3MaxWarps = 8;

// MINB = minimum resident CTAs per SM the register allocation is tuned for: 3 (85 registers, more ILP;
// best for a single launch per tensor) or 4 (64 registers, more CTAs in flight; best for grouped launches).
// IN != kInTable: build the LUT slice of each chunk inside the GEMV from the activation row (with the LUT functions above,
// as preprocessor_kernel, so QLUT bytes, LUT scales and LUT biases are bit-identical to the two-kernel path)
// instead of reading QLUT / LUT_Scales / LUT_Biases.  Requires SYM.  AGQ > 0: activation
// group inside a chunk, scale and bias per chunk by warp shuffles.  AGQ == 0 (integer path, ONE activation group
// = the whole row, BitNet; kInTable and kInRow only): every CTA scans the row once (K * 4 bytes, L2-resident) for the row-wide
// abs-sum maximum -- cheaper than a cluster-wide exchange, which costs a rendezvous -- and the cluster leader also forms
// the row's LUT bias in the reference's order (addv tree per 32 activations, serial over the blocks).
// The LUT input of row n is the row itself (kInRow) or a transform of the activation rows -- kInNorm a[k] = rms_scale(h[k], inv_n,
// w[k]), kInGlu a[k] = swiglu(g[k], u[k]), kInGluNorm a[k] = rms_scale(s[k], inv_n, w[k]) with s[k] = swiglu(g[k], u[k]) and inv_n
// from the sum of squares of s, kInRelu2Norm the same with s[k] = relu2(g[k], u[k]), kInNormBias kInNorm's -- built into the chunk's
// slice with lut_slice as a plain input; on the fp path the leader adds io.res (when not null) to the row sums before the store, and
// kInNormBias adds its tensor's bias there instead: C = fadd_rn(row sum, bias[z][row]), rounded once at the store.
// Routed experts: slot z = i * topk + j of token n takes its tensor from the pointer table at
// i * n_experts + ids[n][j], read after the dependency wait, so the slot's first block request waits for it too.  kInExperts reads row
// n and stores row n * topk + j of C[i]; kInExpertsGlu reads row n * topk + j of g and u, stores its rows into io.ws and counts
// itself in io.cnt, and the leader that completes a (token, row super-block) combines the topk rows in ascending j into C.  A slot
// whose id is outside [0, n_experts) streams no block and yields quiet NaN rows.
template <int PB, bool SYM, int QCH, int AGQ, int MINB, int IN>
__global__ void __launch_bounds__(kG3MaxWarps * 32, MINB) gemv3_kernel(const Gemv3Params p, const uint32_t wtx, const uint32_t wty,
                                                                       const Gemv3Io io) {
    static_assert(IN == kInTable || SYM, "a LUT built from activation rows is symmetric");
    static_assert(IN == kInTable || IN == kInRow || AGQ > 0, "input transforms and experts: fp path only");
    constexpr bool EXPERTS = in_experts(IN);
    constexpr int RW = 8 / PB;
    constexpr int RSB = 32 * RW;
    constexpr int TB = SYM ? 8 : 16;              // table bytes per group in shared memory
    constexpr bool INT_PATH = (AGQ == 0);
    constexpr int NAG = INT_PATH ? 1 : QCH / AGQ; // activation groups per chunk
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int WPC = p.wpc;
    const int rank = (p.cs > 1) ? (int)cluster_ctarank() : 0;
    const int rsb = blockIdx.x / p.cs, n = blockIdx.y;
    // shared memory: cl [CS][RSB] (cluster partials, leader only) | per warp: stage (blk_bytes) + table
    // (QCH*4*TB).  The CTA reduction buffer red [WPC][RSB] aliases the stages once they are consumed.
    float *cl = reinterpret_cast<float *>(smem);
    const int tab_bytes = QCH * 4 * TB;
    const int nbuf = p.nbuf;                      // 2 = double-buffered stage when a warp walks several chunks, 1 = single
    const int per_warp = nbuf * p.blk_bytes + tab_bytes;
    unsigned char *wbase = smem + (size_t)p.cs * RSB * 4;
    unsigned char *stage0 = wbase + (size_t)warp * per_warp;
    unsigned char *tab = stage0 + nbuf * p.blk_bytes;
    float *red = reinterpret_cast<float *>(wbase);
    // warp-private mbarriers (one per stage buffer) behind the region that red aliases
    const size_t wregion = max((size_t)WPC * per_warp, (size_t)WPC * RSB * 4);
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbase + ((wregion + 15) & ~(size_t)15)) + warp * 2;

    if (tid == 0) { TMAC_TRACE(0); }
    if (p.cs > 1) cluster_arrive_relaxed();       // phase 1: "I am running" (waited for right before the DSMEM stores)
    if (!p.pdl_late) pdl_launch_dependents();     // the next launch may start its weight stream now

    const int c_first = (rank * WPC + warp) * p.bpw;
    int c_end = min(p.nchunk, c_first + p.bpw);
    const unsigned char *Wb = p.W;
    const int8_t *qb = p.qlut;
    const float *lsb = p.lut_scales, *lbb = p.lut_biases;
    void *Cb = p.C;
    const int xj = EXPERTS ? (int)blockIdx.z % io.topk : 0;   // experts: the slot's rank j among the token's topk and its tensor i
    const int xi = EXPERTS ? (int)blockIdx.z / io.topk : 0;
    if (p.nbatch > 0) {
        const int z = blockIdx.z;
        if (EXPERTS) Cb = p.Cv[xi * io.n_experts];
        else { Wb = p.Wv[z]; Cb = p.Cv[z]; }
        if (IN == kInTable) { qb = p.qlutv[z]; lsb = p.lsv[z]; lbb = p.lbv[z]; }   // else the tensors of the group share the activation rows
    }
    const unsigned char *rsb_base = Wb + (size_t)rsb * p.rsb_stride;
    const int nag = p.K / p.ags;
    const int arow = IN == kInExpertsGlu ? n * io.topk + xj : n;   // the activation row of this CTA
    // row inputs: the 4 activations from element k of the row of act (p.act, or the GLU's u), fp32 or fp16
    auto load_group = [&](size_t k, float4 &x, const void *act = nullptr) {
        const size_t k0 = (size_t)arow * p.K + k;
        if (!act) act = p.act;
        if (p.act_f16) {
            const uint2 h = __ldg(reinterpret_cast<const uint2 *>(reinterpret_cast<const __half *>(act) + k0));
            const float2 f01 = __half22float2(*reinterpret_cast<const __half2 *>(&h.x)), f23 = __half22float2(*reinterpret_cast<const __half2 *>(&h.y));
            x.x = f01.x; x.y = f01.y; x.z = f23.x; x.w = f23.y;
        } else {
            x = __ldg(reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(act) + k0));
        }
    };

    // ---- first chunk: HBM -> shared, issued before the dependency wait -------------------------
    if (lane == 0) {
        mbar_init(mbar, 1); mbar_init(mbar + 1, 1);
        mbar_fence_init();
        fence_proxy_async();
        if (!EXPERTS && c_first < c_end) {
            bulk_load(stage0, rsb_base + (size_t)c_first * p.blk_bytes, (uint32_t)p.blk_bytes, mbar);
            if (p.Wnext)                           // pull the next tensor's blocks of this warp into L2
                l2_prefetch_bulk(p.Wnext + (size_t)rsb * p.rsb_stride + (size_t)c_first * p.blk_bytes,
                                 (uint32_t)((c_end - c_first) * p.blk_bytes));
        }
    }
    __syncwarp();
    if (tid == 0) TMAC_TRACE(1);
    pdl_wait();                                   // LUT / LUT scales come from the previous kernel
    if (tid == 0) TMAC_TRACE(2);
    bool bad = false;                             // experts: the slot's id is outside [0, n_experts)
    if (EXPERTS) {
        const int id = io.ids[(size_t)n * io.topk + xj];
        bad = (unsigned)id >= (unsigned)io.n_experts;
        if (bad) c_end = c_first;                  // no block: the sums stay 0 and the rows become NaN in the epilogue
        else rsb_base = p.Wv[xi * io.n_experts + id] + (size_t)rsb * p.rsb_stride;
        if (lane == 0 && c_first < c_end) bulk_load(stage0, rsb_base + (size_t)c_first * p.blk_bytes, (uint32_t)p.blk_bytes, mbar);
    }

    float cacc[RW];
    int iacc[RW];
#pragma unroll
    for (int i = 0; i < RW; ++i) { cacc[i] = 0.f; iacc[i] = 0; }
    float row_scale = 0.f, row_ts = 0.f;          // fused integer path: LUT scale of the row and its reciprocal
    float *iscr = reinterpret_cast<float *>(smem + p.ioff);   // [K/32] block sums (leader) | [8] warp maxima | [1] bias
    bool scan_split = false;                      // fused integer path: the cluster splits the row scan (else every CTA scans the row)
    if (IN != kInTable && INT_PATH) {
        // Row-wide LUT scale and bias (lut_ctor.cc:232-260 partial_max over the whole row, :157 bias) without a preprocessor launch.
        // Short rows (one round of four 16-byte loads per thread covers the row, K = 3200): every CTA scans the whole row itself,
        // no exchange.  Long rows (K = 8640): that is 200 CTAs x 34 KB of reads on the same few L2 lines, several serial rounds;
        // the cluster splits the row instead, maxima go to every peer and the block sums of LUT[0] to the last rank through
        // distributed shared memory, one cluster barrier (whole-row scan for short rows, split for long ones).  The last rank's last warp (idle or lightest: warps beyond the last chunk have no block)
        // forms the bias serially; the leader needs it only in the epilogue.
        const int nblk = p.K >> 5, ngrp = p.K >> 2, nth = WPC * 32;
        float *wmax = iscr + nblk, *bias_out = wmax + kG3MaxWarps, *cmax = bias_out + 4;
        scan_split = p.cs > 1 && ngrp > 4 * nth;
        const bool bias_cta = rank == p.cs - 1;
        // K-groups [gbeg, gend): LUT[0] of every group, addv8 per block of 32 activations = 8 lanes, block sums -> the bias CTA;
        // returns the abs-sum maximum
        auto scan = [&](int gbeg, int gend, bool want_max, bool remote) {
            float mm = 0.f;
            for (int g0 = gbeg + warp * 32; g0 < gend; g0 += nth) {   // lane = K-group (coalesced 16-byte loads)
                const int gi = g0 + lane;
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gi < gend) load_group((size_t)gi * 4, x);
                if (want_max) mm = fmaxf(mm, lut_abs_sum(x.x, x.y, x.z, x.w));
                float od[8];
                lut_odd_entries(x.x, x.y, x.z, x.w, od);
                const float v = lut_addv8(-od[7]);
                if ((lane & 7) == 0 && gi < gend) {
                    if (remote) st_cluster_f32(iscr + (gi >> 3), p.cs - 1, v); else iscr[gi >> 3] = v;
                }
            }
            return mm;
        };
        float m = 0.f;
        if (scan_split) {
            const int per = ((nblk + p.cs - 1) / p.cs) * 8;      // K-groups per CTA, whole blocks
            cluster_wait();                                      // phase 1 ("every CTA of the cluster runs"): DSMEM may be written
            m = scan(rank * per, min(ngrp, rank * per + per), true, true);
        } else {
            // four independent loads per thread in one round; every CTA starts at its own offset (the L2 serves a hot line one
            // request at a time)
            const int off = (int)(((long long)blockIdx.x * 160) % ngrp);
            for (int g = tid; g < ngrp; g += 4 * nth) {
                float4 b[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int gj = g + j * nth;
                    b[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (gj < ngrp) { int gi = gj + off; if (gi >= ngrp) gi -= ngrp; load_group((size_t)gi * 4, b[j]); }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) m = fmaxf(m, lut_abs_sum(b[j].x, b[j].y, b[j].z, b[j].w));
            }
            if (bias_cta) scan(0, ngrp, false, false);           // L1 hits
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) wmax[warp] = m;
        __syncthreads();
        m = wmax[0];
        for (int w = 1; w < WPC; ++w) m = fmaxf(m, wmax[w]);
        if (scan_split) {
            if (tid < p.cs) st_cluster_f32(cmax + rank, tid, m);   // this CTA's maximum -> slot `rank` of every CTA of the cluster
            cluster_sync_all();
            m = cmax[0];
            for (int r = 1; r < p.cs; ++r) m = fmaxf(m, cmax[r]);
        }
        row_scale = lut_scale(m);
        row_ts = lut_ts(row_scale);
        if (bias_cta && warp == WPC - 1) {
            // serial over the blocks of the (single) activation group, from 0 (:157).  32 values per shared-memory round trip,
            // the 32 shuffles of a round issued ahead of the dependent adds (fixed trip count); the tail is padded with +0.0,
            // an exact no-op: an accumulator that starts at +0.0 is never -0.0
            float bias = 0.0f;
            for (int k0 = 0; k0 < nblk; k0 += 32) {
                const float v = (k0 + lane < nblk) ? iscr[k0 + lane] : 0.f;
#pragma unroll
                for (int k = 0; k < 32; ++k) bias = __fadd_rn(bias, __shfl_sync(0xffffffffu, v, k));
            }
            if (lane == 0) *bias_out = bias;       // forwarded to the leader with the partial sums below
        }
    }
    float inv = 0.f;                              // in_norm: 1 / rms of the row
    if (in_norm(IN)) {
        // Every CTA computes inv itself.  All threads stage the row (kInGluNorm / kInRelu2Norm: its swiglu / relu2 of the row of g
        // and the row of u), widened to fp32, in shared memory (iscr [K] | inv), with their loads in flight together; warp 0 then
        // sums its squares in the order of rms_sumsq / rms_warp_sum.
        const int ngrp = p.K >> 2, nth = WPC * 32;
        float4 *hrow = reinterpret_cast<float4 *>(iscr);
        for (int g0 = tid; g0 < ngrp; g0 += 4 * nth) {
            float4 b[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (g0 + j * nth < ngrp) load_group((size_t)(g0 + j * nth) * 4, b[j]);
            if (in_gate(IN) != kGateNone) {
                const auto act = [](float g, float u) { return in_gate(IN) == kGateRelu2 ? relu2(g, u) : swiglu(g, u); };
                float4 u[4];
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (g0 + j * nth < ngrp) load_group((size_t)(g0 + j * nth) * 4, u[j], io.act2);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (g0 + j * nth < ngrp)
                        b[j] = make_float4(act(b[j].x, u[j].x), act(b[j].y, u[j].y), act(b[j].z, u[j].z), act(b[j].w, u[j].w));
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (g0 + j * nth < ngrp) hrow[g0 + j * nth] = b[j];
        }
        __syncthreads();
        if (warp == 0) {
            float s = 0.f;
#pragma unroll 8
            for (int g = lane; g < ngrp; g += 32) { const float4 h = hrow[g]; s = rms_sumsq(s, h.x, h.y, h.z, h.w); }
            s = rms_warp_sum(s);
            if (lane == 0) iscr[p.K] = rms_inv(s, p.K, io.eps);
        }
        __syncthreads();
        inv = iscr[p.K];
    }
    const uint4 *qrow = reinterpret_cast<const uint4 *>(qb + (size_t)n * p.K * 4);
    const float *lsg = lsb + (size_t)n * nag, *lbg = lbb + (size_t)n * nag;

    for (int c = c_first; c < c_end; ++c) {
        // ---- LUT slice of this chunk -> warp-private table (lane = group) ---------------------
        float lsv[NAG], lbsum = 0.f;
        if (IN != kInTable) {
            constexpr int NG = QCH * 4;            // lane = K-group of the chunk
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in_norm(IN)) {
                if (lane < NG) {
                    const size_t g = (size_t)c * NG + lane;
                    const float4 h = reinterpret_cast<const float4 *>(iscr)[g], w = __ldg(reinterpret_cast<const float4 *>(io.nw) + g);
                    x = make_float4(rms_scale(h.x, inv, w.x), rms_scale(h.y, inv, w.y), rms_scale(h.z, inv, w.z), rms_scale(h.w, inv, w.w));
                }
            } else if (in_gate(IN) != kGateNone) {
                if (lane < NG) {
                    float4 gv, uv;
                    load_group(((size_t)c * NG + lane) * 4, gv);
                    load_group(((size_t)c * NG + lane) * 4, uv, io.act2);
                    x = make_float4(swiglu(gv.x, uv.x), swiglu(gv.y, uv.y), swiglu(gv.z, uv.z), swiglu(gv.w, uv.w));
                }
            } else if (lane < NG) load_group(((size_t)c * NG + lane) * 4, x);
            if (INT_PATH) {
                uint32_t lo, hi;
                lut_stored(x.x, x.y, x.z, x.w, row_ts, lo, hi);
                if (lane < NG) reinterpret_cast<uint2 *>(tab)[lane] = make_uint2(lo, hi);
            } else {
                lbsum = lut_slice<(AGQ ? AGQ : 1) * 4, NAG>(x.x, x.y, x.z, x.w, lane, tab, lsv);
            }
        } else {
            if (lane < QCH * 4) {
                const uint4 L = __ldg(qrow + (size_t)c * QCH * 4 + lane);
                if (SYM) reinterpret_cast<uint2 *>(tab)[lane] = make_uint2(L.x, L.y);
                else reinterpret_cast<uint4 *>(tab)[lane] = make_uint4(L.x, L.y, __byte_perm(L.w, 0, 0x0123), __byte_perm(L.z, 0, 0x0123));
            }
            if (!INT_PATH) {
#pragma unroll
                for (int a = 0; a < NAG; ++a) { lsv[a] = __ldg(lsg + c * NAG + a); lbsum += __ldg(lbg + c * NAG + a); }
            }
        }
        const int li = c - c_first, buf = li & (nbuf - 1);
        unsigned char *stage = stage0 + (size_t)buf * p.blk_bytes;
        if (nbuf == 2) {
            if (c + 1 < c_end && lane == 0) {      // request chunk c+1 into the other buffer (consumed at c-1, see the __syncwarp below)
                fence_proxy_async();
                bulk_load(stage0 + (size_t)((li + 1) & 1) * p.blk_bytes, rsb_base + (size_t)(c + 1) * p.blk_bytes, (uint32_t)p.blk_bytes, mbar + ((li + 1) & 1));
            }
        } else if (li > 0 && lane == 0) {          // single buffer: the other resident warps cover this warp's load latency
            fence_proxy_async();
            bulk_load(stage0, rsb_base + (size_t)c * p.blk_bytes, (uint32_t)p.blk_bytes, mbar);
        }
        mbar_wait_parity(mbar + buf, nbuf == 2 ? ((li >> 1) & 1) : (li & 1));
        __syncwarp();
        if (tid == 0 && c == c_first) TMAC_TRACE(3);
        float facc[RW];
        TMAC_BLOCK_LOOKUPS(PB, SYM, QCH, AGQ, stage, tab, lane, wtx, wty, lsv, iacc, facc);
        if (!INT_PATH) TMAC_BLOCK_SCALES(PB, QCH, stage, lane, p.one_scale, p.scale0, p.sd, p.zp, facc, lbsum, cacc);
        __syncwarp();                              // stage / table are rewritten by a later chunk
    }
    if (tid == 0) TMAC_TRACE(4);
    if (p.pdl_late) pdl_launch_dependents();

    // ---- CTA reduction (fixed warp order); red aliases the consumed stages ----------------------
    __syncthreads();
    {
        float *r = red + (size_t)warp * RSB + lane * RW;
#pragma unroll
        for (int i = 0; i < RW; ++i) r[i] = INT_PATH ? __int_as_float(iacc[i]) : cacc[i];
    }
    __syncthreads();
    if (tid == 0) TMAC_TRACE(5);
    const int nthreads = WPC * 32;
    if (p.cs > 1 && !scan_split) cluster_wait();  // every CTA of the cluster has started: its shared memory may be written
    if (IN != kInTable && INT_PATH && p.cs > 1 && rank == p.cs - 1 && tid == (WPC - 1) * 32) {
        float *bias_out = iscr + (p.K >> 5) + kG3MaxWarps;
        st_cluster_f32(bias_out, 0, *bias_out);    // written by this thread after the row scan
    }
    for (int t = tid; t < RSB; t += nthreads) {
        float fsum = 0.f; int isum = 0;
        for (int w = 0; w < WPC; ++w) {
            const float v = red[(size_t)w * RSB + t];
            if (INT_PATH) isum += __float_as_int(v); else fsum += v;
        }
        const float mine = INT_PATH ? __int_as_float(isum) : fsum;
        if (p.cs > 1) st_cluster_f32(cl + (size_t)rank * RSB + t, 0, mine);   // into the leader's shared memory
        else cl[t] = mine;
    }
    if (p.cs > 1) cluster_sync_all(); else __syncthreads();
    if (tid == 0) TMAC_TRACE(6);
    if (rank != 0) return;
    for (int t = tid; t < RSB; t += nthreads) {
        float fsum = 0.f; int isum = 0;
        for (int k2 = 0; k2 < p.cs; ++k2) {
            const float v = cl[(size_t)k2 * RSB + t];
            if (INT_PATH) isum += __float_as_int(v); else fsum += v;
        }
        const int row = (p.rsb0 + rsb) * RSB + t;
        if (row >= p.row_begin && row < p.row_end) {
            float out;
            if (INT_PATH)
                out = int_path_out(isum, IN != kInTable ? row_scale : __ldg(lsg), IN != kInTable ? iscr[(p.K >> 5) + kG3MaxWarps] : __ldg(lbg), p.scale0);
            else
                out = fsum;
            if (EXPERTS) {                          // row n * topk + j of C[i] / of the workspace (c_row0 = 0)
                const size_t o = (size_t)(n * io.topk + xj) * p.ldc + row;
                if (bad) out = __int_as_float(0x7fffffff);
                if (IN == kInExperts) store_out(Cb, o, out, p.out_f16);
                else io.ws[o] = out;
            } else {
                const size_t o = (size_t)n * p.ldc + (size_t)(row - p.c_row0);
                if (IN != kInTable && !INT_PATH && io.res)   // read, then written by this thread: the residual may be C itself
                    out = __fadd_rn(out, p.out_f16 ? __half2float(reinterpret_cast<const __half *>(io.res)[o]) : reinterpret_cast<const float *>(io.res)[o]);
                if (in_bias(IN)) out = __fadd_rn(out, __ldg(io.biasv[blockIdx.z] + (row - p.c_row0)));
                store_out(Cb, o, out, p.out_f16);
                for (int q = 0; q < p.npeer; ++q)        // the all-gather, fused into the epilogue: one store per peer and row
                    store_out(p.Cpeer[q], o, out, p.out_f16);
            }
        }
    }
    if (IN == kInExpertsGlu) {
        // The combine.  This slot's rows are in io.ws; thread 0 counts the slot in (release, for every thread's stores: they precede
        // it by the barrier) and learns whether it completes the token's row super-block (acquire, for the other slots' rows).  The
        // leader that completes it adds the topk rows in ascending j -- not in arrival order -- and resets the counter for the next
        // launch, which touches it only after its dependency wait.
        unsigned *last = reinterpret_cast<unsigned *>(red);   // red is free once the CTA and cluster sums are done
        __syncthreads();
        if (tid == 0) {
            unsigned *c = io.cnt + (size_t)n * p.nrsb + rsb, prev;
            asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(c) : "memory");
            *last = prev == (unsigned)io.topk - 1;
            if (*last) *c = 0;
        }
        __syncthreads();
        if (!*last) return;
        const float *wn = io.wts + (size_t)n * io.topk;
        for (int t = tid; t < RSB; t += nthreads) {
            const int row = (p.rsb0 + rsb) * RSB + t;
            if (row < p.row_begin || row >= p.row_end) continue;
            const float *y = io.ws + (size_t)n * io.topk * p.ldc + row;
            float acc = __fmul_rn(wn[0], __ldcg(y));
            for (int j = 1; j < io.topk; ++j) acc = __fadd_rn(acc, __fmul_rn(wn[j], __ldcg(y + (size_t)j * p.ldc)));
            const size_t o = (size_t)n * p.ldc + row;
            if (io.res)                            // read, then written by this thread: the residual may be C itself
                acc = __fadd_rn(acc, p.out_f16 ? __half2float(reinterpret_cast<const __half *>(io.res)[o]) : reinterpret_cast<const float *>(io.res)[o]);
            store_out(Cb, o, acc, p.out_f16);
        }
    }
    if (tid == 0) TMAC_TRACE(7);
}

typedef void (*gemv3_fn)(const Gemv3Params, const uint32_t, const uint32_t, const Gemv3Io);
// gemv3_kernel<PB, SYM, QCH, AGQ, MINB, IN> for a tensor's (pb, qch, agq), the LUT's symmetry (kInTable; the other kinds are
// symmetric) and minb; null for a grouping that is not instantiated.  Each kind's kernels are compiled in the one translation unit
// that instantiates pick_gemv3_in for it, so that the kinds compile in parallel: kInTable in tmac_b200.cu, kInRow, kInNorm, kInGlu,
// kInGluNorm, kInRelu2Norm and kInNormBias in tmac_gemv_io.cu, kInExperts and kInExpertsGlu in tmac_gemv_experts.cu.
template <int IN> gemv3_fn pick_gemv3_in(int pb, bool sym, int qch, int agq, int minb) {
    const auto pick = [&](auto SYM, auto MINB) {
        return with_pb<gemv3_fn>(pb, [&](auto PB) {
            const auto kernel = [&](auto QCH, auto AGQ) -> gemv3_fn { return gemv3_kernel<PB, SYM, QCH, AGQ, MINB, IN>; };
            if constexpr (IN == kInTable || IN == kInRow) {
                if (!agq) return IntGroupings::find<gemv3_fn>(qch, agq, kernel);
            }
            return FpGroupings::find<gemv3_fn>(qch, agq, kernel);
        });
    };
    using Minb3 = std::integral_constant<int, 3>;
    using Minb4 = std::integral_constant<int, 4>;
    if constexpr (IN == kInTable) {
        if (!sym) return minb == 3 ? pick(std::false_type{}, Minb3{}) : pick(std::false_type{}, Minb4{});
    }
    return minb == 3 ? pick(std::true_type{}, Minb3{}) : pick(std::true_type{}, Minb4{});
}
extern template gemv3_fn pick_gemv3_in<kInTable>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInRow>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInNorm>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInGlu>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInGluNorm>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInRelu2Norm>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInNormBias>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInExperts>(int, bool, int, int, int);
extern template gemv3_fn pick_gemv3_in<kInExpertsGlu>(int, bool, int, int, int);

// ------------------------------------------------------------------------------------------
// cbits_kernel (debug / parity gate G2): per-plane int32 sums in the reference plane layout.
// One thread per (row, plane); straightforward lookups in the full 16-entry table, decoding the
// stream layout with row_codes.  Not a performance path.
// ------------------------------------------------------------------------------------------
static __global__ void cbits_kernel(const unsigned char *W, const int8_t *qlut, int32_t *cbits, int Mout, int K, int bits,
                             int pb, int qch, int nchunk, size_t rsb_stride, size_t blk_stride, int N) {
    const int rw = 8 / pb, rsbsz = 32 * rw;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)N * Mout * bits;
    if (t >= total) return;
    const int n = (int)(t / ((long long)Mout * bits));
    const int rem = (int)(t % ((long long)Mout * bits));
    const int row = rem / bits, b = rem % bits;
    const int rsb = row / rsbsz, lane = (row % rsbsz) / rw, i = (row % rsbsz) % rw;
    const int8_t *lut = qlut + (size_t)n * K * 4;
    int sum = 0;
    for (int c = 0; c < nchunk; ++c) {
        const uint32_t *wq = reinterpret_cast<const uint32_t *>(W + (size_t)rsb * rsb_stride + (size_t)c * blk_stride);
        for (int q = 0; q < qch; ++q) {
            const uint32_t *w4 = wq + ((size_t)q * 32 + lane) * 4;
            for (int k = 0; k < 4; ++k) {
                const int g = (c * qch + q) * 4 + k;
                uint32_t codes;
                switch (pb) {
                case 4: codes = row_codes<4>(w4, k, i); break;
                case 2: codes = row_codes<2>(w4, k, i); break;
                default: codes = row_codes<1>(w4, k, i); break;
                }
                const uint32_t code = (codes >> (4 * b)) & 15u, j = code & 7u;
                const uint32_t idx = (code & 8u) ? (8u | (j ^ 7u)) : j;
                sum += lut[(size_t)g * 16 + idx];
            }
        }
    }
    const int p = (row / 8) * 8 * bits + b * 8 + row % 8;
    cbits[(size_t)n * Mout * bits + p] = sum;
}

// ------------------------------------------------------------------------------------------
// preprocessor_kernel.  grid = (ceil(nag / agb), N); block = 256.
// Each CTA handles `agb` consecutive activation groups of one activation row (agb == nag when
// act_group_size == K, i.e. a single CTA per row).  Entries and scales by the LUT functions above.
// ------------------------------------------------------------------------------------------
constexpr int kPreThreads = 256;

template <typename TIn>
__device__ __forceinline__ float ld_act(const TIn *p, size_t i);
template <> __device__ __forceinline__ float ld_act<float>(const float *p, size_t i) { return p[i]; }
template <> __device__ __forceinline__ float ld_act<__half>(const __half *p, size_t i) { return __half2float(p[i]); }

template <typename TIn>
__global__ void __launch_bounds__(kPreThreads) preprocessor_kernel(const TIn *B, float *lut_scales, float *lut_biases,
                                                                    int8_t *qlut, int K, int ags, int agb) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int n = blockIdx.y;
    const int nag = K / ags;
    const int a_begin = blockIdx.x * agb;
    const int a_end = min(nag, a_begin + agb);
    const int gpa = ags / 4;                              // groups per act group
    const int g_begin = a_begin * gpa, g_end = a_end * gpa;
    const int ng = g_end - g_begin;
    int *smax = reinterpret_cast<int *>(smem);            // [agb] max abs-sum (float bits, >= 0)
    float *l0 = reinterpret_cast<float *>(smax + agb);    // [ng] LUT[0] of every group
    float *blk = l0 + ng;                                 // [ng/8] addv8 of every 32-activation block
    const TIn *b = B + (size_t)n * K;
    const int tid = threadIdx.x;

    // Programmatic dependent launch: let the consumer GEMV start streaming its (static) weights now;
    // the activations and the output buffers belong to the stream order, so wait before touching them.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    for (int a = tid; a < a_end - a_begin; a += kPreThreads) smax[a] = 0;
    asm volatile("griddepcontrol.wait;" ::: "memory");
    __syncthreads();
    // pass 1: abs-sum max per act group
    for (int g = tid; g < ng; g += kPreThreads) {
        const size_t k0 = (size_t)(g_begin + g) * 4;
        const float b0 = ld_act(b, k0), b1 = ld_act(b, k0 + 1), b2 = ld_act(b, k0 + 2), b3 = ld_act(b, k0 + 3);
        atomicMax(&smax[g / gpa], __float_as_int(lut_abs_sum(b0, b1, b2, b3)));
    }
    __syncthreads();
    // pass 2: tables
    for (int g = tid; g < ng; g += kPreThreads) {
        const size_t k0 = (size_t)(g_begin + g) * 4;
        const float b0 = ld_act(b, k0), b1 = ld_act(b, k0 + 1), b2 = ld_act(b, k0 + 2), b3 = ld_act(b, k0 + 3);
        const float ts = lut_ts(lut_scale(__int_as_float(smax[g / gpa])));
        float od[8], lut[16];
        lut_odd_entries(b0, b1, b2, b3, od);
#pragma unroll
        for (int e = 0; e < 16; e += 2) { lut[e + 1] = od[e / 2]; lut[e] = -od[(15 - e) / 2]; }
        l0[g] = lut[0];
        uint32_t packed[4];
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            uint32_t acc = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) acc |= (uint32_t)(lut_q8(lut[4 * w + e], ts) & 0xff) << (8 * e);
            packed[w] = acc;
        }
        reinterpret_cast<uint4 *>(qlut + (size_t)n * K * 4)[g_begin + g] = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    }
    __syncthreads();
    // biases: per 32-activation block the _mm256_addv_ps tree (:24-31), then a serial sum over
    // the blocks of the act group (:157), starting from 0.
    for (int bi = tid; bi < ng / 8; bi += kPreThreads) {
        const float *v = l0 + bi * 8;
        const float r0 = __fadd_rn(v[4], v[0]), r1 = __fadd_rn(v[5], v[1]);
        const float r2 = __fadd_rn(v[6], v[2]), r3 = __fadd_rn(v[7], v[3]);
        blk[bi] = __fadd_rn(__fadd_rn(r0, r2), __fadd_rn(r1, r3));
    }
    __syncthreads();
    const int bpa = ags / 32;                              // blocks per act group
    for (int a = tid; a < a_end - a_begin; a += kPreThreads) {
        float bias = 0.0f;
        for (int k = 0; k < bpa; ++k) bias = __fadd_rn(bias, blk[a * bpa + k]);
        lut_biases[(size_t)n * nag + a_begin + a] = bias;
        lut_scales[(size_t)n * nag + a_begin + a] = lut_scale(__int_as_float(smax[a]));
    }
}


// ------------------------------------------------------------------------------------------
// peer_barrier_kernel: "every rank's launches before this point have completed" as a stream-ordered fact on every rank,
// without a collective library call.  flags[0..world) are written by the peers (slot q by rank q), flags[world] is this
// rank's own barrier count.  One block; thread q handles peer q.  Stores issued by EARLIER kernels of this stream
// (e.g. the GEMV epilogues' peer stores) are complete when this kernel starts, so publishing the count after them
// orders them before any peer's wake-up.  Bounded wait; *err != 0 if a peer never arrived.
// ------------------------------------------------------------------------------------------
static __global__ void peer_barrier_kernel(unsigned *flags, unsigned *const *peer_flags, int rank, int world, int *err) {
    __shared__ unsigned s_epoch;
    if (threadIdx.x == 0) { s_epoch = flags[world] + 1u; flags[world] = s_epoch; }
    __syncthreads();
    const unsigned epoch = s_epoch;
    const int q = threadIdx.x;
    if (q >= world || q == rank) return;
    __threadfence_system();
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(peer_flags[q] + rank), "r"(epoch) : "memory");
    unsigned v;
    int spins = 0;
    do {
        asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + q) : "memory");
    } while ((int)(v - epoch) < 0 && ++spins < (1 << 22));
    if ((int)(v - epoch) < 0) atomicExch(err, 1);
    __threadfence_system();
}

}  // namespace tmac_b200
