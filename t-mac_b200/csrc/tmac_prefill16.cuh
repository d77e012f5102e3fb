// tmac_prefill16.cuh -- the prefill tile of the fp path (N >= 64): both scales folded into fp16 operands, fp32 accumulation over the
// whole K in registers (wgmma), stream-K over the SMs when there are fewer tiles than SMs.
//
//   C[m][n] = sum_{g,e} (0.5*scale[m][wg(g)] * S[m][g][e]) * (lut_scale[n][ag(g)] * T8[n][g][e])            (main term)
//           + sum_wg (0.5*scale[m][wg] + zero[m][wg]) * LB[n][wg],  LB[n][wg] = sum_{ag in chunk wg} lut_bias[n][ag]   (bias term)
//
// The int8 tile (tmac_prefill.cuh) keeps the reference's integer sums exact but has to rescale the accumulator after every
// activation group.  Here both factors ride in the operands: A = fp16(0.5*s*S) is expanded by the producers from the packed
// codes, B = fp16(ls*T8) is laid out once per call by lut_tile16_kernel, the accumulator stays in registers for the whole K and
// is read once.  The bias term is one more contraction step with exact operands: A columns (0.5s, 0.5s, z, z) against B columns
// (LBhi, LBlo, LBhi, LBlo), LB split into two fp16 so that their sum carries 22 bits.  Operand rounding (2^-11 per B entry)
// keeps the result inside north_star's 1e-3 of the CPU kernel (tools/sim_fp16_prefill.py: 1.4e-4 W2, 2.2-2.7e-4 W3/W4) -- NOT inside
// the 2e-5 the exact paths hold, so this tile has its own tolerance and never serves the int32 (BitNet) path.
//
// Tile: 128 weight rows x 256 tokens per CTA, wgmma.mma_async m64n256k16.f32.f16.f16, 8 MMAs per warpgroup per 64-K step.
//   warpgroups 0, 1 : consumers (rows 64*wg .. 64*wg+63, 128 fp32 accumulators per thread), then the epilogue.
//   warpgroup  2    : producers (thread = weight row, the step's 16 K-groups): plane codes -> 8 fp16 entries fp16(k * hs), hs of the
//                     group's own chunk, one 16-byte store per group into the K-major canonical A tile; thread 0 also issues the
//                     step's 64 KB B tile as one bulk copy (TMA).
// Supported: W2 (PB 2) and W3/W4 (PB 4: a 128-row tile is two 64-row super-blocks), K % 128 == 0, the int8 tile's fp-path
// groupings (chunk ck = 128, 64 or 32 K: QCH 8, 4, 2; act group ags = 128, 64 or 32 K <= ck: AGQ 8, 4, 2), per-row scales
// (+ zero points), symmetric LUT; routed instantiations of their own (ONE) also one-scale tensors at K % 128 == 0 (blocks without
// scales, hs = fp16(0.5 * scale0), no zero point; tmac_prefill.cuh).  The producers take their row, 128-K window staging, code decode, PB 4 table, grouping constants
// and scale offset from the int8 tile's shared code (tmac_prefill.cuh: PF_PRODUCER_ROW, PF_STAGE_BLOCKS, row_codes, pf_build_xtab,
// PfGroups, pf_scale_off); the expansion into fp16 A entries is this tile's own.  Each stream-K fragment is staged as one run.
#pragma once
#include "tmac_prefill.cuh"

namespace tmac_b200 {

constexpr int kP16NT = 256;                          // tokens per CTA (MMA N)
constexpr int kP16ABytes = 128 * 128 * 2;            // A tile: 128 rows x 128 contraction entries, fp16
constexpr int kP16BBytes = kP16NT * 128 * 2;         // B tile: 256 tokens x 128 entries, fp16 = one record
constexpr int kP16SubA = kP16ABytes, kP16SubB = kP16BBytes;   // the pipeline moves whole steps: 16 K-groups = 8 MMAs
constexpr int kP16NA = 2, kP16NB = 2;                // ring depth: one stage = A tile + B tile (2 x 96 KB)
constexpr int kP16ConsWarps = 8, kP16ProdWarps = 4;
constexpr int kP16Threads = (kP16ConsWarps + kP16ProdWarps) * 32;

struct Prefill16Params {
    const unsigned char *W;
    void *C;
    int N, K, Mout, ldc, out_f16;
    int nchunk, zp, sd, blk_bytes;
    int nmain, nextra;                               // 64-K steps, bias steps (128 columns = 32 weight groups each)
    size_t rsb_stride;
    const unsigned char *tiles;                      // lut_tile16_kernel output: [token tile][nmain + nextra][kP16BBytes]
    int nrsb, ntiles, streamk;                       // row super-blocks, tiles = nrt * token tiles, stream-K split (see the kernel)
    int nrt, bits;                                   // row tiles of 128 rows (PB 2: nrsb, PB 4: ceil(nrsb / 2)), bit width
    float *scratch;                                  // [2][grid][256 tokens][128 rows] fp32 partial tiles (stream-K): published parts, finishers' own parts
    int *flags;                                      // [grid] partial tile ready
    float scale0;                                    // ROUTE, sd == 0: the one-scale tensor's weight scale
};

#define WG_D128(T, d) WG_D64(T, d), WG_D8(T, d, 64), WG_D8(T, d, 72), WG_D8(T, d, 80), WG_D8(T, d, 88), WG_D8(T, d, 96), WG_D8(T, d, 104), \
                      WG_D8(T, d, 112), WG_D8(T, d, 120)
// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, f16 x f16 -> f32, both operands K-major; acc == 0 overwrites D
__device__ __forceinline__ void wg_mma_f16_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}"
                 ", %128, %129, p, 1, 1, 0, 0;\n\t}\n"
                 : WG_D128(WG_FW, d)
                 : "l"(da), "l"(db), "r"(acc));
}

// B tiles.  grid = (nmain + nextra, token tiles of 256), block = 256 (thread = token).
//   step < nmain : entries (lut_scale[n][ag(16*step + g)] * T8[n][16*step + g][e]) as fp16, token t, group g at
//                  ((g*32 + t/8)*128 + (t%8)*16), ag(g) = the activation group of K-group g
//   bias steps   : column 4*wg + {0,1,2,3} = {LBhi, LBlo, LBhi, LBlo}, LB = the sum of lut_bias[n][ag] over the activation groups
//                  ag of chunk wg in order (ck 128, ags 64: lut_bias[n][2wg] + lut_bias[n][2wg+1]); 8 columns per chunk
// Record `tile` of B tiles [tile][nmain + nextra]: token row n (live: the token exists, else zero) at position t, the body of both
// B-tile kernels.
template <int QCH, int AGQ>
__device__ __forceinline__ void lut_tile16_rec(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int tile, int n, bool live,
                                               int K, int nmain, int nextra, int step, int t) {
    using G = PfGroups<QCH, AGQ>;
    const int nag = K / (16 * AGQ), nwg = K / (16 * QCH);
    unsigned char *rec = out + ((size_t)tile * (nmain + nextra) + step) * kP16BBytes;
    if (step < nmain) {
        float ll[G::NLS];                            // the LUT scales of the step's activation groups
#pragma unroll
        for (int i = 0; i < G::NLS; ++i) ll[i] = live ? ls[(size_t)n * nag + step * 4 / AGQ + i] : 0.f;
        const uint2 *src = reinterpret_cast<const uint2 *>(qlut) + ((size_t)n * (K / 4) + (size_t)step * 16) * 2;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
            const float l = ll[g * G::NLS / 16];
            uint2 q = make_uint2(0, 0);
            if (live) q = __ldg(src + g * 2);        // the 8 stored entries of the group
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t word = k < 2 ? q.x : q.y;
                const float a = (float)(int)(int8_t)((word >> (16 * (k & 1))) & 0xff) * l;
                const float b = (float)(int)(int8_t)((word >> (16 * (k & 1) + 8)) & 0xff) * l;
                const __half2 h = __floats2half2_rn(a, b);
                o[k] = *reinterpret_cast<const uint32_t *>(&h);
            }
            *reinterpret_cast<uint4 *>(rec + ((size_t)(g * 32 + (t >> 3)) * 128 + (t & 7) * 16)) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    } else {
        const int e = step - nmain;                  // bias step: weight groups 32e .. 32e+31, two per 16-byte chunk
#pragma unroll
        for (int kc = 0; kc < 16; ++kc) {
            uint32_t o[4];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int wg = e * 32 + kc * 2 + u;
                float LB = 0.f;
                if (live && wg < nwg) {
                    LB = lb[(size_t)n * nag + G::APC * wg];
#pragma unroll
                    for (int a = 1; a < G::APC; ++a) LB += lb[(size_t)n * nag + G::APC * wg + a];
                }
                const __half hi = __float2half_rn(LB);
                const __half lo = __float2half_rn(LB - __half2float(hi));
                const __half2 h = __halves2half2(hi, lo);
                o[2 * u] = o[2 * u + 1] = *reinterpret_cast<const uint32_t *>(&h);
            }
            *reinterpret_cast<uint4 *>(rec + ((size_t)(kc * 32 + (t >> 3)) * 128 + (t & 7) * 16)) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}
template <int QCH = 8, int AGQ = 4>
__global__ void __launch_bounds__(256) lut_tile16_kernel(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int N, int K,
                                                         int nmain, int nextra) {
    const int step = blockIdx.x, tile = blockIdx.y, t = threadIdx.x, n = tile * kP16NT + t;
    lut_tile16_rec<QCH, AGQ>(qlut, ls, lb, out, tile, n, n < N, K, nmain, nextra, step, t);
}
// grid = (nmain + nextra, table entries): the B tiles of the routed fp16 tile, [entry][step], token position t = perm position
// start + t of the entry (PfRoute, lut_tile_gather_kernel); an unused entry's tiles are not written.
template <int QCH, int AGQ>
__global__ void __launch_bounds__(256) lut_tile16_gather_kernel(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int K,
                                                                int nmain, int nextra, const int4 *tiles, const int *perm, int div) {
    const int step = blockIdx.x, k = blockIdx.y, t = threadIdx.x;
    const int4 e = __ldg(tiles + k);
    if (e.z == 0) return;
    const bool live = t < e.z;
    const int n = live ? __ldg(perm + e.y + t) / div : 0;
    lut_tile16_rec<QCH, AGQ>(qlut, ls, lb, out, k, n, live, K, nmain, nextra, step, t);
}

// One CTA walks a contiguous run [L0, L1) of the linear (tile, step) sequence -- tile = (row super-block, token tile), nsteps
// contraction steps per tile.  streamk == 0: L0 = cta * nsteps, one whole tile per CTA (grid = tiles).  streamk == 1: grid = SMs,
// [L0, L1) = [S*cta/G, S*(cta+1)/G): at most the tail of one tile and the head of the next.  A tile cut
// by CTA boundaries is finished by the CTA that holds its LAST step, the others store their fp32 partial tile to `scratch[cta]` and
// raise `flags[cta]`; the finisher adds the partials in ascending K order (deterministic), stores C and clears the flags.  The
// accumulator lives in registers, so a CTA computes its fragments one after the other, the head of the next tile first: no CTA
// waits for a partial before publishing its own.
//
// Pipeline.  One 2-deep ring; a stage holds the A tile (producers) and the B tile (TMA) of one step, released by the consumers once
// the step's MMAs have completed.
//
// Row tile = 128 rows.  PB 2 (W2): one super-block.  PB 4 (W3/W4): super-blocks 2*rt and 2*rt + 1 (64 rows each), producer
// threads 0..63 / 64..127 and consumer warpgroups 0 / 1; when nrsb is odd the last tile's second super-block does not exist and
// its A rows are zero.
//
// ROUTE (routed experts and the dense prefill_* forms, prefill16_experts_kernel): grid = (row tiles, table entries, count), no
// stream-K.  As in the int8 tile (prefill_body): the CTA of entry k = blockIdx.y and tensor i = blockIdx.z exits at once when the
// entry is unused, else runs tile k * nrt + blockIdx.x on the weights W[i * n_experts + expert], the B tiles of entry k, and stores
// token t's row at row perm[start + t] of C[i * n_experts + expert], plus the residual route.R when there is one.  ONE (ROUTE, QCH 8): a
// one-scale tensor, whose blocks carry no scales: hs = fp16(0.5 * scale0), no zero point.  A template parameter rather than a test of
// p.sd: the run-time test made the producers of the per-row-scale instantiations slower.  BIAS (ROUTE, prefill16_bias_kernel): no
// residual; each output takes route.bias's row (PfBias).
template <int PB, int QCH, int AGQ, bool ROUTE, bool ONE = false, bool BIAS = false>
__device__ __forceinline__ void prefill16_body(const Prefill16Params &p, const PfRoute &route) {
    static_assert(PB == 2 || PB == 4, "prefill tile: W2 or W3/W4 stream layout");
    static_assert(!ONE || (ROUTE && QCH == 8), "one-scale tensors: routed, 128-K chunks");
    static_assert(!BIAS || ROUTE, "biases: routed tiles only");
    using PG = PfGroups<QCH, AGQ>;
    constexpr int RSB = 32 * (8 / PB);                                     // rows per super-block
    constexpr int NSB = 128 / RSB;                                         // super-blocks per row tile
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *sA = smem;                                              // [NA][32 KB]
    unsigned char *sB = sA + kP16NA * kP16SubA;                            // [NB][64 KB]
    unsigned char *raw = sB + kP16NB * kP16SubB;                           // [2][NSB][WB * blk] packed 128-K windows (codes + scales)
    const int rawsz = (PG::WB * p.blk_bytes + 127) & ~127;
    uint64_t *xtab = reinterpret_cast<uint64_t *>(raw + 2 * NSB * rawsz);  // PB 4: [512] expansion table (pf_build_xtab, biased)
    uint64_t *bars = xtab + (PB == 4 ? 512 : 0);
    uint64_t *full = bars, *empty = full + kP16NA;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nsteps = p.nmain + p.nextra;
    int4 ent = make_int4(0, 0, 0, 0);                                      // ROUTE: {expert, start, ntok, 0} of the CTA's entry
    if constexpr (ROUTE) {
        ent = __ldg(route.tiles + blockIdx.y);
        if (ent.z == 0) return;
    }
    const int G = gridDim.x, cta = ROUTE ? blockIdx.y * p.nrt + blockIdx.x : blockIdx.x;
    const unsigned char *W = ROUTE ? route.W[blockIdx.z * route.n_experts + ent.x] : p.W;
    const long long Stot = (long long)p.ntiles * nsteps;
    const int L0 = p.streamk ? (int)(Stot * cta / G) : cta * nsteps, L1 = p.streamk ? (int)(Stot * (cta + 1) / G) : (cta + 1) * nsteps;
    // fragments: f = 0 -> [L0, min(L1, end of L0's tile)), f = 1 -> the rest (head of the next tile)
    int ft[2], fs0[2], fs1[2], nfrag = 0;
    for (int L = L0; L < L1 && nfrag < 2;) {
        const int t = L / nsteps, s0 = L - t * nsteps, s1 = min(nsteps, s0 + (L1 - L));
        ft[nfrag] = t; fs0[nfrag] = s0; fs1[nfrag] = s1; ++nfrag;
        L += s1 - s0;
    }
    if (nfrag == 2) {                                // computed in the order (1, 0): keep the arrays in registers, index 0 = first
        int x = ft[0]; ft[0] = ft[1]; ft[1] = x;
        x = fs0[0]; fs0[0] = fs0[1]; fs0[1] = x;
        x = fs1[0]; fs1[0] = fs1[1]; fs1[1] = x;
    }

    if constexpr (PB == 4) pf_build_xtab<4>(xtab, p.bits, true, tid, kP16Threads);
    if (tid == 0) {
        for (int i = 0; i < kP16NA; ++i) { mbar_init(full + i, kP16ProdWarps + 1); mbar_init(empty + i, kP16ConsWarps); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp >= kP16ConsWarps) {
        // ======================= producers: thread = weight row, all 16 K-groups of the step =======================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");           // registers go to the consumers' accumulators
        PF_PRODUCER_ROW(PB, tid - kP16ConsWarps * 32);
        const int srow = wl * (8 / PB) + wi;         // row within the super-block = scale index
        constexpr bool one = ONE;                    // a one-scale tensor: scale0, nothing read at pf_scale_off
        int it = 0;                                  // running step counter over both fragments
        auto stage_in = [&](int f, int u) {          // wait for a free stage, request its B tile; returns the A tile
            const int s = it % kP16NA;
            mbar_wait_parity(empty + s, ((it / kP16NA) & 1) ^ 1);   // the MMAs that read this stage have completed
            if (r == 0) {
                bulk_load(sB + (size_t)s * kP16SubB, p.tiles + ((size_t)(ft[f] / p.nrt) * nsteps + u) * kP16BBytes, kP16SubB, full + s);
            }
            return sA + (size_t)s * kP16SubA;
        };
        auto stage_out = [&]() {
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(full + it % kP16NA);
            __syncwarp();
            ++it;
        };
#pragma unroll
        for (int f = 0; f < 2; ++f) {
            if (f == nfrag) break;
            const int rt = ft[f] % p.nrt;
            const unsigned char *rsb_base = W + (size_t)rt * NSB * p.rsb_stride;     // first super-block of the row tile
            const bool live = PB == 2 || rt * NSB + sb < p.nrsb;
            const unsigned char *sb_base = rsb_base + (size_t)sb * p.rsb_stride;
            const int s0 = fs0[f], s1m = min(fs1[f], p.nmain);
            if (s0 < s1m) {
                const int c_first = s0 >> 1, c_last = (s1m - 1) >> 1;
                asm volatile("bar.sync 1, 128;" ::: "memory");             // the previous fragment's last block is dead
                PF_STAGE_BLOCKS(PB, PG::WB, c, blk, c_first, c_last, {
                    const uint32_t *words = reinterpret_cast<const uint32_t *>(blk);
                    // hs = fp16(0.5 * scale) of block b's chunk.  PB 2: the row's 8 A entries of one K-group are +-hs at entry j0
                    // (plane 0) plus +-2hs at entry j1 (plane 1), built in registers: (+-hs) + (+-2hs) is one fp16 rounding of the
                    // exact k * hs.  A step holds the groups of NCS chunks: their hs, c1 = hs, c2 = 2hs (ck 128: once per window).
                    auto hs_of = [&](int b) {
                        return __float2half_rn(live ? 0.5f * (one ? p.scale0 : load_scale(blk + (size_t)b * p.blk_bytes + pf_scale_off(QCH), p.sd, srow)) : 0.f);
                    };
                    __half hsv[PG::NCS];
                    uint32_t c1[PG::NCS], c2[PG::NCS];
                    if constexpr (QCH == 8) {
                        hsv[0] = hs_of(0);
                        c1[0] = __half_as_ushort(hsv[0]); c2[0] = __half_as_ushort(__hadd(hsv[0], hsv[0]));
                    }
                    const int u0 = (c == c_first) ? (s0 & 1) : 0, u1 = (c == c_last) ? ((s1m - 1) & 1) : 1;   // steps of this window
                    _Pragma("unroll 1") for (int u = u0; u <= u1; ++u) {
                        if constexpr (QCH != 8) {
                            _Pragma("unroll") for (int i = 0; i < PG::NCS; ++i) {
                                hsv[i] = hs_of(u * PG::NCS + i);
                                c1[i] = __half_as_ushort(hsv[i]); c2[i] = __half_as_ushort(__hadd(hsv[i], hsv[i]));
                            }
                        }
                        unsigned char *a_dst = stage_in(f, 2 * c + u);
                        _Pragma("unroll") for (int gl = 0; gl < 16; ++gl) {    // group within the step = 16-byte chunk index
                            const int gqc = u * 16 + gl;                       // group within the window (0..31)
                            // its block in the window (= its chunk in the step: ci) and its quad / word there
                            const int ci = gl * PG::NCS / 16, b = PG::WB == 1 ? 0 : gqc / (4 * QCH), gb = PG::WB == 1 ? gqc : gqc % (4 * QCH);
                            const int q = gb >> 2, k = gb & 3;
                            const uint32_t cw = row_codes<PB>(words + (size_t)b * (p.blk_bytes >> 2) + ((size_t)q * 32 + wl) * 4, k, wi);
                            uint32_t o4[4];
                            if constexpr (PB == 2) {
                                // cw = j0 | neg0 << 3 | j1 << 4 | neg1 << 7
                                const uint32_t v0 = (c1[ci] ^ ((cw & 8u) << 12)) << ((cw & 1u) * 16), v1 = (c2[ci] ^ ((cw & 0x80u) << 8)) << (((cw >> 4) & 1u) * 16);
                                _Pragma("unroll") for (int e = 0; e < 4; ++e) {
                                    const uint32_t a = (cw & 6u) == 2u * e ? v0 : 0u, b = (cw & 0x60u) == 32u * e ? v1 : 0u;
                                    const __half2 x = __hadd2(*reinterpret_cast<const __half2 *>(&a), *reinterpret_cast<const __half2 *>(&b));
                                    o4[e] = *reinterpret_cast<const uint32_t *>(&x);
                                }
                            } else {
                                // PB 4: the integer k = S[e] (|S| <= 15) of the row's four planes from the two biased table halves: the plain
                                // 32-bit add holds k + 16 in [1, 31] per byte.  fp16 bits 0x6400 | m are 1024 + m, minus 1040 is
                                // k exactly; k and hs are exact fp16 values, so the HMUL2 rounds the exact product k * hs once.
                                const uint64_t lo = xtab[cw & 0xffu], hi = xtab[256 + (cw >> 8)];
                                const uint32_t sk[2] = {(uint32_t)lo + (uint32_t)hi, (uint32_t)(lo >> 32) + (uint32_t)(hi >> 32)};
                                const __half2 hs2 = __halves2half2(hsv[ci], hsv[ci]), off = __float2half2_rn(1040.f);
                                _Pragma("unroll") for (int e = 0; e < 4; ++e) {
                                    const uint32_t m = __byte_perm(sk[e >> 1], 0x64u, (e & 1) ? 0x4342u : 0x4140u);   // entries 2e, 2e + 1
                                    const __half2 kk = __hsub2(*reinterpret_cast<const __half2 *>(&m), off);
                                    const __half2 x = __hmul2(kk, hs2);
                                    o4[e] = *reinterpret_cast<const uint32_t *>(&x);
                                }
                            }
                            *reinterpret_cast<uint4 *>(a_dst + ((size_t)(gl * 16 + (r >> 3)) * 128 + (r & 7) * 16)) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
                        }
                        stage_out();
                    }
                });
            }
            // bias steps: A columns 4*wg + {0,1,2,3} = {0.5s, 0.5s, z, z} of weight group wg (= chunk index), 2 groups per 16-byte chunk
            for (int step = max(fs0[f], p.nmain); step < fs1[f]; ++step) {
                const int e = step - p.nmain;
                unsigned char *a_dst = stage_in(f, step);
#pragma unroll 4
                for (int kc = 0; kc < 16; ++kc) {
                    uint32_t o[4];
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int wg = e * 32 + kc * 2 + u;
                        float hs = 0.f, zz = 0.f;
                        if (live && wg < p.nchunk) {
                            const unsigned char *sp = sb_base + (size_t)wg * p.blk_bytes + pf_scale_off(QCH);
                            hs = 0.5f * (one ? p.scale0 : load_scale(sp, p.sd, srow));
                            if (p.zp) zz = load_scale(sp + (size_t)RSB * p.sd, p.sd, srow);
                        }
                        const __half2 a = __floats2half2_rn(hs, hs), b = __floats2half2_rn(zz, zz);
                        o[2 * u] = *reinterpret_cast<const uint32_t *>(&a); o[2 * u + 1] = *reinterpret_cast<const uint32_t *>(&b);
                    }
                    *reinterpret_cast<uint4 *>(a_dst + ((size_t)(kc * 16 + (r >> 3)) * 128 + (r & 7) * 16)) = make_uint4(o[0], o[1], o[2], o[3]);
                }
                stage_out();
            }
        }
    } else {
        // ======================= consumers: MMAs, then the epilogue of each fragment =======================
        // register j = 4*c8 + 2*h + e holds row 64*wg + 16*(warp%4) + lane/4 + 8*h, token 8*c8 + 2*(lane%4) + e
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");          // 2 x 128 x 224 + 128 x 56 = the 384 x 168 of the launch
        const int wg = warp >> 2;
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), tc = 2 * (lane & 3);
        float acc[128];
        int it = 0;
#pragma unroll
        for (int f = 0; f < 2; ++f) {
            if (f == nfrag) break;
            for (int u = fs0[f]; u < fs1[f]; ++u, ++it) {
                const int s = it % kP16NA;
                mbar_wait_parity(full + s, (it / kP16NA) & 1);
                const uint32_t a0 = smem_u32(sA + (size_t)s * kP16SubA) + wg * 1024, b0 = smem_u32(sB + (size_t)s * kP16SubB);
                wg_fence();
#pragma unroll
                for (int i = 0; i < 8; ++i)         // K = 16 entries = two 16-byte chunks per MMA
                    wg_mma_f16_n256(acc, wg_desc(a0 + i * 2 * 2048, 2048), wg_desc(b0 + i * 2 * 4096, 4096), (u > fs0[f] || i > 0) ? 1u : 0u);
                wg_commit();
                wg_wait0();
                wg_fence_acc(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty + s);              // both tiles of the stage are free
                __syncwarp();
            }
            if constexpr (ROUTE) {                   // one whole tile per CTA
                void *const Cr = route.C[blockIdx.z * route.n_experts + ent.x];
                const int row0 = (int)blockIdx.x * 128 + r0;
                const auto stores = [&](auto res) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = row0 + 8 * h;
#pragma unroll
                        for (int c8 = 0; c8 < 32; ++c8)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int t = 8 * c8 + tc + e;
                                if (t < ent.z && row < p.Mout)
                                    pf_route_store<decltype(res)::value>(route, Cr, (size_t)__ldg(route.perm + ent.y + t) * p.ldc + row,
                                                                         pf_bias_add(res, row, acc[4 * c8 + 2 * h + e]), p.out_f16);
                            }
                    }
                };
                if constexpr (BIAS) stores(PfBias{route.bias[blockIdx.z * route.n_experts + ent.x]});
                else if (route.R) stores(PfRes<true>{});
                else stores(PfRes<false>{});
                continue;
            }
            const bool whole = fs0[f] == 0 && fs1[f] == nsteps, last = fs1[f] == nsteps;
            const int rt = ft[f] % p.nrt, tile = ft[f] / p.nrt, n0 = tile * kP16NT, ntok = min(kP16NT, p.N - n0);
            if (whole) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = rt * 128 + r0 + 8 * h;
#pragma unroll
                    for (int c8 = 0; c8 < 32; ++c8)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int t = 8 * c8 + tc + e;
                            if (t < ntok && row < p.Mout) store_out(p.C, (size_t)(n0 + t) * p.ldc + row, acc[4 * c8 + 2 * h + e], p.out_f16);
                        }
                }
                continue;
            }
            // a tile cut between CTAs: this CTA's part -> scratch[0][cta][t][row] (published), scratch[1][cta][t][row] (finisher)
            float *mine = p.scratch + (size_t)(last ? G + cta : cta) * kP16NT * 128;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c8 = 0; c8 < 32; ++c8)
#pragma unroll
                    for (int e = 0; e < 2; ++e) mine[(size_t)(8 * c8 + tc + e) * 128 + r0 + 8 * h] = acc[4 * c8 + 2 * h + e];
            if (!last) {                             // publish: every thread's stores, then the flag
                __threadfence();
                asm volatile("bar.sync 2, 256;" ::: "memory");
                if (tid == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p.flags + cta), "r"(1) : "memory");
                continue;
            }
            // the finisher: wait for the CTAs that hold steps [0, s0) of this tile, add the parts in ascending K order
            // (deterministic; this CTA's part last), store C, clear the flags for the next launch
            const long long lin0 = (long long)ft[f] * nsteps;
            int c_first = (int)(lin0 * G / Stot);
            while ((int)(Stot * (c_first + 1) / G) <= lin0) ++c_first;
            while ((int)(Stot * c_first / G) > lin0) --c_first;
            if (tid == 0)
                for (int c2 = c_first; c2 < cta; ++c2) {
                    int v, spins = 0;
                    do { asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p.flags + c2) : "memory"); } while (v == 0 && ++spins < (1 << 24));
                }
            asm volatile("bar.sync 2, 256;" ::: "memory");
            for (int i = tid; i < ntok * 128; i += kP16ConsWarps * 32) {
                const int t = i >> 7, er = i & 127, row = rt * 128 + er;
                float sum = 0.f;
                for (int c2 = c_first; c2 < cta; ++c2) sum += __ldcg(p.scratch + ((size_t)c2 * kP16NT + t) * 128 + er);
                sum += __ldcg(mine + (size_t)t * 128 + er);
                if (row < p.Mout) store_out(p.C, (size_t)(n0 + t) * p.ldc + row, sum, p.out_f16);
            }
            asm volatile("bar.sync 2, 256;" ::: "memory");                 // all partial reads done: the flags can be reused by the next launch
            if (tid == 0) for (int c2 = c_first; c2 < cta; ++c2) asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p.flags + c2), "r"(0) : "memory");
        }
    }
}
template <int PB, int QCH = 8, int AGQ = 4>
__global__ void __launch_bounds__(kP16Threads, 1) prefill16_kernel(const Prefill16Params p) {
    prefill16_body<PB, QCH, AGQ, false>(p, PfRoute{});
}
template <int PB, int QCH, int AGQ, bool ONE = false>
__global__ void __launch_bounds__(kP16Threads, 1) prefill16_experts_kernel(const Prefill16Params p, const PfRoute route) {
    prefill16_body<PB, QCH, AGQ, true, ONE>(p, route);
}
// prefill16_experts_kernel with a bias on every output (tmac_b200_prefill_rmsnorm_bias), as prefill_bias_kernel
template <int PB, int QCH, int AGQ, bool ONE = false>
__global__ void __launch_bounds__(kP16Threads, 1) prefill16_bias_kernel(const Prefill16Params p, const PfRoute route) {
    prefill16_body<PB, QCH, AGQ, true, ONE, true>(p, route);
}

// The routed launches (tmac_b200_prefill_experts / _glu, and the dense tmac_b200_prefill_rmsnorm / _glu / _residual as one expert):
// the kernels of one tensor kind (PB) and fp grouping, instantiated in tmac_prefill_experts.cu (one: a one-scale tensor, whose fp16
// tile is its own instantiation; unit1: the int8 tile alone, staging one 64-K chunk per unit, for one-scale tensors with K % 128 == 64).  route sorts the slots by expert
// (or writes the identity routing) and the tile table; swiglu (or relu2) and rmsnorm materialise the GLU and norm inputs; combine adds the
// GLU experts' slot rows.
struct PfExpertKernels {
    void (*tile)(const PrefillParams, const PfRoute);
    void (*lut)(const int8_t *, const float *, const float *, unsigned char *, int, const int4 *, const int *, int);
    void (*tile16)(const Prefill16Params, const PfRoute);
    void (*lut16)(const int8_t *, const float *, const float *, unsigned char *, int, int, int, const int4 *, const int *, int);
};
// bias: the tiles are prefill_bias_kernel / prefill16_bias_kernel (tmac_b200_prefill_rmsnorm_bias)
PfExpertKernels pick_pf_experts(int pb, int qch, int agq, bool one, bool unit1, bool bias = false);
void pf_route_launch(const int32_t *ids, int S, int E, int T, int cap, int4 *tiles, int *perm, void *const *Cnan, int count, int ldc,
                     int out_f16, cudaStream_t st);
void pf_swiglu_launch(const void *G, const void *U, int f16, size_t n, float *a, cudaStream_t st, bool relu2 = false);
void pf_rmsnorm_launch(const void *H, int f16, const float *w, float eps, int N, int K, float *a, cudaStream_t st);
void pf_combine_launch(const float *ys, const int32_t *ids, const float *w, int topk, int E, const void *R, void *C, int N, int Mout,
                       int out_f16, cudaStream_t st);

}  // namespace tmac_b200
