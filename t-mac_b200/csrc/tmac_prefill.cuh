// tmac_prefill.cuh -- the N>1 (prefill) tile of qgemm_lut on the Hopper tensor cores (wgmma).
//
// Why tensor cores are legitimate here and how parity is kept (SURVEY.md section 7, hard part 1):
// the reference rounds the *group-of-4 partial sums* (the LUT entries), so a plain int8 GEMM of
// quantised activations is different arithmetic.  The contraction is therefore taken over the LUT
// itself.  With the odd symmetry LUT[15-i] = -LUT[i] (lut_ctor.cc:153-155) the 8 stored entries T8[n][g][0..7]
// of token n, K-group g are enough, and for one weight row m
//     sum_planes 2*alpha_b * sign * LUT_g[idx_b]  =  sum_{e<8} T8[n][g][e] * S[m][g][e],
//     S[m][g][e] = sum_b 2*alpha_b * sign(m,b,g) * [j(m,b,g) == e]          (int8, |S| <= 15)
// i.e. an exact dense int8 contraction of length 8 per K-group:  I[m][n] = S[m][:] . T8[n][:]  -- a true
// int8 GEMM with int32 accumulation, bit-identical to the integer sums of the GEMV path.  It runs as
// wgmma.mma_async m64n128k32.s32.s8.s8 (two consumer warpgroups = 128 weight rows, N = 128 tokens), accumulator in
// registers.  Per activation group (64 K positions = 128 contraction bytes = 4 MMAs per warpgroup) the int32 tile is
// folded into fp32 registers with lut_scale[n][ag] * 0.5*scale[m][wg]; the LUT-bias / zero-point terms are a
// rank-(K/group_size) correction added once per chunk.
//
//   warpgroups 0, 1  consumers: 4 wgmma per step on rows 64*wg .. 64*wg+63, int32 -> fp32 fold, final store.
//   warpgroup  2     producers: cp.async the (row super-block, chunk) block(s), expand the packed codes of "their"
//                    weight row into S (one 64-bit one-hot-signed vector per (row, group), through a 256-entry (W2) or
//                    512-entry (W3/W4: two planes per lookup, two lookups added byte-wise) shared-memory table) in the
//                    K-major no-swizzle canonical layout; fence.proxy.async; arrive full[s].  Thread 0 also issues the
//                    step's LUT record as one bulk copy (TMA) into the same stage.
//
// Shared with the fp16 tile (tmac_prefill16.cuh): the producer's row (PF_PRODUCER_ROW), the double-buffered block staging
// (PF_STAGE_BLOCKS), the code decode (row_codes, tmac_kernels.cuh), the expansion table (pf_build_xtab) and the scale offset
// in a block (kPfScaleOff).  Each tile keeps its own expansion of a chunk's codes into A entries.
//
// Integer path (INT_PATH, BitNet: one weight scale, one activation group per row): the int32 accumulator sums over the whole K
// with no fold, and one epilogue per output applies the token's LUT scale and bias and the tensor's scale in the GEMV's order
// (int_path_out).  The int32 sum is the GEMV's integer (|S| <= 15, |T8| <= 127: no overflow at any K a row can have), converted to
// fp32 the same way, so the output is bit-identical to the GEMV and to the reference.  Its LUT records are the table entries only.
//
// Supported: PB == 2 (W2: a 128-row tile is one super-block) and PB == 4 (W3/W4: two 64-row super-blocks, one per consumer
// warpgroup), with a symmetric LUT and either
//   fp path: chunk = 128 K (QCH 8), act group 64 (AGQ 4), per-row scales (+ zero points), or
//   integer path: one scale, act group = K, chunk = 128 K (QCH 8) or 64 K (QCH 4).
// Everything else takes the GEMV kernel once per activation row.
#pragma once
#include "tmac_kernels.cuh"

namespace tmac_b200 {

struct PrefillParams {
    const unsigned char *W;        // stream layout of the tensor (first super-block)
    const int8_t *qlut;            // [N][K/4][16]
    const float *lut_scales, *lut_biases;   // [N][K/64]; integer path: [N][1]
    void *C;                       // [N][ldc]
    int N, K, Mout, ldc, out_f16;
    int nchunk, zp, sd, blk_bytes;
    size_t rsb_stride;
    const unsigned char *lut_tiles; // output of lut_tile_kernel: [token tile][step][kPfRec]
    long long *dbg;                // optional trace [role][step][4] (TMAC_ENABLE_TRACE builds)
    int nrsb, bits;                // row super-blocks of the tensor (PB 4: the last row tile may hold only one), bit width
    int qch;                       // quads of 16 K per chunk: 8, or 4 (integer path only)
    float scale0;                  // integer path: the tensor's one weight scale
};
#ifdef TMAC_ENABLE_TRACE
#define PF_TRACE(role, step, k) do { if (p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && (step) < 32) p.dbg[((role) * 32 + (step)) * 4 + (k)] = clock64(); } while (0)
#else
#define PF_TRACE(role, step, k) do { } while (0)
#endif

constexpr int kPfNT = 128;                       // tokens per CTA pass (MMA N)
constexpr int kPfStageBytes = 128 * 128;         // one operand tile: 128 rows x 128 contraction bytes

// wgmma shared-memory descriptor, K-major, no swizzle: core matrix = 8 rows x 16 B (128 B) at (kc*G + rn)*128 for K chunk kc,
// row group rn (G row groups per chunk); leading byte offset = distance between K chunks (G*128), stride byte offset = 128.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo) {
    uint64_t d = (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(128u >> 4) << 32;
    return d;                                    // bits 62-63 = 0: no swizzle
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// after wg_wait0: the accumulator registers are defined here, not at the wgmma that named them
template <int R> __device__ __forceinline__ void wg_fence_acc(uint32_t (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
template <int R> __device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
#define WG_D8(T, d, b) T(d[b]), T(d[b + 1]), T(d[b + 2]), T(d[b + 3]), T(d[b + 4]), T(d[b + 5]), T(d[b + 6]), T(d[b + 7])
#define WG_D64(T, d) WG_D8(T, d, 0), WG_D8(T, d, 8), WG_D8(T, d, 16), WG_D8(T, d, 24), WG_D8(T, d, 32), WG_D8(T, d, 40), WG_D8(T, d, 48), WG_D8(T, d, 56)
#define WG_RW(x) "+r"(x)
#define WG_FW(x) "+f"(x)
// D[64 x 128] (+)= A[64 x 32] . B[128 x 32]^T, s8 x s8 -> s32; acc == 0 overwrites D
__device__ __forceinline__ void wg_mma_s8_n128(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {"
                 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
                 ", %64, %65, p;\n\t}\n"
                 : WG_D64(WG_RW, d)
                 : "l"(da), "l"(db), "r"(acc));
}

// ---------------------------------------------------------------------------------------------------
// lut_tile_kernel: QLUT [N][K/4][16] + LUT_Scales/Biases [N][K/64]  ->  per (token tile of 128, activation group) one
// contiguous 17920-byte record that the GEMM stage receives with ONE bulk copy (TMA):
//     [16384 B]  the 8 stored LUT entries of the 16 groups of the step for 128 tokens, already in the K-major
//                canonical order: chunk kc (groups 2kc, 2kc+1), token t at ((kc*16 + t/8)*128 + (t%8)*16)
//     [  512 B]  lut_scale[token][step]
//     [ 1024 B]  (lut_bias[token][2c], lut_bias[token][2c+1]) of the step's chunk c = step/2
// Tokens >= N are zero.  grid = (steps, token tiles), block = 128 (thread = token).
// INT_PATH: the record is the 16384 bytes of table entries alone (the consumers read the token's one LUT scale and bias of
// [N][1] in their epilogue); ls and lb are not read.
// ---------------------------------------------------------------------------------------------------
constexpr int kPfTab = 16384;
constexpr int kPfRec = kPfTab + 512 + 1024;
__host__ __device__ constexpr int pf_rec_bytes(bool int_path) { return int_path ? kPfTab : kPfRec; }
template <bool INT_PATH>
__global__ void __launch_bounds__(128) lut_tile_kernel(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int N, int K) {
    constexpr int REC = pf_rec_bytes(INT_PATH);
    const int step = blockIdx.x, tile = blockIdx.y, t = threadIdx.x, n = tile * 128 + t;
    const int nag = K / 64;
    unsigned char *rec = out + ((size_t)tile * nag + step) * REC;
    const uint2 *src = reinterpret_cast<const uint2 *>(qlut) + ((size_t)n * (K / 4) + (size_t)step * 16) * 2;
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
        uint2 lo = make_uint2(0, 0), hi = make_uint2(0, 0);
        if (n < N) { lo = __ldg(src + kc * 4); hi = __ldg(src + kc * 4 + 2); }
        *reinterpret_cast<uint4 *>(rec + ((size_t)(kc * 16 + (t >> 3)) * 128 + (t & 7) * 16)) = make_uint4(lo.x, lo.y, hi.x, hi.y);
    }
    if constexpr (INT_PATH) return;
    float l = 0.f; float2 b2 = make_float2(0.f, 0.f);
    if (n < N) { l = ls[(size_t)n * nag + step]; b2 = make_float2(lb[(size_t)n * nag + (step & ~1)], lb[(size_t)n * nag + (step | 1)]); }
    reinterpret_cast<float *>(rec + 16384)[t] = l;
    reinterpret_cast<float2 *>(rec + 16384 + 512)[t] = b2;
}

constexpr int kPfStages = 4;                     // stages: A tile 16 KB (expanded by the producers) + record 17.5 KB (TMA)
constexpr int kPfConsWarps = 8;                  // two consumer warpgroups
constexpr int kPfProdWarps = 4;                  // one producer warpgroup
constexpr int kPfThreads2 = (kPfConsWarps + kPfProdWarps) * 32;

constexpr int kPfScaleOff = 8 * 512;            // a block's scales follow its QCH 8 quads of 512 B of codes

// Expansion table: 128*PB entries, each indexed by one byte of row_codes<PB> (two planes, nibble = neg << 3 | j),
//   [0, 256)    planes 0, 1: +-w0 at byte j0 plus +-w1 at byte j1
//   [256, 512)  PB 4 only, planes 2, 3: +-w2 at byte j2 plus +-w3 at byte j3
// w_b = 2*alpha_b from plane_weight_regs: W2 {1, 2}, W4 {1, 2, 4, 8}, W3 {1, 2, 4, 0} (its padded fourth plane is code 0 and must
// add nothing).  biased == false: signed bytes; W2: one entry is S[e], PB 4: one entry of each half added byte-wise (__vadd4) is
// S[e].  biased == true (PB 4): the bytes of the two halves carry +3 and +13 (|w0| + |w1| <= 3, |w2| + |w3| <= 12), so every byte
// is non-negative and a plain 32-bit add of one entry of each half holds S[e] + 16 in [1, 31] per byte without a carry between bytes.
template <int PB>
__device__ __forceinline__ void pf_build_xtab(uint64_t *xtab, int bits, bool biased, int tid, int nthreads) {
    uint32_t wtx, wty;
    plane_weight_regs(bits, true, &wtx, &wty);
    for (int e = tid; e < 128 * PB; e += nthreads) {
        const int h = e >> 8, wa = (int)((wtx >> (16 * h)) & 0xff), wb = (int)((wtx >> (16 * h + 8)) & 0xff);
        const int bias = biased ? (h ? 13 : 3) : 0;
        const int ja = e & 7, jb = (e >> 4) & 7, va = (e & 8) ? -wa : wa, vb = (e & 0x80) ? -wb : wb;
        uint64_t x = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) x |= (uint64_t)(uint8_t)(bias + (i == ja ? va : 0) + (i == jb ? vb : 0)) << (8 * i);
        xtab[e] = x;
    }
}

// The producer warpgroup of both tiles.  These two are macros: written as inline functions (or a struct and a template that
// takes the expansion as a lambda) the same code is ordered differently by the compiler, and the fp16 tile's consumers spill more.
//
// PF_PRODUCER_ROW declares the row of producer thread r < 128 (weight row r of the 128-row tile).  PB 2: the tile is one
// super-block, stream lane wl = r / 4, row-in-lane wi = r % 4 (RW = 4).  PB 4: super-block sb = r / 64 of the tile, lane
// wl = (r % 64) / 2, row-in-lane wi = r % 2 (RW = 2).
#define PF_PRODUCER_ROW(PB, r_)                                                                                              \
    const int r = (r_), sb = (PB) == 4 ? r >> 6 : 0, wl = (PB) == 4 ? (r & 63) >> 1 : r >> 2, wi = (PB) == 4 ? r & 1 : r & 3

// PF_STAGE_BLOCKS runs the expansion (the variadic argument) once per chunk c of [c_first, c_last], with blk = the thread's
// super-block's block of chunk c in shared memory (codes, then the scales at kPfScaleOff).  The blocks come from rsb_base (the row
// tile's first super-block) and sb_base (super-block sb) through raw, a double buffer [2][NSB][rawsz] with chunk c in half c & 1:
// cp.async fetches chunk c + 1 while chunk c is expanded.  The 128 / NSB threads of a super-block stage its blocks; a super-block
// that is not live stages nothing.  Named barrier 1 (the 128 producer threads) makes block c visible to every producer and retires
// block c - 1, whose half then takes chunk c + 1.  The block of c_last may still be read when the loop ends: a producer that stages
// another run passes barrier 1 before it.  Besides PF_PRODUCER_ROW's names it reads p, live, rsb_base, sb_base, raw, rawsz and NSB
// of the kernel.
#define PF_STAGE_BLOCKS(PB, c, blk, c_first, c_last, ...)                                                                    \
    do {                                                                                                                     \
        const int pf_c0 = (c_first), pf_c1 = (c_last), n16 = p.blk_bytes >> 4;                                             \
        auto load_blocks = [&](int c_, unsigned char *dst) {   /* chunk c_ of the tile's super-block(s) -> dst [NSB][rawsz] */ \
            if constexpr ((PB) == 2) {                                                                                       \
                for (int i = r; i < n16; i += 128) cp_async16_plain(dst + i * 16, rsb_base + (size_t)c_ * p.blk_bytes + i * 16); \
            } else if (live) {                                                                                               \
                for (int i = r & 63; i < n16; i += 64)                                                                       \
                    cp_async16_plain(dst + (size_t)sb * rawsz + i * 16, sb_base + (size_t)c_ * p.blk_bytes + i * 16);        \
            }                                                                                                                \
        };                                                                                                                   \
        load_blocks(pf_c0, raw + (size_t)(pf_c0 & 1) * NSB * rawsz);                                                        \
        cp_async_commit();                                                                                                   \
        for (int c = pf_c0; c <= pf_c1; ++c) {                                                                               \
            unsigned char *rb = raw + (size_t)(c & 1) * NSB * rawsz;                                                         \
            cp_async_wait_all();                                                                                             \
            asm volatile("bar.sync 1, 128;" ::: "memory");             /* block c visible to all producers; block c-1 dead */ \
            if (c + 1 <= pf_c1) {                                                                                            \
                load_blocks(c + 1, raw + (size_t)((c + 1) & 1) * NSB * rawsz);                                               \
                cp_async_commit();                                                                                           \
            }                                                                                                                \
            const unsigned char *blk = rb + (size_t)sb * rawsz;                                                              \
            __VA_ARGS__                                                                                                      \
        }                                                                                                                    \
    } while (0)

// grid = (row tiles of 128 rows, ceil(N / 128)), block = 384 threads, 1 CTA per SM.
//   warps 0..7  : consumers, warpgroup wg = rows 64*wg .. 64*wg+63 of the tile (wgmma accumulator layout)
//   warps 8..11 : producers, thread = weight row; thread 0 also issues the record copy of each step
// PB 2 (W2): a row tile is one 128-row super-block.  PB 4 (W3/W4): two 64-row super-blocks 2*tile + wg, one per consumer
// warpgroup; when nrsb is odd the last tile's second super-block does not exist and its A rows are zero.
// INT_PATH: the integer path (see the header); a step is 64 K, QCH / 4 of them per chunk.
template <int PB, bool INT_PATH>
__global__ void __launch_bounds__(kPfThreads2, 1) prefill_kernel(const PrefillParams p) {
    static_assert(PB == 2 || PB == 4, "prefill tile: W2 or W3/W4 stream layout");
    constexpr int RSB = 32 * (8 / PB);                                     // rows per super-block
    constexpr int NSB = 128 / RSB;                                         // super-blocks per row tile
    constexpr int REC = pf_rec_bytes(INT_PATH);
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *sA = smem;                                              // [S][16 KB]
    unsigned char *sR = sA + kPfStages * kPfStageBytes;                    // [S][REC] B tile (+ lut scales + lut bias pairs)
    unsigned char *raw = sR + kPfStages * REC;                             // [2][NSB][blk_bytes] packed blocks (codes + scales)
    const int rawsz = (p.blk_bytes + 127) & ~127;
    uint64_t *xtab = reinterpret_cast<uint64_t *>(raw + 2 * NSB * rawsz);  // [128 * PB] expansion table
    uint64_t *bars = xtab + 128 * PB;
    uint64_t *full = bars, *empty = bars + kPfStages;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rt = blockIdx.x, tile = blockIdx.y, n0 = tile * kPfNT;
    const int ntok = min(kPfNT, p.N - n0);
    const int nag = p.K / 64;

    pf_build_xtab<PB>(xtab, p.bits, false, tid, kPfThreads2);
    if (tid == 0) {
        for (int i = 0; i < kPfStages; ++i) { mbar_init(full + i, kPfProdWarps + 1); mbar_init(empty + i, kPfConsWarps); }
        mbar_fence_init();
    }
    __syncthreads();
    const unsigned char *rsb_base = p.W + (size_t)rt * NSB * p.rsb_stride;   // first super-block of the row tile
    const int spc = INT_PATH ? p.qch >> 2 : 2;       // steps (64 K) per chunk
    const int nsteps = spc * p.nchunk;               // fp path: activation groups (two per chunk)

    if (warp >= kPfConsWarps) {
        // ======================= producers: thread = weight row of the tile =======================
        PF_PRODUCER_ROW(PB, tid - kPfConsWarps * 32);
        const bool live = PB == 2 || rt * NSB + sb < p.nrsb;
        const unsigned char *rec_src = p.lut_tiles + (size_t)tile * nag * REC;
        const unsigned char *sb_base = rsb_base + (size_t)sb * p.rsb_stride;
        PF_STAGE_BLOCKS(PB, c, blk, 0, p.nchunk - 1, {
            const uint32_t *words = reinterpret_cast<const uint32_t *>(blk);
            _Pragma("unroll 1") for (int h = 0; h < spc; ++h) {
                const int step = spc * c + h, s = step % kPfStages;
                if (r == 0) PF_TRACE(0, step, 0);
                mbar_wait_parity(empty + s, ((step / kPfStages) & 1) ^ 1);     // stage released by the consumers of step - S
                if (r == 0) {
                    PF_TRACE(0, step, 1);
                    bulk_load(sR + (size_t)s * REC, rec_src + (size_t)step * REC, REC, full + s);
                }
                unsigned char *a_dst = sA + (size_t)s * kPfStageBytes;
                _Pragma("unroll") for (int kc = 0; kc < 8; ++kc) {
                    uint64_t v2[2];
                    _Pragma("unroll") for (int u = 0; u < 2; ++u) {
                        const int gq = h * 16 + kc * 2 + u;                // group within the chunk (0..31)
                        const int q = gq >> 2, k = gq & 3;
                        const uint32_t cw = row_codes<PB>(words + ((size_t)q * 32 + wl) * 4, k, wi);
                        if constexpr (PB == 2) {
                            v2[u] = xtab[cw];
                        } else {
                            // planes (0, 1) and (2, 3) index the two table halves, added byte-wise (|S| <= 15: no byte overflows,
                            // no borrow crosses into the next entry)
                            const uint64_t lo = xtab[cw & 0xffu], hi = xtab[256 + (cw >> 8)];
                            const uint32_t s0 = __vadd4((uint32_t)lo, (uint32_t)hi), s1 = __vadd4((uint32_t)(lo >> 32), (uint32_t)(hi >> 32));
                            v2[u] = live ? ((uint64_t)s1 << 32 | s0) : 0ull;
                        }
                    }
                    *reinterpret_cast<uint4 *>(a_dst + ((size_t)(kc * 16 + (r >> 3)) * 128 + (r & 7) * 16)) =
                        make_uint4((uint32_t)v2[0], (uint32_t)(v2[0] >> 32), (uint32_t)v2[1], (uint32_t)(v2[1] >> 32));
                }
                if (r == 0) PF_TRACE(0, step, 2);
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) mbar_arrive(full + s);
                __syncwarp();
            }
        });
    } else {
        // ======================= consumers: wgmma accumulator fragment of warpgroup wg =======================
        // register j = 4*c8 + 2*h + e holds row 64*wg + 16*(warp%4) + lane/4 + 8*h, token 8*c8 + 2*(lane%4) + e
        const int wg = warp >> 2;
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), tc = 2 * (lane & 3);
        float accf[64];
        uint32_t acc[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) accf[j] = 0.f;
        // weight scale / zero point of (row, chunk), prefetched one chunk ahead (L2 hits, latency off the critical path).
        // PB 4: the warpgroup's super-block, row r & 63 in it; zero for the missing second super-block of the last tile.
        const unsigned char *wg_base = rsb_base + (size_t)(PB == 4 ? wg : 0) * p.rsb_stride;
        const bool live = PB == 2 || rt * NSB + wg < p.nrsb;
        auto ld_s = [&](int c, int r) {
            return live ? 0.5f * load_scale(wg_base + (size_t)c * p.blk_bytes + kPfScaleOff, p.sd, PB == 2 ? r : r & (RSB - 1)) : 0.f;
        };
        auto ld_z = [&](int c, int r) {
            return (p.zp && live) ? load_scale(wg_base + (size_t)c * p.blk_bytes + kPfScaleOff + (size_t)RSB * p.sd, p.sd, PB == 2 ? r : r & (RSB - 1)) : 0.f;
        };
        float hs[2], zz[2], hs_n[2], zz_n[2];
        if constexpr (!INT_PATH) {               // the integer path's blocks carry no scales
#pragma unroll
            for (int h = 0; h < 2; ++h) { hs[h] = hs_n[h] = ld_s(0, r0 + 8 * h); zz[h] = zz_n[h] = ld_z(0, r0 + 8 * h); }
        }
        for (int step = 0; step < nsteps; ++step) {
            const int c = step >> 1, s = step % kPfStages;
            if (!INT_PATH && !(step & 1) && c + 1 < p.nchunk) {
#pragma unroll
                for (int h = 0; h < 2; ++h) { hs_n[h] = ld_s(c + 1, r0 + 8 * h); zz_n[h] = ld_z(c + 1, r0 + 8 * h); }
            }
            if (tid == 0) PF_TRACE(1, step, 0);
            mbar_wait_parity(full + s, (step / kPfStages) & 1);
            if (tid == 0) PF_TRACE(1, step, 1);
            const uint32_t a0 = smem_u32(sA + (size_t)s * kPfStageBytes) + wg * 1024, b0 = smem_u32(sR + (size_t)s * REC);
            wg_fence();
            // fp path: each step's int32 tile is folded below, the next step overwrites it; integer path: one int32 sum over K
#pragma unroll
            for (int i = 0; i < 4; ++i)
                wg_mma_s8_n128(acc, wg_desc(a0 + i * 4096, 2048), wg_desc(b0 + i * 4096, 2048), (i > 0 || (INT_PATH && step > 0)) ? 1u : 0u);
            wg_commit();
            wg_wait0();
            wg_fence_acc(acc);
            if (tid == 0) PF_TRACE(1, step, 2);
            if constexpr (!INT_PATH) {
                const unsigned char *rec = sR + (size_t)s * REC;
                const float2 *ls2 = reinterpret_cast<const float2 *>(rec + 16384);                 // (ls[t], ls[t+1]) pairs
#pragma unroll
                for (int c8 = 0; c8 < 16; ++c8) {
                    const float2 l = ls2[(8 * c8 + tc) >> 1];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int j = 4 * c8 + 2 * h;
                        accf[j] = fmaf(hs[h] * l.x, (float)(int)acc[j], accf[j]);
                        accf[j + 1] = fmaf(hs[h] * l.y, (float)(int)acc[j + 1], accf[j + 1]);
                    }
                }
                if (step & 1) {
                    // LUT-bias / zero-point term of the chunk: (0.5*s + z)[row] * (lb[2c] + lb[2c+1])[token]
                    const float4 *lb4 = reinterpret_cast<const float4 *>(rec + 16384 + 512);  // two tokens: (lb0, lb1), (lb0, lb1)
#pragma unroll
                    for (int c8 = 0; c8 < 16; ++c8) {
                        const float4 l = lb4[(8 * c8 + tc) >> 1];
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int j = 4 * c8 + 2 * h;
                            const float wz = hs[h] + zz[h];
                            accf[j] = fmaf(wz, l.x + l.y, accf[j]);
                            accf[j + 1] = fmaf(wz, l.z + l.w, accf[j + 1]);
                        }
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) { hs[h] = hs_n[h]; zz[h] = zz_n[h]; }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + s);        // A tile and record of this step are dead: the stage may be refilled
            __syncwarp();
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rt * 128 + r0 + 8 * h;
            if (row >= p.Mout) continue;
#pragma unroll
            for (int c8 = 0; c8 < 16; ++c8)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int t = 8 * c8 + tc + e, j = 4 * c8 + 2 * h + e;
                    // integer path: the token's one LUT scale and bias ([N][1]) and the tensor's scale, in the GEMV's order
                    if (t < ntok)
                        store_out(p.C, (size_t)(n0 + t) * p.ldc + row,
                                  INT_PATH ? int_path_out((int)acc[j], __ldg(p.lut_scales + n0 + t), __ldg(p.lut_biases + n0 + t), p.scale0) : accf[j],
                                  p.out_f16);
                }
        }
    }
}

}  // namespace tmac_b200
