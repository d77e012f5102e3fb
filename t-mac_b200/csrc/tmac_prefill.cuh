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
// registers.  A step is 64 K positions = 128 contraction bytes = 4 MMAs per warpgroup.  Once per activation group (ags 32: after
// MMAs {0, 1} and {2, 3} of a step; ags 64: after the step; ags 128: after every second step) the int32 tile is folded into fp32
// registers with lut_scale[n][ag] * 0.5*scale[m][wg] -- the layout keeps an activation group inside one weight chunk, so the fold
// has one weight scale; the LUT-bias / zero-point terms are a rank-(K/group_size) correction added once per chunk.
//
//   warpgroups 0, 1  consumers: 4 wgmma per step on rows 64*wg .. 64*wg+63, int32 -> fp32 fold, final store.
//   warpgroup  2     producers: cp.async the (row super-block, 128-K window) blocks, expand the packed codes of "their"
//                    weight row into S (one 64-bit one-hot-signed vector per (row, group), through a 256-entry (W2) or
//                    512-entry (W3/W4: two planes per lookup, two lookups added byte-wise) shared-memory table) in the
//                    K-major no-swizzle canonical layout; fence.proxy.async; arrive full[s].  Thread 0 also issues the
//                    step's LUT record as one bulk copy (TMA) into the same stage.
//
// Shared with the fp16 tile (tmac_prefill16.cuh): the producer's row (PF_PRODUCER_ROW), the double-buffered block staging
// (PF_STAGE_BLOCKS), the code decode (row_codes, tmac_kernels.cuh), the expansion table (pf_build_xtab), the grouping constants
// (PfGroups) and the scale offset in a block (pf_scale_off).  Each tile keeps its own expansion of a chunk's codes into A entries.
//
// Integer path (INT_PATH, BitNet: one weight scale, one activation group per row): the int32 accumulator sums over the whole K
// with no fold, and one epilogue per output applies the token's LUT scale and bias and the tensor's scale in the GEMV's order
// (int_path_out).  The int32 sum is the GEMV's integer (|S| <= 15, |T8| <= 127: no overflow at any K a row can have), converted to
// fp32 the same way, so the output is bit-identical to the GEMV and to the reference.  Its LUT records are the table entries only.
//
// Supported: PB == 2 (W2: a 128-row tile is one super-block) and PB == 4 (W3/W4: two 64-row super-blocks, one per consumer
// warpgroup), with a symmetric LUT and either
//   fp path: K % 128 == 0, per-row scales (+ zero points), chunk ck = 128, 64 or 32 K (template QCH 8, 4, 2) and act group
//            ags = 128, 64 or 32 K (template AGQ 8, 4, 2) with ags <= ck: (128, 128), (128, 64), (128, 32), (64, 64), (64, 32),
//            (32, 32) -- the last is ggml Q4_0 and GPTQ g32.  The producers stage a 128-K window (128 / ck consecutive chunk
//            blocks, one contiguous run of the stream layout) per two steps, whatever the chunk; or
//   integer path: one scale, act group = K, chunk = 128 K or 64 K (p.qch at run time; QCH and AGQ are not used).
// The routed instantiations (ROUTE) also take one-scale fp-path tensors (act group 128, 64 or 32 K < K): their blocks carry no
// scales (sd == 0), and the fold's weight scale is the tensor's scale0 with no zero point -- the same operations on the same values
// as a tensor whose per-row scales all equal scale0.  At K % 128 == 0 the chunk is 128 K; at K % 128 == 64 it is 64 K (an odd chunk
// count is possible), and the producers stage one chunk per unit (UNIT1, QCH 4), as on the integer path.
// Everything else takes the GEMV kernel once per activation row.
#pragma once
#include "tmac_kernels.cuh"

namespace tmac_b200 {

struct PrefillParams {
    const unsigned char *W;        // stream layout of the tensor (first super-block)
    const int8_t *qlut;            // [N][K/4][16]
    const float *lut_scales, *lut_biases;   // [N][K/ags]; integer path: [N][1]
    void *C;                       // [N][ldc]
    int N, K, Mout, ldc, out_f16;
    int nchunk, zp, sd, blk_bytes;
    size_t rsb_stride;
    const unsigned char *lut_tiles; // output of lut_tile_kernel: [token tile][step][pf_rec_bytes]
    long long *dbg;                // optional trace [role][step][4] (TMAC_ENABLE_TRACE builds)
    int nrsb, bits;                // row super-blocks of the tensor (PB 4: the last row tile may hold only one), bit width
    int qch;                       // quads of 16 K per chunk: 8, or 4 (integer path only)
    float scale0;                  // the tensor's one weight scale (integer path; routed tiles: one-scale fp-path tensors)
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

// The fp path's grouping: QCH quads of 16 K per weight chunk, AGQ quads per activation group (AGQ <= QCH, both 8, 4 or 2).  A
// step is 64 K; a window, the producers' staging unit, is 128 K = WB chunk blocks (two steps).
template <int QCH, int AGQ> struct PfGroups {
    static_assert((QCH == 8 || QCH == 4 || QCH == 2) && (AGQ == 8 || AGQ == 4 || AGQ == 2) && QCH % AGQ == 0, "prefill grouping");
    static constexpr int WB = 8 / QCH;                   // chunk blocks per window
    static constexpr int SPC = QCH == 8 ? 2 : 1;         // steps per chunk set: the NCS chunks whose scales a consumer holds
    static constexpr int NCS = QCH == 2 ? 2 : 1;         // chunks per chunk set (a step never straddles two sets)
    static constexpr int APC = QCH / AGQ;                // activation groups per chunk
    static constexpr int NLS = AGQ == 2 ? 2 : 1;         // LUT scales per token in a step's record: the step's activation groups
    static constexpr int NLB = NCS * APC;                // LUT biases per token in a step's record: those of the step's chunk set
};
__host__ __device__ constexpr int pf_scale_off(int qch) { return qch * 512; }   // a block's scales follow its QCH quads of codes

// ---------------------------------------------------------------------------------------------------
// lut_tile_kernel: QLUT [N][K/4][16] + LUT_Scales/Biases [N][K/ags]  ->  per (token tile of 128, 64-K step) one contiguous
// record that the GEMM stage receives with ONE bulk copy (TMA):
//     [16384 B]      the 8 stored LUT entries of the 16 groups of the step for 128 tokens, already in the K-major
//                    canonical order: chunk kc (groups 2kc, 2kc+1), token t at ((kc*16 + t/8)*128 + (t%8)*16)
//     [NLS * 512 B]  per token the LUT scales of the step's activation groups (ags 128: the group that holds the step)
//     [NLB * 512 B]  per token the LUT biases of the activation groups of the step's chunk set (ck 128: chunk step/2)
// (ck 128, ags 64: 17920 bytes: lut_scale[t][step], then (lut_bias[t][2c], lut_bias[t][2c+1]) of chunk c = step/2.)
// Tokens >= N are zero.  grid = (steps, token tiles), block = 128 (thread = token).
// INT_PATH: the record is the 16384 bytes of table entries alone (the consumers read the token's one LUT scale and bias of
// [N][1] in their epilogue); ls and lb are not read.
// ---------------------------------------------------------------------------------------------------
constexpr int kPfTab = 16384;
__host__ __device__ constexpr int pf_rec_bytes(bool int_path, int qch = 8, int agq = 4) {
    return int_path ? kPfTab : kPfTab + 512 * ((agq == 2 ? 2 : 1) + (qch == 2 ? 2 : 1) * (qch / agq));   // PfGroups NLS + NLB
}
//
// Routed experts (tmac_prefill_experts.cu) gather their records: the record of table entry k (PfRoute) at token position t holds
// LUT row perm[start + t] / div (div = topk: a token's slots share its row; div = 1: one row per slot); positions >= ntok are zero.
// Both record kernels of a tile share the body of one record (token row n, `live` = the token exists).
struct PfRoute {
    const int4 *tiles;                   // [cap] {expert, first position in perm, ntok (0 = unused entry), 0}; tiles never straddle experts
    const int *perm;                     // [N * topk] the valid slots s = n * topk + j sorted by expert, ascending s inside an expert
    const unsigned char *const *W;       // W[i * n_experts + e]: tensor i of expert e (the grouped pointer table)
    void *const *C;                      // C[i * n_experts + e]: where tensor i stores slot s's row, at row s of [N * topk][Mout]
    int n_experts;
    const void *R;                       // null, or the residual added to every output: R[s][row] of C's type (the dense forms)
    const float *const *bias;            // the BIAS tiles (prefill_rmsnorm_bias): bias[i * n_experts + e] fp32 [Mout], indexed like C
};
// A routed tile's output element C[o] = v (RES: + R[o], fp16 R widened).  R is read, then C written, by the same thread: R may be C.
// The epilogues branch on route.R once and run a store loop per case, so the experts' loop (no R) stores as it did without it.
template <bool RES>
__device__ __forceinline__ void pf_route_store(const PfRoute &route, void *const &C, size_t o, float v, int out_f16) {
    if constexpr (RES) v = __fadd_rn(v, out_f16 ? __half2float(reinterpret_cast<const __half *>(route.R)[o]) : reinterpret_cast<const float *>(route.R)[o]);
    store_out(C, o, v, out_f16);
}
template <bool V> struct PfRes { static constexpr bool value = V; };
// The BIAS tiles' case: no residual, and every output of tensor i is fadd_rn(v, b[row]) with b its bias, rounded once at the store.
struct PfBias { static constexpr bool value = false; const float *b; };
// The epilogues' output value of (row, v): v, or PfBias's sum.
template <typename E> __device__ __forceinline__ float pf_bias_add(const E &e, int row, float v) {
    if constexpr (std::is_same_v<E, PfBias>) return __fadd_rn(v, __ldg(e.b + row));
    else return v;
}
template <bool INT_PATH, int QCH, int AGQ>
__device__ __forceinline__ void lut_tile_rec(const int8_t *qlut, const float *ls, const float *lb, unsigned char *rec, int n, bool live,
                                             int K, int step, int t) {
    using G = PfGroups<QCH, AGQ>;
    const uint2 *src = reinterpret_cast<const uint2 *>(qlut) + ((size_t)n * (K / 4) + (size_t)step * 16) * 2;
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
        uint2 lo = make_uint2(0, 0), hi = make_uint2(0, 0);
        if (live) { lo = __ldg(src + kc * 4); hi = __ldg(src + kc * 4 + 2); }
        *reinterpret_cast<uint4 *>(rec + ((size_t)(kc * 16 + (t >> 3)) * 128 + (t & 7) * 16)) = make_uint4(lo.x, lo.y, hi.x, hi.y);
    }
    if constexpr (INT_PATH) return;
    const int nag = K / (16 * AGQ);                                      // activation groups per row
    const int ag0 = step * 4 / AGQ;                                      // the step's first activation group
    const int lb0 = (QCH == 8 ? step >> 1 : step * G::NCS) * G::APC;     // first activation group of the step's chunk set
    float *lsd = reinterpret_cast<float *>(rec + 16384) + t * G::NLS, *lbd = reinterpret_cast<float *>(rec + 16384 + 512 * G::NLS) + t * G::NLB;
#pragma unroll
    for (int i = 0; i < G::NLS; ++i) lsd[i] = live ? ls[(size_t)n * nag + ag0 + i] : 0.f;
#pragma unroll
    for (int i = 0; i < G::NLB; ++i) lbd[i] = live ? lb[(size_t)n * nag + lb0 + i] : 0.f;
}
template <bool INT_PATH, int QCH = 8, int AGQ = 4>
__global__ void __launch_bounds__(128) lut_tile_kernel(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int N, int K) {
    constexpr int REC = pf_rec_bytes(INT_PATH, QCH, AGQ);
    static_assert(INT_PATH || REC == kPfTab + 512 * (PfGroups<QCH, AGQ>::NLS + PfGroups<QCH, AGQ>::NLB), "record size");
    const int step = blockIdx.x, tile = blockIdx.y, t = threadIdx.x, n = tile * 128 + t;
    const int nsteps = K / 64;
    lut_tile_rec<INT_PATH, QCH, AGQ>(qlut, ls, lb, out + ((size_t)tile * nsteps + step) * REC, n, n < N, K, step, t);
}
// grid = (steps, table entries): the records of the routed int8 tile, [entry][step]; an unused entry's records are not written
// (its tile CTAs exit without reading them).  fp path only.
template <int QCH, int AGQ>
__global__ void __launch_bounds__(128) lut_tile_gather_kernel(const int8_t *qlut, const float *ls, const float *lb, unsigned char *out, int K,
                                                              const int4 *tiles, const int *perm, int div) {
    constexpr int REC = pf_rec_bytes(false, QCH, AGQ);
    const int step = blockIdx.x, k = blockIdx.y, t = threadIdx.x;
    const int4 e = __ldg(tiles + k);
    if (e.z == 0) return;
    const bool live = t < e.z;
    const int n = live ? __ldg(perm + e.y + t) / div : 0;
    lut_tile_rec<false, QCH, AGQ>(qlut, ls, lb, out + ((size_t)k * (K / 64) + step) * REC, n, live, K, step, t);
}

// NV consecutive floats of shared memory (NV = 2, 4 or 8, aligned to their size) as vector loads
template <int NV> __device__ __forceinline__ void pf_ld_floats(const float *src, float (&v)[NV]) {
    if constexpr (NV == 2) {
        const float2 a = *reinterpret_cast<const float2 *>(src);
        v[0] = a.x; v[1] = a.y;
    } else {
#pragma unroll
        for (int i = 0; i < NV / 4; ++i) {
            const float4 a = reinterpret_cast<const float4 *>(src)[i];
            v[4 * i] = a.x; v[4 * i + 1] = a.y; v[4 * i + 2] = a.z; v[4 * i + 3] = a.w;
        }
    }
}

constexpr int kPfStages = 4;                     // stages: A tile 16 KB (expanded by the producers) + record 17.5 KB (TMA)
constexpr int kPfConsWarps = 8;                  // two consumer warpgroups
constexpr int kPfProdWarps = 4;                  // one producer warpgroup
constexpr int kPfThreads2 = (kPfConsWarps + kPfProdWarps) * 32;

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

// PF_STAGE_BLOCKS runs the expansion (the variadic argument) once per staging unit c of [c_first, c_last] -- WB consecutive chunk
// blocks, which are contiguous in the stream layout: a 128-K window on the fp path, one chunk on the integer path -- with blk = the
// thread's super-block's first block of unit c in shared memory (each block: codes, then the scales at pf_scale_off(QCH)).  The
// blocks come from rsb_base (the row tile's first super-block) and sb_base (super-block sb) through raw, a double buffer
// [2][NSB][rawsz] with unit c in half c & 1: cp.async fetches unit c + 1 while unit c is expanded.  The 128 / NSB threads of a
// super-block stage its blocks; a super-block that is not live stages nothing.  Named barrier 1 (the 128 producer threads) makes
// unit c visible to every producer and retires unit c - 1, whose half then takes unit c + 1.  The blocks of c_last may still be
// read when the loop ends: a producer that stages another run passes barrier 1 before it.  Besides PF_PRODUCER_ROW's names it reads
// p, live, rsb_base, sb_base, raw, rawsz and NSB of the kernel.
#define PF_STAGE_BLOCKS(PB, WB, c, blk, c_first, c_last, ...)                                                                \
    do {                                                                                                                     \
        const int pf_c0 = (c_first), pf_c1 = (c_last), n16 = ((WB) * p.blk_bytes) >> 4;                                     \
        auto load_blocks = [&](int c_, unsigned char *dst) {   /* unit c_ of the tile's super-block(s) -> dst [NSB][rawsz] */ \
            const size_t src0 = (size_t)c_ * (WB) * p.blk_bytes;                                                             \
            if constexpr ((PB) == 2) {                                                                                       \
                for (int i = r; i < n16; i += 128) cp_async16_plain(dst + i * 16, rsb_base + src0 + i * 16);                 \
            } else if (live) {                                                                                               \
                for (int i = r & 63; i < n16; i += 64)                                                                       \
                    cp_async16_plain(dst + (size_t)sb * rawsz + i * 16, sb_base + src0 + i * 16);                            \
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
// fp path: a step is 64 K, two per 128-K window.  INT_PATH: the integer path (see the header); a step is 64 K, p.qch / 4 of them
// per chunk, and the staging unit is one chunk.
// ROUTE (routed experts and the dense prefill_* forms, fp path, prefill_experts_kernel): grid = (row tiles, table entries, count);
// the CTA of entry k = blockIdx.y and tensor i = blockIdx.z exits at once when the entry is unused, else takes the weights
// W[i * n_experts + expert] of the pointer table, the records of entry k (lut_tile_gather_kernel) and stores token t's row at row
// perm[start + t] of C[i * n_experts + expert], plus the residual route.R when there is one (pf_route_store).  A tensor with
// p.sd == 0 has one scale (see the header).  UNIT1 (ROUTE, QCH 4, one-scale tensors with K % 128 == 64): a staging unit is one
// 64-K chunk, one step.  BIAS (ROUTE, prefill_bias_kernel): no residual; each output takes route.bias's row (PfBias).
template <int PB, bool INT_PATH, int QCH, int AGQ, bool ROUTE, bool UNIT1 = false, bool BIAS = false>
__device__ __forceinline__ void prefill_body(const PrefillParams &p, const PfRoute &route) {
    static_assert(PB == 2 || PB == 4, "prefill tile: W2 or W3/W4 stream layout");
    static_assert(!(ROUTE && INT_PATH), "routed experts: fp path only");
    static_assert(!UNIT1 || (ROUTE && QCH == 4), "one-chunk staging: routed 64-K chunks only");
    static_assert(!BIAS || ROUTE, "biases: routed tiles only");
    using G = PfGroups<QCH, AGQ>;
    constexpr int RSB = 32 * (8 / PB);                                     // rows per super-block
    constexpr int NSB = 128 / RSB;                                         // super-blocks per row tile
    constexpr int REC = pf_rec_bytes(INT_PATH, QCH, AGQ);
    constexpr int WB = (INT_PATH || UNIT1) ? 1 : G::WB;                    // chunk blocks per staging unit
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *sA = smem;                                              // [S][16 KB]
    unsigned char *sR = sA + kPfStages * kPfStageBytes;                    // [S][REC] B tile (+ lut scales + lut biases)
    unsigned char *raw = sR + kPfStages * REC;                             // [2][NSB][WB * blk_bytes] packed blocks (codes + scales)
    const int rawsz = (WB * p.blk_bytes + 127) & ~127;
    uint64_t *xtab = reinterpret_cast<uint64_t *>(raw + 2 * NSB * rawsz);  // [128 * PB] expansion table
    uint64_t *bars = xtab + 128 * PB;
    uint64_t *full = bars, *empty = bars + kPfStages;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rt = blockIdx.x, tile = blockIdx.y, n0 = tile * kPfNT;
    int4 ent = make_int4(0, 0, 0, 0);                                      // ROUTE: {expert, start, ntok, 0} of the CTA's entry
    if constexpr (ROUTE) {
        ent = __ldg(route.tiles + tile);
        if (ent.z == 0) return;
    }
    const int ntok = ROUTE ? ent.z : min(kPfNT, p.N - n0);
    const int nag = p.K / 64;

    pf_build_xtab<PB>(xtab, p.bits, false, tid, kPfThreads2);
    if (tid == 0) {
        for (int i = 0; i < kPfStages; ++i) { mbar_init(full + i, kPfProdWarps + 1); mbar_init(empty + i, kPfConsWarps); }
        mbar_fence_init();
    }
    __syncthreads();
    // first super-block of the row tile
    const unsigned char *rsb_base = (ROUTE ? route.W[blockIdx.z * route.n_experts + ent.x] : p.W) + (size_t)rt * NSB * p.rsb_stride;
    const int spc = INT_PATH ? p.qch >> 2 : UNIT1 ? 1 : 2;   // steps (64 K) per staging unit
    const int nunits = p.nchunk / WB;                // fp path: 128-K windows; integer path: chunks
    const int nsteps = spc * nunits;

    if (warp >= kPfConsWarps) {
        // ======================= producers: thread = weight row of the tile =======================
        PF_PRODUCER_ROW(PB, tid - kPfConsWarps * 32);
        const bool live = PB == 2 || rt * NSB + sb < p.nrsb;
        const unsigned char *rec_src = p.lut_tiles + (size_t)tile * nag * REC;
        const unsigned char *sb_base = rsb_base + (size_t)sb * p.rsb_stride;
        PF_STAGE_BLOCKS(PB, WB, c, blk, 0, nunits - 1, {
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
                        const int gq = h * 16 + kc * 2 + u;                // group within the unit (0..31)
                        // its block in the window and its quad / word there
                        const int b = WB == 1 ? 0 : gq / (4 * QCH), gb = WB == 1 ? gq : gq % (4 * QCH);
                        const int q = gb >> 2, k = gb & 3;
                        const uint32_t cw = row_codes<PB>(words + (size_t)b * (p.blk_bytes >> 2) + ((size_t)q * 32 + wl) * 4, k, wi);
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
        // one-scale tensors (routed tiles): scale0, and nothing is read at pf_scale_off (their blocks are codes only)
        const bool one = ROUTE && (UNIT1 || p.sd == 0);
        auto ld_s = [&](int c, int r) {
            return live ? 0.5f * (one ? p.scale0 : load_scale(wg_base + (size_t)c * p.blk_bytes + pf_scale_off(QCH), p.sd, PB == 2 ? r : r & (RSB - 1))) : 0.f;
        };
        auto ld_z = [&](int c, int r) {
            return (p.zp && live) ? load_scale(wg_base + (size_t)c * p.blk_bytes + pf_scale_off(QCH) + (size_t)RSB * p.sd, p.sd, PB == 2 ? r : r & (RSB - 1)) : 0.f;
        };
        // the scales of the chunk set (G::NCS chunks) of the step and of the next set
        float hs[G::NCS][2], zz[G::NCS][2], hs_n[G::NCS][2], zz_n[G::NCS][2];
        if constexpr (!INT_PATH) {               // the integer path's blocks carry no scales
#pragma unroll
            for (int i = 0; i < G::NCS; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h) { hs[i][h] = hs_n[i][h] = ld_s(i, r0 + 8 * h); zz[i][h] = zz_n[i][h] = ld_z(i, r0 + 8 * h); }
        }
        // MMAs {0..3} of a step in NF runs of 4 / NF; the fp path folds after each run (ags 32: two activation groups per step)
        constexpr int NF = (!INT_PATH && AGQ == 2) ? 2 : 1, MPF = 4 / NF;
        // ags 128: the two steps of a window run as one unrolled pair (su), so which one folds is known at compile time
        constexpr int SU = (!INT_PATH && AGQ == 8) ? 2 : 1;
        for (int step0 = 0; step0 < nsteps; step0 += SU)
#pragma unroll
        for (int su = 0; su < SU; ++su) {
            const int step = step0 + su;
            const bool set_first = SU == 2 ? su == 0 : step % G::SPC == 0, set_last = SU == 2 ? su == 1 : step % G::SPC == G::SPC - 1;
            const int cs = step / G::SPC, s = step % kPfStages;
            if (!INT_PATH && set_first && (cs + 1) * G::NCS < p.nchunk) {
#pragma unroll
                for (int i = 0; i < G::NCS; ++i)
#pragma unroll
                    for (int h = 0; h < 2; ++h) { hs_n[i][h] = ld_s((cs + 1) * G::NCS + i, r0 + 8 * h); zz_n[i][h] = ld_z((cs + 1) * G::NCS + i, r0 + 8 * h); }
            }
            if (tid == 0) PF_TRACE(1, step, 0);
            mbar_wait_parity(full + s, (step / kPfStages) & 1);
            if (tid == 0) PF_TRACE(1, step, 1);
            const uint32_t a0 = smem_u32(sA + (size_t)s * kPfStageBytes) + wg * 1024, b0 = smem_u32(sR + (size_t)s * REC);
            const unsigned char *rec = sR + (size_t)s * REC;
#pragma unroll
            for (int f = 0; f < NF; ++f) {
                wg_fence();
                // fp path: each run's int32 tile is folded below and the next run overwrites it, except that ags 128 carries it
                // into the step's odd partner; integer path: one int32 sum over K
#pragma unroll
                for (int i = 0; i < MPF; ++i) {
                    const int m = f * MPF + i;
                    wg_mma_s8_n128(acc, wg_desc(a0 + m * 4096, 2048), wg_desc(b0 + m * 4096, 2048),
                                   (i > 0 || (INT_PATH && step > 0) || (SU == 2 && su == 1)) ? 1u : 0u);
                }
                wg_commit();
                wg_wait0();
                wg_fence_acc(acc);
                if (tid == 0 && f == NF - 1) PF_TRACE(1, step, 2);
                if constexpr (!INT_PATH) {
                    if (SU == 1 || su == 1) {
                        // the activation group ends here: accf += 0.5*s[row] * ls[token] * acc, s of the group's chunk
                        const float *lsp = reinterpret_cast<const float *>(rec + 16384);
                        const int ci = G::NCS == 2 ? f : 0;
#pragma unroll
                        for (int c8 = 0; c8 < 16; ++c8) {
                            float lv[2 * G::NLS];                                  // tokens t, t + 1: their NLS LUT scales each
                            pf_ld_floats(lsp + ((8 * c8 + tc) >> 1) * 2 * G::NLS, lv);
                            const float lx = lv[G::NLS == 2 ? f : 0], ly = lv[G::NLS + (G::NLS == 2 ? f : 0)];
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int j = 4 * c8 + 2 * h;
                                accf[j] = fmaf(hs[ci][h] * lx, (float)(int)acc[j], accf[j]);
                                accf[j + 1] = fmaf(hs[ci][h] * ly, (float)(int)acc[j + 1], accf[j + 1]);
                            }
                        }
                    }
                }
            }
            if constexpr (!INT_PATH) {
                if (set_last) {
                    // the chunk set ends here: LUT-bias / zero-point term of each chunk, (0.5*s + z)[row] * (sum of the chunk's
                    // activation groups' lb)[token]
                    const float *lbp = reinterpret_cast<const float *>(rec + 16384 + 512 * G::NLS);
#pragma unroll
                    for (int c8 = 0; c8 < 16; ++c8) {
                        float lv[2 * G::NLB];                                      // tokens t, t + 1: their NLB LUT biases each
                        pf_ld_floats(lbp + ((8 * c8 + tc) >> 1) * 2 * G::NLB, lv);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int j = 4 * c8 + 2 * h;
#pragma unroll
                            for (int i = 0; i < G::NCS; ++i) {
                                float bx = lv[i * G::APC], by = lv[G::NLB + i * G::APC];
#pragma unroll
                                for (int a = 1; a < G::APC; ++a) { bx += lv[i * G::APC + a]; by += lv[G::NLB + i * G::APC + a]; }
                                const float wz = hs[i][h] + zz[i][h];
                                accf[j] = fmaf(wz, bx, accf[j]);
                                accf[j + 1] = fmaf(wz, by, accf[j + 1]);
                            }
                        }
                    }
#pragma unroll
                    for (int i = 0; i < G::NCS; ++i)
#pragma unroll
                        for (int h = 0; h < 2; ++h) { hs[i][h] = hs_n[i][h]; zz[i][h] = zz_n[i][h]; }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + s);        // A tile and record of this step are dead: the stage may be refilled
            __syncwarp();
        }
        if constexpr (ROUTE) {
            void *const Cr = route.C[blockIdx.z * route.n_experts + ent.x];
            const auto stores = [&](auto res) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = rt * 128 + r0 + 8 * h;
                    if (row >= p.Mout) continue;
#pragma unroll
                    for (int c8 = 0; c8 < 16; ++c8)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int t = 8 * c8 + tc + e;
                            if (t < ntok)
                                pf_route_store<decltype(res)::value>(route, Cr, (size_t)__ldg(route.perm + ent.y + t) * p.ldc + row,
                                                                     pf_bias_add(res, row, accf[4 * c8 + 2 * h + e]), p.out_f16);
                        }
                }
            };
            if constexpr (BIAS) stores(PfBias{route.bias[blockIdx.z * route.n_experts + ent.x]});
            else if (route.R) stores(PfRes<true>{});
            else stores(PfRes<false>{});
            return;
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
template <int PB, bool INT_PATH, int QCH = 8, int AGQ = 4>
__global__ void __launch_bounds__(kPfThreads2, 1) prefill_kernel(const PrefillParams p) {
    prefill_body<PB, INT_PATH, QCH, AGQ, false>(p, PfRoute{});
}
template <int PB, int QCH, int AGQ, bool UNIT1 = false>
__global__ void __launch_bounds__(kPfThreads2, 1) prefill_experts_kernel(const PrefillParams p, const PfRoute route) {
    prefill_body<PB, false, QCH, AGQ, true, UNIT1>(p, route);
}
// prefill_experts_kernel with a bias on every output (tmac_b200_prefill_rmsnorm_bias): kernels of their own, so that the routed
// kernels' epilogues are not touched
template <int PB, int QCH, int AGQ, bool UNIT1 = false>
__global__ void __launch_bounds__(kPfThreads2, 1) prefill_bias_kernel(const PrefillParams p, const PfRoute route) {
    prefill_body<PB, false, QCH, AGQ, true, UNIT1, true>(p, route);
}

}  // namespace tmac_b200
