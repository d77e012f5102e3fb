// tmac_seq.cuh -- the decode SEQUENCE kernel: a whole chain of dependent table-lookup GEMVs (the quantised linears of
// a token step, in model order) executed by ONE persistent launch, one CTA per SM.
//
// Why: a chain of per-GEMV launches loses, per launch, the time for griddepcontrol.wait to return, the exposed weight
// stream (one launch fills the register file, so the next one cannot co-reside and prefetch), a cluster barrier on the
// slowest CTA and the final store -- several microseconds for a 12.7 MB GEMV whose HBM time is 3.8 us at 3.35 TB/s.  The reference has the same structure on the CPU: ggml's graph loop runs one
// mul_mat node after the other on a persistent thread pool (3rdparty/llama.cpp/ggml/src/ggml.c:12562-12706 per node,
// workers parked between nodes, never re-created).  This kernel is the GPU form of that loop:
//
//   * the weight stream never stops: one producer thread per CTA walks the CTA's blocks of op 0, 1, 2, ... and
//     requests each (4.6 KB, contiguous) with one cp.async.bulk (TMA) into a ring of ~40 shared-memory slots; a
//     slot is reused when every consumer warp has published a progress counter beyond it.  HBM therefore runs
//     ~2 GEMVs ahead of the arithmetic, across the data dependencies, because weights do not depend on activations;
//   * 20 consumer warps per CTA do, per op: (A) build the LUT slices of the CTA's K chunks from the op's input
//     vector (lut_group, lut_addv8 and lut_bias of tmac_kernels.cuh, the LUT functions preprocessor_kernel uses
//     -> bit-identical tables), (B) the lookups of gemv3 and chain_kernel (TMAC_QUAD_LOOKUP and TMAC_GROUP_FOLD of
//     tmac_kernels.cuh) over an arithmetic "stream-K" share of the op's blocks -- CTA c owns blocks
//     [T*c/G, T*(c+1)/G), a warp owns a contiguous run of activation-group units inside them, so a warp's run can
//     start and end inside a block --, (C) reduce the warps through shared memory in fixed order and finish the rows;
//   * rows whose K range is split between CTAs are finished by the LAST CTA that touches them: the earlier ones
//     publish their partial sums through 8-byte {value, epoch} slots in global memory (one store, one polling load
//     per row; no fence, no atomic; ascending CTA order -> deterministic);
//   * the data dependency between ops is carried the same way: the finished row is stored as {value, epoch} into the
//     op's output vector, and the LUT build of a consumer op polls exactly the elements it needs.  An op can also
//     take an external (plain) vector as input and can write a plain copy of its output (C) for the caller.  A GLU op reads
//     two producers (gate, up) and builds its LUT from swiglu(gate, up) (tmac_kernels.cuh).
//   Every wait is bounded (~1 s) and raises an error flag instead of hanging the GPU.
#pragma once
#include "tmac_kernels.cuh"

namespace tmac_b200 {

constexpr int kSeqWarps = 19;                         // consumer warps per CTA
constexpr int kSeqThreads = (kSeqWarps + 1) * 32;     // + 1 producer warp
constexpr int kSeqMaxRsb = 256;                       // rows per super-block, PB = 1
constexpr int kSeqDescWords = 64;                     // SeqOp (words 0..) + SeqCta (words 40..55) staged in shared memory
constexpr int kSeqSpinLimit = 1 << 20;           // x ~0.3 us per poll: every wait gives up after ~0.3 s

struct SeqOp {                            // one GEMV; read-only for the kernel
    const unsigned char *W;               // stream layout of the tensor (tmac_layout.h)
    const float *x_ext;                   // input: external fp32 vector [K] ...
    const uint2 *x_ll;                    // ... or {value, epoch} elements of an earlier op's output (already offset)
    void *C;                              // optional plain output [Mout] (f32 / f16)
    uint2 *y;                             // this op's output vector as {value, epoch} [nrsb * RSB]
    uint2 *xchg;                          // [grid][RSB] partial-sum exchange slots of this op
    // LUT hand-over (optional): the CTA that finishes a row super-block also builds the LUT of those rows -- the consumer op's
    // preprocessor, fused into the producer's epilogue -- as {lo, epoch, hi, epoch} per K-group and {scale, epoch, bias, epoch}
    // per activation group; a consumer whose input is this op's output then only fetches its slices.
    uint4 *lut_out, *ag_out;              // this op's output as LUT records [nrsb*RSB/4], [nrsb*RSB/ags] (or null)
    const uint4 *lut_in, *ag_in;          // input LUT records (already offset) or null: build the LUT from x_ext / x_ll
    unsigned long long rsb_stride;
    int K, Mout, nrsb, nchunk;
    int blk_bytes, total;                 // bytes per block; nrsb * nchunk
    int zp, one_scale, sd, out_f16;
    float scale0;
    int geff;                             // CTAs that take part in this op = min(grid, total): every one of them owns >= 1 block
    const uint2 *x_ll2;                   // GLU op (seq_kernel<..., true> only): the up producer's elements (x_ll: the gate's); the
                                          // input is swiglu(gate, up).  Never takes the LUT hand-over.  NULL: a plain op
};

// Per (op, CTA) work description, precomputed by the host (tmac_b200_seq_build) so that no warp spends instructions on
// integer divisions: CTA c of an op with T blocks and G participating CTAs owns blocks [T*c/G, T*(c+1)/G) in
// (row super-block, K chunk) order.
struct SeqCta {
    int b0, nb;                           // first block, number of blocks (0: the CTA sits the op out)
    int sb_first, c0;                     // row super-block / chunk of block b0
    int nseg, nck;                        // row super-blocks touched; distinct K chunks touched = min(nb, nchunk)
    int npass, P;                         // the share is walked in npass passes of <= P blocks (P <= half the ring)
    int fc;                               // first CTA that contributes to my first super-block (== own index: it starts here)
    int last_open;                        // 1: my last super-block continues in the next CTA (its partial sum is published)
    int pad_[6];
};

struct SeqParams {
    const SeqOp *ops;
    const SeqCta *ctas;                   // [nops][grid]
    int nops;
    int nslots, slot_bytes;               // weight ring
    int red_off, tab_off, lsb_off, bar_off, prog_off, yfin_off, desc_off;   // shared-memory offsets (bytes)
    unsigned int *epochs;                 // [grid] launch counter of every CTA (incremented by that CTA at exit)
    int *err;                             // != 0: a wait expired
    long long *trace;                     // optional [nops][grid][16] globaltimer stamps, followed by [nops][grid][NW][16] per-warp clock64 stamps
};

__device__ __forceinline__ void seq_publish(uint2 *slot, uint32_t bits, uint32_t epoch) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(slot), "r"(bits), "r"(epoch) : "memory");
}
// Waiting for N = 1, 2 or 4 consecutive {value, epoch} words at src per active lane; val = their values (0 in inactive lanes and
// after LIMIT polls: error `code`), separate references because an array or a returned vector changes chain_kernel's SASS.  While
// some are stale, every stale lane reloads all its words, so the round trip that sees the last epoch also brings the values.
// (Polling one lane's first epoch and then reloading costs a second L2 round trip per wait after the data has landed: on an H100
// that made the dependent bench chain 0.18 us per GEMV slower, and seq_kernel 0.67; the extra poll traffic did not show.)  All 32
// lanes must call.
template <int LIMIT, typename... F>
__device__ __forceinline__ void wait_words(const uint2 *src, bool active, uint32_t epoch, int *err, int code, F &...val) {
    constexpr int N = sizeof...(F);
    static_assert(N == 1 || N == 2 || N == 4, "words per lane");
    uint4 v0 = make_uint4(0u, epoch, 0u, epoch), v1 = v0;      // words 0, 1 | 2, 3 (absent words read as current)
    auto load = [&]() {
        if constexpr (N == 1) asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v0.x), "=r"(v0.y) : "l"(src) : "memory");
        else asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v0.x), "=r"(v0.y), "=r"(v0.z), "=r"(v0.w) : "l"(src) : "memory");
        if constexpr (N == 4) asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v1.x), "=r"(v1.y), "=r"(v1.z), "=r"(v1.w) : "l"(src + 2) : "memory");
    };
    if (active) load();
    int spins = 0;
    for (;;) {
        const bool stale = active && (v0.y != epoch || v0.w != epoch || v1.y != epoch || v1.w != epoch);
        if (__ballot_sync(0xffffffffu, stale) == 0) break;
        if (++spins >= LIMIT) { if ((threadIdx.x & 31) == 0) atomicExch(err, code); v0.x = v0.z = v1.x = v1.z = 0u; break; }
        if (stale) load();
    }
    const float w[4] = {__uint_as_float(v0.x), __uint_as_float(v0.z), __uint_as_float(v1.x), __uint_as_float(v1.z)};
    int i = 0;
    ((val = w[i++]), ...);
}
__device__ __forceinline__ void seq_bar(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(kSeqWarps * 32) : "memory"); }
__device__ __forceinline__ int ld_volatile_s32(const int *p) { int v; asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory"); return v; }
__device__ __forceinline__ void st_volatile_s32(int *p, int v) { asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory"); }

__device__ __forceinline__ void seq_publish16(uint4 *slot, uint32_t a, uint32_t b, uint32_t epoch) {
    // two 8-byte {value, epoch} words written by ONE 16-byte store; each half is valid on its own
    asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1, %2, %3, %2};" ::"l"(slot), "r"(a), "r"(epoch), "r"(b) : "memory");
}

// N (2, 4 or 8) consecutive fp16 values -> fp32 with one shared-memory vector load
template <int N> __device__ __forceinline__ void load_half_vec(const unsigned char *p, float *out) {
    static_assert(N == 2 || N == 4 || N == 8, "rows per lane");
    uint32_t w[N / 2];
    if (N == 2) w[0] = *reinterpret_cast<const uint32_t *>(p);
    else if (N == 4) { const uint2 v = *reinterpret_cast<const uint2 *>(p); w[0] = v.x; w[1] = v.y; }
    else { const uint4 v = *reinterpret_cast<const uint4 *>(p); w[0] = v.x; w[1] = v.y; w[N / 2 - 2] = v.z; w[N / 2 - 1] = v.w; }
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
        out[2 * i] = f.x; out[2 * i + 1] = f.y;
    }
}

// The LUT record of a K-group (lane = K-group, x0..x3 = its activations, WL lanes per activation group): the stored entries
// lo | hi and the group's LUT scale; returns the group's LUT bias.  All 32 lanes must call it.
template <int WL>
__device__ __forceinline__ float lut_record(float x0, float x1, float x2, float x3, int lane, uint32_t &lo, uint32_t &hi, float &scale) {
    return lut_bias<WL>(lut_addv8(lut_group<WL>(x0, x1, x2, x3, lo, hi, scale)), lane & ~(WL - 1));
}
// LUT hand-over: the record of K-group g of an op's output from its four rows x, published as {lo, epoch, hi, epoch} to
// lut_out[g] and, by the activation group's first lane, {scale, epoch, bias, epoch} to ag_out[g / WL] (`valid` lanes only).
// All 32 lanes must call it.
template <int WL>
__device__ __forceinline__ void publish_lut_record(float4 x, int lane, bool valid, size_t g, uint4 *lut_out, uint4 *ag_out, uint32_t epoch) {
    uint32_t lo, hi;
    float scale;
    const float bias = lut_record<WL>(x.x, x.y, x.z, x.w, lane, lo, hi, scale);
    if (valid) {
        seq_publish16(lut_out + g, lo, hi, epoch);
        if ((lane & (WL - 1)) == 0) seq_publish16(ag_out + g / WL, __float_as_uint(scale), __float_as_uint(bias), epoch);
    }
}

// PB planes per word, QCH quads per chunk, AGQ quads per activation group (fp path: AGQ > 0).  GLU: the sequence has GLU ops
// (SeqOp::x_ll2), a separate instantiation so that sequences without them keep their code.
template <int PB, int QCH, int AGQ, bool GLU>
__global__ void __launch_bounds__(kSeqThreads, 1) seq_kernel(const SeqParams p, const uint32_t wtx, const uint32_t wty) {
    constexpr int RW = 8 / PB, RSB = 32 * RW;
    constexpr int NAG = QCH / AGQ;                 // activation groups per chunk = work units per block
    constexpr int NG = QCH * 4;                    // K-groups per chunk
    constexpr int WL = AGQ * 4;                    // lanes (K-groups) per activation group
    constexpr int TAB = NG * 8;                    // table bytes per chunk (8 stored entries per group)
    constexpr int NW = kSeqWarps;
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    unsigned char *ring = smem;
    float *red = reinterpret_cast<float *>(smem + p.red_off);          // [nseg][NW][RSB]
    unsigned char *tabs = smem + p.tab_off;                            // [ntab][TAB]
    float *lsb = reinterpret_cast<float *>(smem + p.lsb_off);          // [ntab][2 * NAG]: LUT scale, LUT bias per activation group
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + p.bar_off);   // [nslots]
    int *prog = reinterpret_cast<int *>(smem + p.prog_off);            // [NW] lowest block sequence number the warp still needs
    int *issued = prog + NW;
                                           // blocks requested so far by the producer
    uint32_t *desc = reinterpret_cast<uint32_t *>(smem + p.desc_off);  // [2][kSeqDescWords] op + share descriptors of the current / next op
    float *yfin = reinterpret_cast<float *>(smem + p.yfin_off);        // [nseg][RSB] finished rows of this op (LUT hand-over)
    const uint32_t epoch = p.epochs[cta] + 1u;

    if (tid == 0) {
        for (int s = 0; s < p.nslots; ++s) mbar_init(full + s, 1);
        mbar_fence_init();
        fence_proxy_async();
    }
    if (tid <= NW) prog[tid] = 0;                  // prog[NW] = issued
    static_assert(sizeof(SeqOp) <= 160 && sizeof(SeqCta) == 64, "descriptor staging layout");
    auto desc_word = [&](int op, int i) -> uint32_t {   // word i of the staged descriptor of `op` for this CTA
        return i < 40 ? (i < (int)(sizeof(SeqOp) / 4) ? reinterpret_cast<const uint32_t *>(p.ops + op)[i] : 0u)
                      : reinterpret_cast<const uint32_t *>(p.ctas + (size_t)op * G + cta)[i - 40];
    };
    if (tid < 56) desc[tid] = desc_word(0, tid);
    __syncthreads();

    // =========================================== producer warp ===========================================
    if (warp == NW) {
        if (lane != 0) return;
        int seq = 0, slot = 0, known_min = 0;
        for (int op = 0; op < p.nops; ++op) {
            const SeqOp &o = p.ops[op];
            const SeqCta &q = p.ctas[(size_t)op * G + cta];
            const int b0 = q.b0, b1 = b0 + q.nb;
            if (b1 == b0) continue;
            const int nchunk = o.nchunk, blk = o.blk_bytes;
            const unsigned char *W = o.W;
            const unsigned long long rs = o.rsb_stride;
            int sb = q.sb_first, c = q.c0;
            if (p.trace) p.trace[((size_t)op * G + cta) * 16 + 8] = globaltimer_ns();  // producer reaches this op
            for (int b = b0; b < b1; ++b, ++seq) {
                if (seq >= p.nslots) {                         // slot still holds block seq - nslots: wait until nobody needs it
                    const int need = seq - p.nslots + 1;
                    int spins = 0;
                    while (known_min < need) {
                        int m = 0x7fffffff;
                        for (int w = 0; w < NW; ++w) m = min(m, ld_volatile_s32(prog + w));
                        known_min = m;
                        if (known_min >= need) break;
                        __nanosleep(200);                      // a spinning producer would take issue slots from 5 consumer warps
                        if (++spins > kSeqSpinLimit) { atomicExch(p.err, 1); return; }
                    }
                }
                fence_proxy_async();
                bulk_load(ring + (size_t)slot * p.slot_bytes, W + (size_t)sb * rs + (size_t)c * blk, (uint32_t)blk, full + slot);
                st_volatile_s32(issued, seq + 1);              // the phase parity of `full` is only meaningful once the request is out
                if (++slot == p.nslots) slot = 0;
                if (++c == nchunk) { c = 0; ++sb; }
            }
            if (p.trace) p.trace[((size_t)op * G + cta) * 16 + 9] = globaltimer_ns();  // ... and has requested all of its blocks
        }
        return;
    }

    // =========================================== consumer warps ===========================================
    int seq_base = 0, slot_base = 0, par_base = 0;     // sequence number / ring slot / phase parity of the op's first block
    for (int op = 0; op < p.nops; ++op) {
        // descriptors come from shared memory (staged one op ahead): a global load per field would put ~1 us of L2 latency in
        // front of every op
        const SeqOp &o = *reinterpret_cast<const SeqOp *>(desc + (op & 1) * kSeqDescWords);
        const SeqCta &qc = *reinterpret_cast<const SeqCta *>(desc + (op & 1) * kSeqDescWords + 40);
        const int nb = qc.nb;
        uint32_t next_word = 0;
        if (tid < 56 && op + 1 < p.nops) next_word = desc_word(op + 1, tid);      // in flight during this op
        if (nb == 0) {                                     // more CTAs than blocks: this CTA sits the op out
            if (tid < 56) desc[((op + 1) & 1) * kSeqDescWords + tid] = next_word;
            seq_bar(2);
            continue;
        }
        const int nchunk = o.nchunk;
        // op fields live in registers: `o` is global memory and every asm volatile below would force a reload
        const int zp = o.zp, sd = o.sd, one_scale = o.one_scale, Mout = o.Mout, out_f16 = o.out_f16;
        const float scale0 = o.scale0;
        void *const Cout = o.C;
        uint2 *const yv = o.y, *const xchg = o.xchg;
        uint4 *const lut_out = o.lut_out, *const ag_out = o.ag_out;
        const int sb_first = qc.sb_first, c0 = qc.c0, nseg = qc.nseg, nck = qc.nck;
        // Work split inside the CTA: the share is walked in passes of at most half a ring (so that the blocks the warps
        // work on are resident together); inside a pass every warp owns a contiguous run of units.
        const int npass = qc.npass, P = qc.P, fc = qc.fc, last_open = qc.last_open;
        if (lane == 0) st_volatile_s32(prog + warp, seq_base);
        long long *tr = p.trace ? p.trace + ((size_t)op * G + cta) * 16 : nullptr;
        long long *tw = (p.trace && lane == 0) ? p.trace + (size_t)p.nops * G * 16 + (((size_t)op * G + cta) * NW + warp) * 16 : nullptr;
        if (tw) { tw[0] = clock64(); tw[12] = globaltimer_ns(); }
        if (tr && tid == 0) { tr[0] = globaltimer_ns(); tr[10] = 0; }
        if (tr && warp == NW - 1 && lane == 0) tr[11] = 0;

        // ---- (A) LUT slices of my chunks: thread = K-group.  Either fetched ready-made (built by the CTAs that finished the
        //      producer's rows) or built here from the input vector. ----
        {
            const float *xe = o.x_ext;
            const uint2 *xl = o.x_ll;
            const uint2 *xl2 = nullptr;
            if constexpr (GLU) xl2 = o.x_ll2;
            const uint4 *li = o.lut_in, *ai = o.ag_in;
            const int ngroups = nck * NG;
            for (int t0 = warp * 32; t0 < ngroups; t0 += NW * 32) {
                const int t = t0 + lane;
                const bool valid = t < ngroups;
                const int ci = valid ? t / NG : 0, gl = t % NG;
                int c = c0 + ci; if (c >= nchunk) c -= nchunk;
                float *d = lsb + (size_t)ci * (2 * NAG);
                if (li) {
                    float lo, hi, scale, bias;
                    wait_words<kSeqSpinLimit>(reinterpret_cast<const uint2 *>(li + (size_t)c * NG + gl), valid, epoch, p.err, 5, lo, hi);
                    const bool first = valid && (gl % WL) == 0;
                    wait_words<kSeqSpinLimit>(reinterpret_cast<const uint2 *>(ai + (size_t)c * NAG + gl / WL), first, epoch, p.err, 5, scale, bias);
                    if (valid) reinterpret_cast<uint2 *>(tabs + (size_t)ci * TAB)[gl] = make_uint2(__float_as_uint(lo), __float_as_uint(hi));
                    if (first) {
                        d[gl / WL] = scale;
                        d[NAG + gl / WL] = bias;
                    }
                    continue;
                }
                float x0 = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f;
                {
                    const size_t k0 = ((size_t)c * NG + gl) * 4;
                    if (xe) {
                        if (valid) {
                            const float4 f = *reinterpret_cast<const float4 *>(xe + k0);
                            x0 = f.x; x1 = f.y; x2 = f.z; x3 = f.w;
                        }
                    } else {
                        wait_words<kSeqSpinLimit>(xl + k0, valid, epoch, p.err, 3, x0, x1, x2, x3);
                        if constexpr (GLU)
                            if (xl2) {
                                float u0, u1, u2, u3;
                                wait_words<kSeqSpinLimit>(xl2 + k0, valid, epoch, p.err, 3, u0, u1, u2, u3);
                                x0 = swiglu(x0, u0); x1 = swiglu(x1, u1); x2 = swiglu(x2, u2); x3 = swiglu(x3, u3);
                            }
                    }
                }
                uint32_t lo, hi;
                float scale;
                const float bias = lut_record<WL>(x0, x1, x2, x3, lane, lo, hi, scale);
                if (valid) reinterpret_cast<uint2 *>(tabs + (size_t)ci * TAB)[gl] = make_uint2(lo, hi);
                if (valid && (gl % WL) == 0) {
                    d[gl / WL] = scale;
                    d[NAG + gl / WL] = bias;
                }
            }
        }
        if (tr && tid == 0) tr[1] = globaltimer_ns();   // (stamps right after a bar.sync would show its issue, not its release)
        if (tw) tw[1] = clock64();
        seq_bar(1);
        long long ck1 = 0;
        if (tw) { const int dummy = ld_volatile_s32(prog + NW); ck1 = clock64() + (dummy == -12345); tw[2] = ck1; }

        // ---- (B) lookups over my units (unit = one activation group of one block) ----
        for (int s = 0; s < nseg; ++s) {                       // rows of super-blocks I do not touch must read as zero
            float *r = red + ((size_t)s * NW + warp) * RSB + lane * RW;
#pragma unroll
            for (int i = 0; i < RW; ++i) r[i] = 0.f;
        }
        {
            float cacc[RW];
            int iacc[RW];
#pragma unroll
            for (int i = 0; i < RW; ++i) { cacc[i] = 0.f; iacc[i] = 0; }
            int cur_seg = -1;
            for (int pass = 0; pass < npass; ++pass) {
            const int pb0 = pass * P, pb1 = min(nb, pb0 + P);
            const int nu = (pb1 - pb0) * NAG;
            const int u1 = pb0 * NAG + (nu * (warp + 1)) / NW;
            int u = pb0 * NAG + (nu * warp) / NW;
            int j = u / NAG;
            int sb = sb_first, c = c0 + j;
            while (c >= nchunk) { c -= nchunk; ++sb; }
            int slot = slot_base + j, par = par_base;
            while (slot >= p.nslots) { slot -= p.nslots; par ^= 1; }
            if (u < u1 && lane == 0) st_volatile_s32(prog + warp, seq_base + j);
            while (u < u1) {
                const int a0 = u - j * NAG, a1 = min(NAG, a0 + (u1 - u));
                const int seg = sb - sb_first;
                if (seg != cur_seg) {
                    if (cur_seg >= 0) {
                        float *r = red + ((size_t)cur_seg * NW + warp) * RSB + lane * RW;
#pragma unroll
                        for (int i = 0; i < RW; ++i) { r[i] = cacc[i]; cacc[i] = 0.f; }
                    }
                    cur_seg = seg;
                }
                int ci = c - c0; if (ci < 0) ci += nchunk;
                const unsigned char *tab = tabs + (size_t)ci * TAB;
                const float *ls = lsb + (size_t)ci * (2 * NAG);
                {
                    const long long tw0 = tr ? clock64() : 0;
                    if (tw && ck1) tw[3] = tw0;
                    int spins = 0;
                    while (ld_volatile_s32(issued) <= seq_base + j && ++spins < kSeqSpinLimit) __nanosleep(100);
                    if (spins >= kSeqSpinLimit || !mbar_wait_bounded<kSeqSpinLimit>(full + slot, (uint32_t)par)) atomicExch(p.err, 4);
                    if (tr && lane == 0 && (warp == 0 || warp == NW - 1)) tr[warp == 0 ? 10 : 11] += clock64() - tw0;   // cycles waiting for weights
                }
                if (tr && tid == 0 && u == 0) tr[2] = globaltimer_ns();   // first block of the share is resident
                if (tw && ck1) { tw[4] = clock64(); ck1 = 0; }           // my first block is resident
                const unsigned char *stage = ring + (size_t)slot * p.slot_bytes;
                const uint4 *wp = reinterpret_cast<const uint4 *>(stage) + lane;
                float facc[RW];
#pragma unroll
                for (int i = 0; i < RW; ++i) facc[i] = 0.f;
                float lbp = 0.f;                                // LUT biases of the activation groups [a0, a1)
                for (int a = a0; a < a1; ++a) {
#pragma unroll
                    for (int qq = 0; qq < AGQ; ++qq) TMAC_QUAD_LOOKUP(PB, true, wp, tab, a * AGQ + qq, wtx, wty, iacc);
                    TMAC_GROUP_FOLD(PB, ls[a], iacc, facc);
                    lbp += ls[NAG + a];
                }
                {
                    // TMAC_BLOCK_SCALES's arithmetic with lbsum = lbp, but the fp16 scales read with one vector load per lane:
                    // the macro's per-row load_scale made this kernel ~5% slower on the 32 x 11008x4096 W2 chain (H100 SXM, 700 W)
                    const unsigned char *sp = stage + (size_t)QCH * 512;
                    float sv[RW], zv[RW];
                    if (one_scale) {
#pragma unroll
                        for (int i = 0; i < RW; ++i) { sv[i] = scale0; zv[i] = 0.f; }
                    } else if (sd == 2) {                  // fp16 scales: the lane's RW values with one vector load
                        load_half_vec<RW>(sp + (size_t)lane * RW * 2, sv);
                        if (zp) load_half_vec<RW>(sp + (size_t)RSB * 2 + (size_t)lane * RW * 2, zv);
                    } else {
#pragma unroll
                        for (int i = 0; i < RW; ++i) {
                            sv[i] = reinterpret_cast<const float *>(sp)[lane * RW + i];
                            if (zp) zv[i] = reinterpret_cast<const float *>(sp + (size_t)RSB * 4)[lane * RW + i];
                        }
                    }
#pragma unroll
                    for (int i = 0; i < RW; ++i) {
                        float v = fmaf(0.5f * sv[i], facc[i] + lbp, cacc[i]);
                        if (zp) v = fmaf(zv[i], lbp, v);
                        cacc[i] = v;
                    }
                }
                u += a1 - a0;
                if (a1 == NAG) {                                // on to the next block
                    ++j;
                    if (++c == nchunk) { c = 0; ++sb; }
                    if (++slot == p.nslots) { slot = 0; par ^= 1; }
                    if (u < u1 && lane == 0) st_volatile_s32(prog + warp, seq_base + j);
                }
            }
            __syncwarp();
            if (lane == 0) st_volatile_s32(prog + warp, seq_base + pb1);
            }
            if (cur_seg >= 0) {
                float *r = red + ((size_t)cur_seg * NW + warp) * RSB + lane * RW;
#pragma unroll
                for (int i = 0; i < RW; ++i) r[i] = cacc[i];
            }
        }
        if (tr && lane == 0 && (warp == 0 || warp == NW / 2 || warp == NW - 1)) tr[warp == 0 ? 3 : (warp == NW - 1 ? 4 : 5)] = globaltimer_ns();
        if (tw) tw[5] = clock64();
        if (tid < 56) desc[((op + 1) & 1) * kSeqDescWords + tid] = next_word;
        seq_bar(2);

        // ---- (C) per (super-block, row): sum the warps in fixed order, then publish the partial sum or finish the row ----
        for (int item = tid; item < nseg * RSB; item += NW * 32) {
            const int s = item / RSB, t = item - s * RSB;
            const int sb = sb_first + s;
            const bool ends_here = !(last_open && s == nseg - 1);
            float mine = 0.f;
#pragma unroll 4
            for (int w = 0; w < NW; ++w) mine += red[((size_t)s * NW + w) * RSB + t];
            if (tr && item == 0) tr[6] = globaltimer_ns() + (mine == 1.2345e-30f); // after the barrier released and the sums are in
            if (tw && item < NW * 32) tw[6] = clock64() + (mine == 1.2345e-30f);
            if (!ends_here) {                                   // continues in the next CTA (always my last super-block)
                seq_publish(xchg + (size_t)cta * RSB + t, __float_as_uint(mine), epoch);
                continue;
            }
            float fsum = 0.f;
            if (s == 0) {                                       // started in earlier CTAs: their partial sums, ascending K order
                for (int k2 = fc; k2 < cta; ++k2) {             // (RSB is a multiple of 32: the whole warp is in this branch)
                    float part;
                    wait_words<kSeqSpinLimit>(xchg + (size_t)k2 * RSB + t, true, epoch, p.err, 2, part);
                    fsum += part;
                }
            }
            fsum += mine;
            if (tw && item < NW * 32) tw[7] = clock64() + (fsum == 1.2345e-30f);
            const int row = sb * RSB + t;
            if (row < Mout) {
                if (Cout) store_out(Cout, row, fsum, out_f16);
                seq_publish(yv + row, __float_as_uint(fsum), epoch);
            }
            if (lut_out) yfin[item] = row < Mout ? fsum : 0.f;
            if (tw && item < NW * 32) tw[8] = clock64();
        }
        if (lut_out) {
            // the consumer's preprocessor for the rows finished here (row super-blocks that end in this CTA): thread = K-group of
            // 4 consecutive rows, built as on the consumer side
            const int nfin = nseg - last_open;
            constexpr int GPS = RSB / 4;                        // K-groups per row super-block
            constexpr int GPSW = (GPS + 31) & ~31;              // ... rounded up to whole warps
            if (nseg * RSB <= NW * 32) {
                // one loop iteration above: super-block s was finished by threads [s*RSB, (s+1)*RSB) -- whole warps -- so only
                // they synchronise (named barrier 4 + s), not the CTA
                if (tid < nfin * RSB) {
                    const int s = tid / RSB, t = tid - s * RSB;
                    asm volatile("bar.sync %0, %1;" ::"r"(4 + s), "r"(RSB) : "memory");
                    if (t < GPSW) {
                        const bool valid = t < GPS;
                        const float4 f = valid ? reinterpret_cast<const float4 *>(yfin)[s * GPS + t] : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (tw) tw[9] = clock64() + (f.x == 1.2345e-30f);
                        publish_lut_record<WL>(f, lane, valid, (size_t)(sb_first + s) * GPS + t, lut_out, ag_out, epoch);
                        if (tw) tw[10] = clock64();
                    }
                }
            } else {
                seq_bar(3);
                for (int t0 = warp * 32; t0 < nfin * GPS; t0 += NW * 32) {
                    const int t = t0 + lane;
                    const bool valid = t < nfin * GPS;
                    const float4 f = valid ? reinterpret_cast<const float4 *>(yfin)[t] : make_float4(0.f, 0.f, 0.f, 0.f);
                    // finished super-blocks are my first nfin ones
                    publish_lut_record<WL>(f, lane, valid, (size_t)sb_first * GPS + t, lut_out, ag_out, epoch);
                }
            }
        }
        if (tr && tid == 0) tr[7] = globaltimer_ns();
        if (tw) tw[11] = clock64();
        seq_base += nb;
        slot_base += nb;
        while (slot_base >= p.nslots) { slot_base -= p.nslots; par_base ^= 1; }
    }
    if (tid == 0) p.epochs[cta] = epoch;
}

typedef void (*seq_fn)(const SeqParams, const uint32_t, const uint32_t);
// Defined in tmac_seq.cu (its own translation unit); nullptr = chunking not instantiated.
seq_fn pick_seq(int pb, int qch, int agq, bool glu);

}  // namespace tmac_b200
