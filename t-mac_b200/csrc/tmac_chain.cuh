// tmac_chain.cuh -- the dependent chain of GEMVs as ONE persistent launch, second form: gemv3's decomposition kept resident.
//
// tmac_seq.cuh (stream-K shares, partial sums and LUT records exchanged through HBM words) turned out latency-bound at the
// granularity of one 12.7 MB GEMV: three CTA-wide phases and two inter-CTA hops per op (DESIGN.md section 3.4).  This kernel
// keeps what measured well in the launch chain -- gemv3's decomposition: cluster of 4 CTAs x 4 warps per 128-row super-block,
// one (super-block, chunk) block per warp, LUT slice built by the warp itself, K slices summed in the leader's shared memory
// in rank order -- and removes what the launch chain loses per launch:
//   * the kernel boundary becomes DATA FLOW: the leader of each cluster writes its rows as {value, epoch} words next to C, and a
//     warp of the next op waits for exactly the 128 input values of its chunk (one producer cluster), not for a grid barrier;
//   * the cluster-wide rendezvous of the reduction becomes one DSMEM hop: peers send their partial sums with st.async, whose
//     completion bytes are counted on the leader's mbarrier (data and signal travel together); a split-phase cluster barrier,
//     waited for a whole op later, only guards the re-use of the buffers;
//   * the exposed weight stream: a warp's blocks over the whole chain form one sequence (op 0's chunks of this warp, then op 1's,
//     ...), loaded by one cp.async.bulk each (4.6 KB) into a per-warp ring of ChainParams::nstage stages.  When the warp starts
//     the lookups of block j it requests block j + nstage - 1 into the stage block j - 1 has vacated -- weights do not depend on
//     activations -- so the stream overlaps the ALU-bound phase and is out of the way of the latency-critical words (requesting
//     earlier, across the hand-over, puts 12.7 MB of bulk traffic in front of the words everybody waits for).  With nstage =
//     bpw + 1 every block is requested one full op before it is consumed; the host picks the deepest ring that keeps every
//     cluster resident.  The copies carry an L2 evict_first policy: a block is read once per launch, and its lines should leave
//     L2 before the {value, epoch} words, inputs and outputs that the ops after it read;
//   * CTA placement is fixed for the whole chain (344 CTAs of 128 threads for 11008 rows, all resident).
// bench.py times it on the bench chain (32 x 11008x4096 W2, x[i+1] = first K outputs of op i) beside the launch chain and
// tmac_seq.cuh; flags bit 0 selects the grid-barrier form this kernel started as, kept for comparison.  Per-phase stamps
// (ChainParams::trace) are read by tools/seq_bench.py --trace.
// The LUT slices are built by lut_slice, the code gemv3's fused path runs, and the blocks by TMAC_BLOCK_LOOKUPS /
// TMAC_BLOCK_SCALES (tmac_kernels.cuh), gemv3's block step, so LUT bytes, scales and biases are identical
// to the preprocessor's and a block's fp32 operation order is gemv3's; fp32 sums in fixed (warp, then cluster rank) order;
// the K split differs from the lone launch's, so results equal tmac_b200_gemv's up to fp32 re-association.  Waits are
// bounded (error flag): mbar_wait_bounded, and wait_words of tmac_seq.cuh for the producer's {value, epoch} words.
// A GLU op (the down projection of a SwiGLU FFN) reads two producers, gate and up: its warps wait for both producers' words of
// the chunk (flow form) or load both (barrier form) and build the LUT slice of swiglu(gate, up).
// Decode-ahead (template QD > 0): the weight part of a block's first QD quads (quad_decode) needs only the block, which the ring
// has staged an op earlier, so a warp waits for the block and decodes those quads before it waits for the chunk's input, while
// its ALU pipe is otherwise idle; after the LUT slice it runs only their table part.  The decoded quads live in registers, so
// this instantiation is bounded to 3 CTAs per SM; seq_build_chain falls back to QD = 0 (5 CTAs per SM) when a sequence needs
// more.  Both compute the same bits.
// The decode-ahead instantiation also loads the input words of a warp's next chunk as the current chunk's lookups start
// (load_words4): when its producer has published by then, the next chunk's wait costs no L2 round trip (wait_loaded_words4).
// QD = 0 does not: its registers are what lets 11008-row W3 / W4 chains (688 CTAs) keep 6 CTAs per SM.
#pragma once
#include "tmac_kernels.cuh"
#include "tmac_seq.cuh"     // {value, epoch} words: seq_publish, wait_words

namespace tmac_b200 {

constexpr int kChainCS = 4;                 // CTAs per cluster (K slices of one row super-block): 4 keeps the 86 clusters of an
                                            // 11008-row op resident on 132 SMs (8 would need 688 CTAs, 5 fit per SM)
constexpr int kChainWarps = 4;              // warps per CTA
constexpr int kChainSpin = 1 << 22;
constexpr int kChainBarrier = 1;            // ChainParams::flags bit 0: grid barrier between ops instead of data flow
constexpr int kChainAhead = 4;              // quads per block decoded ahead by the decode-ahead instantiation: 16 registers each,
                                            // 137 registers in chain_kernel<2,8,4> (2, 5, 6 and 8 quads measured slower)

struct ChainOp {
    const unsigned char *W;                 // stream layout of the tensor
    const float *x;                         // input vector [K] (external, or an earlier op's C + offset)
    void *C;                                // output [Mout]
    unsigned long long rsb_stride;
    int K, Mout, nrsb, nchunk;
    int blk_bytes, bpw;                     // bytes per block; chunks per warp = ceil(nchunk / (kChainCS * kChainWarps))
    int zp, one_scale, sd, out_f16;
    float scale0;
    int in_op;                              // producer op of x, or -1 (external input)
    uint2 *ll_out;                          // [rows] {value bits, epoch} words written next to C
    const uint2 *ll_in;                     // the producer's words, already offset (NULL: external input, plain loads)
    // multi-GPU row sharding (as Gemv3Params::Cpeer): the finished rows are also stored straight into the peers' output vectors
    int npeer, pad_;
    void *Cpeer[7];
};

// The second input of a GLU op (read by chain_kernel<..., true> only): the op's input is swiglu(x[k], x2[k]) -- ChainOp::x / ll_in /
// in_op name the gate producer, these the up producer; x2 == NULL: a plain op.  Kept out of ChainOp so that the descriptor the
// plain instantiations read keeps its 160 bytes.
struct ChainGlu {
    const float *x2;
    const uint2 *ll_in2;
    int in_op2, pad_;
};

struct ChainParams {
    const ChainOp *ops;
    int nops;
    int max_blk;                            // bytes per stage
    int nstage;                             // stages per warp (>= 2): blocks are requested nstage - 1 blocks ahead
    unsigned int *bar;                      // grid barrier counter (barrier form; monotonic over launches)
    unsigned int *epochs;                   // [grid] launches seen by each CTA
    int *err;
    int flags;                              // kChainBarrier
    long long *trace;                       // debug: [nops][grid][16] globaltimer stamps of thread 0, or NULL
    const ChainGlu *glu;                    // [nops] second inputs of GLU ops (chain_kernel<..., true>), or NULL
};

// partial sum -> the leader's shared memory, completion counted on the leader's mbarrier
__device__ __forceinline__ void st_async_f32(float *local_ptr, uint64_t *local_bar, uint32_t rank, float v) {
    uint32_t ra, rb;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(local_ptr)), "r"(rank));
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(smem_u32(local_bar)), "r"(rank));
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra), "r"(__float_as_uint(v)), "r"(rb) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

// GLU: the sequence has GLU ops (ChainOp::x2).  A separate instantiation, so that the plain input path of the sequences without
// them keeps its code and registers.
// QD: the first QD quads of every block are decoded ahead (see the chunk loop): 0 in the instantiation that fits 5 CTAs per SM,
// kChainAhead in the one for 3 CTAs per SM.
template <int PB, int QCH, int AGQ, bool GLU, int QD>
__global__ void __launch_bounds__(kChainWarps * 32, QD ? 3 : 5) chain_kernel(const ChainParams p, const uint32_t wtx, const uint32_t wty) {
    constexpr int RW = 8 / PB, RSB = 32 * RW;
    constexpr int QA = QD < QCH ? QD : QCH;                        // quads decoded ahead
    constexpr int NAG = QCH / AGQ, NG = QCH * 4, WL = AGQ * 4;
    constexpr int WPC = kChainWarps, CS = kChainCS;
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = (int)cluster_ctarank(), rsb = blockIdx.x / CS;
    const int nclusters = gridDim.x / CS;
    const bool flow = !(p.flags & kChainBarrier);
    const int NS = p.nstage;
    // shared memory: cl [CS][RSB] (cluster partials, leader) | red [WPC][RSB] | per warp: NS stages (max_blk) + table (NG * 8) |
    //                mbar [WPC][NS] (bulk copies) | rmbar (leader: the peers' partial sums have landed)
    float *cl = reinterpret_cast<float *>(smem);
    float *red = cl + CS * RSB;
    unsigned char *wbase = reinterpret_cast<unsigned char *>(red + WPC * RSB);
    const int per_warp = NS * p.max_blk + NG * 8;
    unsigned char *stage0 = wbase + (size_t)warp * per_warp;
    unsigned char *tab = stage0 + (size_t)NS * p.max_blk;
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbase + (size_t)WPC * per_warp) + NS * warp;
    uint64_t *rmbar = reinterpret_cast<uint64_t *>(wbase + (size_t)WPC * per_warp) + NS * WPC;
    int nred = 0;                                                  // leader: reductions waited for (mbarrier phase)
    const unsigned epoch0 = p.epochs[blockIdx.x];                 // launches before this one
    const unsigned bar_base = epoch0 * (unsigned)p.nops * (unsigned)nclusters;

    if (lane == 0) {
        for (int s = 0; s < NS; ++s) mbar_init(mbar + s, 1);
        if (warp == 0) mbar_init(rmbar, 1);
        mbar_fence_init();
        fence_proxy_async();
    }
    __syncwarp();
    cluster_sync_all();                                            // every CTA of the cluster runs: its shared memory may be written

    // The warp's block sequence: for op 0, 1, ... the chunks c_slot * bpw .. min(nchunk, (c_slot + 1) * bpw) - 1 (none where the CTA
    // or the warp has no chunk).  Block j goes to stage j % NS, whose mbarrier it completes; stages are filled and consumed in ring
    // order, so the consumer's mbarrier phase flips once per lap.
    const int c_slot = rank * WPC + warp;
    int rop = -1, rc = 0, rc_end = 0, rs = 0;                      // sequence position: op, chunk, end of the op's chunks; stage
    // The ChainOp fields of the next block to request are loaded one request ahead and only combined at the request: the request
    // is made as a block's lookups start, and waiting there for global loads would delay the lookups once per block.
    const unsigned char *nw = nullptr;                             // the next block to request: tensor (NULL: none left), super-
    unsigned long long nstride = 0;                                // block stride, bytes per block, chunk
    int nbytes = 0, nc = 0;
    auto advance = [&]() {
        nw = nullptr;
        while (rc >= rc_end) {
            if (rop + 1 >= p.nops) return;
            const ChainOp &o = p.ops[++rop];
            rc = c_slot * o.bpw;
            rc_end = rsb < o.nrsb ? min(o.nchunk, rc + o.bpw) : rc;
        }
        const ChainOp &o = p.ops[rop];
        nw = o.W; nstride = o.rsb_stride; nbytes = o.blk_bytes; nc = rc;
        ++rc;
    };
    // stage rs <- the next block of the sequence (one bulk copy), if there is one
    auto request_next = [&]() {
        if (!nw) return;
        if (lane == 0) {
            fence_proxy_async();
            bulk_load_hint(stage0 + (size_t)rs * p.max_blk, nw + (size_t)rsb * nstride + (size_t)nc * nbytes, (uint32_t)nbytes, mbar + rs,
                           policy_evict_first());
        }
        if (++rs == NS) rs = 0;
        advance();
    };
    advance();
    for (int s = 1; s < NS; ++s) request_next();                   // blocks 0 .. NS - 2
    int cs = 0;                                                    // stage of the next block to consume
    uint32_t cph = 0;                                              // its mbarrier phase

    for (int op = 0; op < p.nops; ++op) {
        const ChainOp &o = p.ops[op];
        const int nchunk = o.nchunk, bpw = o.bpw, zp = o.zp, sd = o.sd, one_scale = o.one_scale;
        const float scale0 = o.scale0;
        const float *x = o.x;
        // read once per op, before the waits: every asm volatile below (polls, mbarrier waits, barriers) would otherwise force a
        // reload of the ChainOp field right where the waited-for data has arrived
        const uint2 *const ll_in = o.ll_in;
        uint2 *const ll_out = o.ll_out;
        void *const C = o.C;
        const int Mout = o.Mout, out_f16 = o.out_f16, npeer = o.npeer;
        const bool active = rsb < o.nrsb;
        const int c_first = c_slot * bpw, c_end = min(nchunk, c_first + bpw);
        const uint32_t ep_in = epoch0 * (uint32_t)p.nops + (uint32_t)o.in_op + 1u, ep_out = epoch0 * (uint32_t)p.nops + (uint32_t)op + 1u;
        const float *x2 = nullptr;                                 // GLU op: the up producer's rows (x, ll_in: the gate's)
        const uint2 *ll_in2 = nullptr;
        uint32_t ep_in2 = 0;
        if constexpr (GLU) {
            const ChainGlu &q = p.glu[op];
            x2 = q.x2; ll_in2 = q.ll_in2; ep_in2 = epoch0 * (uint32_t)p.nops + (uint32_t)q.in_op2 + 1u;
        }
        long long *tr = (p.trace && tid == 0) ? p.trace + ((size_t)op * gridDim.x + blockIdx.x) * 16 : nullptr;
        if (tr) tr[0] = globaltimer_ns();
        if (op > 0 && !flow) {
            // ---- barrier form: every cluster has stored op-1's rows (release-increment by its leader); one polling thread per CTA ----
            if (tid == 0) {
                const unsigned target = bar_base + (unsigned)op * (unsigned)nclusters;
                int spins = 0;
                while ((int)(ld_acquire_u32(p.bar) - target) < 0 && ++spins < kChainSpin) { }
                if (spins >= kChainSpin) atomicExch(p.err, 1);
            }
            if (tr) tr[1] = globaltimer_ns();
            __syncthreads();
        }
        if (tr) tr[2] = globaltimer_ns();
        float cacc[RW];
        int iacc[RW];
#pragma unroll
        for (int i = 0; i < RW; ++i) { cacc[i] = 0.f; iacc[i] = 0; }
        // the input words of the warp's next chunk, loaded as the current chunk's lookups start (preloaded: they were)
        uint4 nw0 = make_uint4(0u, ep_in, 0u, ep_in), nw1 = nw0;
        bool preloaded = false;
        if (active)
            for (int c = c_first; c < c_end; ++c) {
                // ---- decode ahead: the weight part of the block's first QA quads, which reads only the block, goes before the
                // input wait, where the ALU pipe is idle; the lookups then run only the table part of those quads ----
                QuadCodes qc[QA ? QA : 1];
                if constexpr (QA > 0) {
                    if (!mbar_wait_bounded<kChainSpin>(mbar + cs, cph)) atomicExch(p.err, 2);
                    const uint4 *wp = reinterpret_cast<const uint4 *>(stage0 + (size_t)cs * p.max_blk) + lane;
#pragma unroll
                    for (int q = 0; q < QA; ++q) qc[q] = quad_decode<true>(wp[q * 32], wtx);
                }
                // ---- LUT slice of this chunk -> warp-private table (lane = group) ----
                float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
                if (flow && ll_in) {                               // the producer's rows, as soon as they exist
                    if (preloaded)
                        wait_loaded_words4<kChainSpin>(ll_in + ((size_t)c * NG + lane) * 4, lane < NG, ep_in, p.err, 5, nw0, nw1, b0, b1, b2, b3);
                    else
                        wait_words<kChainSpin>(ll_in + ((size_t)c * NG + lane) * 4, lane < NG, ep_in, p.err, 5, b0, b1, b2, b3);
                    if constexpr (GLU)
                        if (ll_in2) {
                            float u0, u1, u2, u3;
                            wait_words<kChainSpin>(ll_in2 + ((size_t)c * NG + lane) * 4, lane < NG, ep_in2, p.err, 5, u0, u1, u2, u3);
                            b0 = swiglu(b0, u0); b1 = swiglu(b1, u1); b2 = swiglu(b2, u2); b3 = swiglu(b3, u3);
                        }
                    if (lane >= NG) b0 = b1 = b2 = b3 = 0.f;
                } else if (lane < NG) {
                    const float4 f = __ldcg(reinterpret_cast<const float4 *>(x + ((size_t)c * NG + lane) * 4));   // L2: written by other SMs
                    b0 = f.x; b1 = f.y; b2 = f.z; b3 = f.w;
                    if constexpr (GLU)
                        if (x2) {
                            const float4 u = __ldcg(reinterpret_cast<const float4 *>(x2 + ((size_t)c * NG + lane) * 4));
                            b0 = swiglu(b0, u.x); b1 = swiglu(b1, u.y); b2 = swiglu(b2, u.z); b3 = swiglu(b3, u.w);
                        }
                }
                float lsv[NAG];
                const float lbsum = lut_slice<WL, NAG>(b0, b1, b2, b3, lane, tab, lsv);
                if (tr) tr[3] = globaltimer_ns();
                if constexpr (QA == 0)
                    if (!mbar_wait_bounded<kChainSpin>(mbar + cs, cph)) atomicExch(p.err, 2);
                __syncwarp();
                if (tr) tr[4] = globaltimer_ns();
                // block j + NS - 1 is requested as block j's lookups start, into the stage of block j - 1 (its lookups ended with the
                // __syncwarp at the end of the previous chunk; the proxy fence in request_next orders them before the bulk copy)
                request_next();
                // the next chunk's words, while the lookups run: if its producer has published by then, its wait is one ballot
                preloaded = QA > 0 && flow && ll_in && c + 1 < c_end;
                if (preloaded && lane < NG) load_words4(ll_in + ((size_t)(c + 1) * NG + lane) * 4, nw0, nw1);
                const unsigned char *stage = stage0 + (size_t)cs * p.max_blk;
                float facc[RW];
                TMAC_BLOCK_LOOKUPS_AHEAD(PB, true, QCH, AGQ, QA, qc, stage, tab, lane, wtx, wty, lsv, iacc, facc);
                TMAC_BLOCK_SCALES(PB, QCH, stage, lane, one_scale, scale0, sd, zp, facc, lbsum, cacc);
                __syncwarp();                                      // stage / table are rewritten by later chunks
                if (++cs == NS) { cs = 0; cph ^= 1u; }
            }
        if (tr) tr[5] = globaltimer_ns();

        // ---- CTA reduction (fixed warp order), cluster reduction in the leader's shared memory (rank order), leader stores the rows ----
        if (flow && op > 0) cluster_wait();                        // every thread of the cluster is past op-1's reduction: red / cl may be rewritten
        {
            float *r = red + (size_t)warp * RSB + lane * RW;
#pragma unroll
            for (int i = 0; i < RW; ++i) r[i] = cacc[i];
        }
        __syncthreads();
        if (tr) tr[6] = globaltimer_ns();
        if (flow) {
            // peers send their partial with st.async (completion bytes counted on the leader's mbarrier); the leader sums in rank
            // order once (CS-1) x RSB floats have landed: one DSMEM hop instead of a cluster-wide rendezvous
            if (active) {
                if (rank == 0 && tid == 0)
                    expect_tx(rmbar, (uint32_t)((CS - 1) * RSB * 4));
                for (int t = tid; t < RSB; t += WPC * 32) {
                    float fsum = 0.f;
#pragma unroll
                    for (int w = 0; w < WPC; ++w) fsum += red[(size_t)w * RSB + t];
                    if (rank == 0) cl[t] = fsum;                   // read back by the same thread below
                    else st_async_f32(cl + (size_t)rank * RSB + t, rmbar, 0, fsum);
                }
                if (tr) tr[7] = globaltimer_ns();
                if (rank == 0) {
                    if (!mbar_wait_bounded<kChainSpin>(rmbar, nred & 1)) atomicExch(p.err, 6);
                    ++nred;
                    for (int t = tid; t < RSB; t += WPC * 32) {
                        float fsum = 0.f;
#pragma unroll
                        for (int k2 = 0; k2 < CS; ++k2) fsum += cl[(size_t)k2 * RSB + t];
                        const int row = rsb * RSB + t;
                        if (row < Mout) {
                            seq_publish(ll_out + row, __float_as_uint(fsum), ep_out);
                            store_out(C, row, fsum, out_f16);
                            for (int q = 0; q < npeer; ++q)          // the all-gather, fused into the epilogue: one store per peer and row
                                store_out(o.Cpeer[q], row, fsum, out_f16);
                        }
                    }
                    if (tr) tr[8] = globaltimer_ns();
                }
            }
            cluster_arrive_relaxed();                              // split-phase: waited for before the next op's partials are written
        } else {
            for (int t = tid; t < RSB; t += WPC * 32) {
                float fsum = 0.f;
#pragma unroll
                for (int w = 0; w < WPC; ++w) fsum += red[(size_t)w * RSB + t];
                st_cluster_f32(cl + (size_t)rank * RSB + t, 0, fsum);
            }
            cluster_sync_all();
            if (tr) tr[7] = globaltimer_ns();
            if (rank == 0) {
                if (active)
                    for (int t = tid; t < RSB; t += WPC * 32) {
                        float fsum = 0.f;
#pragma unroll
                        for (int k2 = 0; k2 < CS; ++k2) fsum += cl[(size_t)k2 * RSB + t];
                        const int row = rsb * RSB + t;
                        if (row < Mout) {
                            store_out(C, row, fsum, out_f16);
                            for (int q = 0; q < npeer; ++q) store_out(o.Cpeer[q], row, fsum, out_f16);
                        }
                    }
                __syncthreads();                                   // the release below is cumulative over the CTA's stores
                if (tid == 0) asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p.bar), "r"(1u) : "memory");
                if (tr) tr[8] = globaltimer_ns();
            }
        }
    }
    if (tid == 0) {
        if (!flow) {
            // the last increments must be in before the next launch computes its base from its own epoch: every CTA passes one final
            // barrier so that no cluster of a later launch can see a counter that is still being incremented by this one
            const unsigned target = bar_base + (unsigned)p.nops * (unsigned)nclusters;
            int spins = 0;
            while ((int)(ld_acquire_u32(p.bar) - target) < 0 && ++spins < kChainSpin) { }
            if (spins >= kChainSpin) atomicExch(p.err, 3);
        }
        p.epochs[blockIdx.x] = epoch0 + 1u;
    }
    if (flow) cluster_wait();                                      // completes the last split-phase barrier
    cluster_sync_all();                                            // nobody leaves while a peer may still write its shared memory
}

typedef void (*chain_fn)(const ChainParams, const uint32_t, const uint32_t);
// ahead: the decode-ahead instantiation (QD = kChainAhead, bounded to 3 CTAs per SM), else QD = 0 (5 CTAs per SM)
chain_fn pick_chain(int pb, int qch, int agq, bool glu, bool ahead);

}  // namespace tmac_b200
