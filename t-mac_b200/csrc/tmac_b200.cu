// tmac_b200.cu -- host side of libtmac_b200.so: context, resident-weight registry, kcfg registry,
// pointer-domain handling and the C ABI declared in include/tmac_b200.h.
//
// Mirrors, for the hot path only:
//   * the generated dispatchers qgemm_lut_int8 / preprocessor_int8 (deploy/compile.py:60-67),
//   * TMAC::TMACGeMMWrapper::{llama_cpp_init, llama_cpp_compute, get_kcfg}
//     (include/t-mac/tmac_gemm_wrapper.h:173-255),
//   * the ggml hook (3rdparty/llama.cpp/ggml/src/ggml-tmac.cpp).
// There is no CPU fallback anywhere in this file: every compute entry point launches CUDA
// kernels or fails with -1.
#include "../../include/tmac_b200.h"

#include <algorithm>
#include <atomic>
#include <functional>
#include <thread>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sys/mman.h>
#include <map>
#include <mutex>
#include <shared_mutex>
#include <set>
#include <string>
#include <tuple>
#include <vector>

#include "tmac_kernels.cuh"
#include "tmac_prefill.cuh"
#include "tmac_prefill16.cuh"
#include "tmac_seq.cuh"
#include "tmac_chain.cuh"
#include "tmac_layout.h"
#include "tmac_gguf.h"

using namespace tmac_b200;

namespace tmac_b200 {
template gemv3_fn pick_gemv3_in<kInTable>(int, bool, int, int, int);   // the other kinds: tmac_gemv_io.cu, tmac_gemv_experts.cu
}

namespace {

thread_local std::string t_err;
int fail(const std::string &m) { t_err = m; return -1; }
#define CUDA_OK(expr)                                                                              \
    do {                                                                                           \
        cudaError_t e_ = (expr);                                                                   \
        if (e_ != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(e_));    \
    } while (0)

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = std::max(n, (size_t)4096);
        if (cudaMalloc(&p, want) != cudaSuccess) return -1;
        cap = want;
        return 0;
    }
};
struct PinBuf {
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return 0;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = std::max(n, (size_t)65536);
        if (cudaMallocHost(&p, want) != cudaSuccess) return -1;
        cap = want;
        return 0;
    }
};

struct Resident {
    tmac_b200_kcfg cfg{};
    StreamLayout L{};
    unsigned char *d = nullptr;          // stream layout in HBM
    const unsigned char *host_a = nullptr;  // alias key: reference-layout host range
    size_t host_a_bytes = 0;
    int row0 = 0;                        // first row of the full tensor held here (row shards)
    void *reserved = nullptr;            // address range reserved (PROT_NONE, no memory) to serve as the host alias key
    size_t reserved_bytes = 0;
    float *host_scales = nullptr;        // scales in the reference's run-time order, owned here (tmac_tensor_extra::scales)
    int64_t id = 0;                      // its handle
};

// A LUT that lives in CALLER host memory (the reference's workspace, ref:ggml.c:12566-12576) and its device-resident copy.
// ggml writes the LUT once per mat-vec (task_init) and then calls task_compute once per weight tile with the same pointers
// (ref:ggml.c:12662-12691): the copy is keyed by the host QLUT pointer AND compared with the bytes the call passes, so a caller that
// rewrites the table is never served stale data, and the first tile call computes the whole tensor once (`res`), later tile
// calls of the same (LUT bytes, tensor) copy their rows out.
struct HostLut {
    const void *hq = nullptr;
    std::vector<unsigned char> copy;     // the bytes the device copy was made from: QLUT || LUT_Scales || LUT_Biases (empty = invalid)
    size_t qb = 0, sb = 0;
    int N = 0;
    DevBuf dq, dls, dlb;
    bool sym = false;
    int64_t res_id = 0;                  // tensor whose full result `res` holds (0 = none)
    int res_dtype = 0;
    PinBuf res;                          // [N][Mout] in page-locked host memory, written by the kernel itself
    uint64_t stamp = 0;
};

struct Context {
    bool inited = false;
    int device = 0, sms = 132;
    cudaStream_t own = nullptr, user = nullptr;
    bool use_user = false;
    int float_type = TMAC_B200_F32;
    int lut_mode = 0;                    // 0 auto, 1 general, 2 symmetric
    int use_pdl = 1;
    int cs_override = 0, wpc_override = 0, pdl_late = -1, minb_override = 0, nbuf_override = 0;
    int last_launch[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int use_fused = 1;
    int seq_impl = 2;                    // decode sequences: 0 = stream-K sequence kernel (tmac_seq.cuh), 1 = resident gemv3 chain (tmac_chain.cuh), 2 = chain when the sequence qualifies
    int seq_smem_kb = 200;               // decode sequences: shared-memory budget; the rest of the 228 KB stays L1 (descriptor / polling loads, spills)
    int seq_grid = 0;                    // decode sequences: grid override (tests: CTA-boundary placements); 0 = one CTA per SM
    int seq_handover = 1;                // stream-K sequence kernel: producers hand their consumers built LUT records; 0 = consumers build them
    int scales_f32 = 0;                  // weight uploads: store scales as fp32 even when every one is fp16-exact
    int use_prefill16 = 1;               // fp16-operand prefill tile for N >= 64 (tmac_prefill16.cuh); 0 = the exact int8 tile for every N >= tile_min_n
    int pf_streamk = 0;                  // stream-K over all SMs when a prefill call has fewer tiles than SMs (measured slower: B delivery from L2 is the bound)
    int use_prefill = 1, prefill_min_n = 0;    // N >= prefill_min_n: the wgmma tiles (W2, W3/W4, takes_prefill_tile); 0 = by shape (tile_min_n)
    int npeer = 0; void *peer_out[7] = {};   // one-shot: peer output vectors of the next N = 1 launch (tmac_b200_peer_outputs)
    int64_t next_hint = 0;               // one-shot: tensor whose blocks the next launch prefetches into L2
    std::map<int64_t, Resident> res;
    int64_t next_handle = 1;
    std::vector<tmac_b200_kcfg> kcfgs;
    HostLut hluts[4];
    uint64_t hlut_clock = 0;
    std::set<const void *> sym_qluts;    // device QLUT buffers last written by our preprocessor
    std::vector<std::pair<std::vector<const void *>, void *>> ptr_tables;   // grouped-launch pointer tables
    // workspaces
    DevBuf d_b, d_qlut, d_ls, d_lb, d_c, d_cbits, d_trace, d_tiles, d_pf_scratch, d_pf_flags;
    DevBuf d_moe_ws, d_moe_cnt;          // tmac_b200_gemv_experts_glu: the slots' rows and the arrival counters (zero between launches)
    DevBuf d_moe_route, d_moe_act;       // tmac_b200_prefill_experts / _glu: tile table + sorted slots; the GLU form's fp32 inputs
    int trace = 0, trace_ctas = 0, trace_seq = 0;
    int chain_flags = 0;                 // resident chain (tmac_chain.cuh): bit 0 = grid-barrier form (comparison); default: data flow
    int chain_ahead = 1;                 // resident chain: 0 = never the decode-ahead instantiation (comparison); default: when it fits
    PinBuf h_in, h_out;
    cudaEvent_t stage_ev = nullptr;      // last H2D that read h_in
    bool stage_pending = false;
    cudaStream_t stream() const { return use_user ? user : own; }
};

// Tuning / A-B knobs: read from TMAC_B200_<KEY in upper case> at init, settable with tmac_b200_debug_set(key) afterwards.
struct Knob { const char *key; int Context::*field; };
const Knob kKnobs[] = {
    {"lut_mode", &Context::lut_mode}, {"pdl", &Context::use_pdl}, {"pdl_late", &Context::pdl_late}, {"cs", &Context::cs_override},
    {"wpc", &Context::wpc_override}, {"minb", &Context::minb_override}, {"nbuf", &Context::nbuf_override},
    {"fused", &Context::use_fused}, {"prefill", &Context::use_prefill}, {"prefill16", &Context::use_prefill16},
    {"pf_streamk", &Context::pf_streamk}, {"prefill_min_n", &Context::prefill_min_n}, {"scales_f32", &Context::scales_f32},
    {"trace", &Context::trace}, {"seq_impl", &Context::seq_impl}, {"seq_handover", &Context::seq_handover},
    {"seq_grid", &Context::seq_grid}, {"seq_smem_kb", &Context::seq_smem_kb}, {"chain_flags", &Context::chain_flags},
    {"chain_ahead", &Context::chain_ahead},
};

Context g;
std::shared_mutex g_mu;     // exclusive for everything that launches or mutates; shared for the read-only tile fast path
std::map<int64_t, GgufFile *> g_gguf;    // open GGUF files (tmac_b200_gguf_*)
int64_t g_next_gguf = 1;

std::map<int64_t, cudaGraphExec_t> g_graphs;   // tmac_b200_graph_*
int64_t g_next_graph = 1;

// decode sequences (tmac_b200_seq_*)
// in_op2 >= 0: a GLU op (tmac_b200_seq_add_gemv_glu), input swiglu(output of in_op at in_off, output of in_op2 at in_off2)
// nw != NULL: a norm op (tmac_b200_seq_add_gemv_rmsnorm) over the whole output of in_op; res: a residual (tmac_b200_seq_residual),
// the external vector r or the output of op r_op
struct SeqOpHost {
    int64_t handle; const void *x_ext; int in_op, in_off; void *C; int out_f16; int npeer = 0; void *peer[7] = {}; int in_op2 = -1, in_off2 = 0;
    const float *nw = nullptr; float eps = 0.f; bool res = false; const float *r = nullptr; int r_op = -1;
    bool layer() const { return nw || res; }
};
// The launch shape of a sequence kernel: grid CTAs of `threads` threads with smem bytes of dynamic shared memory, and one launch
// attribute (the chain kernel's clusters, the stream-K kernel's cooperative launch).
struct SeqLaunch {
    int grid = 0, threads = 0;
    size_t smem = 0;
    cudaLaunchAttribute attr{};
    cudaLaunchConfig_t config(cudaStream_t st) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cfg.attrs = &attr; cfg.numAttrs = 1;
        return cfg;
    }
};
// chain_kernel's: grid CTAs in clusters of kChainCS
SeqLaunch chain_launch(int grid, size_t smem) {
    SeqLaunch l{grid, kChainWarps * 32, smem};
    l.attr.id = cudaLaunchAttributeClusterDimension;
    l.attr.val.clusterDim.x = kChainCS; l.attr.val.clusterDim.y = 1; l.attr.val.clusterDim.z = 1;
    return l;
}
struct Sequence {
    std::vector<SeqOpHost> ops;
    bool built = false;
    int pb = 0, qch = 0, agq = 0, bits = 0;
    int nb = 1;                           // activation rows (tmac_b200_seq_set_batch)
    SeqLaunch launch;
    seq_fn fn = nullptr;
    SeqParams params{};
    int impl = 0;                         // 1: chain_kernel
    chain_fn cfn = nullptr;
    ChainParams cparams{};
    void *d_mem = nullptr;                // the one device allocation: descriptors, words, flags and trace of the built kernel
    int *d_err = nullptr;                 // views into d_mem: the error flag, the trace (null: not traced)
    long long *d_trace = nullptr;
    void release() {
        if (d_mem) cudaFree(d_mem);
        d_mem = nullptr; d_err = nullptr; d_trace = nullptr; built = false;
    }
};
// Bytes of a sequence's trace: [ops][grid][16] stamps, then the stream-K kernel's [ops][grid][kSeqWarps][16] per-warp stamps
size_t seq_trace_bytes(size_t nops, int grid) { return nops * grid * (16 + 16 * kSeqWarps) * sizeof(long long); }
std::map<int64_t, Sequence> g_seqs;
int64_t g_next_seq = 1;

bool is_device_ptr(const void *p) {
    if (!p) return false;
    // ggml calls in once per weight tile with pointers into the same few host buffers: remember which 4 KB pages were ORDINARY
    // HOST memory (a page of host address space never becomes device memory; one that gets page-locked later is still valid to
    // treat as pageable), so that cudaPointerGetAttributes (~0.5 us) is not paid 4 times per tile
    static thread_local uintptr_t host_pages[64];
    const uintptr_t page = (uintptr_t)p >> 12, slot = page & 63;
    if (host_pages[slot] == page) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    if (a.type == cudaMemoryTypeUnregistered) host_pages[slot] = page;
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The entry whose device copy was made from exactly these host bytes (memcmp of ~17 KB: ~0.1 us), or null.
HostLut *hlut_find(const void *hq, const void *ls, const void *lb, size_t qb, size_t sb) {
    for (HostLut &e : g.hluts)
        if (e.hq == hq && e.qb == qb && e.sb == sb && e.copy.size() == qb + 2 * sb && !std::memcmp(e.copy.data(), hq, qb) &&
            !std::memcmp(e.copy.data() + qb, ls, sb) && !std::memcmp(e.copy.data() + qb + sb, lb, sb)) { e.stamp = ++g.hlut_clock; return &e; }
    return nullptr;
}
HostLut *hlut_slot(const void *hq) {     // the entry of this host pointer, else the least recently used one
    HostLut *best = &g.hluts[0];
    for (HostLut &e : g.hluts) {
        if (e.hq == hq) { best = &e; break; }
        if (e.stamp < best->stamp) best = &e;
    }
    best->hq = hq; best->copy.clear(); best->res_id = 0; best->stamp = ++g.hlut_clock;
    return best;
}

// 0 = ordinary host memory, 1 = page-locked host memory the device can address (dev = its device alias), 2 = device / managed
int ptr_kind(const void *p, void **dev = nullptr) {
    if (!p) return 0;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return 0; }
    if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return 2;
    if (a.type == cudaMemoryTypeHost && a.devicePointer) { if (dev) *dev = a.devicePointer; return 1; }
    return 0;
}

int ensure_init() {
    if (g.inited) {   // the CUDA current device is per host thread (ggml worker threads enter here too)
        static thread_local int t_dev = -1;
        if (t_dev != g.device) { if (cudaSetDevice(g.device) != cudaSuccess) { cudaGetLastError(); return fail("cudaSetDevice failed"); } t_dev = g.device; }
        return 0;
    }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return fail("no CUDA device: libtmac_b200 has no CPU fallback"); }
    int dev = 0;
    if (const char *e = getenv("TMAC_B200_DEVICE")) dev = atoi(e);
    else { int cur = 0; if (cudaGetDevice(&cur) == cudaSuccess) dev = cur; }
    CUDA_OK(cudaSetDevice(dev));
    g.device = dev;
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) return fail("libtmac_b200 is built for sm_90a only (found sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ")");
    g.sms = prop.multiProcessorCount;
    CUDA_OK(cudaStreamCreate(&g.own));   // blocking stream: ordered after the legacy default stream (safe default for torch/ggml callers)
    for (const Knob &k : kKnobs) {
        std::string name = "TMAC_B200_";
        for (const char *c = k.key; *c; ++c) name += (char)std::toupper((unsigned char)*c);
        if (const char *e = getenv(name.c_str())) g.*k.field = atoi(e);
    }
    g.inited = true;
    return 0;
}

// ---- kernel dispatch ---------------------------------------------------------------------
gemv3_fn pick_gemv3(int pb, bool sym, int qch, int agq, int minb, int in) {
    switch (in) {
        case kInTable: return pick_gemv3_in<kInTable>(pb, sym, qch, agq, minb);
        case kInRow: return pick_gemv3_in<kInRow>(pb, sym, qch, agq, minb);
        case kInNorm: return pick_gemv3_in<kInNorm>(pb, sym, qch, agq, minb);
        case kInGlu: return pick_gemv3_in<kInGlu>(pb, sym, qch, agq, minb);
        case kInGluNorm: return pick_gemv3_in<kInGluNorm>(pb, sym, qch, agq, minb);
        case kInRelu2Norm: return pick_gemv3_in<kInRelu2Norm>(pb, sym, qch, agq, minb);
        case kInNormBias: return pick_gemv3_in<kInNormBias>(pb, sym, qch, agq, minb);
        case kInExperts: return pick_gemv3_in<kInExperts>(pb, sym, qch, agq, minb);
        case kInExpertsGlu: return pick_gemv3_in<kInExpertsGlu>(pb, sym, qch, agq, minb);
        default: return nullptr;
    }
}

// Decomposition of one launch: cluster size CS (K slices of a super-block), warps per CTA, chunks
// per warp.  Minimises the work of the busiest SM (CTAs are spread round-robin over SMs), then
// prefers more warps in flight.
void choose_decomposition(int nrsb, int nchunk, int N, int *cs_out, int *wpc_out, int *bpw_out) {
    double best_cost = 1e30; int bcs = 1, bwpc = 1, bbpw = nchunk;
    for (int cs : {1, 2, 4, 8})
        for (int wpc = 1; wpc <= kG3MaxWarps; ++wpc) {
            if (cs * wpc > nchunk && !(cs == 1 && wpc == 1)) { if (cs * (wpc - 1) >= nchunk) continue; }
            const int bpw = (nchunk + cs * wpc - 1) / (cs * wpc);
            if ((cs - 1) * wpc * bpw >= nchunk) continue;              // an entirely idle CTA
            const long ctas = (long)nrsb * cs * N;
            const int res = std::max(1, std::min(32, 2048 / (wpc * 32)));   // resident CTAs per SM (threads)
            const long per_sm = (ctas + g.sms - 1) / g.sms;
            const long waves = (per_sm + res - 1) / res;
            double cost = (double)per_sm * wpc * bpw;                  // chunk-slots on the busiest SM
            cost *= 1.0 + 0.15 * (waves - 1);                          // later waves lose the overlap
            cost += 0.02 * bpw * wpc + 0.2 * bpw;                      // prefer short per-warp chains ...
            cost += 0.5 * std::max(0L, 8 - per_sm * wpc);              // ... and at least 8 warps per SM
            if (cost < best_cost) { best_cost = cost; bcs = cs; bwpc = wpc; bbpw = bpw; }
        }
    *cs_out = bcs; *wpc_out = bwpc; *bpw_out = bbpw;
}

// Production launch: clusters + DSMEM reduction + PDL (gemv3_kernel).
struct BatchPtrs { int n = 0; const unsigned char *const *W = nullptr; const int8_t *const *q = nullptr; const float *const *ls = nullptr,
                   *const *lb = nullptr; void *const *C = nullptr; const float *const *bias = nullptr; };

// What a launch reads: LUT tables (kInTable; a grouped launch takes them from its pointer table), or activation rows [N][K] from
// which the kernel builds a symmetric LUT (the other kinds), with the kind's Gemv3Io.
struct Gemv3In {
    int kind = kInTable;
    bool sym = false;                              // kInTable: symmetric tables (8 stored entries)
    const int8_t *qlut = nullptr;                  // kInTable, single launches
    const float *ls = nullptr, *lb = nullptr;
    const void *act = nullptr;                     // the other kinds
    int act_f16 = 0;
    Gemv3Io io{};
    static Gemv3In tables(const int8_t *qlut, const float *ls, const float *lb, bool sym) { return {kInTable, sym, qlut, ls, lb}; }
    static Gemv3In rows(int kind, const void *act, int act_f16, const Gemv3Io &io = Gemv3Io{}) {
        return {kind, false, nullptr, nullptr, nullptr, act, act_f16, io};
    }
};

int launch_gemv3(const Resident &R, int row_begin, int row_end, int N, const Gemv3In &in, void *C, int ldc, int c_row0, int out_f16,
                 const BatchPtrs *batch = nullptr) {
    const StreamLayout &L = R.L;
    if (row_begin < 0 || row_end > L.Mout || row_begin >= row_end) return fail("qgemm_lut: bad row range");
    const int rsb0 = row_begin / L.rsb, rsb1 = (row_end + L.rsb - 1) / L.rsb, nrsb = rsb1 - rsb0;
    Gemv3Params p{};
    p.W = R.d + (size_t)rsb0 * L.rsb_stride;
    p.Wnext = nullptr;
    if (g.next_hint) {
        auto it = g.res.find(g.next_hint);
        if (it != g.res.end() && it->second.L.total == L.total && it->second.L.blk == L.blk) p.Wnext = it->second.d + (size_t)rsb0 * L.rsb_stride;
        g.next_hint = 0;
    }
    const bool sym = in.kind != kInTable || in.sym;
    p.qlut = in.qlut; p.lut_scales = in.ls; p.lut_biases = in.lb; p.C = C;
    p.act = in.act; p.act_f16 = in.act_f16;
    p.K = L.K; p.ldc = ldc; p.row_begin = row_begin; p.row_end = row_end; p.c_row0 = c_row0; p.bits = L.bits;
    p.nrsb = nrsb; p.rsb0 = rsb0; p.nchunk = L.nchunk;
    p.ags = L.act_group_size;
    p.zp = L.zp; p.one_scale = L.one_scale; p.sd = L.sd; p.out_f16 = out_f16;
    p.blk_bytes = (int)L.blk; p.scale0 = L.scale0; p.rsb_stride = L.rsb_stride;
    if (g.npeer) {
        if (N != 1 || batch) { g.npeer = 0; return fail("peer outputs: N = 1, single-tensor launches only"); }
        p.npeer = g.npeer;
        for (int q = 0; q < g.npeer; ++q) p.Cpeer[q] = g.peer_out[q];
        g.npeer = 0;
    }
    p.pdl_late = (g.pdl_late >= 0) ? g.pdl_late : (in.kind != kInTable ? 0 : 1);   // measured: row inputs prefer the early trigger
    const int nb = batch ? batch->n : 0;
    if (batch) { p.nbatch = nb; p.Wv = batch->W; p.qlutv = batch->q; p.lsv = batch->ls; p.lbv = batch->lb; p.Cv = batch->C; }
    choose_decomposition(nrsb, L.nchunk, N * std::max(1, nb), &p.cs, &p.wpc, &p.bpw);
    // A lone launch per tensor is latency bound and prefers fewer, fatter
    // CTAs with more registers (ILP); grouped / batched launches are ALU-pipe bound and prefer more CTAs.
    const bool lone = (N * std::max(1, nb) == 1);
    // 85-register variant (more ILP) for lone launches and for grouped W1/W2 launches (shared memory caps residency at 3
    // CTAs per SM anyway; measured +6 %); grouped W3/W4 launches measured better with the 64-register variant.
    int minb = (lone || L.pb != 4) ? 3 : 4;
    if (lone && p.cs == 8 && p.wpc == 4 && p.bpw == 1) { p.cs = 4; p.wpc = 8; }
    if (!lone && (long)nrsb * N * std::max(1, nb) >= 4L * g.sms) {   // machine already full of whole super-blocks: no K split
        p.cs = 1; p.wpc = std::min(kG3MaxWarps, L.nchunk); p.bpw = (L.nchunk + p.wpc - 1) / p.wpc;
    }
    if (g.minb_override > 0) minb = g.minb_override;
    if (g.cs_override > 0) { p.cs = g.cs_override; }
    if (g.wpc_override > 0) { p.wpc = std::min(g.wpc_override, kG3MaxWarps); }
    if (g.cs_override > 0 || g.wpc_override > 0) p.bpw = (L.nchunk + p.cs * p.wpc - 1) / (p.cs * p.wpc);
    g.last_launch[0] = p.cs; g.last_launch[1] = p.wpc; g.last_launch[2] = p.bpw; g.last_launch[3] = minb;
    g.last_launch[4] = nrsb * p.cs; g.last_launch[5] = L.pb; g.last_launch[6] = sym ? 1 : 0; g.last_launch[7] = std::max(1, nb);
    if (g.trace) {   // ring of 8 launches
        const size_t per = (size_t)nrsb * p.cs * 8;
        if (g.d_trace.ensure(per * 8 * sizeof(long long))) return fail("out of device memory (trace)");
        p.trace = (long long *)g.d_trace.p + per * (size_t)(g.trace_seq++ % 8);
        g.trace_ctas = nrsb * p.cs;
    }
    const int agq = L.agq();
    gemv3_fn fn = pick_gemv3(L.pb, sym, L.qch, agq, minb, in.kind);
    if (!fn) return fail("qgemm_lut: unsupported chunking (qch=" + std::to_string(L.qch) + ", agq=" + std::to_string(agq) + ")");
    p.nbuf = (p.bpw > 1) ? 2 : 1;
    if (g.nbuf_override > 0) p.nbuf = std::min(p.nbuf, g.nbuf_override);
    const size_t wregion = std::max((size_t)p.wpc * (p.nbuf * L.blk + (size_t)L.qch * 4 * (sym ? 8 : 16)), (size_t)p.wpc * L.rsb * 4);
    size_t smem = (size_t)p.cs * L.rsb * 4 + ((wregion + 15) & ~(size_t)15) + (size_t)p.wpc * 16;   // + warp-private mbarriers
    if (in.kind != kInTable && L.int_path()) { p.ioff = (int)smem; smem += (size_t)(L.K / 32 + kG3MaxWarps + 4 + 8) * 4; }   // row scan: block sums, warp maxima, bias, cluster maxima
    if (in_norm(in.kind)) { p.ioff = (int)smem; smem += (size_t)(L.K + 4) * 4; }   // the norm's row in fp32, then inv
    if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    uint32_t wtx, wty;
    plane_weight_regs(L.bits, sym, &wtx, &wty);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(nrsb * p.cs, N, std::max(1, nb));
    cfg.blockDim = dim3(p.wpc * 32, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = g.stream();
    cudaLaunchAttribute attr[2];
    int na = 0;
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = g.use_pdl ? 1 : 0;
    ++na;
    if (p.cs > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = p.cs; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
        ++na;
    }
    cfg.attrs = attr; cfg.numAttrs = na;
    CUDA_OK(cudaLaunchKernelEx(&cfg, fn, p, wtx, wty, in.io));
    return 0;
}

// Smallest N that takes a prefill tile (unless set with the prefill_min_n knob).  W2: 32.  W3/W4: 32 as well, but a tensor of fewer
// than 64 row tiles of 128 rows (the 4096-row Llama-2 projections: 32) fills a quarter of the SMs with one token tile, and there the
// tiles overtake the W4 GEMV only between N = 64 and 128 (H100 SXM at 400 W, DESIGN.md 3.3): 128.
// The integer path (one scale): 128 below 64 row tiles, 64 from there.  A tile then sums the whole K alone, so a tensor of few row
// tiles runs long serial tiles: on BitNet-3B's 3200-row projections (25 row tiles) the GEMV wins at N = 64 and loses at 128, on the
// 8640-row one (68 row tiles) the tile wins from N = 64 against both GEMV call forms (H100 SXM at 700 W, DESIGN.md 3.3).
// The other fp groupings follow the same rule, with one exception: a 32-K chunk (ggml Q4_0, GPTQ g32) makes the W3/W4 GEMV slower,
// and on the 4096-row Llama-2 projections (32 row tiles) the tiles win from N = 64 against both call forms, so W3/W4 g32 tensors of
// 32 to 63 row tiles take them from 64 (H100 SXM at 700 W, DESIGN.md 3.3).  Fewer row tiles keep 128 (not measured).
int tile_min_n(const StreamLayout &L) {
    if (g.prefill_min_n > 0) return g.prefill_min_n;
    if (L.one_scale) return (L.nrsb * L.rsb + 127) / 128 < 64 ? 128 : 64;
    const int nrt = (L.nrsb + 1) / 2;
    if (L.pb == 4 && nrt < 64) return (L.ck == 32 && nrt >= 32) ? 64 : 128;
    return 32;
}

// The fp-path tensors both tiles take, dense and routed: W2 or W3/W4 streams with per-row scales, K % 128 == 0, chunk 128, 64 or
// 32 K, and the act group (128, 64 or 32 K) inside the chunk.
static bool tiles_take_fp(const StreamLayout &L) {
    return !L.one_scale && L.K % 128 == 0 && (L.qch == 8 || L.qch == 4 || L.qch == 2) && L.ck % L.act_group_size == 0 && (L.pb == 2 || L.pb == 4);
}

// The tensors the routed tiles take (the prefill_* forms, tmac_prefill_experts.cu): those of tiles_take_fp, and one-scale fp-path
// W2/W3/W4 tensors (act group 128, 64 or 32 K < K) with K % 128 == 0 (chunk 128 K, both tiles) or K % 128 == 64 (chunk 64 K, the
// int8 tile only: TilePlan::fits16 is false).
static bool routed_tiles_take(const StreamLayout &L) {
    if (tiles_take_fp(L)) return true;
    return L.one_scale && !L.int_path() && (L.pb == 2 || L.pb == 4) &&
           ((L.K % 128 == 0 && L.qch == 8) || (L.K % 128 == 64 && L.qch == 4));
}

// Whether N activation rows against this tensor take a prefill tile (with a symmetric LUT): N >= tile_min_n, and either an fp-path
// tensor the tiles take or the integer path (W2 or W3/W4 streams, one scale, act group K, chunk 128 or 64).
bool takes_prefill_tile(const StreamLayout &L, int N) {
    return g.use_prefill && N >= tile_min_n(L) && (tiles_take_fp(L) || (L.int_path() && (L.pb == 2 || L.pb == 4) && (L.qch == 8 || L.qch == 4)));
}

// Both tiles' geometry and shared memory for a tensor (int_path: the int8 tile's integer-path form), dense and routed alike.
constexpr size_t kP16MaxSmem = 227 * 1024, kPfMaxSmem = 225 * 1024;   // the largest carve-up each tile is launched with
struct TilePlan {
    int nrt, nmain, nextra;        // row tiles of 128 rows; the 64-K steps, and the fp16 tile's bias steps
    size_t rec, smem16, smem8;     // the int8 tile's LUT record bytes; both tiles' dynamic shared memory
    bool fits16, fits8;
    TilePlan(const StreamLayout &L, bool int_path) {
        // the producers stage a 128-K window of 128 / ck chunk blocks (integer path, K % 128 == 64: one chunk)
        const bool unit1 = int_path || L.K % 128;
        const size_t rawsz = ((unit1 ? 1 : 8 / L.qch) * L.blk + 127) & ~(size_t)127;
        // a row tile is 128 rows: one W2 super-block, two W3/W4 super-blocks (64 rows each) whose blocks the producers stage together
        const int nsb = 128 / L.rsb;
        const size_t rawall = 2 * (size_t)nsb * rawsz, xtab = (size_t)128 * L.pb * 8;   // + the expansion table (fp16 tile: PB 4 only)
        nrt = (L.nrsb + nsb - 1) / nsb; nmain = L.K / 64; nextra = (L.nchunk + 31) / 32;
        rec = pf_rec_bytes(int_path, L.qch, L.agq());
        smem16 = (size_t)kP16NA * kP16SubA + (size_t)kP16NB * kP16SubB + rawall + (L.pb == 4 ? xtab : 0) + (2 * kP16NA + 2 * kP16NB + 2) * 8 + 1024;
        smem8 = (size_t)kPfStages * (kPfStageBytes + rec) + rawall + xtab + (2 * kPfStages + 4) * 8 + 1024;
        fits16 = smem16 <= kP16MaxSmem && L.K % 128 == 0; fits8 = smem8 <= kPfMaxSmem;
    }
};

// The fields of a tile's parameters (Prefill16Params or PrefillParams) that come from the tensor and the call; the callers set the
// pointers, the tile count and (dense fp16 tile) the stream-K split.
template <class P> static P tile_params(const StreamLayout &L, const TilePlan &t, int N, int ldc, int out_f16) {
    P p{};
    p.N = N; p.K = L.K; p.Mout = L.Mout; p.ldc = ldc; p.out_f16 = out_f16;
    p.nchunk = L.nchunk; p.zp = L.zp; p.sd = L.sd; p.blk_bytes = (int)L.blk; p.rsb_stride = L.rsb_stride; p.nrsb = L.nrsb; p.bits = L.bits;
    p.scale0 = L.scale0;
    if constexpr (std::is_same_v<P, PrefillParams>) p.qch = L.qch;
    else { p.nrt = t.nrt; p.nmain = t.nmain; p.nextra = t.nextra; }
    return p;
}

// Launch the fp16 tile (fp16) or the int8 tile with its shared memory from the plan, and report it in last_launch: {16 or 1, warps, chunks,
// split, grid.x, PB, 1, -rows} (a batch < 0 marks the tensor-core prefill tile).
template <class F, class... P>
static int launch_tile(bool fp16, F fn, dim3 grid, const TilePlan &t, int split, const StreamLayout &L, int rows, const P &...args) {
    const int threads = fp16 ? kP16Threads : kPfThreads2;
    const size_t smem = fp16 ? t.smem16 : t.smem8;
    CUDA_OK(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fn<<<grid, threads, smem, g.stream()>>>(args...);
    CUDA_OK(cudaGetLastError());
    const int rep[8] = {fp16 ? 16 : 1, threads / 32, L.nchunk, split, (int)grid.x, L.pb, 1, -rows};
    std::memcpy(g.last_launch, rep, sizeof rep);
    return 0;
}

// The fp path's kernels of one grouping (QCH quads per chunk, AGQ quads per activation group): int8 tile, its LUT records,
// fp16 tile, its B tiles.
struct PfKernels {
    void (*tile)(const PrefillParams);
    void (*lut)(const int8_t *, const float *, const float *, unsigned char *, int, int);
    void (*tile16)(const Prefill16Params);
    void (*lut16)(const int8_t *, const float *, const float *, unsigned char *, int, int, int, int);
};
template <int PB> PfKernels pick_pf(int qch, int agq) {
    return FpGroupings::find<PfKernels>(qch, agq, [](auto QCH, auto AGQ) -> PfKernels {
        return {prefill_kernel<PB, false, QCH, AGQ>, lut_tile_kernel<false, QCH, AGQ>, prefill16_kernel<PB, QCH, AGQ>, lut_tile16_kernel<QCH, AGQ>};
    });
}

// Prefill tile on the tensor cores (wgmma, tmac_prefill.cuh).  Returns 1 if the shape is not covered (caller falls back to the GEMV
// kernel per activation row), 0 on launch, -1 on error.
int launch_prefill(const Resident &R, int N, const int8_t *qlut, const float *ls, const float *lb, void *C, int ldc, int out_f16, bool sym) {
    const StreamLayout &L = R.L;
    if (!sym || !takes_prefill_tile(L, N)) return 1;
    const bool int_path = L.int_path();
    PfKernels fk{};
    if (!int_path) {
        fk = L.pb == 4 ? pick_pf<4>(L.qch, L.agq()) : pick_pf<2>(L.qch, L.agq());
        if (!fk.tile) return fail("prefill: no tile for chunk " + std::to_string(L.ck) + ", act group " + std::to_string(L.act_group_size));
    }
    const TilePlan t(L, int_path);
    // fp path: scales folded into fp16 operands, fp32 accumulation over K in registers (tmac_prefill16.cuh).  Not exact, so the
    // integer path never takes it.
    if (g.use_prefill16 && N >= 64 && !int_path && t.fits16) {
        const int nsteps = t.nmain + t.nextra, ntile16 = (N + kP16NT - 1) / kP16NT;
        if (g.d_tiles.ensure((size_t)ntile16 * nsteps * kP16BBytes)) return fail("out of device memory (LUT tiles)");
        fk.lut16<<<dim3(nsteps, ntile16), 256, 0, g.stream()>>>(qlut, ls, lb, (unsigned char *)g.d_tiles.p, N, L.K, t.nmain, t.nextra);
        CUDA_OK(cudaGetLastError());
        auto q = tile_params<Prefill16Params>(L, t, N, ldc, out_f16);
        q.W = R.d; q.C = C; q.tiles = (const unsigned char *)g.d_tiles.p; q.ntiles = t.nrt * ntile16;
        // fewer tiles than SMs (e.g. 86 at N = 256): stream-K over all SMs, partial tiles through `scratch`
        q.streamk = (g.pf_streamk && q.ntiles < g.sms && (long)q.ntiles * nsteps >= 2L * g.sms) ? 1 : 0;
        const int grid = q.streamk ? g.sms : q.ntiles;
        if (q.streamk) {
            const size_t sb = (size_t)2 * grid * kP16NT * 128 * sizeof(float);
            if (g.d_pf_scratch.ensure(sb)) return fail("out of device memory (stream-K scratch)");
            if (g.d_pf_flags.cap < (size_t)grid * sizeof(int)) {
                if (g.d_pf_flags.ensure((size_t)grid * sizeof(int))) return fail("out of device memory (stream-K flags)");
                CUDA_OK(cudaMemsetAsync(g.d_pf_flags.p, 0, g.d_pf_flags.cap, g.stream()));
            }
            q.scratch = (float *)g.d_pf_scratch.p; q.flags = (int *)g.d_pf_flags.p;
        }
        return launch_tile(true, fk.tile16, dim3(grid), t, q.streamk, L, N, q);
    }
    if (!t.fits8) return 1;
    const int ntile = (N + kPfNT - 1) / kPfNT;   // records: one per 64-K step
    if (g.d_tiles.ensure((size_t)ntile * t.nmain * t.rec)) return fail("out of device memory (LUT tiles)");
    if (int_path) lut_tile_kernel<true><<<dim3(t.nmain, ntile), 128, 0, g.stream()>>>(qlut, nullptr, nullptr, (unsigned char *)g.d_tiles.p, N, L.K);
    else fk.lut<<<dim3(t.nmain, ntile), 128, 0, g.stream()>>>(qlut, ls, lb, (unsigned char *)g.d_tiles.p, N, L.K);
    CUDA_OK(cudaGetLastError());
    auto p = tile_params<PrefillParams>(L, t, N, ldc, out_f16);
    p.W = R.d; p.qlut = qlut; p.lut_scales = ls; p.lut_biases = lb; p.C = C;
    p.lut_tiles = (const unsigned char *)g.d_tiles.p;
    if (g.trace) {
        if (g.d_trace.ensure(8192)) return fail("out of device memory (trace)");
        CUDA_OK(cudaMemsetAsync(g.d_trace.p, 0, 3 * 32 * 4 * sizeof(long long), g.stream()));
        p.dbg = (long long *)g.d_trace.p; g.trace_ctas = 12;   // 96 rows of 4 = 48 rows of 8
    }
    const auto fn = int_path ? (L.pb == 4 ? prefill_kernel<4, true> : prefill_kernel<2, true>) : fk.tile;
    return launch_tile(false, fn, dim3(t.nrt, ntile), t, 1, L, N, p);
}

// Launch qgemm_lut over rows [row_begin,row_end) (relative to the resident tensor): the tensor-core tile for whole-tensor batches,
// else gemv3_kernel.  All pointers are device pointers; C is [N][ldc] with C[n][row - c_row0].
int launch_gemv(const Resident &R, int row_begin, int row_end, int N, const int8_t *qlut, const float *ls,
                const float *lb, void *C, int ldc, int c_row0, int out_f16, bool sym) {
    if (row_begin == 0 && row_end == R.L.Mout && c_row0 == 0 && ldc == R.L.Mout) {
        const int rc = launch_prefill(R, N, qlut, ls, lb, C, ldc, out_f16, sym);
        if (rc <= 0) return rc;
    }
    return launch_gemv3(R, row_begin, row_end, N, Gemv3In::tables(qlut, ls, lb, sym), C, ldc, c_row0, out_f16);
}

int launch_preprocessor(int K, int N, int ags, int dtype, const void *B, float *ls, float *lb, int8_t *qlut) {
    if (ags <= 0 || ags > K) ags = K;
    if (K % 32 || ags % 32 || K % ags) return fail("preprocessor: K and act_group_size must be multiples of 32, K % act_group_size == 0");
    const int nag = K / ags;
    int agb = (ags == K) ? 1 : std::max(1, 1024 / ags);
    const int gx = (nag + agb - 1) / agb;
    const int ng = agb * (ags / 4);
    const size_t smem = (size_t)agb * 4 + (size_t)ng * 4 + (size_t)(ng / 8 + 1) * 4;
    if (smem > 200 * 1024) return fail("preprocessor: activation group too large");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(gx, N, 1);
    cfg.blockDim = dim3(kPreThreads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = g.stream();
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = g.use_pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (dtype == TMAC_B200_F16) {
        if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute((const void *)preprocessor_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_OK(cudaLaunchKernelEx(&cfg, preprocessor_kernel<__half>, (const __half *)B, ls, lb, qlut, K, ags, agb));
    } else {
        if (smem > 48 * 1024) CUDA_OK(cudaFuncSetAttribute((const void *)preprocessor_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_OK(cudaLaunchKernelEx(&cfg, preprocessor_kernel<float>, (const float *)B, ls, lb, qlut, K, ags, agb));
    }
    CUDA_OK(cudaGetLastError());
    if (g.sym_qluts.size() > 4096) g.sym_qluts.clear();
    g.sym_qluts.insert(qlut);
    return 0;
}

bool host_lut_symmetric(const int8_t *q, size_t groups) {
    for (size_t g2 = 0; g2 < groups; ++g2) {
        const int8_t *t = q + g2 * 16;
        for (int i = 0; i < 8; ++i)
            if ((int)t[15 - i] != -(int)t[i]) return false;
    }
    return true;
}

int validate_cfg(const tmac_b200_kcfg &c) {
    if (c.bits < 1 || c.bits > 4) return fail("kcfg: bits must be 1..4");
    if (c.M <= 0 || c.K <= 0 || c.K % 32) return fail("kcfg: bad M/K");
    if (c.bm <= 0 || (c.M * c.bits) % c.bm || c.bm % 32 || c.bm % c.bits) return fail("kcfg: bm must divide M*bits and be a multiple of 32 and of bits");
    if (c.kfactor <= 0 || (c.K / 4) % c.kfactor) return fail("kcfg: kfactor must divide K/4");
    if (c.simd_n_in != 16 || c.simd_n_out != 8) return fail("kcfg: only simd_n_in=16, simd_n_out=8 (the reference's only instantiation)");
    if (!c.one_scale && (c.group_size <= 0 || c.K % c.group_size || c.group_size % 32)) return fail("kcfg: group_size must be a positive multiple of 32 that divides K");
    return 0;
}

int64_t register_resident(const tmac_b200_kcfg &cfg, const PlainWeights &P, const void *host_alias, size_t alias_bytes, int row0) {
    StreamLayout L;
    bool fp16_ok = true;
    if (!cfg.one_scale)
        fp16_ok = !g.scales_f32 && all_fp16_exact(P.scales.data(), P.scales.size()) && (P.zeros.empty() || all_fp16_exact(P.zeros.data(), P.zeros.size()));
    if (!make_layout(P.Mout, cfg.K, cfg.bits, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale, fp16_ok ? 2 : 4, &L))
        return fail("unsupported shape / grouping for the stream layout");
    if (cfg.one_scale) L.scale0 = P.scales.empty() ? 0.f : P.scales[0];
    std::vector<uint8_t> host(L.total);
    encode_stream(P, L, host.data());
    Resident R;
    R.cfg = cfg; R.L = L; R.row0 = row0;
    if (cudaMalloc((void **)&R.d, L.total) != cudaSuccess) { cudaGetLastError(); return fail("out of device memory for resident weights"); }
    if (cudaMemcpy(R.d, host.data(), L.total, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(R.d); return fail("weight upload failed"); }
    R.host_a = (const unsigned char *)host_alias;
    R.host_a_bytes = alias_bytes;
    const int64_t h = g.next_handle++;
    R.id = h;
    g.res[h] = R;
    return h;
}

Resident *find_by_alias(const void *A, size_t *offset) {
    const unsigned char *a = (const unsigned char *)A;
    for (auto &kv : g.res) {
        Resident &R = kv.second;
        if (R.host_a && a >= R.host_a && a < R.host_a + R.host_a_bytes) { *offset = (size_t)(a - R.host_a); return &R; }
        if (a == R.d) { *offset = 0; return &R; }
    }
    return nullptr;
}

const tmac_b200_kcfg *find_kcfg_locked(int m_times_bits, int k, int bits) {
    const tmac_b200_kcfg *tile_match = nullptr;
    for (const auto &c : g.kcfgs) {
        if (c.K != k || c.bits != bits) continue;
        if (c.M * c.bits == m_times_bits) return &c;
        if (m_times_bits % c.bm == 0 && m_times_bits < c.M * c.bits && !tile_match) tile_match = &c;
    }
    return tile_match;
}

// Stage helpers for host pointers ---------------------------------------------------------
// h_in is written by the host at call time and read by an async H2D: before reusing it wait for
// the previous call's copy; after enqueuing this call's copies record the event again.
void stage_wait() {
    if (g.stage_pending) { cudaEventSynchronize(g.stage_ev); g.stage_pending = false; }
}
void stage_mark() {
    if (!g.stage_ev) cudaEventCreateWithFlags(&g.stage_ev, cudaEventDisableTiming);
    cudaEventRecord(g.stage_ev, g.stream());
    g.stage_pending = true;
}
int h2d(DevBuf &dst, PinBuf &pin, size_t pin_off, const void *src, size_t bytes) {
    if (dst.ensure(bytes)) return fail("out of device memory");
    std::memcpy((char *)pin.p + pin_off, src, bytes);
    CUDA_OK(cudaMemcpyAsync(dst.p, (char *)pin.p + pin_off, bytes, cudaMemcpyHostToDevice, g.stream()));
    return 0;
}

size_t esize(int dtype) { return dtype == TMAC_B200_F16 ? 2 : 4; }

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int tmac_b200_init(int device) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!g.inited && device >= 0) {
        if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return fail("cudaSetDevice failed"); }
    }
    return ensure_init();
}

void tmac_b200_shutdown(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!g.inited) return;
    cudaStreamSynchronize(g.stream());
    for (auto &kv : g_seqs) kv.second.release();
    g_seqs.clear();
    for (auto &kv : g_graphs) cudaGraphExecDestroy(kv.second);
    g_graphs.clear();
    for (auto &e : g.ptr_tables) if (e.second) cudaFree(e.second);
    g.ptr_tables.clear();
    for (auto &kv : g_gguf) delete kv.second;
    g_gguf.clear();
    for (auto &kv : g.res) {
        cudaFree(kv.second.d);
        if (kv.second.reserved) munmap(kv.second.reserved, kv.second.reserved_bytes);
        std::free(kv.second.host_scales);
    }
    g.res.clear();
    for (DevBuf *b : {&g.d_b, &g.d_qlut, &g.d_ls, &g.d_lb, &g.d_c, &g.d_cbits, &g.d_trace, &g.d_tiles, &g.d_pf_scratch, &g.d_pf_flags,
                      &g.d_moe_route, &g.d_moe_act}) { if (b->p) cudaFree(b->p); b->p = nullptr; b->cap = 0; }
    for (HostLut &e : g.hluts) {
        for (DevBuf *b : {&e.dq, &e.dls, &e.dlb}) { if (b->p) cudaFree(b->p); b->p = nullptr; b->cap = 0; }
        if (e.res.p) cudaFreeHost(e.res.p);
        e = HostLut();
    }
    for (PinBuf *b : {&g.h_in, &g.h_out}) { if (b->p) cudaFreeHost(b->p); b->p = nullptr; b->cap = 0; }
    if (g.stage_ev) cudaEventDestroy(g.stage_ev);
    g.stage_ev = nullptr; g.stage_pending = false;
    if (g.own) cudaStreamDestroy(g.own);
    g.own = nullptr; g.sym_qluts.clear();
    g.user = nullptr; g.use_user = false; g.trace_ctas = 0; g.trace_seq = 0; g.next_hint = 0;
    g.inited = false;
}

const char *tmac_b200_last_error(void) { return t_err.c_str(); }
int tmac_b200_version(void) { return 100; }

int tmac_b200_set_stream(void *stream) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    g.user = (cudaStream_t)stream;
    g.use_user = stream != nullptr;
    return 0;
}

int tmac_b200_set_float_type(int dtype) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (dtype != TMAC_B200_F32 && dtype != TMAC_B200_F16) return fail("bad dtype");
    g.float_type = dtype;
    return 0;
}

int tmac_b200_register_kcfg(const tmac_b200_kcfg *cfg) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!cfg) return fail("null kcfg");
    tmac_b200_kcfg c = *cfg;
    if (c.simd_n_in == 0) c.simd_n_in = 16;
    if (c.simd_n_out == 0) c.simd_n_out = 8;
    if (c.act_group_size <= 0 || c.act_group_size > c.K) c.act_group_size = c.K;
    if (validate_cfg(c)) return -1;
    for (auto &o : g.kcfgs)
        if (o.M == c.M && o.K == c.K && o.bits == c.bits) { o = c; return 0; }
    g.kcfgs.push_back(c);
    return 0;
}

void tmac_b200_clear_kcfg(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    g.kcfgs.clear();
}

int tmac_b200_find_kcfg(int m_times_bits, int k, int bits, tmac_b200_kcfg *out) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    const tmac_b200_kcfg *c = find_kcfg_locked(m_times_bits, k, bits);
    if (!c) return fail("no kcfg for m=" + std::to_string(m_times_bits) + " k=" + std::to_string(k) + " b=" + std::to_string(bits));
    if (out) *out = *c;
    return 0;
}

// Minimal INI reader for the reference's kcfg.ini (deploy/compile.py:156-165,203-204).
int tmac_b200_load_kcfg_file(const char *path) {
    FILE *f = path ? fopen(path, "r") : nullptr;
    if (!f) return fail(std::string("cannot open kcfg file ") + (path ? path : "(null)"));
    struct Sec { std::string name; std::map<std::string, long> kv; };
    std::vector<Sec> secs;
    char line[512];
    while (fgets(line, sizeof line, f)) {
        std::string s(line);
        size_t a = s.find_first_not_of(" \t\r\n");
        if (a == std::string::npos || s[a] == ';' || s[a] == '#') continue;
        size_t b = s.find_last_not_of(" \t\r\n");
        s = s.substr(a, b - a + 1);
        if (s.front() == '[' && s.back() == ']') { secs.push_back({s.substr(1, s.size() - 2), {}}); continue; }
        size_t eq = s.find('=');
        if (eq == std::string::npos || secs.empty()) continue;
        std::string k = s.substr(0, eq), v = s.substr(eq + 1);
        k.erase(k.find_last_not_of(" \t") + 1);
        v.erase(0, v.find_first_not_of(" \t"));
        secs.back().kv[k] = atol(v.c_str());
    }
    fclose(f);
    int count = 0;
    for (auto &s : secs) {
        int t, m, k, n, b;
        if (sscanf(s.name.c_str(), "qgemm_lut_t%d_int8_m%d_k%d_n%d_b%d", &t, &m, &k, &n, &b) != 5) continue;
        if (b < 1 || b > 4) continue;                    // not a section this library can serve (and m / b below)
        auto get = [&](const char *key, long dflt) { auto it = s.kv.find(key); return it == s.kv.end() ? dflt : it->second; };
        tmac_b200_kcfg c{};
        c.M = m / b; c.K = k; c.bits = b;
        c.bm = (int)get("bm", 0); c.kfactor = (int)get("kfactor", 16);
        c.simd_n_in = (int)get("simd_n_in", 16); c.simd_n_out = (int)get("simd_n_out", 8);
        c.group_size = (int)get("group_size", 128);
        const long lss = get("lut_scales_size", 0), ss = get("scales_size", 0);
        c.act_group_size = (int)get("act_group_size", lss > 0 ? (long)k * n / lss : 64);
        const long per_group = (long)c.M * (k / std::max(1, c.group_size));
        c.one_scale = (int)get("m_groups", ss > 0 && ss < c.M ? 1 : -1) > 0 ? 1 : 0;
        c.zero_point = (int)get("zero_point", (!c.one_scale && ss == 2 * per_group) ? 1 : 0);
        if (tmac_b200_register_kcfg(&c) == 0) ++count;
    }
    return count;
}

int64_t tmac_b200_upload_weights(const tmac_b200_kcfg *cfg_in, const void *A, const void *scales, int scales_dtype) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!cfg_in || !A || !scales) return fail("upload_weights: null argument");
    if (is_device_ptr(A)) return fail("upload_weights: A must be a host pointer (reference layout)");
    tmac_b200_kcfg cfg = *cfg_in;
    if (cfg.simd_n_in == 0) cfg.simd_n_in = 16;
    if (cfg.simd_n_out == 0) cfg.simd_n_out = 8;
    if (cfg.act_group_size <= 0 || cfg.act_group_size > cfg.K) cfg.act_group_size = cfg.K;
    if (validate_cfg(cfg)) return -1;
    const size_t nsc = cfg.one_scale ? 1 : (size_t)cfg.M * (cfg.K / cfg.group_size) * (cfg.zero_point ? 2 : 1);
    std::vector<float> s32(nsc);
    if (scales_dtype == TMAC_B200_F16) {
        const uint16_t *h = (const uint16_t *)scales;
        for (size_t i = 0; i < nsc; ++i) s32[i] = f16_bits_to_f32(h[i]);
    } else
        std::memcpy(s32.data(), scales, nsc * 4);
    PlainWeights P;
    plain_from_reference((const uint8_t *)A, s32.data(), cfg.M, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size,
                         cfg.zero_point, cfg.one_scale, &P);
    return register_resident(cfg, P, A, (size_t)cfg.M * cfg.K * cfg.bits / 8, 0);
}

int64_t tmac_b200_upload_plain_rows(const tmac_b200_kcfg *cfg_in, const uint8_t *w, const float *scales, const float *zeros,
                                    int row0, int rows) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!cfg_in || !w || !scales) return fail("upload_plain: null argument");
    tmac_b200_kcfg cfg = *cfg_in;
    if (cfg.simd_n_in == 0) cfg.simd_n_in = 16;
    if (cfg.simd_n_out == 0) cfg.simd_n_out = 8;
    if (cfg.act_group_size <= 0 || cfg.act_group_size > cfg.K) cfg.act_group_size = cfg.K;
    if (cfg.bits < 1 || cfg.bits > 4 || cfg.M <= 0 || cfg.K <= 0 || cfg.K % 32) return fail("upload_plain: bad shape");
    if (!cfg.one_scale && (cfg.group_size <= 0 || cfg.K % cfg.group_size || cfg.group_size % 32)) return fail("upload_plain: group_size must be a positive multiple of 32 that divides K");
    if (row0 < 0 || rows <= 0 || row0 + rows > cfg.M) return fail("upload_plain: bad row range");
    if (cfg.zero_point && !zeros && !cfg.one_scale) return fail("upload_plain: zero_point set but zeros == NULL");
    PlainWeights P;
    plain_from_w(w, cfg.M, cfg.K, cfg.bits, row0, rows, &P);
    if (cfg.one_scale) P.scales.assign(1, scales[0]);
    else {
        const int NG = cfg.K / cfg.group_size;
        P.scales.assign(scales + (size_t)row0 * NG, scales + (size_t)(row0 + rows) * NG);
        if (cfg.zero_point) P.zeros.assign(zeros + (size_t)row0 * NG, zeros + (size_t)(row0 + rows) * NG);
    }
    return register_resident(cfg, P, nullptr, 0, row0);
}

int64_t tmac_b200_upload_plain(const tmac_b200_kcfg *cfg, const uint8_t *w, const float *scales, const float *zeros) {
    if (!cfg) return fail("upload_plain: null kcfg");
    return tmac_b200_upload_plain_rows(cfg, w, scales, zeros, 0, cfg->M);
}

// GPTQ checkpoint tensors (safetensors: qweight, scales, qzeros) -> resident weights, the C form of
// unpack_gptqv2 + preprocess_weights + upload (model_utils.py:95-129, :262-271; convert_hf_to_gguf.py:300-320).
// cfg gives M, K, bits, group_size, bm, kfactor, act_group_size; zero_point is implied.
int64_t tmac_b200_upload_gptq(const tmac_b200_kcfg *cfg_in, const int32_t *qweight, const uint16_t *scales_f16, const int32_t *qzeros,
                              int gptq_v2) {
    if (!cfg_in || !qweight || !scales_f16 || !qzeros) return fail("upload_gptq: null argument");
    tmac_b200_kcfg cfg = *cfg_in;
    cfg.zero_point = 1; cfg.one_scale = 0;
    if (cfg.group_size <= 0 || cfg.K % cfg.group_size) return fail("upload_gptq: bad group_size");
    const size_t NG = (size_t)cfg.K / cfg.group_size;
    std::vector<uint8_t> w((size_t)cfg.M * cfg.K);
    std::vector<float> sc((size_t)cfg.M * NG), zr((size_t)cfg.M * NG);
    if (!unpack_gptq(qweight, scales_f16, qzeros, cfg.K, cfg.M, cfg.bits, cfg.group_size, gptq_v2 != 0, w.data(), sc.data(), zr.data()))
        return fail("upload_gptq: unsupported packing (bits must divide 32; K, M multiples of 32/bits)");
    return tmac_b200_upload_plain(&cfg, w.data(), sc.data(), zr.data());
}
// Host-only: the unpack step alone (CPU suite).  w [M][K], scales / zeros [M][K/group_size].
int tmac_b200_debug_unpack_gptq(const int32_t *qweight, const uint16_t *scales_f16, const int32_t *qzeros, int K, int M, int bits,
                                int group_size, int gptq_v2, uint8_t *w, float *scales, float *zeros) {
    if (!qweight || !scales_f16 || !qzeros || !w || !scales || !zeros) return fail("debug_unpack_gptq: null argument");
    if (!unpack_gptq(qweight, scales_f16, qzeros, K, M, bits, group_size, gptq_v2 != 0, w, scales, zeros)) return fail("debug_unpack_gptq: unsupported packing");
    return 0;
}

// Host-only converter-side quantisers (tmac_layout.h): fp weights -> codes + scales (+ zeros) in the T-MAC convention, ready for
// tmac_b200_upload_plain.  0 or -1.
int tmac_b200_quantize_bitdistiller(const float *w, int rows, int cols, int bits, int group_size, uint8_t *codes, float *scales, float *zeros) {
    if (!w || !codes || !scales || !zeros) return fail("quantize_bitdistiller: null argument");
    if (!quantize_bitdistiller(w, rows, cols, bits, group_size, codes, scales, zeros)) return fail("quantize_bitdistiller: bad shape / bits / group size");
    return 0;
}
int tmac_b200_quantize_bitnet(const float *w, int rows, int cols, uint8_t *codes, float *scale) {
    if (!w || !codes || !scale || rows <= 0 || cols <= 0) return fail("quantize_bitnet: bad argument");
    quantize_bitnet(w, (size_t)rows * cols, codes, scale);
    return 0;
}

// Host-only: run the reference-layout -> stream-layout transform without touching the GPU and
// return the stream bytes (used by the CPU test-suite to pin the layout).  dst may be NULL to
// query the size.  Returns the byte count or -1.
int64_t tmac_b200_debug_encode(const tmac_b200_kcfg *cfg_in, const void *A, const void *scales, void *dst, size_t cap,
                               int *layout_out /* int[12] */) {
    if (!cfg_in || !A || !scales) return fail("debug_encode: null argument");
    tmac_b200_kcfg cfg = *cfg_in;
    if (cfg.simd_n_in == 0) cfg.simd_n_in = 16;
    if (cfg.simd_n_out == 0) cfg.simd_n_out = 8;
    if (cfg.act_group_size <= 0 || cfg.act_group_size > cfg.K) cfg.act_group_size = cfg.K;
    if (validate_cfg(cfg)) return -1;
    PlainWeights P;
    plain_from_reference((const uint8_t *)A, (const float *)scales, cfg.M, cfg.K, cfg.bits, cfg.bm, cfg.kfactor, cfg.group_size,
                         cfg.zero_point, cfg.one_scale, &P);
    bool fp16_ok = true;
    if (!cfg.one_scale) fp16_ok = all_fp16_exact(P.scales.data(), P.scales.size()) && (P.zeros.empty() || all_fp16_exact(P.zeros.data(), P.zeros.size()));
    StreamLayout L;
    if (!make_layout(P.Mout, cfg.K, cfg.bits, cfg.group_size, cfg.act_group_size, cfg.zero_point, cfg.one_scale, fp16_ok ? 2 : 4, &L))
        return fail("unsupported shape / grouping for the stream layout");
    if (layout_out) {
        const int v[12] = {L.pb, L.rw, L.rsb, L.nrsb, L.ck, L.qch, L.nchunk, L.sd, L.zp, L.one_scale, (int)L.blk, (int)L.wbytes};
        std::memcpy(layout_out, v, sizeof v);
    }
    if (dst) {
        if (cap < L.total) return fail("debug_encode: destination too small");
        encode_stream(P, L, (uint8_t *)dst);
    }
    return (int64_t)L.total;
}

int tmac_b200_free_weights(int64_t handle) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g.res.find(handle);
    if (it == g.res.end()) return fail("bad handle");
    cudaStreamSynchronize(g.stream());
    for (HostLut &e : g.hluts) if (e.res_id == handle) e.res_id = 0;
    cudaFree(it->second.d);
    if (it->second.reserved) munmap(it->second.reserved, it->second.reserved_bytes);
    std::free(it->second.host_scales);
    g.res.erase(it);
    return 0;
}

size_t tmac_b200_weights_nbytes(int64_t handle) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g.res.find(handle);
    return it == g.res.end() ? 0 : it->second.L.total;
}

// Second resident copy of the same tensor in its own HBM allocation (benchmarks rotate through
// distinct buffers so that weights stream from HBM, not L2; multi-layer models with tied shapes).
int64_t tmac_b200_clone_weights(int64_t handle) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g.res.find(handle);
    if (it == g.res.end()) return fail("clone: bad handle");
    Resident R = it->second;
    R.host_a = nullptr; R.host_a_bytes = 0;
    R.reserved = nullptr; R.reserved_bytes = 0; R.host_scales = nullptr;   // owned by the original only (no double munmap / free)
    if (cudaMalloc((void **)&R.d, R.L.total) != cudaSuccess) { cudaGetLastError(); return fail("out of device memory for clone"); }
    if (cudaMemcpy(R.d, it->second.d, R.L.total, cudaMemcpyDeviceToDevice) != cudaSuccess) { cudaFree(R.d); return fail("clone copy failed"); }
    const int64_t h = g.next_handle++;
    R.id = h;
    g.res[h] = R;
    return h;
}

// ---- CUDA-graph helpers: capture a sequence of library calls (device pointers only; run the
// sequence once eagerly first so that every workspace is allocated) and replay it. -------------

int tmac_b200_graph_begin(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    CUDA_OK(cudaStreamBeginCapture(g.stream(), cudaStreamCaptureModeThreadLocal));
    return 0;
}
int64_t tmac_b200_graph_end(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    cudaGraph_t graph = nullptr;
    CUDA_OK(cudaStreamEndCapture(g.stream(), &graph));
    cudaGraphExec_t exec = nullptr;
    cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
    const int64_t h = g_next_graph++;
    g_graphs[h] = exec;
    return h;
}
int tmac_b200_graph_launch(int64_t graph, int times) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_graphs.find(graph);
    if (it == g_graphs.end()) return fail("graph_launch: bad handle");
    for (int i = 0; i < times; ++i) CUDA_OK(cudaGraphLaunch(it->second, g.stream()));
    return 0;
}
int tmac_b200_graph_free(int64_t graph) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_graphs.find(graph);
    if (it == g_graphs.end()) return fail("graph_free: bad handle");
    cudaGraphExecDestroy(it->second);
    g_graphs.erase(it);
    return 0;
}
int tmac_b200_sync(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!g.inited) return 0;
    CUDA_OK(cudaStreamSynchronize(g.stream()));
    return 0;
}

// Debug / reporting: {cluster size, warps per CTA, chunks per warp, min blocks variant, grid.x, PB, sym, batch}
// of the last qgemm_lut launch.
int tmac_b200_debug_last_launch(int *out8) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!out8) return fail("null");
    std::memcpy(out8, g.last_launch, sizeof g.last_launch);
    return 0;
}

// One-shot hint: the tensor that will be multiplied next.  The next qgemm_lut launch prefetches its
// blocks into L2 (cp.async.bulk.prefetch.L2) while it computes, so that the HBM stream of launch
// i+1 overlaps launch i.  Ignored unless the tensor has the same stream geometry.
int tmac_b200_hint_next_weights(int64_t handle) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    g.next_hint = handle;
    return 0;
}

// Debug: per-CTA clock64 stamps of the last gemv3 launch ([ctas][8]); returns #ctas or -1.
int tmac_b200_debug_trace(long long *dst, int cap_ctas) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (!g.trace || !g.d_trace.p) return fail("trace disabled (TMAC_B200_TRACE=1)");
    CUDA_OK(cudaStreamSynchronize(g.stream()));
    const int n = std::min(cap_ctas, g.trace_ctas * 8);   // ring of 8 launches x ctas
    CUDA_OK(cudaMemcpy(dst, g.d_trace.p, (size_t)n * 8 * sizeof(long long), cudaMemcpyDeviceToHost));
    return g.trace_ctas;
}

// Tuning / A-B knobs at run time (kKnobs: the TMAC_B200_* environment variables, lower case, without the prefix).
int tmac_b200_debug_set(const char *key, int value) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    const std::string k = key ? key : "";
    for (const Knob &kn : kKnobs)
        if (k == kn.key) { g.*kn.field = value; return 0; }
    return fail("tmac_b200_debug_set: unknown key '" + k + "'");
}

int tmac_b200_set_lut_mode(int mode) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    g.lut_mode = mode;
    return 0;
}

int tmac_b200_preprocessor(int K, int N, int act_group_size, int dtype, const void *B, void *LUT_Scales, void *LUT_Biases, void *QLUT) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!B || !LUT_Scales || !LUT_Biases || !QLUT || N <= 0) return fail("preprocessor: null/empty argument");
    const int ags = (act_group_size <= 0 || act_group_size > K) ? K : act_group_size;
    if (K % 32 || ags % 32 || K % ags) return fail("preprocessor: bad K / act_group_size");
    const int nag = K / ags;
    const bool dev_in = is_device_ptr(B), dev_out = is_device_ptr(QLUT);
    if (dev_out != is_device_ptr(LUT_Scales) || dev_out != is_device_ptr(LUT_Biases)) return fail("preprocessor: outputs must live in one memory domain");
    const void *dB = B;
    if (!dev_in) {
        const size_t bytes = (size_t)N * K * esize(dtype);
        stage_wait();
        if (g.h_in.ensure(bytes)) return fail("out of pinned memory");
        if (h2d(g.d_b, g.h_in, 0, B, bytes)) return -1;
        stage_mark();
        dB = g.d_b.p;
    }
    float *dls = (float *)LUT_Scales, *dlb = (float *)LUT_Biases;
    int8_t *dq = (int8_t *)QLUT;
    const size_t qb = (size_t)N * K * 4, sb = (size_t)N * nag * 4;
    HostLut *hl = nullptr;
    if (!dev_out) {          // the LUT goes to the caller's host workspace AND stays on the device for the compute calls that follow
        hl = hlut_slot(QLUT);
        if (hl->dq.ensure(qb) || hl->dls.ensure(sb) || hl->dlb.ensure(sb)) return fail("out of device memory");
        dls = (float *)hl->dls.p; dlb = (float *)hl->dlb.p; dq = (int8_t *)hl->dq.p;
    }
    if (launch_preprocessor(K, N, ags, dtype, dB, dls, dlb, dq)) return -1;
    if (!dev_out) {
        if (g.h_out.ensure(qb + 2 * sb)) return fail("out of pinned memory");
        char *ho = (char *)g.h_out.p;
        CUDA_OK(cudaMemcpyAsync(ho, dq, qb, cudaMemcpyDeviceToHost, g.stream()));
        CUDA_OK(cudaMemcpyAsync(ho + qb, dls, sb, cudaMemcpyDeviceToHost, g.stream()));
        CUDA_OK(cudaMemcpyAsync(ho + qb + sb, dlb, sb, cudaMemcpyDeviceToHost, g.stream()));
        CUDA_OK(cudaStreamSynchronize(g.stream()));
        std::memcpy(QLUT, ho, qb);
        std::memcpy(LUT_Scales, ho + qb, sb);
        std::memcpy(LUT_Biases, ho + qb + sb, sb);
        hl->copy.assign((const unsigned char *)ho, (const unsigned char *)ho + qb + 2 * sb);
        hl->qb = qb; hl->sb = sb; hl->N = N; hl->sym = true; hl->res_id = 0;
    }
    return 0;
}

static int qgemm_impl(Resident &R, int row0, int rows, int N, int dtype, const void *QLUT, const void *LUT_Scales,
                      const void *LUT_Biases, void *C) {
    const StreamLayout &L = R.L;
    if (N <= 0 || rows <= 0) return fail("qgemm_lut: empty problem");
    if (!QLUT || !LUT_Scales || !LUT_Biases || !C) return fail("qgemm_lut: null argument");
    const int nag = L.K / L.act_group_size;
    const size_t qb = (size_t)N * L.K * 4, sb = (size_t)N * nag * 4;
    const bool dev_lut = is_device_ptr(QLUT);
    if (dev_lut != is_device_ptr(LUT_Scales) || dev_lut != is_device_ptr(LUT_Biases)) return fail("qgemm_lut: LUT inputs must live in one memory domain");
    const bool dev_c = is_device_ptr(C);
    const int8_t *dq = (const int8_t *)QLUT;
    const float *dls = (const float *)LUT_Scales, *dlb = (const float *)LUT_Biases;
    bool sym;
    HostLut *hl = nullptr;
    if (!dev_lut) {
        // device-resident copy keyed by (host pointer, content hash): written by the preprocessor call that filled this host
        // workspace, or uploaded here once when the caller brings a table of its own
        hl = hlut_find(QLUT, LUT_Scales, LUT_Biases, qb, sb);
        if (!hl) {
            hl = hlut_slot(QLUT);
            stage_wait();
            if (g.h_in.ensure(qb + 2 * sb)) return fail("out of pinned memory");
            if (h2d(hl->dq, g.h_in, 0, QLUT, qb) || h2d(hl->dls, g.h_in, qb, LUT_Scales, sb) || h2d(hl->dlb, g.h_in, qb + sb, LUT_Biases, sb)) return -1;
            stage_mark();
            hl->copy.resize(qb + 2 * sb);
            std::memcpy(hl->copy.data(), QLUT, qb); std::memcpy(hl->copy.data() + qb, LUT_Scales, sb); std::memcpy(hl->copy.data() + qb + sb, LUT_Biases, sb);
            hl->qb = qb; hl->sb = sb; hl->N = N; hl->res_id = 0;
            hl->sym = host_lut_symmetric((const int8_t *)QLUT, (size_t)N * L.K / 4);
        }
        sym = hl->sym;
        dq = (const int8_t *)hl->dq.p; dls = (const float *)hl->dls.p; dlb = (const float *)hl->dlb.p;
    } else
        sym = g.sym_qluts.count(QLUT) != 0;
    if (g.lut_mode == 1) sym = false;
    if (g.lut_mode == 2) sym = true;
    const size_t es = esize(dtype);
    if (hl && !dev_c) {
        // host LUT, host output (the reference's callers): the whole tensor is computed ONCE per (LUT bytes, tensor) straight
        // into page-locked host memory; this call and the later tile calls of the same mat-vec copy their rows out
        const bool hit = hl->res_id == R.id && hl->res_dtype == dtype && hl->N == N;
        if (!hit) {
            const size_t full = (size_t)N * L.Mout * es;
            if (hl->res.ensure(full)) return fail("out of pinned memory");
            if (launch_gemv(R, 0, L.Mout, N, dq, dls, dlb, hl->res.p, L.Mout, 0, dtype == TMAC_B200_F16, sym)) return -1;
            CUDA_OK(cudaStreamSynchronize(g.stream()));
            hl->res_id = R.id; hl->res_dtype = dtype; hl->N = N;
        }
        for (int n = 0; n < N; ++n)
            std::memcpy((char *)C + (size_t)n * rows * es, (const char *)hl->res.p + ((size_t)n * L.Mout + row0) * es, (size_t)rows * es);
        return 0;
    }
    void *dC = C;
    const size_t cb = (size_t)N * rows * es;
    if (!dev_c) {
        if (g.d_c.ensure(cb)) return fail("out of device memory");
        dC = g.d_c.p;
    }
    if (launch_gemv(R, row0, row0 + rows, N, dq, dls, dlb, dC, rows, row0, dtype == TMAC_B200_F16, sym)) return -1;
    if (!dev_c) {
        if (g.h_out.ensure(cb)) return fail("out of pinned memory");
        CUDA_OK(cudaMemcpyAsync(g.h_out.p, dC, cb, cudaMemcpyDeviceToHost, g.stream()));
        CUDA_OK(cudaStreamSynchronize(g.stream()));
        std::memcpy(C, g.h_out.p, cb);
    }
    return 0;
}

int tmac_b200_qgemm_lut(int64_t handle, int row0, int rows, int N, int dtype, const void *QLUT, const void *LUT_Scales,
                        const void *LUT_Biases, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    auto it = g.res.find(handle);
    if (it == g.res.end()) return fail("qgemm_lut: bad weight handle");
    return qgemm_impl(it->second, row0, rows, N, dtype, QLUT, LUT_Scales, LUT_Biases, C);
}

// The setup both grouped launches share: the tensors of `handles`, which must share one geometry (*first: the first of them), and the
// device pointer table {W, QLUT, LUT_Scales, LUT_Biases, C[i / per_c]}[count] of the call (null q / ls / lb: null entries), followed
// by {bias[i / per_c]}[count] when bias is given.  Pointer tables: one device allocation per distinct call signature (stable under
// graph capture), at most 256.
static int grouped_setup(const char *what, const int64_t *handles, int count, const void *const *q, const void *const *ls,
                         const void *const *lb, void *const *C, const Resident **first, BatchPtrs *bp, int per_c = 1,
                         const float *const *bias = nullptr) {
    std::vector<const void *> tab((bias ? 6 : 5) * (size_t)count, nullptr);
    for (int i = 0; i < count; ++i) {
        auto it = g.res.find(handles[i]);
        if (it == g.res.end()) return fail(std::string(what) + ": bad weight handle");
        if (i == 0) *first = &it->second;
        const StreamLayout &a = (*first)->L, &b = it->second.L;
        if (a.Mout != b.Mout || a.K != b.K || a.bits != b.bits || a.blk != b.blk || a.nchunk != b.nchunk || a.zp != b.zp ||
            a.one_scale != b.one_scale || a.sd != b.sd || a.act_group_size != b.act_group_size || a.scale0 != b.scale0)
            return fail(std::string(what) + ": all tensors must share one geometry");
        tab[i] = it->second.d; tab[4 * count + i] = C[i / per_c];
        if (bias) tab[5 * count + i] = bias[i / per_c];
        if (q) { tab[count + i] = q[i]; tab[2 * count + i] = ls[i]; tab[3 * count + i] = lb[i]; }
    }
    void *dtab = nullptr;
    for (auto &e : g.ptr_tables)
        if (e.first == tab) { dtab = e.second; break; }
    if (!dtab) {
        if (cudaMalloc(&dtab, tab.size() * sizeof(void *)) != cudaSuccess) { cudaGetLastError(); return fail("out of device memory (pointer table)"); }
        CUDA_OK(cudaMemcpy(dtab, tab.data(), tab.size() * sizeof(void *), cudaMemcpyHostToDevice));
        if (g.ptr_tables.size() >= 256) {          // bounded: evict the oldest table (its launches are complete or enqueued before this sync)
            cudaStreamSynchronize(g.stream());
            cudaFree(g.ptr_tables.front().second);
            g.ptr_tables.erase(g.ptr_tables.begin());
        }
        g.ptr_tables.emplace_back(tab, dtab);
    }
    const void **dt = (const void **)dtab;
    bp->n = count;
    bp->W = (const unsigned char *const *)dt; bp->q = (const int8_t *const *)(dt + count);
    bp->ls = (const float *const *)(dt + 2 * count); bp->lb = (const float *const *)(dt + 3 * count); bp->C = (void *const *)(dt + 4 * count);
    if (bias) bp->bias = (const float *const *)(dt + 5 * count);
    return 0;
}

// Grouped launch: `count` qgemm_lut problems with identical geometry (same M, K, bits, grouping;
// e.g. the q/k/v or gate/up projections of a layer, the experts of an MoE layer, or any set of
// GEMVs whose LUTs are already available) in ONE kernel launch.  Device pointers only.
// QLUT[i], LUT_Scales[i], LUT_Biases[i], C[i] are per-problem device pointers (host arrays of pointers).
int tmac_b200_qgemm_lut_grouped(const int64_t *handles, int count, int N, int dtype, const void *const *QLUT,
                                const void *const *LUT_Scales, const void *const *LUT_Biases, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!handles || count <= 0 || count > 65535 || !QLUT || !LUT_Scales || !LUT_Biases || !C) return fail("grouped: bad arguments");
    for (int i = 0; i < count; ++i)
        if (!is_device_ptr(QLUT[i]) || !is_device_ptr(C[i])) return fail("grouped: device pointers only");
    const Resident *R = nullptr;
    BatchPtrs bp;
    if (grouped_setup("grouped", handles, count, QLUT, LUT_Scales, LUT_Biases, C, &R, &bp)) return -1;
    bool sym = true;
    for (int i = 0; i < count; ++i) sym = sym && g.sym_qluts.count(QLUT[i]) != 0;
    if (g.lut_mode == 1) sym = false;
    if (g.lut_mode == 2) sym = true;
    const StreamLayout &L = R->L;
    return launch_gemv3(*R, 0, L.Mout, N, Gemv3In::tables(nullptr, nullptr, nullptr, sym), nullptr, L.Mout, 0, dtype == TMAC_B200_F16, &bp);
}

/* q/k/v or gate/up in ONE launch with the LUT built inside it: `count` tensors of one geometry applied to the SAME activation
 * rows B [N][K] (device), outputs C[i] [N][Mout] (device).  The one-call form of preprocessor + tmac_b200_qgemm_lut_grouped. */
int tmac_b200_gemv_grouped(const int64_t *handles, int count, int N, int dtype, const void *B, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!handles || count <= 0 || count > 65535 || !B || !C || N <= 0) return fail("gemv_grouped: bad arguments");
    if (!is_device_ptr(B)) return fail("gemv_grouped: device pointers only");
    for (int i = 0; i < count; ++i)
        if (!is_device_ptr(C[i])) return fail("gemv_grouped: device pointers only");
    const Resident *R = nullptr;
    BatchPtrs bp;
    if (grouped_setup("gemv_grouped", handles, count, nullptr, nullptr, nullptr, C, &R, &bp)) return -1;
    const StreamLayout &L = R->L;
    if (!(L.int_path() || L.act_group_size <= L.ck)) return fail("gemv_grouped: the activation group must lie inside a chunk (or be the whole row)");
    return launch_gemv3(*R, 0, L.Mout, N, Gemv3In::rows(kInRow, B, dtype == TMAC_B200_F16), nullptr, L.Mout, 0, dtype == TMAC_B200_F16, &bp);
}

// What a transformed-input call computes (tmac_b200_gemv_* and tmac_b200_prefill_* of rmsnorm, rmsnorm_bias, glu, residual,
// subnorm and subnorm_relu2, and of the routed experts), filled in by its entry points and read by both of its forms: the input row
// is A, or gate(A, U) when the call has a gate; then its RMS norm with w and eps when it has a norm.  Its output C[i] takes R when R
// is given (required when needs_R), or bias[i] when it has a bias.  Routed calls pick each slot's tensor from the count * n_experts
// tensors of handles by ids, topk slots per token; the GLU form combines the slots' rows with wts.
struct IoCall {
    const char *name;                              // the call without its form, as messages name it
    const int64_t *handles;
    int count, N, dtype;
    const void *A;
    void *const *C;
    int gate = kGateNone;                          // kGateSilu / kGateRelu2: gate(A, U) with the second input U
    const void *U = nullptr;
    bool norm = false;
    const float *w = nullptr;                      // norm: fp32 [K], 16-byte aligned
    float eps = 0.f;
    bool needs_R = false;
    const void *R = nullptr;
    bool bias = false;
    const float *const *biasv = nullptr;           // bias: count fp32 [Mout], 16-byte aligned
    bool routed = false;
    const int32_t *ids = nullptr;                  // routed: [N][topk]
    const float *wts = nullptr;                    // routed with a gate: [N][topk]
    int topk = 1, n_experts = 1;
    IoCall(const char *name, const int64_t *handles, int count, int N, int dtype, const void *A, void *const *C)
        : name(name), handles(handles), count(count), N(N), dtype(dtype), A(A), C(C) {}
};

// Every argument check of both forms of the calls IoCall describes (form: "gemv" or "prefill").
static int io_check(const std::string &form, const IoCall &c) {
    const std::string what = form + "_" + c.name;
    if (c.gate == kGateRelu2 && !c.U) return fail(what + ": U must not be null (" + form + "_subnorm is the call for the attn sub-norm)");
    if (c.needs_R && !c.R) return fail(what + ": R must not be null");
    if (c.norm) {
        if (!c.w || ((uintptr_t)c.w & 15)) return fail(what + ": w must be a 16-byte aligned device vector");
        if (!(c.eps >= 0.f) || !std::isfinite(c.eps)) return fail(what + ": eps must be finite and >= 0");
    }
    if (!c.handles || c.count <= 0 || c.N <= 0 || !c.A || !c.C || (c.gate != kGateNone && !c.U) ||
        (c.dtype != TMAC_B200_F32 && c.dtype != TMAC_B200_F16) ||
        (c.routed ? c.n_experts <= 0 || !c.ids || (c.gate != kGateNone && (!c.wts || !c.C[0])) : c.count > 65535))
        return fail(what + ": bad arguments");
    if (c.routed) {
        if (c.topk < 1 || c.topk > 8) return fail(what + ": topk must be 1..8");
        if ((long long)c.count * c.n_experts > 65535) return fail(what + ": count * n_experts must be <= 65535");
    }
    if (!is_device_ptr(c.A) || (c.U && !is_device_ptr(c.U)) || (c.w && !is_device_ptr(c.w)) || (c.R && !is_device_ptr(c.R)) ||
        (c.ids && !is_device_ptr(c.ids)) || (c.wts && !is_device_ptr(c.wts)))
        return fail(what + ": device pointers only");
    for (int i = 0; i < c.count; ++i)
        if (!is_device_ptr(c.C[i])) return fail(what + ": device pointers only");
    if (!c.bias) return 0;
    // count fp32 [Mout] vectors (Mout of handles[0]; grouped_setup checks the geometry) that overlap no C[j] ([N][Mout] of dtype)
    if (!c.biasv) return fail(what + ": bias must not be null");
    auto it = g.res.find(c.handles[0]);
    if (it == g.res.end()) return fail(what + ": bad weight handle");
    const size_t bb = (size_t)it->second.L.Mout * sizeof(float), cb = (size_t)c.N * it->second.L.Mout * (c.dtype == TMAC_B200_F16 ? 2 : 4);
    for (int i = 0; i < c.count; ++i) {
        if (!c.biasv[i] || ((uintptr_t)c.biasv[i] & 15) || !is_device_ptr(c.biasv[i]))
            return fail(what + ": each bias must be a 16-byte aligned device vector");
        const uintptr_t b0 = (uintptr_t)c.biasv[i];
        for (int j = 0; j < c.count; ++j) {
            const uintptr_t c0 = (uintptr_t)c.C[j];
            if (b0 < c0 + cb && c0 < b0 + bb) return fail(what + ": a bias must not overlap an output");
        }
    }
    return 0;
}

// The gemv3_kernel input kind of a call: the one whose properties are the call's.
static int io_kind(const IoCall &c) {
    for (int k = kInRow; k <= kInNormBias; ++k)
        if (in_experts(k) == c.routed && in_gate(k) == c.gate && in_norm(k) == c.norm && in_bias(k) == c.bias) return k;
    return -1;
}

// The gemv_* form: tmac_b200_gemv_grouped's launch (same decomposition, so the same sums) of the gemv3_kernel of the call's kind, whose
// input is built in the LUT build.  Routed calls launch count * topk slots (so each slot's sums are those of gemv_grouped at
// N * count * topk) with a pointer table of every tensor, count * n_experts entries.  Everything is checked before anything is launched.
static int gemv_io(const IoCall &c) {
    const std::string what = std::string("gemv_") + c.name;
    const Resident *R = nullptr;
    BatchPtrs bp;
    if (io_check("gemv", c) ||
        grouped_setup(what.c_str(), c.handles, c.count * c.n_experts, nullptr, nullptr, nullptr, c.C, &R, &bp, c.n_experts, c.biasv))
        return -1;
    const StreamLayout &L = R->L;
    if (L.int_path() || L.act_group_size > L.ck) return fail(what + ": fp-path tensors with the activation group inside a chunk only");
    const int kind = io_kind(c);
    Gemv3Io io{};
    io.act2 = c.U; io.nw = c.w; io.eps = c.eps; io.res = c.R; io.ids = c.ids; io.wts = c.wts; io.biasv = bp.bias;
    if (c.routed) {
        bp.n = c.count * c.topk;                   // grid.z: the slots
        io.topk = c.topk; io.n_experts = c.n_experts;
    }
    if (kind == kInExpertsGlu) {
        const size_t cnt_bytes = (size_t)c.N * ((L.Mout + L.rsb - 1) / L.rsb) * sizeof(unsigned);
        if (g.d_moe_ws.ensure((size_t)c.N * c.topk * L.Mout * sizeof(float))) return fail(what + ": out of device memory (workspace)");
        if (g.d_moe_cnt.cap < cnt_bytes) {
            if (g.d_moe_cnt.ensure(cnt_bytes)) return fail(what + ": out of device memory (workspace)");
            CUDA_OK(cudaMemsetAsync(g.d_moe_cnt.p, 0, g.d_moe_cnt.cap, g.stream()));
        }
        io.ws = (float *)g.d_moe_ws.p; io.cnt = (unsigned *)g.d_moe_cnt.p;
    }
    const int f16 = c.dtype == TMAC_B200_F16;
    return launch_gemv3(*R, 0, L.Mout, c.N, Gemv3In::rows(kind, c.A, f16, io), nullptr, L.Mout, 0, f16, &bp);
}

int tmac_b200_gemv_rmsnorm(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                           void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("rmsnorm", handles, count, N, dtype, H, C);
    c.norm = true; c.w = w; c.eps = eps;
    return gemv_io(c);
}

int tmac_b200_gemv_rmsnorm_bias(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                                const float *const *bias, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("rmsnorm_bias", handles, count, N, dtype, H, C);
    c.norm = true; c.w = w; c.eps = eps; c.bias = true; c.biasv = bias;
    return gemv_io(c);
}

int tmac_b200_gemv_glu(int64_t handle, int N, int dtype, const void *G, const void *U, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("glu", &handle, 1, N, dtype, G, &C);
    c.gate = kGateSilu; c.U = U; c.R = R;
    return gemv_io(c);
}

int tmac_b200_gemv_residual(int64_t handle, int N, int dtype, const void *B, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("residual", &handle, 1, N, dtype, B, &C);
    c.needs_R = true; c.R = R;
    return gemv_io(c);
}

int tmac_b200_gemv_subnorm(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps, const void *R,
                           void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("subnorm", &handle, 1, N, dtype, G, &C);
    c.gate = U ? kGateSilu : kGateNone; c.U = U; c.norm = true; c.w = w; c.eps = eps; c.R = R;
    return gemv_io(c);
}

int tmac_b200_gemv_subnorm_relu2(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps,
                                 const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("subnorm_relu2", &handle, 1, N, dtype, G, &C);
    c.gate = kGateRelu2; c.U = U; c.norm = true; c.w = w; c.eps = eps; c.R = R;
    return gemv_io(c);
}

int tmac_b200_gemv_experts(const int64_t *handles, int count, int n_experts, int N, int dtype, const void *B, const int32_t *ids,
                           int topk, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("experts", handles, count, N, dtype, B, C);
    c.routed = true; c.ids = ids; c.topk = topk; c.n_experts = n_experts;
    return gemv_io(c);
}

int tmac_b200_gemv_experts_glu(const int64_t *handles, int n_experts, int N, int dtype, const void *G, const void *U,
                               const int32_t *ids, const float *weights, int topk, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("experts_glu", handles, 1, N, dtype, G, &C);
    c.routed = true; c.gate = kGateSilu; c.U = U; c.ids = ids; c.wts = weights; c.topk = topk; c.n_experts = n_experts; c.R = R;
    return gemv_io(c);
}

// The tile of a routed launch: the fp16 tile when it is on and the average expert fills one of its 256-token tiles,
// N * topk >= 256 * n_experts, else the int8 tile.  On Mixtral-8x7B's FFN (8 experts, top-2, W2 and W4) the int8 tile is up to 1.5x
// faster at N = 256 and 512, the fp16 tile faster at N = 2048 and with uniform routing at 1024 (H100 SXM at 700 W, DESIGN.md 3.3).
static bool experts_take_tile16(int N, int topk, int n_experts) { return g.use_prefill16 && (long long)N * topk >= 256LL * n_experts; }

// An armed tmac_b200_peer_outputs makes a prefill-sized call fail, and is disarmed.
static int refuse_peer(const std::string &what) {
    if (!g.npeer) return 0;
    g.npeer = 0;
    return fail(what + ": peer outputs are for N = 1 single-tensor launches");
}

// The prefill_* form: the routed tile launch.  Routed calls: route the slots on the device (pf_route_kernel).  The others: the
// identity routing (one expert, topk = 1), one table entry per token tile.  Then build the LUT of every input row once (A's N rows;
// a gate: the N * topk rows gate(A[s], U[s]), swiglu or relu2; a norm: the N rows rms_scale(A[n], inv_n, w); both: the RMS norm of
// the gated rows, all materialised in fp32), gather each table entry's LUT records and run the routed tile over (row tiles, table
// entries, count).  wts (the routed GLU form): the tile stores the slots' fp32 rows and the combine adds them (+ R); otherwise the
// tile adds R (when not null) in its epilogue, or with a bias the BIAS tiles add bias[i] to tensor i's outputs.  Everything is
// checked and every workspace allocated before anything is launched.
static int prefill_io(const IoCall &c) {
    const std::string what = std::string("prefill_") + c.name;
    if (refuse_peer(what) || io_check("prefill", c)) return -1;
    const bool combine = c.wts != nullptr, slot_rows = c.gate != kGateNone;   // slot_rows: one input row per slot (GLU), else per token
    const int N = c.N, topk = c.topk, n_experts = c.n_experts, count = c.count;
    if (n_experts > 256) return fail(what + ": n_experts must be 1..256");   // the routing kernel's shared arrays
    auto it0 = g.res.find(c.handles[0]);
    if (it0 == g.res.end()) return fail(what + ": bad weight handle");
    const StreamLayout &L = it0->second.L;
    if (!routed_tiles_take(L))
        return fail(what + ": the tiles take W2/W3/W4 fp-path tensors with the act group inside the chunk: per-row scales with K % 128 "
                    "== 0 (chunk 128/64/32 K), or one scale with act group < K and K % 128 == 0 or 64; use gemv_" + c.name + " for the others");
    const int S = N * topk, Mout = L.Mout, K = L.K, f16 = c.dtype == TMAC_B200_F16;
    // combine: the table's C is the slots' fp32 rows, so the workspace is allocated before the table is built
    if (combine && g.d_moe_ws.ensure((size_t)S * Mout * sizeof(float))) return fail(what + ": out of device memory (workspace)");
    const Resident *R = nullptr;
    BatchPtrs bp;
    if (grouped_setup(what.c_str(), c.handles, count * n_experts, nullptr, nullptr, nullptr, combine ? &g.d_moe_ws.p : c.C, &R, &bp, n_experts,
                      c.biasv))
        return -1;
    const PfExpertKernels fk = pick_pf_experts(L.pb, L.qch, L.agq(), L.one_scale, L.K % 128 != 0, c.bias);
    if (!fk.tile) return fail(what + ": no tile for chunk " + std::to_string(L.ck) + ", act group " + std::to_string(L.act_group_size));
    const TilePlan t(L, false);
    // the tile rule: routed experts as experts_take_tile16, the dense forms as the dense calls (launch_prefill)
    const bool t16 = (c.routed ? experts_take_tile16(N, topk, n_experts) : g.use_prefill16 && N >= 64) && t.fits16;
    if (!t16 && !t.fits8) return fail(what + ": the tensor's blocks do not fit the int8 tile's shared memory");
    const int T = t16 ? kP16NT : kPfNT;
    const long long cap = S / T + std::min(n_experts, S);
    if (cap > 65535) return fail(what + ": N * topk too large for one launch");
    const int rows = slot_rows ? S : N, nag = K / L.act_group_size, nsteps = t16 ? t.nmain + t.nextra : t.nmain;
    const bool act = c.gate != kGateNone || c.norm;   // a materialised fp32 input
    const size_t recb = t16 ? (size_t)kP16BBytes : t.rec;
    if (g.d_moe_route.ensure((size_t)cap * sizeof(int4) + (size_t)S * sizeof(int)) || (act && g.d_moe_act.ensure((size_t)rows * K * sizeof(float))) ||
        g.d_qlut.ensure((size_t)rows * K * 4) || g.d_ls.ensure((size_t)rows * nag * 4) || g.d_lb.ensure((size_t)rows * nag * 4) ||
        g.d_tiles.ensure((size_t)cap * nsteps * recb))
        return fail(what + ": out of device memory (workspace)");
    int4 *tiles = (int4 *)g.d_moe_route.p;
    int *perm = (int *)(tiles + cap);
    const int8_t *qlut = (const int8_t *)g.d_qlut.p;
    const float *ls = (const float *)g.d_ls.p, *lb = (const float *)g.d_lb.p;
    unsigned char *recs = (unsigned char *)g.d_tiles.p;
    const cudaStream_t st = g.stream();

    pf_route_launch(c.ids, S, n_experts, T, (int)cap, tiles, perm, c.routed && !combine ? bp.C : nullptr, count, Mout, f16, st);
    CUDA_OK(cudaGetLastError());
    if (act) {
        if (slot_rows) pf_swiglu_launch(c.A, c.U, f16, (size_t)rows * K, (float *)g.d_moe_act.p, st, c.gate == kGateRelu2);
        if (c.norm)   // after a gate: in place
            pf_rmsnorm_launch(slot_rows ? g.d_moe_act.p : c.A, slot_rows ? 0 : f16, c.w, c.eps, rows, K, (float *)g.d_moe_act.p, st);
        CUDA_OK(cudaGetLastError());
        if (launch_preprocessor(K, rows, L.act_group_size, TMAC_B200_F32, g.d_moe_act.p, (float *)ls, (float *)lb, (int8_t *)qlut)) return -1;
    } else if (launch_preprocessor(K, rows, L.act_group_size, c.dtype, c.A, (float *)ls, (float *)lb, (int8_t *)qlut)) return -1;
    const PfRoute route{tiles, perm, bp.W, bp.C, n_experts, combine ? nullptr : c.R, bp.bias};
    const int div = slot_rows ? 1 : topk, out_f16 = combine ? 0 : f16;
    const dim3 grid(t.nrt, (unsigned)cap, count);
    if (t16) {
        fk.lut16<<<dim3(nsteps, (unsigned)cap), 256, 0, st>>>(qlut, ls, lb, recs, K, t.nmain, t.nextra, tiles, perm, div);
        CUDA_OK(cudaGetLastError());
        auto q = tile_params<Prefill16Params>(L, t, N, Mout, out_f16);
        q.tiles = recs; q.ntiles = t.nrt * (int)cap;   // no stream-K split
        if (launch_tile(true, fk.tile16, grid, t, 0, L, S, q, route)) return -1;
    } else {
        fk.lut<<<dim3(nsteps, (unsigned)cap), 128, 0, st>>>(qlut, ls, lb, recs, K, tiles, perm, div);
        CUDA_OK(cudaGetLastError());
        auto p = tile_params<PrefillParams>(L, t, N, Mout, out_f16);
        p.lut_tiles = recs;   // qlut, lut_scales and lut_biases are read on the integer path only; scale0 by one-scale tensors
        if (launch_tile(false, fk.tile, grid, t, 1, L, S, p, route)) return -1;
    }
    if (combine) {
        pf_combine_launch((const float *)g.d_moe_ws.p, c.ids, c.wts, topk, n_experts, c.R, c.C[0], N, Mout, f16, st);
        CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int tmac_b200_prefill_experts(const int64_t *handles, int count, int n_experts, int N, int dtype, const void *B, const int32_t *ids,
                              int topk, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("experts", handles, count, N, dtype, B, C);
    c.routed = true; c.ids = ids; c.topk = topk; c.n_experts = n_experts;
    return prefill_io(c);
}

int tmac_b200_prefill_experts_glu(const int64_t *handles, int n_experts, int N, int dtype, const void *G, const void *U,
                                  const int32_t *ids, const float *weights, int topk, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("experts_glu", handles, 1, N, dtype, G, &C);
    c.routed = true; c.gate = kGateSilu; c.U = U; c.ids = ids; c.wts = weights; c.topk = topk; c.n_experts = n_experts; c.R = R;
    return prefill_io(c);
}

int tmac_b200_prefill_rmsnorm(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                              void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("rmsnorm", handles, count, N, dtype, H, C);
    c.norm = true; c.w = w; c.eps = eps;
    return prefill_io(c);
}

int tmac_b200_prefill_rmsnorm_bias(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                                   const float *const *bias, void *const *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("rmsnorm_bias", handles, count, N, dtype, H, C);
    c.norm = true; c.w = w; c.eps = eps; c.bias = true; c.biasv = bias;
    return prefill_io(c);
}

int tmac_b200_prefill_glu(int64_t handle, int N, int dtype, const void *G, const void *U, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("glu", &handle, 1, N, dtype, G, &C);
    c.gate = kGateSilu; c.U = U; c.R = R;
    return prefill_io(c);
}

int tmac_b200_prefill_residual(int64_t handle, int N, int dtype, const void *B, const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("residual", &handle, 1, N, dtype, B, &C);
    c.needs_R = true; c.R = R;
    return prefill_io(c);
}

int tmac_b200_prefill_subnorm(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps, const void *R,
                              void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("subnorm", &handle, 1, N, dtype, G, &C);
    c.gate = U ? kGateSilu : kGateNone; c.U = U; c.norm = true; c.w = w; c.eps = eps; c.R = R;
    return prefill_io(c);
}

int tmac_b200_prefill_subnorm_relu2(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps,
                                    const void *R, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    IoCall c("subnorm_relu2", &handle, 1, N, dtype, G, &C);
    c.gate = kGateRelu2; c.U = U; c.norm = true; c.w = w; c.eps = eps; c.R = R;
    return prefill_io(c);
}

int tmac_b200_gemv(int64_t handle, int N, int dtype, const void *B, void *C) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    auto it = g.res.find(handle);
    if (it == g.res.end()) return fail("gemv: bad weight handle");
    Resident &R = it->second;
    const StreamLayout &L = R.L;
    if (!B || !C || N <= 0) return fail("gemv: null/empty argument");
    const int nag = L.K / L.act_group_size;
    const size_t qb = (size_t)N * L.K * 4, sb = (size_t)N * nag * 4;
    const size_t bb = (size_t)N * L.K * esize(dtype), cb = (size_t)N * L.Mout * esize(dtype);
    void *pinB = nullptr, *pinC = nullptr;
    const int kind_b = ptr_kind(B, &pinB), kind_c = ptr_kind(C, &pinC);
    const bool dev_b = kind_b == 2, dev_c = kind_c == 2;
    const bool can_fuse = g.use_fused && (L.int_path() || L.act_group_size <= L.ck) && g.lut_mode != 1 && !takes_prefill_tile(L, N);
    auto launch_compute = [&](const void *dB, void *dC) -> int {
        if (can_fuse)   // one launch: the GEMV builds each chunk's LUT slice itself (bit-identical tables)
            return launch_gemv3(R, 0, L.Mout, N, Gemv3In::rows(kInRow, dB, dtype == TMAC_B200_F16), dC, L.Mout, 0, dtype == TMAC_B200_F16);
        if (g.d_qlut.ensure(qb) || g.d_ls.ensure(sb) || g.d_lb.ensure(sb)) return fail("out of device memory");
        if (launch_preprocessor(L.K, N, L.act_group_size, dtype, dB, (float *)g.d_ls.p, (float *)g.d_lb.p, (int8_t *)g.d_qlut.p)) return -1;
        return launch_gemv(R, 0, L.Mout, N, (const int8_t *)g.d_qlut.p, (const float *)g.d_ls.p, (const float *)g.d_lb.p, dC, L.Mout, 0,
                           dtype == TMAC_B200_F16, g.lut_mode != 1);
    };
    // The (small) output is stored by the kernel straight into page-locked host memory the device can address -- the
    // caller's own buffer when it is page-locked, else our staging buffer -- instead of a device buffer + D2H copy.
    void *dC = C;
    if (kind_c == 1) dC = pinC;
    else if (kind_c == 0) { if (g.h_out.ensure(cb)) return fail("out of pinned memory"); dC = g.h_out.p; }

    const void *dB = B;
    if (!dev_b) {
        stage_wait();
        if (kind_b == 1 && !dev_c) {
            // page-locked caller buffer as the copy source itself -- only when this call synchronises before returning (host
            // output); with a device output the call returns early and the caller may overwrite B at once: stage it instead
            if (g.d_b.ensure(bb)) return fail("out of device memory");
            CUDA_OK(cudaMemcpyAsync(g.d_b.p, pinB, bb, cudaMemcpyHostToDevice, g.stream()));
        } else {
            if (g.h_in.ensure(bb)) return fail("out of pinned memory");
            if (h2d(g.d_b, g.h_in, 0, B, bb)) return -1;
            stage_mark();
        }
        dB = g.d_b.p;
    }
    if (launch_compute(dB, dC)) return -1;
    if (!dev_c) {
        CUDA_OK(cudaStreamSynchronize(g.stream()));
        if (kind_c == 0) std::memcpy(C, g.h_out.p, cb);
    }
    return 0;
}

// ---- multi-GPU row sharding without a collective launch (SURVEY 8e) --------------------------------------------------
// Rows shard naturally (ref:ggml.c:12636-12691: tiles are independent given the replicated activation row), so the
// "all-gather" of a sharded GEMV is every rank storing its finished rows into every rank's output vector.  The next
// N = 1 launch (tmac_b200_gemv / tmac_b200_qgemm_lut) stores its rows, besides C, at ptrs[q] + the same index as C --
// device pointers into PEER memory (cudaIpcOpenMemHandle), each already offset to this shard's first row.  One-shot.
int tmac_b200_peer_outputs(void *const *ptrs, int count) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (count < 0 || count > 7 || (count && !ptrs)) return fail("peer_outputs: 0..7 peers");
    g.npeer = count;
    for (int q = 0; q < count; ++q) g.peer_out[q] = ptrs[q];
    return 0;
}
// One tiny launch: all launches this rank enqueued before it are complete, and so are the peers' up to their matching call --
// the flag / barrier per fused group of a row-sharded model (peer stores into `flags` of every rank; see peer_barrier_kernel).
// flags: this rank's (world + 1) x u32 array inside an ipc allocation; peer_flags[q]: rank q's array as mapped here.
int tmac_b200_peer_barrier(void *flags, void *const *peer_flags, int rank, int world) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (!flags || !peer_flags || world < 1 || world > 8 || rank < 0 || rank >= world) return fail("peer_barrier: bad arguments");
    // the pointer table lives in device memory (stable under graph capture): cached per (flags) key
    static std::map<void *, void *> tables;
    void *&dt = tables[flags];
    if (!dt) {
        if (cudaMalloc(&dt, 10 * sizeof(void *)) != cudaSuccess) { cudaGetLastError(); dt = nullptr; return fail("peer_barrier: out of device memory"); }
        void *host[9] = {};
        for (int q = 0; q < world; ++q) host[q] = peer_flags[q];
        CUDA_OK(cudaMemcpy(dt, host, sizeof host, cudaMemcpyHostToDevice));
    }
    peer_barrier_kernel<<<1, 32, 0, g.stream()>>>((unsigned *)flags, (unsigned *const *)dt, rank, world, (int *)((void **)dt + 8));
    CUDA_OK(cudaGetLastError());
    return 0;
}

// Device allocations that other processes of the node can map: alloc returns the pointer and a 64-byte handle to send to the
// peers; open maps a peer's allocation (peer access is enabled on demand); close / free undo them.
void *tmac_b200_ipc_alloc(size_t bytes, void *handle64) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return nullptr;
    void *p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); fail("ipc_alloc: out of device memory"); return nullptr; }
    cudaMemset(p, 0, bytes);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    if (cudaIpcGetMemHandle((cudaIpcMemHandle_t *)handle64, p) != cudaSuccess) { cudaGetLastError(); cudaFree(p); fail("cudaIpcGetMemHandle failed"); return nullptr; }
    return p;
}
void *tmac_b200_ipc_open(const void *handle64) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return nullptr;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle64, sizeof h);
    void *p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { cudaGetLastError(); fail(std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e)); return nullptr; }
    return p;
}
int tmac_b200_ipc_close(void *peer_ptr) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    CUDA_OK(cudaIpcCloseMemHandle(peer_ptr));
    return 0;
}
int tmac_b200_ipc_free(void *ptr) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (g.inited) cudaStreamSynchronize(g.stream());
    CUDA_OK(cudaFree(ptr));
    return 0;
}

// ---- decode sequences: a chain of dependent GEMVs in ONE persistent launch (tmac_seq.cuh) ---------------------------
// The reference runs a token step as ggml's graph loop over mul_mat nodes on a persistent thread pool
// (3rdparty/llama.cpp/ggml/src/ggml.c:12562-12706 per node); a sequence is that loop for the quantised linears.

int64_t tmac_b200_seq_create(void) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    const int64_t h = g_next_seq++;
    g_seqs[h];
    return h;
}

int tmac_b200_seq_set_batch(int64_t seq, int n) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_set_batch: bad sequence");
    Sequence &S = it->second;
    if (S.built || !S.ops.empty()) return fail("seq_set_batch: call before the first op is added");
    if (n < 1 || n > 4) return fail("seq_set_batch: 1 <= n <= 4 activation rows");
    S.nb = n;
    return 0;
}

// The checks both seq_add_gemv* entry points make: the sequence exists and is not built yet, the tensor exists, each of the
// nin inputs {op, offset} reads [offset, offset + K) of an earlier op's output at an even offset, and C is a device pointer or null.
static int seq_add_check(const char *what, int64_t seq, int64_t handle, const std::pair<int, int> *in, int nin, const void *C, Sequence **out) {
    const std::string w(what);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail(w + ": bad sequence");
    Sequence &S = it->second;
    if (S.built) return fail(w + ": sequence already built");
    auto rt = g.res.find(handle);
    if (rt == g.res.end()) return fail(w + ": bad weight handle");
    const StreamLayout &L = rt->second.L;
    for (int i = 0; i < nin; ++i) {
        const auto [src, off] = in[i];
        if (src < 0 || src >= (int)S.ops.size()) return fail(w + ": an input op must name an earlier op of the sequence");
        const auto pt = g.res.find(S.ops[src].handle);
        if (pt == g.res.end()) return fail(w + ": a producer's weight handle was freed");
        if (off < 0 || off % 2 || off + L.K > pt->second.L.Mout) return fail(w + ": [offset, offset + K) must lie inside the producer's output (even offset)");
    }
    if (C && !is_device_ptr(C)) return fail(w + ": C must be a device pointer (or NULL)");
    *out = &S;
    return 0;
}

int tmac_b200_seq_add_gemv(int64_t seq, int64_t handle, const void *x, int in_op, int in_offset, void *C, int dtype) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    const std::pair<int, int> in{in_op, in_offset};
    Sequence *S = nullptr;
    if (seq_add_check("seq_add_gemv", seq, handle, &in, x ? 0 : 1, C, &S)) return -1;
    if (x) {
        if (!is_device_ptr(x)) return fail("seq_add_gemv: the external input must be a device pointer");
        if ((uintptr_t)x % 16) return fail("seq_add_gemv: the external input must be 16-byte aligned");
    }
    S->ops.push_back({handle, x, x ? -1 : in_op, in_offset, C, dtype == TMAC_B200_F16});
    return (int)S->ops.size() - 1;
}

int tmac_b200_seq_add_gemv_glu(int64_t seq, int64_t handle, int gate_op, int gate_offset, int up_op, int up_offset, void *C, int dtype) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    const std::pair<int, int> in[2] = {{gate_op, gate_offset}, {up_op, up_offset}};
    Sequence *S = nullptr;
    if (seq_add_check("seq_add_gemv_glu", seq, handle, in, 2, C, &S)) return -1;
    SeqOpHost o{handle, nullptr, gate_op, gate_offset, C, dtype == TMAC_B200_F16};
    o.in_op2 = up_op; o.in_off2 = up_offset;
    S->ops.push_back(o);
    return (int)S->ops.size() - 1;
}

int tmac_b200_seq_add_gemv_rmsnorm(int64_t seq, int64_t handle, int in_op, const float *w, float eps, void *C, int dtype) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    const std::pair<int, int> in{in_op, 0};
    Sequence *S = nullptr;
    if (seq_add_check("seq_add_gemv_rmsnorm", seq, handle, &in, 1, C, &S)) return -1;
    if (g.res.find(handle)->second.L.K != g.res.find(S->ops[in_op].handle)->second.L.Mout)
        return fail("seq_add_gemv_rmsnorm: K must equal the producer's Mout (the norm is over its whole output)");
    if (!is_device_ptr(w) || (uintptr_t)w % 16) return fail("seq_add_gemv_rmsnorm: w must be a 16-byte aligned device pointer");
    if (!std::isfinite(eps) || eps < 0.f) return fail("seq_add_gemv_rmsnorm: eps must be finite and >= 0");
    SeqOpHost o{handle, nullptr, in_op, 0, C, dtype == TMAC_B200_F16};
    o.nw = w; o.eps = eps;
    S->ops.push_back(o);
    return (int)S->ops.size() - 1;
}

int tmac_b200_seq_residual(int64_t seq, int op, const float *r, int r_op) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_residual: bad sequence");
    Sequence &S = it->second;
    if (S.built) return fail("seq_residual: sequence already built");
    if (op < 0 || op >= (int)S.ops.size()) return fail("seq_residual: bad op");
    if (S.ops[op].res) return fail("seq_residual: the op already has a residual");
    if (r) {
        if (r_op != -1) return fail("seq_residual: give either r or r_op");
        if (!is_device_ptr(r) || (uintptr_t)r % 16) return fail("seq_residual: r must be a 16-byte aligned device pointer");
    } else {
        if (r_op < 0 || r_op >= op) return fail("seq_residual: r_op must name an earlier op of the sequence");
        const auto a = g.res.find(S.ops[op].handle), b = g.res.find(S.ops[r_op].handle);
        if (a == g.res.end() || b == g.res.end()) return fail("seq_residual: a weight handle was freed");
        if (a->second.L.Mout != b->second.L.Mout) return fail("seq_residual: r_op must have the op's Mout");
    }
    S.ops[op].res = true; S.ops[op].r = r; S.ops[op].r_op = r ? -1 : r_op;
    return 0;
}

/* Multi-GPU row sharding inside a sequence (as tmac_b200_peer_outputs for single launches): op `op` also stores its finished rows
 * at ptrs[q][row] -- device pointers into PEER memory, each already offset to this shard's first row.  Before seq_build. */
int tmac_b200_seq_peer_outputs(int64_t seq, int op, void *const *ptrs, int count) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_peer_outputs: bad sequence");
    Sequence &S = it->second;
    if (S.built) return fail("seq_peer_outputs: sequence already built");
    if (op < 0 || op >= (int)S.ops.size() || count < 0 || count > 7 || (count && !ptrs)) return fail("seq_peer_outputs: bad op / 0..7 peers");
    if (!S.ops[op].C) return fail("seq_peer_outputs: the op has no output vector");
    S.ops[op].npeer = count;
    for (int q = 0; q < count; ++q) S.ops[op].peer[q] = ptrs[q];
    return 0;
}

// Reserves `bytes` at an `align` boundary after the `total` bytes laid out so far; returns their offset.
static size_t reserve(size_t &total, size_t bytes, size_t align = 256) {
    const size_t off = (total + align - 1) & ~(align - 1);
    total = off + bytes;
    return off;
}
// A sequence's allocation starts with its {value, epoch} words (and the stream-K kernel's exchange slots and LUT records); the
// descriptors, flags and trace start on the next 2 MB page.  Against a separate allocation per buffer, bench.py's dependent
// resident-chain step took 1-1.5% longer with the descriptors right behind the words, 0-0.4% longer this way (H100 SXM 80 GB, 700 W).
constexpr size_t kSeqPage = (size_t)2 << 20;

// Raises fn's dynamic shared-memory limit to smem, and never lowers it: sequences built earlier on the same kernel with more
// shared memory keep launching.
static cudaError_t raise_smem_limit(const void *fn, size_t smem) {
    cudaFuncAttributes fa{};
    cudaError_t e = cudaFuncGetAttributes(&fa, fn);
    if (e == cudaSuccess && (int)smem > fa.maxDynamicSharedSizeBytes) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    return e;
}

// Zeroes the sequence's allocation of `bytes`, copies the host arrays {device address, host data, bytes} into it and waits (on the
// library's stream: the legacy default stream does not order against a non-blocking stream).  On failure the allocation is freed,
// so that the next seq_build starts clean.
static int seq_upload(Sequence &S, size_t bytes, std::initializer_list<std::tuple<void *, const void *, size_t>> copies) {
    cudaError_t e = cudaMemsetAsync(S.d_mem, 0, bytes, g.stream());
    for (const auto &[dst, src, n] : copies) if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, g.stream());
    if (e == cudaSuccess) e = cudaStreamSynchronize(g.stream());
    if (e == cudaSuccess) return 0;
    S.release();
    return fail(std::string("seq_build: ") + cudaGetErrorString(e));
}

// Resident gemv3 chain (tmac_chain.cuh) of a sequence whose format tmac_b200_seq_build has checked and set; R[i] is op i's tensor.
// 1 = built, 0 = the sequence does not qualify (caller falls back), -1 = error.
static int seq_build_chain(Sequence &S, const std::vector<const Resident *> &R) {
    const int n = (int)S.ops.size();
    std::vector<ChainOp> ops(n);
    std::vector<ChainGlu> glus(n);
    std::vector<SeqLayer> lays(n);
    std::vector<size_t> coff(n, (size_t)-1), lloff(n, 0);
    size_t ctot = 0, max_blk = 0, lltot = 0;
    int max_nrsb = 0, max_bpw = 0, rsbsz = 0;
    bool glu = false, layer = false;
    auto chain_bpw = [](int nchunk) { return (nchunk + kChainCS * kChainWarps - 1) / (kChainCS * kChainWarps); };
    // float4 loads (16-byte word pairs in data-flow mode) of an fp32 producer; in a batch, of every row of it
    auto loadable = [&](int src, int off) {
        return off % ((g.chain_flags & kChainBarrier) ? 4 : 2) == 0 && !S.ops[src].out_f16 && (S.nb == 1 || R[src]->L.Mout % 4 == 0);
    };
    for (int i = 0; i < n; ++i) {
        const StreamLayout &L = R[i]->L;
        rsbsz = L.rsb;                   // one bit width: one super-block size
        if (S.ops[i].x_ext) { if ((uintptr_t)S.ops[i].x_ext % 16) return 0; }
        else if (!loadable(S.ops[i].in_op, S.ops[i].in_off)) return 0;
        if (S.ops[i].in_op2 >= 0) {
            if (!loadable(S.ops[i].in_op2, S.ops[i].in_off2)) return 0;
            glu = true;
        }
        if (S.ops[i].r_op >= 0 && S.ops[S.ops[i].r_op].out_f16) return 0;   // the barrier form reads the residual op's fp32 C
        layer = layer || S.ops[i].layer() || S.nb > 1;   // batches: the layer instantiation
        max_blk = std::max(max_blk, (L.blk + 127) & ~(size_t)127);
        max_nrsb = std::max(max_nrsb, L.nrsb);
        max_bpw = std::max(max_bpw, chain_bpw(L.nchunk));
        if (!S.ops[i].C) coff[i] = reserve(ctot, (size_t)S.nb * L.nrsb * L.rsb * sizeof(float));
        lloff[i] = reserve(lltot, (size_t)S.nb * L.nrsb * L.rsb * sizeof(uint2));
    }
    const int grid = max_nrsb * kChainCS;
    // The kernel: the decode-ahead instantiation (registers for the decoded quads, bounded to 3 CTAs per SM) when every cluster
    // stays resident with it, else the one without (5 CTAs per SM), e.g. for 18944 rows (592 CTAs on 132 SMs).
    // Ring depth: the deepest per-warp stage ring, up to one op of blocks ahead (max_bpw + 1 stages), with which every cluster is
    // still resident at once -- the waits between clusters spin.
    chain_fn fn = nullptr;
    int nstage = 0;
    SeqLaunch shape;
    for (int ahead = g.chain_ahead && S.nb == 1 ? 1 : 0; ahead >= 0 && !nstage; --ahead) {
        fn = pick_chain(S.pb, S.qch, S.agq, glu, layer, ahead != 0, S.nb);
        if (!fn) return 0;
        cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        for (int s = max_bpw + 1; s >= 2 && !nstage; --s) {
            shape = chain_launch(grid, (size_t)(kChainCS + kChainWarps) * S.nb * rsbsz * 4 +
                                       (size_t)kChainWarps * chain_warp_smem((int)max_blk, s, S.nb, S.qch * 4, rsbsz) + (size_t)kChainWarps * s * 8 + 32);
            const cudaLaunchConfig_t cfg = shape.config(0);
            int nc = 0;
            if (raise_smem_limit((const void *)fn, shape.smem) != cudaSuccess || cudaOccupancyMaxActiveClusters(&nc, (const void *)fn, &cfg) != cudaSuccess) { cudaGetLastError(); continue; }
            if (nc >= max_nrsb) nstage = s;
        }
    }
    if (!nstage) return 0;
    static_assert(sizeof(ChainOp) % alignof(ChainGlu) == 0, "the ChainGlu array follows the ChainOp array");
    static_assert((sizeof(ChainOp) + sizeof(ChainGlu)) % alignof(SeqLayer) == 0, "the SeqLayer array follows the ChainGlu array");
    size_t tot = 0;
    const size_t o_y = reserve(tot, lltot), o_ops = reserve(tot, n * (sizeof(ChainOp) + sizeof(ChainGlu) + sizeof(SeqLayer)), kSeqPage),
                 o_bar = reserve(tot, sizeof(unsigned)), o_epochs = reserve(tot, grid * sizeof(unsigned)), o_err = reserve(tot, sizeof(int)),
                 o_cint = reserve(tot, ctot), o_trace = reserve(tot, g.trace ? seq_trace_bytes(n, grid) : 0);
    if (cudaMalloc(&S.d_mem, tot) != cudaSuccess) { cudaGetLastError(); S.d_mem = nullptr; return fail("seq_build: out of device memory"); }
    char *const d = (char *)S.d_mem;
    char *const cint = d + o_cint, *const y = d + o_y;
    for (int i = 0; i < n; ++i) {
        const StreamLayout &L = R[i]->L;
        ChainOp &o = ops[i];
        o.W = R[i]->d;
        o.C = S.ops[i].C ? S.ops[i].C : (void *)(cint + coff[i]);
        o.x = S.ops[i].x_ext ? (const float *)S.ops[i].x_ext : (const float *)ops[S.ops[i].in_op].C + S.ops[i].in_off;
        o.rsb_stride = L.rsb_stride; o.K = L.K; o.Mout = L.Mout; o.nrsb = L.nrsb; o.nchunk = L.nchunk;
        o.blk_bytes = (int)L.blk; o.bpw = chain_bpw(L.nchunk);
        o.zp = L.zp; o.one_scale = L.one_scale; o.sd = L.sd; o.out_f16 = S.ops[i].out_f16; o.scale0 = L.scale0;
        o.in_op = S.ops[i].x_ext ? -1 : S.ops[i].in_op;
        o.npeer = S.ops[i].npeer; o.pad_ = 0;
        for (int q = 0; q < 7; ++q) o.Cpeer[q] = q < S.ops[i].npeer ? S.ops[i].peer[q] : nullptr;

        o.ll_out = (uint2 *)(y + lloff[i]);
        o.ll_in = S.ops[i].x_ext ? nullptr : (const uint2 *)(y + lloff[S.ops[i].in_op]) + S.ops[i].in_off;
        const int up = S.ops[i].in_op2;
        ChainGlu &q = glus[i];
        q.x2 = up >= 0 ? (const float *)ops[up].C + S.ops[i].in_off2 : nullptr;
        q.ll_in2 = up >= 0 ? (const uint2 *)(y + lloff[up]) + S.ops[i].in_off2 : nullptr;
        q.in_op2 = up; q.pad_ = 0;
        const SeqOpHost &h = S.ops[i];
        lays[i] = SeqLayer{h.nw, h.r ? h.r : h.r_op >= 0 ? (const float *)ops[h.r_op].C : nullptr,
                           h.r_op >= 0 ? (const uint2 *)(y + lloff[h.r_op]) : nullptr, h.eps, h.r_op};
    }
    ChainOp *const d_ops = (ChainOp *)(d + o_ops);
    ChainGlu *const d_glus = (ChainGlu *)(d_ops + n);
    SeqLayer *const d_lays = (SeqLayer *)(d_glus + n);
    // (the words start zeroed: epoch 0 never matches, launches publish epochs >= 1)
    if (seq_upload(S, tot, {{d_ops, ops.data(), n * sizeof(ChainOp)}, {d_glus, glus.data(), n * sizeof(ChainGlu)}, {d_lays, lays.data(), n * sizeof(SeqLayer)}}))
        return -1;
    S.d_err = (int *)(d + o_err); S.d_trace = g.trace ? (long long *)(d + o_trace) : nullptr;
    S.cparams.ops = d_ops; S.cparams.nops = n; S.cparams.max_blk = (int)max_blk; S.cparams.nstage = nstage;
    S.cparams.glu = glu || layer ? d_glus : nullptr;
    S.cparams.bar = (unsigned *)(d + o_bar); S.cparams.epochs = (unsigned *)(d + o_epochs); S.cparams.err = S.d_err;
    S.cparams.flags = g.chain_flags; S.cparams.trace = S.d_trace;
    S.cfn = fn; S.impl = 1; S.launch = shape;
    S.built = true;
    return 1;
}

// Stream-K sequence kernel (tmac_seq.cuh) of a sequence whose format tmac_b200_seq_build has checked and set; R[i] is op i's tensor.
static int seq_build_streamk(Sequence &S, const std::vector<const Resident *> &R) {
    const int G = g.seq_grid > 0 ? std::min(g.seq_grid, g.sms) : g.sms;
    const int n = (int)S.ops.size();
    std::vector<SeqOp> ops(n);
    std::vector<SeqLayer> lays(n);
    std::vector<SeqCta> ct((size_t)n * G);
    std::vector<size_t> yoff(n);
    size_t ytot = 0, red_b = 0, tab_b = 0, lsb_b = 0, slot_b = 0, yfin_b = 0, ltot = 0;
    int rsbmax = 0;
    std::vector<size_t> loff(n, (size_t)-1);       // LUT hand-over records of op i (only if an aligned consumer exists)
    std::vector<char> takes(n, 0);                 // op i takes its producer's LUT records
    bool glu = false, layer = false;
    const bool handover = g.seq_handover != 0;
    for (int i = 0; i < n; ++i) {
        const StreamLayout &L = R[i]->L;
        const long total = (long)L.nrsb * L.nchunk;
        const long ge = std::min<long>(G, total);
        const int per = (int)((total + ge - 1) / ge);
        const int nseg = (per - 1 + L.nchunk - 1) / L.nchunk + 1;
        const int ntab = std::min(per, L.nchunk);
        const int nag = L.qch / S.agq;
        red_b = std::max(red_b, (size_t)nseg * kSeqWarps * L.rsb * 4);
        yfin_b = std::max(yfin_b, (size_t)nseg * L.rsb * 4);
        glu = glu || S.ops[i].in_op2 >= 0;
        layer = layer || S.ops[i].layer();
        // consumer of an earlier op: can it take ready-made LUT records?  (A GLU op builds its LUT from two producers' rows, a
        // norm op from the norm of its producer's whole row.)
        if (!S.ops[i].x_ext && S.ops[i].in_op2 < 0 && !S.ops[i].nw && handover) {
            const int src = S.ops[i].in_op;
            const StreamLayout &PL = R[src]->L;
            takes[i] = S.ops[i].in_off % L.act_group_size == 0 && PL.rsb % L.act_group_size == 0;
            const size_t rows = (size_t)PL.nrsb * PL.rsb;
            if (takes[i] && loff[src] == (size_t)-1) loff[src] = reserve(ltot, (rows / 4 + rows / L.act_group_size) * sizeof(uint4));
        }
        tab_b = std::max(tab_b, (size_t)ntab * L.qch * 4 * 8);
        lsb_b = std::max(lsb_b, (size_t)ntab * 2 * nag * 4);
        slot_b = std::max(slot_b, (L.blk + 127) & ~(size_t)127);
        rsbmax = std::max(rsbmax, L.rsb);
        yoff[i] = reserve(ytot, (size_t)L.nrsb * L.rsb * sizeof(uint2));
    }
    const size_t budget = (size_t)std::max(64, std::min(227, g.seq_smem_kb)) * 1024;
    const size_t fixed = ((red_b + 15) & ~(size_t)15) + ((tab_b + 15) & ~(size_t)15) + ((lsb_b + 15) & ~(size_t)15) + ((yfin_b + 15) & ~(size_t)15) + 64 * 8 + (kSeqWarps + 1) * 4 + 64 + 2 * kSeqDescWords * 4;
    if (fixed + 4 * slot_b > budget) return fail("seq_build: shared-memory budget exceeded");
    const int nslots = (int)std::min<size_t>(64, (budget - fixed) / slot_b);
    const seq_fn fn = pick_seq(S.pb, S.qch, S.agq, glu, layer);
    if (!fn) return fail("seq_build: chunking not instantiated");
    SeqParams &P = S.params;
    P.nops = n; P.nslots = nslots; P.slot_bytes = (int)slot_b;
    size_t off = (size_t)nslots * slot_b;
    P.red_off = (int)off; off += (red_b + 15) & ~(size_t)15;
    P.tab_off = (int)off; off += (tab_b + 15) & ~(size_t)15;
    P.lsb_off = (int)off; off += (lsb_b + 15) & ~(size_t)15;
    P.bar_off = (int)off; off += (size_t)nslots * 8;
    P.prog_off = (int)off; off += (kSeqWarps + 1) * 4;   // + the producer's `issued` counter
    off = (off + 15) & ~(size_t)15;
    P.yfin_off = (int)off; off += (yfin_b + 15) & ~(size_t)15;
    P.desc_off = (int)off; off += 2 * kSeqDescWords * 4;
    CUDA_OK(raise_smem_limit((const void *)fn, off));

    const size_t xper = (size_t)G * rsbmax * sizeof(uint2);
    static_assert(sizeof(SeqOp) % alignof(SeqLayer) == 0, "the SeqLayer array follows the SeqOp array");
    size_t tot = 0;
    const size_t o_y = reserve(tot, ytot), o_xchg = reserve(tot, xper * n), o_lut = reserve(tot, ltot),
                 o_ops = reserve(tot, n * (sizeof(SeqOp) + sizeof(SeqLayer)), kSeqPage), o_ctas = reserve(tot, ct.size() * sizeof(SeqCta)),
                 o_epochs = reserve(tot, G * sizeof(unsigned)), o_err = reserve(tot, sizeof(int)), o_trace = reserve(tot, g.trace ? seq_trace_bytes(n, G) : 0);
    if (cudaMalloc(&S.d_mem, tot) != cudaSuccess) { cudaGetLastError(); S.d_mem = nullptr; return fail("seq_build: out of device memory"); }
    char *const d = (char *)S.d_mem;
    char *const y = d + o_y, *const lut = d + o_lut;
    for (int i = 0; i < n; ++i) {
        const StreamLayout &L = R[i]->L;
        SeqOp &o = ops[i];
        o.W = R[i]->d;
        o.x_ext = (const float *)S.ops[i].x_ext;
        o.x_ll = S.ops[i].x_ext ? nullptr : (const uint2 *)(y + yoff[S.ops[i].in_op]) + S.ops[i].in_off;
        o.x_ll2 = S.ops[i].in_op2 >= 0 ? (const uint2 *)(y + yoff[S.ops[i].in_op2]) + S.ops[i].in_off2 : nullptr;
        o.C = S.ops[i].C;
        o.y = (uint2 *)(y + yoff[i]);
        o.xchg = (uint2 *)(d + o_xchg + xper * i);
        o.rsb_stride = L.rsb_stride;
        o.K = L.K; o.Mout = L.Mout; o.nrsb = L.nrsb; o.nchunk = L.nchunk;
        o.blk_bytes = (int)L.blk; o.total = L.nrsb * L.nchunk;
        o.zp = L.zp; o.one_scale = L.one_scale; o.sd = L.sd; o.out_f16 = S.ops[i].out_f16;
        o.scale0 = L.scale0; o.geff = std::min(G, o.total);
        o.lut_out = o.ag_out = nullptr; o.lut_in = o.ag_in = nullptr;
        if (loff[i] != (size_t)-1) {
            o.lut_out = (uint4 *)(lut + loff[i]);
            o.ag_out = o.lut_out + (size_t)L.nrsb * L.rsb / 4;
        }
        if (takes[i]) {
            const StreamLayout &PL = R[S.ops[i].in_op]->L;
            const uint4 *base = (const uint4 *)(lut + loff[S.ops[i].in_op]);
            o.lut_in = base + S.ops[i].in_off / 4;
            o.ag_in = base + (size_t)PL.nrsb * PL.rsb / 4 + S.ops[i].in_off / L.act_group_size;
        }
        const SeqOpHost &h = S.ops[i];
        lays[i] = SeqLayer{h.nw, h.r, h.r_op >= 0 ? (const uint2 *)(y + yoff[h.r_op]) : nullptr, h.eps, h.r_op};
    }
    const int pmax = std::max(1, nslots / 2);
    for (int i = 0; i < n; ++i) {   // per (op, CTA) shares: blocks [T*c/GE, T*(c+1)/GE) in (row super-block, chunk) order
        const long T = ops[i].total, GE = ops[i].geff, nc = ops[i].nchunk;
        auto first_block = [&](long c) { return T * c / GE; };
        for (int c = 0; c < G; ++c) {
            SeqCta &q = ct[(size_t)i * G + c];
            std::memset(&q, 0, sizeof q);
            q.fc = c;
            if (c >= GE) continue;
            const long b0 = first_block(c), b1 = first_block(c + 1);
            q.b0 = (int)b0; q.nb = (int)(b1 - b0);
            q.sb_first = (int)(b0 / nc); q.c0 = (int)(b0 % nc);
            q.nseg = (int)((b1 - 1) / nc - b0 / nc + 1);
            q.nck = (int)std::min<long>(q.nb, nc);
            q.npass = (q.nb + pmax - 1) / pmax;
            q.P = (q.nb + q.npass - 1) / q.npass;
            q.last_open = (b1 % nc) != 0;                     // my last super-block continues in CTA c + 1
            int fc = c;                                       // CTA that owns the first block of my first super-block
            while (fc > 0 && first_block(fc) > (long)q.sb_first * nc) --fc;
            q.fc = fc;
        }
    }
    SeqOp *const d_ops = (SeqOp *)(d + o_ops);
    if (seq_upload(S, tot, {{d_ops, ops.data(), n * sizeof(SeqOp)}, {d_ops + n, lays.data(), n * sizeof(SeqLayer)}, {d + o_ctas, ct.data(), ct.size() * sizeof(SeqCta)}}))
        return -1;
    S.d_err = (int *)(d + o_err); S.d_trace = g.trace ? (long long *)(d + o_trace) : nullptr;
    P.ops = d_ops; P.ctas = (const SeqCta *)(d + o_ctas);
    P.epochs = (unsigned *)(d + o_epochs); P.err = S.d_err; P.trace = S.d_trace;
    S.fn = fn;
    S.launch = SeqLaunch{G, kSeqThreads, off};
    S.launch.attr.id = cudaLaunchAttributeCooperative;      // every CTA must be resident: CTAs wait for each other's rows
    S.launch.attr.val.cooperative = 1;
    S.built = true;
    return 0;
}

int tmac_b200_seq_build(int64_t seq) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_build: bad sequence");
    Sequence &S = it->second;
    if (S.built) return 0;
    if (S.ops.empty()) return fail("seq_build: empty sequence");
    std::vector<const Resident *> R(S.ops.size());
    for (size_t i = 0; i < S.ops.size(); ++i) {   // both sequence kernels: the fp path, one bit width and grouping for every op
        auto rt = g.res.find(S.ops[i].handle);
        if (rt == g.res.end()) return fail("seq_build: a weight handle was freed");
        R[i] = &rt->second;
        const StreamLayout &L = rt->second.L;
        if (L.int_path() || L.act_group_size > L.ck) return fail("seq_build: activation group must lie inside a chunk (fp path)");
        if (i == 0) { S.pb = L.pb; S.qch = L.qch; S.agq = L.agq(); S.bits = L.bits; }
        else if (S.pb != L.pb || S.qch != L.qch || S.agq != L.agq() || S.bits != L.bits) return fail("seq_build: all tensors of a sequence must share bits / grouping");
    }
    if (S.nb > 1) {   // batches run in the resident chain kernel only
        const char *why = g.seq_impl == 0 ? "seq_impl 0 selects the stream-K kernel" : g.seq_grid > 0 ? "seq_grid selects the stream-K kernel" : nullptr;
        for (auto &o : S.ops) if (o.npeer) why = "peer outputs are not supported";
        if (why) return fail(std::string("seq_build: a batch (seq_set_batch n > 1) needs the resident chain kernel, and ") + why);
        const int rc = seq_build_chain(S, R);
        if (rc != 0) return rc < 0 ? -1 : 0;
        return fail("seq_build: a batch (seq_set_batch n > 1) needs the resident chain kernel, and the sequence does not qualify for it "
                    "(fp32 16-byte aligned inputs, producers' Mout a multiple of 4, all clusters resident with the batch kernel)");
    }
    if (g.seq_impl >= 1 && g.seq_grid == 0) {
        const int rc = seq_build_chain(S, R);
        if (rc != 0) return rc < 0 ? -1 : 0;
        if (g.seq_impl == 1) return fail("seq_build: the sequence does not qualify for the resident chain kernel (fp32 16-byte aligned inputs, clusters resident)");
    }
    for (auto &o : S.ops) if (o.npeer) return fail("seq_build: peer outputs need the resident chain kernel, and this sequence does not qualify for it");
    return seq_build_streamk(S, R);
}

int tmac_b200_seq_launch(int64_t seq) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_launch: bad sequence");
    Sequence &S = it->second;
    if (!S.built) return fail("seq_launch: call tmac_b200_seq_build first");
    uint32_t wtx, wty;
    plane_weight_regs(S.bits, true, &wtx, &wty);
    const cudaLaunchConfig_t cfg = S.launch.config(g.stream());
    if (S.impl == 1) CUDA_OK(cudaLaunchKernelEx(&cfg, S.cfn, S.cparams, wtx, wty));
    else CUDA_OK(cudaLaunchKernelEx(&cfg, S.fn, S.params, wtx, wty));
    return 0;
}

/* Synchronises the stream and returns the sequence's error flag (0 = every wait completed). */
int tmac_b200_seq_status(int64_t seq) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end() || !it->second.built) return fail("seq_status: bad sequence");
    CUDA_OK(cudaStreamSynchronize(g.stream()));
    int e = 0;
    CUDA_OK(cudaMemcpy(&e, it->second.d_err, sizeof(int), cudaMemcpyDeviceToHost));
    if (e) return fail("sequence kernel: a bounded wait expired (code " + std::to_string(e) + ")");
    return 0;
}

/* info[8] = {grid, ring slots, slot bytes, shared memory bytes, ops, planes/word, quads/chunk, quads/act group} */
int tmac_b200_seq_info(int64_t seq, int *out8) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end() || !it->second.built || !out8) return fail("seq_info: bad sequence");
    const Sequence &S = it->second;
    const int v[8] = {S.launch.grid, S.impl == 1 ? -kChainCS : S.params.nslots, S.impl == 1 ? S.cparams.max_blk : S.params.slot_bytes, (int)S.launch.smem, (int)S.ops.size(), S.pb, S.qch, S.agq};
    std::memcpy(out8, v, sizeof v);
    return 0;
}

/* Debug (knob "trace" set before seq_build): globaltimer stamps [ops][grid][8] of the last launch; returns grid. */
int tmac_b200_seq_trace(int64_t seq, long long *dst, size_t cap_bytes) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end() || !it->second.built || !it->second.d_trace) return fail("seq_trace: tracing was not enabled when the sequence was built");
    CUDA_OK(cudaStreamSynchronize(g.stream()));
    const size_t bytes = std::min(cap_bytes, seq_trace_bytes(it->second.ops.size(), it->second.launch.grid));
    CUDA_OK(cudaMemcpy(dst, it->second.d_trace, bytes, cudaMemcpyDeviceToHost));
    return it->second.launch.grid;
}

int tmac_b200_seq_free(int64_t seq) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_seqs.find(seq);
    if (it == g_seqs.end()) return fail("seq_free: bad sequence");
    if (g.inited) cudaStreamSynchronize(g.stream());
    it->second.release();
    g_seqs.erase(it);
    return 0;
}

int tmac_b200_cbits(int64_t handle, int N, const void *QLUT, int32_t *CBits) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    auto it = g.res.find(handle);
    if (it == g.res.end()) return fail("cbits: bad weight handle");
    Resident &R = it->second;
    const StreamLayout &L = R.L;
    if (!QLUT || !CBits || N <= 0) return fail("cbits: null/empty argument");
    const size_t qb = (size_t)N * L.K * 4, ob = (size_t)N * L.Mout * L.bits * 4;
    const int8_t *dq = (const int8_t *)QLUT;
    if (!is_device_ptr(QLUT)) {
        stage_wait();
        if (g.h_in.ensure(qb)) return fail("out of pinned memory");
        if (h2d(g.d_qlut, g.h_in, 0, QLUT, qb)) return -1;
        stage_mark();
        dq = (const int8_t *)g.d_qlut.p;
    }
    const bool dev_o = is_device_ptr(CBits);
    int32_t *dout = CBits;
    if (!dev_o) {
        if (g.d_cbits.ensure(ob)) return fail("out of device memory");
        dout = (int32_t *)g.d_cbits.p;
    }
    const long long total = (long long)N * L.Mout * L.bits;
    cbits_kernel<<<(unsigned)((total + 255) / 256), 256, 0, g.stream()>>>(R.d, dq, dout, L.Mout, L.K, L.bits, L.pb, L.qch, L.nchunk,
                                                                         L.rsb_stride, L.blk, N);
    CUDA_OK(cudaGetLastError());
    if (!dev_o) {
        CUDA_OK(cudaMemcpyAsync(CBits, dout, ob, cudaMemcpyDeviceToHost, g.stream()));
        CUDA_OK(cudaStreamSynchronize(g.stream()));
    }
    return 0;
}

// ---- reference dispatchers ---------------------------------------------------------------
int preprocessor_int8(int m, int k, int n, int b, void *B, void *LUT_Scales, void *LUT_Biases, void *QLUT) {
    int ags, dtype;
    {
        std::unique_lock<std::shared_mutex> lk(g_mu);
        const tmac_b200_kcfg *c = find_kcfg_locked(m, k, b);
        if (!c) return fail("preprocessor_int8: shape not configured (m=" + std::to_string(m) + ", k=" + std::to_string(k) + ", b=" + std::to_string(b) + ")");
        ags = c->act_group_size;
        dtype = g.float_type;
    }
    return tmac_b200_preprocessor(k, n, ags, dtype, B, LUT_Scales, LUT_Biases, QLUT);
}

int qgemm_lut_int8(int m, int k, int n, int b, void *A, void *LUT, void *Scales, void *LUT_Scales, void *LUT_Biases, void *C) {
    (void)Scales;  // the resident copy carries the scales that were uploaded together with A
    if (g.inited && b >= 1 && b <= 4 && m > 0 && m % b == 0 && !is_device_ptr(LUT) && !is_device_ptr(C)) {
        // read-only fast path (shared lock): a tile call of a mat-vec whose whole-tensor result is already in page-locked memory
        // (computed by an earlier tile call with the same LUT bytes) only copies its rows -- ggml's workers do this concurrently
        std::shared_lock<std::shared_mutex> rl(g_mu);
        size_t off = 0;
        Resident *R = find_by_alias(A, &off);
        if (R && R->cfg.K == k && R->cfg.bits == b) {
            const size_t tile_bytes = (size_t)(k / 4) * R->cfg.bm / 2;
            const int row0 = (int)(off / tile_bytes) * (R->cfg.bm / b), rows = m / b;
            const size_t qb = (size_t)n * k * 4, sb = (size_t)n * (k / R->L.act_group_size) * 4, es = esize(g.float_type);
            if (off % tile_bytes == 0 && row0 + rows <= R->L.Mout)
                for (HostLut &e : g.hluts)
                    if (e.hq == LUT && e.res_id == R->id && e.res_dtype == g.float_type && e.N == n && e.qb == qb && e.sb == sb &&
                        e.copy.size() == qb + 2 * sb && !std::memcmp(e.copy.data(), LUT, qb) && !std::memcmp(e.copy.data() + qb, LUT_Scales, sb) &&
                        !std::memcmp(e.copy.data() + qb + sb, LUT_Biases, sb)) {
                        for (int r = 0; r < n; ++r)
                            std::memcpy((char *)C + (size_t)r * rows * es, (const char *)e.res.p + ((size_t)r * R->L.Mout + row0) * es, (size_t)rows * es);
                        return 0;
                    }
        }
    }
    std::unique_lock<std::shared_mutex> lk(g_mu);
    if (ensure_init()) return -1;
    if (b < 1 || b > 4 || m <= 0 || m % b) return fail("qgemm_lut_int8: bad m/b");
    size_t off = 0;
    Resident *R = find_by_alias(A, &off);
    if (!R) return fail("qgemm_lut_int8: A is not a registered weight tensor (call tmac_b200_upload_weights / ggml_tmac_b200_transform_tensor at load time)");
    if (R->cfg.K != k || R->cfg.bits != b) return fail("qgemm_lut_int8: (k, b) do not match the registered tensor");
    const size_t tile_bytes = (size_t)(k / 4) * R->cfg.bm / 2;
    if (off % tile_bytes) return fail("qgemm_lut_int8: A is not at a tile boundary");
    const int row0 = (int)(off / tile_bytes) * (R->cfg.bm / b);
    const int rows = m / b;
    if (row0 + rows > R->L.Mout) return fail("qgemm_lut_int8: tile range exceeds the tensor");
    return qgemm_impl(*R, row0, rows, n, g.float_type, LUT, LUT_Scales, LUT_Biases, C);
}

// ---- ggml hook -----------------------------------------------------------------------------
void ggml_tmac_init(void) {
    if (tmac_b200_init(-1) != 0) { fprintf(stderr, "ggml_tmac_init: %s\n", tmac_b200_last_error()); return; }
    if (const char *f = getenv("TMAC_KCFG_FILE")) {   // tmac_gemm_wrapper.h:40-56
        if (tmac_b200_load_kcfg_file(f) < 0) fprintf(stderr, "ggml_tmac_init: %s\n", tmac_b200_last_error());
    }
}
void ggml_tmac_free(void) { tmac_b200_shutdown(); }

// ggml-tmac.cpp:267-275: ggml's n (output dim) / m (batch) are swapped relative to T-MAC.
void ggml_tmac_mul_mat_task_init(void *src1, void *qlut, void *lut_scales, void *lut_biases, int n, int k, int m, int bits) {
    if (preprocessor_int8(n * bits, k, m, bits, src1, lut_scales, lut_biases, qlut) != 0)
        fprintf(stderr, "ggml_tmac_mul_mat_task_init: %s\n", tmac_b200_last_error());
}
void ggml_tmac_mul_mat_task_compute(void *src0, void *scales, void *qlut, void *lut_scales, void *lut_biases, void *dst, int n, int k,
                                    int m, int bits) {
    if (qgemm_lut_int8(n * bits, k, m, bits, src0, qlut, scales, lut_scales, lut_biases, dst) != 0)
        fprintf(stderr, "ggml_tmac_mul_mat_task_compute: %s\n", tmac_b200_last_error());
}
// Caller emulation for measurements and tests: ggml_compute_forward_mul_mat's T-MAC branch (ref:ggml.c:12562-12706) for one
// activation row, in C++ so that no interpreter overhead sits between the hook calls.  Phase 1: ggml_tmac_mul_mat_task_init
// (one call).  Phase 2: per_tile = 0 -> one ggml_tmac_mul_mat_task_compute for the whole tensor (the TMAC_USE_TVM_THREADPOOL
// branch, :12610-12630); per_tile = 1 -> one call per weight tile of `tile_rows` rows from `threads` host threads that steal
// tiles through an atomic counter (:12632-12703).  All pointers are HOST pointers as in ggml.
int tmac_b200_debug_ggml_mul_mat(void *src0_qweights, void *src0_scales, void *src1_row, void *wdata, void *dst, int ne01, int ne00,
                                 int bits, int tile_rows, int per_tile, int threads) {
    if (!src0_qweights || !src1_row || !wdata || !dst || ne01 <= 0 || ne00 <= 0 || bits < 1 || bits > 4 || tile_rows <= 0 || ne01 % tile_rows)
        return fail("debug_ggml_mul_mat: bad arguments");
    tmac_b200_kcfg c;
    if (tmac_b200_find_kcfg(ne01 * bits, ne00, bits, &c)) return fail("debug_ggml_mul_mat: shape not configured");
    // workspace layout of ggml.c:12566-12576: qlut (K * 4 bytes) || lut_scales || lut_biases
    char *qlut = (char *)wdata;
    float *ls = (float *)(qlut + (size_t)ne00 * 4), *lb = ls + ne00 / c.act_group_size;
    ggml_tmac_mul_mat_task_init(src1_row, qlut, ls, lb, ne01, ne00, 1, bits);
    if (!per_tile) {
        ggml_tmac_mul_mat_task_compute(src0_qweights, src0_scales, qlut, ls, lb, dst, ne01, ne00, 1, bits);
        return 0;
    }
    const int n_tiles = ne01 / tile_rows;
    const size_t w_chunk = (size_t)ne00 * tile_rows * bits / 8;               // bytes of one tile in the permuted blob (:12636)
    const size_t s_chunk = c.one_scale ? 0 : (size_t)tile_rows * (ne00 / c.group_size) * (c.zero_point ? 2 : 1);
    // tile-stealing workers, parked between calls like ggml's thread pool (spawning threads per mat-vec would dominate)
    struct Pool {
        std::vector<std::thread> th;
        std::atomic<int> gen{0}, done{0}, next{0}, stop{0};
        std::function<void()> job;
        ~Pool() { stop = 1; gen++; for (auto &t : th) t.join(); }
    };
    static Pool pool;
    static std::mutex pool_mu;
    std::lock_guard<std::mutex> pl(pool_mu);
    const int extra = std::max(0, std::min(threads, 64) - 1);
    pool.next = 0; pool.done = 0;
    pool.job = [&, n_tiles, w_chunk, s_chunk]() {
        for (int t = pool.next.fetch_add(1); t < n_tiles; t = pool.next.fetch_add(1))
            ggml_tmac_mul_mat_task_compute((char *)src0_qweights + t * w_chunk, src0_scales ? (float *)src0_scales + t * s_chunk : nullptr, qlut, ls, lb,
                                           (float *)dst + (size_t)t * tile_rows, tile_rows, ne00, 1, bits);
    };
    while ((int)pool.th.size() < extra)
        pool.th.emplace_back([&p = pool, my = pool.gen.load()]() mutable {
            for (;;) {
                while (p.gen.load(std::memory_order_acquire) == my) std::this_thread::yield();
                my = p.gen.load();
                if (p.stop) return;
                p.job();
                p.done.fetch_add(1, std::memory_order_release);
            }
        });
    const int nworkers = (int)pool.th.size();
    pool.gen.fetch_add(1, std::memory_order_release);
    pool.job();
    while (pool.done.load(std::memory_order_acquire) < nworkers) std::this_thread::yield();
    return 0;
}

void ggml_tmac_set_n_threads(int n_threads) { (void)n_threads; /* CPU thread pool size is irrelevant on the GPU */ }

int ggml_tmac_get_type_bits(int type) {  // ggml-tmac.cpp:503-522; ids from ggml.h:359,391-396
    switch (type) {
        case 36: return 1;   // GGML_TYPE_I1
        case 37: return 2;   // GGML_TYPE_I2
        case 38: return 3;   // GGML_TYPE_I3
        case 39: return 4;   // GGML_TYPE_I4
        case 2: return 4;    // GGML_TYPE_Q4_0
        case 34: return 2;   // GGML_TYPE_TQ1_0
        case 35: return 2;   // GGML_TYPE_TQ2_0
        default: return 0;
    }
}

int ggml_tmac_b200_can_mul_mat(int src0_type, int src1_is_f32, int dst_is_f32, const char *src0_name) {
    // ggml-tmac.cpp:72-96,238-248 minus the backend check (weights live in HBM here): the pre-permuted I1..I4 types and
    // the block types the reference re-permutes at load time (Q4_0, TQ1_0, TQ2_0).
    const bool supported = (src0_type >= 36 && src0_type <= 39) || ggml_block_elems(src0_type) > 0;
    if (!supported || !src1_is_f32 || !dst_is_f32) return 0;
    if (src0_name && (!strcmp(src0_name, "token_embd.weight") || !strcmp(src0_name, "output.weight"))) return 0;
    return 1;
}

size_t ggml_tmac_b200_mul_mat_get_wsize(int ne01, int ne10, int ne11, int bits) {  // ggml-tmac.cpp:250-265
    tmac_b200_kcfg c;
    if (tmac_b200_find_kcfg(ne01 * bits, ne10, bits, &c)) return 0;
    const size_t lss = (size_t)ne10 / c.act_group_size;
    size_t wsize = (size_t)ne10 * ne11 * 4 + lss * ne11 * 2 * sizeof(float);
    return ((wsize - 1) / 64 + 1) * 64;
}

size_t ggml_tmac_b200_get_nbytes(int ne00, int ne01, int bits) {  // ggml-tmac.cpp:277-288
    tmac_b200_kcfg c;
    if (tmac_b200_find_kcfg(ne01 * bits, ne00, bits, &c)) return 0;
    const size_t ss = c.one_scale ? 1 : (size_t)c.M * (c.K / c.group_size) * (c.zero_point ? 2 : 1);
    return (size_t)ne00 * ne01 / 8 * bits + ss * sizeof(float);
}

int ggml_tmac_b200_transform_tensor(void *data, int ne00, int ne01, int bits, struct tmac_tensor_extra_b200 *extra) {
    // ggml-tmac.cpp:290-354, I1..I4 branch (:336-345): the blob is `permuted weights || fp32 scales`.
    tmac_b200_kcfg c;
    if (tmac_b200_find_kcfg(ne01 * bits, ne00, bits, &c)) return -1;
    if (c.M != ne01) return fail("transform_tensor: kcfg is for a different M");
    uint8_t *qweights = (uint8_t *)data;
    float *scales = (float *)(qweights + (size_t)ne00 * ne01 * bits / 8);
    const int64_t h = tmac_b200_upload_weights(&c, qweights, scales, TMAC_B200_F32);
    if (h < 0) return -1;
    if (extra) {
        extra->lut_scales_size = ne00 / c.act_group_size;
        extra->scales_size = c.one_scale ? 1 : c.M * (c.K / c.group_size) * (c.zero_point ? 2 : 1);
        extra->n_tile_num = c.M * c.bits / c.bm;
        extra->qweights = qweights;
        extra->scales = scales;
    }
    return (int)h;
}

// ggml-tmac.cpp:290-498 for every type it supports: I1..I4 blobs are aliased in place (above); Q4_0 / TQ1_0 / TQ2_0
// blocks are decoded element by element like the reference's accessors and encoded into the stream layout.  The
// reference hands ggml a freshly allocated permuted copy in extra->qweights; here that pointer is only an ADDRESS KEY
// (ggml.c adds tile offsets to it and passes it back), so a PROT_NONE reservation of the same size stands in for it.
int ggml_tmac_b200_transform_tensor_typed(void *data, int ggml_type, int ne00, int ne01, struct tmac_tensor_extra_b200 *extra) {
    const int bits = ggml_tmac_get_type_bits(ggml_type);
    if (!bits || !data) return fail("transform_tensor: unsupported ggml type " + std::to_string(ggml_type));
    if (ggml_type >= 36 && ggml_type <= 39) return ggml_tmac_b200_transform_tensor(data, ne00, ne01, bits, extra);
    tmac_b200_kcfg c;
    if (tmac_b200_find_kcfg(ne01 * bits, ne00, bits, &c)) return -1;
    if (c.M != ne01) return fail("transform_tensor: kcfg is for a different M");
    const int E = ggml_block_elems(ggml_type);
    if (c.one_scale || c.zero_point || c.group_size != E)
        return fail("transform_tensor: block type needs a kcfg with group_size = " + std::to_string(E) + ", no zero point, per-group scales");
    if (validate_cfg(c)) return -1;
    std::vector<uint8_t> w((size_t)ne01 * ne00);
    std::vector<float> sc((size_t)ne01 * (ne00 / E));
    if (!decode_ggml_blocks(ggml_type, data, ne01, ne00, w.data(), sc.data())) return fail("transform_tensor: K is not a multiple of the block size");
    const size_t abytes = (size_t)ne00 * ne01 * bits / 8;
    void *key = mmap(nullptr, abytes, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (key == MAP_FAILED) return fail("transform_tensor: cannot reserve an address range for the tensor");
    // scales in the reference's run-time order [M/bm][K/gs][bm/bits] (ggml-tmac.cpp:464-489)
    const int NG = ne00 / E, rows_per_tile = c.bm / bits;
    float *hs = (float *)std::malloc(sc.size() * sizeof(float));
    if (!hs) { munmap(key, abytes); return fail("out of host memory"); }
    for (int r = 0; r < ne01; ++r)
        for (int gk = 0; gk < NG; ++gk)
            hs[((size_t)(r / rows_per_tile) * NG + gk) * rows_per_tile + r % rows_per_tile] = sc[(size_t)r * NG + gk];
    int64_t h;
    {
        std::unique_lock<std::shared_mutex> lk(g_mu);
        if (ensure_init()) { munmap(key, abytes); std::free(hs); return -1; }
        PlainWeights P;
        plain_from_w(w.data(), ne01, ne00, bits, 0, ne01, &P);
        P.scales = sc;
        h = register_resident(c, P, key, abytes, 0);
        if (h < 0) { munmap(key, abytes); std::free(hs); return -1; }
        Resident &R = g.res[h];
        R.reserved = key; R.reserved_bytes = abytes; R.host_scales = hs;
    }
    if (extra) {
        extra->lut_scales_size = ne00 / c.act_group_size;
        extra->scales_size = ne01 * NG;
        extra->n_tile_num = c.M * c.bits / c.bm;
        extra->qweights = (uint8_t *)key;
        extra->scales = hs;
    }
    return (int)h;
}

// Host-only (no GPU): the decode step of the typed transform, for the CPU suite.  w [ne01][ne00] codes, scales
// [ne01][ne00 / block elems].  Returns the block size or -1.
int tmac_b200_debug_decode_ggml(int ggml_type, const void *data, int ne00, int ne01, uint8_t *w, float *scales) {
    if (!data || !w || !scales) return fail("debug_decode_ggml: null argument");
    if (!decode_ggml_blocks(ggml_type, data, ne01, ne00, w, scales)) return fail("debug_decode_ggml: unsupported type or K");
    return ggml_block_elems(ggml_type);
}

// The reference's default tiling when no tuned kcfg exists (python/t_mac/ops/qgemm.py:98-115: the first candidate of each knob):
// bm = first of {256,128,512,1024,320,640} ({192,384,576,768} for 3 bits) dividing M*bits with bm % bits == 0; kfactor = first
// of {8,16} with (4*kfactor) % act_group_size == 0 and group_size % (4*kfactor) == 0 (any of them on the do_scale_final path).
int tmac_b200_default_kcfg(int M, int K, int bits, int group_size, int act_group_size, int zero_point, int one_scale, tmac_b200_kcfg *out) {
    if (!out || M <= 0 || K <= 0 || bits < 1 || bits > 4) return fail("default_kcfg: bad argument");
    static const int bms3[] = {192, 384, 576, 768}, bmsx[] = {256, 128, 512, 1024, 320, 640};
    const int *bms = bits == 3 ? bms3 : bmsx;
    const int nb = bits == 3 ? 4 : 6;
    int bm = 0;
    for (int i = 0; i < nb && !bm; ++i)
        if ((M * bits) % bms[i] == 0 && bms[i] % bits == 0) bm = bms[i];
    if (!bm) return fail("default_kcfg: no tile size divides M*bits = " + std::to_string(M * bits));
    const int ags = (act_group_size <= 0 || act_group_size > K) ? K : act_group_size;
    const bool scale_final = one_scale && ags == K;
    const int wgs = one_scale ? K : group_size;
    int kf = 0;
    for (int cand : {8, 16})
        if (!kf && (scale_final || ((cand * 4) % ags == 0 && wgs > 0 && wgs % (cand * 4) == 0))) kf = cand;
    if (!kf) {   // act group wider than 64 K positions: the reference has no candidate; the stream layout only needs kfactor | K/4
        for (int cand : {16, 8})
            if (!kf && (K / 4) % cand == 0) kf = cand;
    }
    if (!kf || (K / 4) % kf) return fail("default_kcfg: no kfactor for this grouping");
    std::memset(out, 0, sizeof *out);
    out->M = M; out->K = K; out->bits = bits; out->bm = bm; out->kfactor = kf; out->simd_n_in = 16; out->simd_n_out = 8;
    out->group_size = one_scale ? (group_size > 0 ? group_size : 128) : group_size; out->act_group_size = ags;
    out->zero_point = zero_point ? 1 : 0; out->one_scale = one_scale ? 1 : 0;
    return 0;
}

// ---- GGUF files (tmac_gguf.h) ----------------------------------------------------------------------------------------

int64_t tmac_b200_gguf_open(const char *path) {
    if (!path) return fail("gguf_open: null path");
    GgufFile *f = new GgufFile();
    if (!f->open(path)) { const std::string e = f->error; delete f; return fail("gguf_open: " + e); }
    std::unique_lock<std::shared_mutex> lk(g_mu);
    const int64_t h = g_next_gguf++;
    g_gguf[h] = f;
    return h;
}
int tmac_b200_gguf_close(int64_t gguf) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    auto it = g_gguf.find(gguf);
    if (it == g_gguf.end()) return fail("gguf_close: bad handle");
    // the file is unmapped: weights uploaded from it stay resident, but their host alias keys (ranges inside the mapping)
    // must not survive -- a later mapping can land on the same addresses and would resolve to the old tensor
    const unsigned char *lo = it->second->base, *hi = lo + it->second->size;
    for (auto &kv : g.res)
        if (kv.second.host_a && kv.second.host_a >= lo && kv.second.host_a < hi) { kv.second.host_a = nullptr; kv.second.host_a_bytes = 0; }
    delete it->second;
    g_gguf.erase(it);
    return 0;
}
static GgufFile *gguf_locked(int64_t gguf) {
    auto it = g_gguf.find(gguf);
    return it == g_gguf.end() ? nullptr : it->second;
}
int tmac_b200_gguf_tensor_count(int64_t gguf) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    GgufFile *f = gguf_locked(gguf);
    return f ? (int)f->tensors.size() : fail("gguf: bad handle");
}
int tmac_b200_gguf_tensor_info(int64_t gguf, int index, struct tmac_b200_gguf_tensor *out) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    GgufFile *f = gguf_locked(gguf);
    if (!f || !out) return fail("gguf: bad handle / null argument");
    if (index < 0 || index >= (int)f->tensors.size()) return fail("gguf: tensor index out of range");
    const GgufTensor &T = f->tensors[index];
    std::memset(out, 0, sizeof *out);
    std::strncpy(out->name, T.name.c_str(), sizeof out->name - 1);
    out->ggml_type = T.type; out->n_dims = T.n_dims;
    for (int d = 0; d < 4; ++d) out->ne[d] = T.ne[d];
    out->offset = T.offset; out->nbytes = T.nbytes;
    out->data = f->data(index);
    return 0;
}
int tmac_b200_gguf_find_tensor(int64_t gguf, const char *name) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    GgufFile *f = gguf_locked(gguf);
    if (!f || !name) return fail("gguf: bad handle / null argument");
    const int i = f->find(name);
    return i >= 0 ? i : fail(std::string("gguf: no tensor named '") + name + "'");
}
// Metadata: integers / bools / floats (as double) and strings.  Return 0, or -1 when the key is absent or of another kind.
int tmac_b200_gguf_meta_number(int64_t gguf, const char *key, double *out) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    GgufFile *f = gguf_locked(gguf);
    if (!f || !key || !out) return fail("gguf: bad handle / null argument");
    auto it = f->meta.find(key);
    if (it == f->meta.end() || it->second.type == 8 || it->second.type == 9) return fail(std::string("gguf: no numeric key '") + key + "'");
    *out = it->second.f;
    return 0;
}
int tmac_b200_gguf_meta_string(int64_t gguf, const char *key, char *dst, size_t cap) {
    std::unique_lock<std::shared_mutex> lk(g_mu);
    GgufFile *f = gguf_locked(gguf);
    if (!f || !key || !dst || !cap) return fail("gguf: bad handle / null argument");
    auto it = f->meta.find(key);
    if (it == f->meta.end() || it->second.type != 8) return fail(std::string("gguf: no string key '") + key + "'");
    std::strncpy(dst, it->second.s.c_str(), cap - 1); dst[cap - 1] = 0;
    return (int)it->second.s.size();
}
// Upload one quantised linear of the file (I1..I4, Q4_0, TQ1_0, TQ2_0; 2-D) through the typed transform; the kcfg for its
// shape must be registered (tmac_b200_load_kcfg_file).  The mapped file region serves as the host alias of I-type tensors.
int64_t tmac_b200_gguf_load_tensor(int64_t gguf, int index, struct tmac_tensor_extra_b200 *extra) {
    const uint8_t *data; int type, ne0, ne1; uint64_t nbytes;
    {
        std::unique_lock<std::shared_mutex> lk(g_mu);
        GgufFile *f = gguf_locked(gguf);
        if (!f) return fail("gguf: bad handle");
        if (index < 0 || index >= (int)f->tensors.size()) return fail("gguf: tensor index out of range");
        const GgufTensor &T = f->tensors[index];
        if (T.n_dims != 2) return fail("gguf_load_tensor: '" + T.name + "' is not a matrix");
        data = f->data(index); type = T.type; ne0 = (int)T.ne[0]; ne1 = (int)T.ne[1]; nbytes = T.nbytes;
    }
    const int bits = ggml_tmac_get_type_bits(type);
    if (!bits) return fail("gguf_load_tensor: ggml type " + std::to_string(type) + " is not a T-MAC type");
    uint64_t need;
    if (ggml_block_elems(type)) {
        need = (uint64_t)ne1 * (ne0 / ggml_block_elems(type)) * ggml_block_bytes(type);
        tmac_b200_kcfg c;   // block types fix their grouping themselves: without a tuned kcfg the reference's default tiling will do
        if (tmac_b200_find_kcfg(ne1 * bits, ne0, bits, &c) != 0) {
            const int E = ggml_block_elems(type);
            if (tmac_b200_default_kcfg(ne1, ne0, bits, E, E == 32 ? 32 : 64, 0, 0, &c) != 0 || tmac_b200_register_kcfg(&c) != 0) return -1;
        }
    } else need = ggml_tmac_b200_get_nbytes(ne0, ne1, bits);
    if (need == 0) return -1;                      // no kcfg for the shape (message set by the lookup)
    if (nbytes < need) return fail("gguf_load_tensor: tensor data is shorter than its type and shape require");
    return ggml_tmac_b200_transform_tensor_typed((void *)data, type, ne0, ne1, extra);
}

}  // extern "C"
