// tmac_prefill_experts.cu -- the routed launches at prefill sizes: the routed experts (tmac_b200_prefill_experts / _glu) and the
// dense transformed-input forms (tmac_b200_prefill_rmsnorm / _glu / _residual), which run as one expert with the identity routing.
// The routing kernel that groups the slots by expert, the routed instantiations of both wgmma tiles and their gathered LUT records
// (3 bit widths x 6 fp groupings, plus for one-scale tensors the fp16 tile's 128-K-chunk groupings and the int8 tile's 64-K chunk
// units; tmac_prefill.cuh, tmac_prefill16.cuh), the same tiles once more with a bias on the outputs (tmac_b200_prefill_rmsnorm_bias),
// the RMSNorm, GLU and sub-norm inputs and the GLU combine.  In their
// own translation unit so that they compile in parallel with tmac_b200.cu.
#include "tmac_prefill16.cuh"

namespace tmac_b200 {

namespace {

constexpr int kRouteThreads = 1024, kRouteWarps = kRouteThreads / 32, kRouteMaxE = 256;

// One CTA.  Slot s = n * topk + j of expert e = ids[s] (valid: 0 <= e < E).  A counting sort that depends only on ids: the counts of
// each expert, their exclusive prefix off[e], then rounds of 1024 slots in which a slot's position is off[e] + (the slots of e in
// earlier rounds) + (those in earlier warps of the round) + (those in earlier lanes of its warp) -- ascending s inside an expert.
// Tile table: expert e's rows in runs of T from off[e], entries in expert order, the rest of the cap entries unused (ntok 0).
// Cnan != null (the plain form): the Mout-wide rows of every invalid slot in C_i = Cnan[i * E] are quiet NaN.
// ids == null (the dense forms): every slot is expert 0, so with E = 1 the table is {0, q * T, min(T, S - q * T), 0} and perm[s] = s.
__global__ void __launch_bounds__(kRouteThreads) pf_route_kernel(const int32_t *ids, int S, int E, int T, int cap, int4 *tiles, int *perm,
                                                                 void *const *Cnan, int count, int ldc, int out_f16) {
    __shared__ int cnt[kRouteMaxE], off[kRouteMaxE], tb[kRouteMaxE], run[kRouteMaxE], wc[kRouteWarps][kRouteMaxE];
    __shared__ int used;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int e = tid; e < E; e += kRouteThreads) { cnt[e] = 0; run[e] = 0; }
    __syncthreads();
    for (int s = tid; s < S; s += kRouteThreads) {
        const int e = ids ? ids[s] : 0;
        if ((unsigned)e < (unsigned)E) atomicAdd(&cnt[e], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int o = 0, k = 0;
        for (int e = 0; e < E; ++e) { off[e] = o; tb[e] = k; o += cnt[e]; k += (cnt[e] + T - 1) / T; }
        used = k;
    }
    __syncthreads();
    for (int e = tid; e < E; e += kRouteThreads)
        for (int q = 0; q * T < cnt[e]; ++q) tiles[tb[e] + q] = make_int4(e, off[e] + q * T, min(T, cnt[e] - q * T), 0);
    for (int k = used + tid; k < cap; k += kRouteThreads) tiles[k] = make_int4(0, 0, 0, 0);
    for (int base = 0; base < S; base += kRouteThreads) {
        const int s = base + tid;
        int e = s < S ? (ids ? ids[s] : 0) : -1;
        if ((unsigned)e >= (unsigned)E) e = -1;
        for (int i = tid; i < kRouteWarps * E; i += kRouteThreads) wc[i / E][i % E] = 0;
        __syncthreads();
        const unsigned same = __match_any_sync(0xffffffffu, e);
        const int rank = __popc(same & ((1u << lane) - 1u));
        if (e >= 0 && rank == 0) wc[warp][e] = __popc(same);
        __syncthreads();
        for (int x = tid; x < E; x += kRouteThreads) {   // per expert: the warps' exclusive prefix, on top of the earlier rounds
            int acc = run[x];
            for (int w = 0; w < kRouteWarps; ++w) { const int c = wc[w][x]; wc[w][x] = acc; acc += c; }
            run[x] = acc;
        }
        __syncthreads();
        if (e >= 0) perm[off[e] + wc[warp][e] + rank] = s;
        __syncthreads();
    }
    if (!Cnan) return;
    for (int s = warp; s < S; s += kRouteWarps) {
        if ((unsigned)ids[s] < (unsigned)E) continue;
        for (int i = 0; i < count; ++i) {
            void *const Ci = Cnan[(size_t)i * E];
            for (int r = lane; r < ldc; r += 32) store_out(Ci, (size_t)s * ldc + r, __int_as_float(0x7fffffff), out_f16);
        }
    }
}

// a[i] = swiglu(g[i], u[i]) in fp32, fp16 inputs widened first: the input the GEMV's GLU kinds build their LUT from.  RELU2:
// a[i] = relu2(g[i], u[i]), the squared-ReLU input of kInRelu2Norm (before pf_rmsnorm_kernel in place).
template <typename T, bool RELU2 = false>
__global__ void __launch_bounds__(256) pf_swiglu_kernel(const T *g, const T *u, size_t n, float *a) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        a[i] = RELU2 ? relu2(ld_act(g, i), ld_act(u, i)) : swiglu(ld_act(g, i), ld_act(u, i));
}

// a[n][k] = rms_scale(h[n][k], inv_n, w[k]), fp16 inputs widened first: the input the GEMV's norm kind (kInNorm) builds its LUT from.
// One CTA per row: warp 0 sums the squares in the order rms_sumsq / rms_warp_sum document (lane l: the 4-element groups l, l + 32,
// ...), then every thread scales its elements.  K % 4 == 0.  In place (fp32, h == a) is allowed: a thread writes only elements it has
// just read, after the sum.
template <typename T>
__global__ void __launch_bounds__(256) pf_rmsnorm_kernel(const T *h, const float *w, float eps, int K, float *a) {
    __shared__ float inv;
    const size_t base = (size_t)blockIdx.x * K;
    if (threadIdx.x < 32) {
        float s = 0.f;
        for (int g = threadIdx.x; g < K / 4; g += 32) {
            const size_t k = base + 4 * (size_t)g;
            s = rms_sumsq(s, ld_act(h, k), ld_act(h, k + 1), ld_act(h, k + 2), ld_act(h, k + 3));
        }
        s = rms_warp_sum(s);
        if (threadIdx.x == 0) inv = rms_inv(s, K, eps);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) a[base + k] = rms_scale(ld_act(h, base + k), inv, w[k]);
}

// C[n][row] = fadd_rn(...fadd_rn(fmul_rn(w_0, y_0), fmul_rn(w_1, y_1))..., fmul_rn(w_{topk-1}, y_{topk-1})) (+ R[n][row]), y_j =
// ys[n * topk + j][row]; quiet NaN for a token with an id outside [0, E) (its slots' rows were never computed)
__global__ void __launch_bounds__(256) pf_combine_kernel(const float *ys, const int32_t *ids, const float *w, int topk, int E, const void *R,
                                                         void *C, int N, int Mout, int out_f16) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * Mout) return;
    const int n = (int)(i / Mout), row = (int)(i % Mout);
    bool bad = false;
    for (int j = 0; j < topk; ++j) bad |= (unsigned)ids[n * topk + j] >= (unsigned)E;
    float acc = __int_as_float(0x7fffffff);
    if (!bad) {
        const float *y = ys + (size_t)n * topk * Mout + row, *wn = w + (size_t)n * topk;
        acc = __fmul_rn(wn[0], y[0]);
        for (int j = 1; j < topk; ++j) acc = __fadd_rn(acc, __fmul_rn(wn[j], y[(size_t)j * Mout]));
        if (R)                                   // read, then written by this thread: the residual may be C itself
            acc = __fadd_rn(acc, out_f16 ? __half2float(reinterpret_cast<const __half *>(R)[i]) : reinterpret_cast<const float *>(R)[i]);
    }
    store_out(C, i, acc, out_f16);
}

// BIAS: the same tiles with a bias on the outputs (prefill_bias_kernel, prefill16_bias_kernel)
template <int PB, bool BIAS> PfExpertKernels pick_pf_experts_pb(int qch, int agq, bool one, bool unit1) {
    using Tile = void (*)(const PrefillParams, const PfRoute);
    using Tile16 = void (*)(const Prefill16Params, const PfRoute);
    const auto tile = [](auto QCH, auto AGQ, auto UNIT1) -> Tile {
        if constexpr (BIAS) return prefill_bias_kernel<PB, QCH, AGQ, UNIT1>;
        else return prefill_experts_kernel<PB, QCH, AGQ, UNIT1>;
    };
    const auto tile16 = [](auto QCH, auto AGQ, auto ONE) -> Tile16 {
        if constexpr (BIAS) return prefill16_bias_kernel<PB, QCH, AGQ, ONE>;
        else return prefill16_experts_kernel<PB, QCH, AGQ, ONE>;
    };
    using I4 = std::integral_constant<int, 4>;
    using I8 = std::integral_constant<int, 8>;
    using I2 = std::integral_constant<int, 2>;
    if (unit1) {                                 // one-scale, K % 128 == 64: 64-K chunks staged one per unit, the int8 tile only
        if (qch == 4 && agq == 4) return {tile(I4{}, I4{}, std::true_type{}), lut_tile_gather_kernel<4, 4>, nullptr, nullptr};
        if (qch == 4 && agq == 2) return {tile(I4{}, I2{}, std::true_type{}), lut_tile_gather_kernel<4, 2>, nullptr, nullptr};
        return PfExpertKernels{};
    }
    PfExpertKernels k = FpGroupings::find<PfExpertKernels>(qch, agq, [&](auto QCH, auto AGQ) -> PfExpertKernels {
        return {tile(QCH, AGQ, std::false_type{}), lut_tile_gather_kernel<QCH, AGQ>, tile16(QCH, AGQ, std::false_type{}),
                lut_tile16_gather_kernel<QCH, AGQ>};
    });
    if (one)                                     // one-scale, K % 128 == 0: chunk 128 K, the fp16 tile's own instantiations
        k.tile16 = qch != 8 ? nullptr : agq == 8 ? tile16(I8{}, I8{}, std::true_type{}) : agq == 4 ? tile16(I8{}, I4{}, std::true_type{})
                 : agq == 2 ? tile16(I8{}, I2{}, std::true_type{}) : nullptr;
    return k;
}

}  // namespace

PfExpertKernels pick_pf_experts(int pb, int qch, int agq, bool one, bool unit1, bool bias) {
    if (pb == 4) return bias ? pick_pf_experts_pb<4, true>(qch, agq, one, unit1) : pick_pf_experts_pb<4, false>(qch, agq, one, unit1);
    if (pb == 2) return bias ? pick_pf_experts_pb<2, true>(qch, agq, one, unit1) : pick_pf_experts_pb<2, false>(qch, agq, one, unit1);
    return PfExpertKernels{};
}

void pf_route_launch(const int32_t *ids, int S, int E, int T, int cap, int4 *tiles, int *perm, void *const *Cnan, int count, int ldc,
                     int out_f16, cudaStream_t st) {
    pf_route_kernel<<<1, kRouteThreads, 0, st>>>(ids, S, E, T, cap, tiles, perm, Cnan, count, ldc, out_f16);
}

void pf_swiglu_launch(const void *G, const void *U, int f16, size_t n, float *a, cudaStream_t st, bool relu2) {
    const int grid = (int)std::min<size_t>((n + 255) / 256, 132 * 16);
    if (relu2 && f16) pf_swiglu_kernel<__half, true><<<grid, 256, 0, st>>>((const __half *)G, (const __half *)U, n, a);
    else if (relu2) pf_swiglu_kernel<float, true><<<grid, 256, 0, st>>>((const float *)G, (const float *)U, n, a);
    else if (f16) pf_swiglu_kernel<__half><<<grid, 256, 0, st>>>((const __half *)G, (const __half *)U, n, a);
    else pf_swiglu_kernel<float><<<grid, 256, 0, st>>>((const float *)G, (const float *)U, n, a);
}

void pf_rmsnorm_launch(const void *H, int f16, const float *w, float eps, int N, int K, float *a, cudaStream_t st) {
    if (f16) pf_rmsnorm_kernel<__half><<<N, 256, 0, st>>>((const __half *)H, w, eps, K, a);
    else pf_rmsnorm_kernel<float><<<N, 256, 0, st>>>((const float *)H, w, eps, K, a);
}

void pf_combine_launch(const float *ys, const int32_t *ids, const float *w, int topk, int E, const void *R, void *C, int N, int Mout,
                       int out_f16, cudaStream_t st) {
    const size_t n = (size_t)N * Mout;
    pf_combine_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ys, ids, w, topk, E, R, C, N, Mout, out_f16);
}

}  // namespace tmac_b200
