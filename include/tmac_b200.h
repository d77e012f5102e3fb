/*
 * tmac_b200.h -- C ABI of libtmac_b200.so: the H100-native (sm_90a) drop-in for the
 * preprocessor + qgemm_lut operator pair of microsoft/T-MAC.
 *
 * Plain C: pointers and sizes only, no torch / C++ types.  Every entry point cites the
 * reference interface it replaces (paths relative to the T-MAC tree).
 *
 * Pointer domain: every data pointer may be a DEVICE pointer (native use: benchmarks, a
 * GPU-resident host program) or a HOST pointer (the reference's callers: ggml passes host
 * memory).  The library classifies each pointer (cudaPointerGetAttributes); host activations /
 * outputs are staged through pinned buffers, host weights must be registered once
 * (tmac_b200_upload_weights / ggml_tmac_b200_transform_tensor) so that they stay resident in HBM.
 *
 * Errors: the reference's convention -- 0 = ok, -1 = failure (deploy/tuned/<preset>/kernels.h:27,37).
 * tmac_b200_last_error() returns a static message for the calling thread.  There is NO CPU
 * fallback: without a usable CUDA device every compute entry point returns -1.
 */
#ifndef TMAC_B200_H_
#define TMAC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TMAC_B200_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * Kernel configuration = the reference's per-shape `kcfg.ini` section
 * (TMAC::TMACGeMMConfig, include/t-mac/tmac_gemm_wrapper.h:26-35; written by
 * deploy/compile.py:156-165) plus the compile-time options the reference bakes into each
 * generated kernel (deploy/compile.py:207-229: bits, group_size, act_group_size, zero_point,
 * m_groups).
 * ---------------------------------------------------------------------------------------- */
typedef struct tmac_b200_kcfg {
    int M;               /* output features (rows of the weight matrix), NOT multiplied by bits */
    int K;               /* input features */
    int bits;            /* 1..4 */
    int bm;              /* reference tile of bit-plane rows (kcfg `bm`) -- needed to decode A */
    int kfactor;         /* kcfg `kfactor` */
    int simd_n_in;       /* kcfg `simd_n_in`  (16) */
    int simd_n_out;      /* kcfg `simd_n_out` (8) */
    int group_size;      /* weight quantisation group along K (kcfg `group_size`) */
    int act_group_size;  /* LUT-scale group along K; -1 or K = one scale per activation row */
    int zero_point;      /* scales carry interleaved zero points (GPTQ-like) */
    int one_scale;       /* m_groups == 1: one unified weight scale (BitNet-like) */
} tmac_b200_kcfg;

/* dtype codes for activations / outputs (`T` of the reference: float on x86, fp16 on ARM) */
enum { TMAC_B200_F32 = 0, TMAC_B200_F16 = 1 };

/* ---- library ---------------------------------------------------------------------------- */
TMAC_B200_API int tmac_b200_init(int device);          /* picks the device, creates streams */
TMAC_B200_API void tmac_b200_shutdown(void);
TMAC_B200_API const char *tmac_b200_last_error(void);
TMAC_B200_API int tmac_b200_version(void);
/* All launches go to `stream` (a cudaStream_t passed as void*); NULL = the library's own stream. */
TMAC_B200_API int tmac_b200_set_stream(void *stream);
TMAC_B200_API int tmac_b200_set_float_type(int dtype); /* TMAC_B200_F32 (default) or _F16 */
/* LUT handling in qgemm_lut: 0 = auto (device QLUTs written by tmac_b200_preprocessor and host
 * QLUTs that pass the odd-symmetry check LUT[15-i] == -LUT[i] take the 8-entry fast path, any
 * other QLUT the general 16-entry path), 1 = always general, 2 = always symmetric.
 * A DEVICE QLUT buffer is recognised by address: if a caller overwrites a buffer that tmac_b200_preprocessor filled
 * earlier with a table of its own (the reference never does; its QLUT always comes from preprocessor_int8), it must
 * select mode 1 for that call. */
TMAC_B200_API int tmac_b200_set_lut_mode(int mode);

/* CUDA-graph helpers: capture the library calls issued between begin/end (device pointers only,
 * after one eager warm-up of the same sequence) on the current stream and replay them. */
TMAC_B200_API int tmac_b200_graph_begin(void);
TMAC_B200_API int64_t tmac_b200_graph_end(void);
TMAC_B200_API int tmac_b200_graph_launch(int64_t graph, int times);
TMAC_B200_API int tmac_b200_graph_free(int64_t graph);
TMAC_B200_API int tmac_b200_sync(void);
/* Reporting: eight ints describing the last GEMV or prefill launch (qgemm_lut, gemv and their grouped and fused-input forms).
 * gemv3_kernel: {cluster size cs (1, 2, 4, 8), warps per CTA wpc, chunks per warp bpw, register variant MINB (3 or 4),
 *   grid.x = row super-blocks * cs, planes per word, symmetric LUT (1) or general (0), tensors in the launch (>= 1)}.
 *   Warp w of cluster rank k owns the K chunks [(k*wpc + w)*bpw, +bpw); these three fields fix the fp-path summation order.
 * int8 prefill tile: {1, warps per CTA, K chunks, 1, row tiles, planes per word, 1, -N}.
 * fp16 prefill tile: {16, warps per CTA, K chunks, stream-K (1) or not (0), grid.x, planes per word, 1, -N}.
 * A negative last field marks a prefill tile over N activation rows. */
TMAC_B200_API int tmac_b200_debug_last_launch(int *out8);
/* Tuning / A-B knobs at run time.  Each key is also read once, when the library initialises, from the environment variable
 * TMAC_B200_<key in upper case>; an unknown key fails.
 * ("fused", "prefill", "prefill16", "pf_streamk", "prefill_min_n", "pdl", "pdl_late", "cs", "wpc", "minb", "nbuf", "trace",
 * "lut_mode" (as tmac_b200_set_lut_mode), "scales_f32" 1 = later uploads keep fp32 scales even when they are fp16-exact;
 * decode sequences: "seq_impl" 0 stream-K sequence kernel | 1 resident chain kernel | 2 chain when the sequence qualifies (default),
 * "chain_flags" bit 0 = the chain kernel's grid-barrier form, "chain_ahead" 0 = never the chain kernel's decode-ahead
 * instantiation (default 1: when every cluster stays resident with it), "seq_handover" 0 = the stream-K sequence kernel's
 * consumers build their LUT instead of taking it from the producer, "seq_grid", "seq_smem_kb"). */
TMAC_B200_API int tmac_b200_debug_set(const char *key, int value);
/* Debug (TMAC_B200_TRACE=1): per-CTA clock64 stamps [ctas][8] of the last qgemm_lut launch. */
TMAC_B200_API int tmac_b200_debug_trace(long long *dst, int cap_ctas);

/* ---- configuration (replaces kcfg.ini lookup, tmac_gemm_wrapper.h:230-255) -------------- */
TMAC_B200_API int tmac_b200_register_kcfg(const tmac_b200_kcfg *cfg);
/* Parses a reference kcfg.ini (sections qgemm_lut_t{T}_int8_m{M*bits}_k{K}_n{N}_b{bits}).
 * act_group_size / zero_point / one_scale are derived from lut_scales_size / scales_size unless
 * the (extension) keys `act_group_size`, `zero_point`, `m_groups` are present. Returns #sections or -1. */
TMAC_B200_API int tmac_b200_load_kcfg_file(const char *path);
TMAC_B200_API int tmac_b200_find_kcfg(int m_times_bits, int k, int bits, tmac_b200_kcfg *out);
TMAC_B200_API void tmac_b200_clear_kcfg(void);

/* ---- weights ---------------------------------------------------------------------------- *
 * Replaces the load-time re-permutation ggml_tmac_transform_tensor
 * (3rdparty/llama.cpp/ggml/src/ggml-tmac.cpp:290-501): takes the reference run-time layout
 *   A      uint8 [M*bits/bm][K/4][bm/2]                     (python/t_mac/weights.py:57-73)
 *   Scales T     [M*bits/bm][K/group_size][bm/bits (*2)] or [1]   (weights.py:75-88)
 * (host pointers), re-permutes once into the GPU stream layout, uploads it and registers the
 * host pointer range [A, A+M*K*bits/8) as an alias of the resident copy, so that later
 * qgemm_lut_int8 / ggml_tmac_mul_mat_task_compute calls that pass `A + tile_offset` find it.
 * Returns an opaque handle (>0) or -1. */
TMAC_B200_API int64_t tmac_b200_upload_weights(const tmac_b200_kcfg *cfg, const void *A,
                                               const void *scales, int scales_dtype);
/* Same, from un-permuted quantised weights w uint8 [M][K] in [0,2^bits), scales/zeros fp32
 * [M][K/group_size] (zeros already in the (z - 2^(bits-1))*s convention, weights.py:28-30). */
TMAC_B200_API int64_t tmac_b200_upload_plain(const tmac_b200_kcfg *cfg, const uint8_t *w,
                                             const float *scales, const float *zeros);
/* GPTQ checkpoint tensors as stored in safetensors (qweight int32 [K*bits/32][M], scales fp16 [K/gs][M], qzeros int32
 * [K/gs][M*bits/32]) -> resident weights: unpack_gptqv2 + preprocess_weights of the reference's converter
 * (python/t_mac/model_utils.py:95-129, :262-271; convert_hf_to_gguf.py:300-320) in one call.  cfg: M, K, bits (1, 2 or 4),
 * group_size, bm, kfactor, act_group_size; zero points are implied.  gptq_v2 = 1 for GPTQModel, 0 for AutoGPTQ (zeros + 1). */
TMAC_B200_API int64_t tmac_b200_upload_gptq(const tmac_b200_kcfg *cfg, const int32_t *qweight, const uint16_t *scales_f16,
                                            const int32_t *qzeros, int gptq_v2);
/* Host-only: the unpack alone (w [M][K], scales / zeros [M][K/group_size]); 0 or -1. */
TMAC_B200_API int tmac_b200_debug_unpack_gptq(const int32_t *qweight, const uint16_t *scales_f16, const int32_t *qzeros, int K, int M,
                                              int bits, int group_size, int gptq_v2, uint8_t *w, float *scales, float *zeros);
/* Host-only layout transform (no GPU needed): writes the stream layout of tmac_b200_upload_weights
 * into dst (dst == NULL: size query); layout_out[12] = {pb, rows/lane, rows/super-block,
 * #super-blocks, K/chunk, quads/chunk, #chunks, scale bytes, zp, one_scale, block bytes, weight bytes}. */
TMAC_B200_API int64_t tmac_b200_debug_encode(const tmac_b200_kcfg *cfg, const void *A, const void *scales,
                                             void *dst, size_t cap, int *layout_out);
TMAC_B200_API int tmac_b200_free_weights(int64_t handle);
/* A second resident copy in its own HBM allocation (distinct layers with tied shapes; benchmarks
 * that must stream weights from HBM rather than L2). */
TMAC_B200_API int64_t tmac_b200_clone_weights(int64_t handle);
/* One-shot hint for the next qgemm_lut / gemv call: `handle` is the tensor that will be multiplied
 * after it (next layer).  The launch prefetches that tensor's blocks into L2 while it computes. */
TMAC_B200_API int tmac_b200_hint_next_weights(int64_t handle);
TMAC_B200_API size_t tmac_b200_weights_nbytes(int64_t handle); /* resident bytes in HBM */
/* Row-shard view for multi-GPU (SURVEY 8e): keep only rows [row0,row0+rows) resident. */
TMAC_B200_API int64_t tmac_b200_upload_plain_rows(const tmac_b200_kcfg *cfg, const uint8_t *w,
                                                  const float *scales, const float *zeros,
                                                  int row0, int rows);

/* ---- native operators (explicit configuration, device or host pointers) ------------------ */
/* preprocessor: B [N][K] T -> LUT_Scales [N][K/ags] T, LUT_Biases [N][K/ags] T,
 * QLUT [N][K/4][16] int8.  Bit-exact with lut_ctor_g4_int8_impl / partial_max_g4_int8_k8
 * (python/t_mac/intrins/lut_ctor.cc:38-260) in the generated loop order
 * (deploy/tuned/kernels.cc:1002-1040). */
TMAC_B200_API int tmac_b200_preprocessor(int K, int N, int act_group_size, int dtype, const void *B,
                                         void *LUT_Scales, void *LUT_Biases, void *QLUT);
/* qgemm_lut over rows [row0,row0+rows) of a resident tensor: C [N][rows] T.
 * Same arithmetic as tbl_g4_int8_{float,int32}_update + the generated recombine
 * (python/t_mac/intrins/tbl.cc:323-630; aarch64-llama-2-7b-2bit/kernels.cc:1059-1075). */
TMAC_B200_API int tmac_b200_qgemm_lut(int64_t handle, int row0, int rows, int N, int dtype,
                                      const void *QLUT, const void *LUT_Scales,
                                      const void *LUT_Biases, void *C);
/* Grouped launch: `count` qgemm_lut problems of identical geometry (same M, K, bits, grouping) in
 * ONE kernel launch -- the q/k/v or gate/up projections of a layer, MoE experts, ...  Host arrays of
 * per-problem DEVICE pointers; C[i] is [N][M]. */
TMAC_B200_API int tmac_b200_qgemm_lut_grouped(const int64_t *handles, int count, int N, int dtype,
                                              const void *const *QLUT, const void *const *LUT_Scales,
                                              const void *const *LUT_Biases, void *const *C);
/* The one-call form of a fused group (q/k/v, gate/up: tensors of one geometry applied to the SAME activation rows, the
 * sharing the reference's graph has between ggml_tmac_mul_mat_task_init and the task_compute calls of one op,
 * 3rdparty/llama.cpp/ggml/src/ggml.c:12570-12600): ONE launch, the LUT built inside it.  B [N][K] and C[i] [N][Mout]
 * are device pointers. */
TMAC_B200_API int tmac_b200_gemv_grouped(const int64_t *handles, int count, int N, int dtype, const void *B, void *const *C);
/* tmac_b200_gemv_grouped behind an input transform or before a residual add, so that a decoder layer's linears run as four launches
 * with no other ops between them: gemv_rmsnorm(q/k/v, x, w1), gemv_residual(o, att, x) -> h, gemv_rmsnorm(gate/up, h, w2),
 * gemv_glu(down, gate, up, h).  The rules of tmac_b200_gemv_grouped apply: device pointers only, the LUT built inside the launch,
 * the GEMV kernel at every N (no prefill tile: tmac_b200_prefill_rmsnorm / _rmsnorm_bias / _glu / _residual / _subnorm /
 * _subnorm_relu2 below are the prompt-sized forms), and
 * an armed tmac_b200_peer_outputs makes the call fail.  fp-path tensors with the
 * activation group inside a chunk only.  The transform is applied in fp32 (fp16 inputs widened first) to give the input a, whose
 * LUT is built as for any input.  Each call gives exactly tmac_b200_gemv_grouped(handles, count, N, F32, a, C32) with a
 * materialised in fp32, then y = fadd_rn(C32, R) when there is a residual R (fp16 R widened), rounded once to fp16 when dtype is
 * F16.  Every array is [N][...] of dtype unless said otherwise.
 *   gemv_rmsnorm: C[i] = gemv(handles[i], a) for count >= 1 tensors of one geometry (q/k/v, gate/up), H [N][K],
 *                 a[n][k] = fmul_rn(fmul_rn(H[n][k], inv_n), w[k]), inv_n and its sum of squares as for seq_add_gemv_rmsnorm (every
 *                 CTA computes inv_n itself).  w: fp32 [K], 16-byte aligned; eps finite, >= 0.  C[i] [N][Mout].
 *   gemv_glu:     C = gemv(handle, a) (+ R when R != NULL), a = swiglu(G, U) as for seq_add_gemv_glu.  G, U [N][K], R and C [N][Mout].
 *   gemv_residual: C = fadd_rn(gemv(handle, B), R), B [N][K], R and C [N][Mout].
 *   gemv_subnorm: the two sub-norms of a BitNet b1.58 layer, so that its linears run as four launches too: gemv_rmsnorm(q/k/v, x, w1),
 *                 gemv_subnorm(o, att, NULL, w_as, x) -> h, gemv_rmsnorm(gate/up, h, w2), gemv_subnorm(down, gate, up, w_fs, h).
 *                 C = gemv(handle, a) (+ R when R != NULL), a = rmsnorm(X) * w, X = G when U == NULL (attn_sub_norm before wo),
 *                 X = swiglu(G, U) when U != NULL (ffn_sub_norm before ffn_down).  a[n][k] = fmul_rn(fmul_rn(X[n][k], inv_n), w[k]),
 *                 X[n][k] in fp32 (swiglu rounded as for seq_add_gemv_glu), inv_n and its sum of squares of X as for gemv_rmsnorm.
 *                 G, U [N][K], R and C [N][Mout]; w and eps as for gemv_rmsnorm.
 *   gemv_subnorm_relu2: gemv_subnorm's ffn_sub_norm for a squared-ReLU FFN (BitNet b1.58 2B4T, HF hidden_act "relu2"):
 *                 gemv_subnorm_relu2(down, gate, up, w_fs, h).  The arguments, rules and output of gemv_subnorm with U != NULL, but
 *                 X[n][k] = fmul_rn(fmul_rn(r, r), U[n][k]) with r = G[n][k] when G[n][k] > 0 or is NaN (torch's relu), else +0.
 *                 U must not be NULL (gemv_subnorm is the attn sub-norm's call).  Decode sequences (seq_add_gemv_glu) and the routed
 *                 experts' GLU forms stay SiLU-only.
 *   gemv_rmsnorm_bias: gemv_rmsnorm for projections that carry a bias (Qwen2's q_proj, k_proj and v_proj; HF Qwen2Attention has
 *                 bias=True there and nowhere else): gemv_rmsnorm_bias(q/k/v, x, w1, b).  The arguments, rules, decomposition and
 *                 rejections of gemv_rmsnorm, plus bias: a host array of count device pointers, bias[i] fp32 [Mout], non-null, 16-byte
 *                 aligned, overlapping no C[j].  C[i][n][row] = fadd_rn(y, bias[i][row]), y the fp32 value gemv_rmsnorm gives that row,
 *                 rounded once to fp16 when dtype is F16 (so with F32 it equals gemv_rmsnorm followed by a float32 add of the bias, bit
 *                 for bit).  GQA models pass the stacked q/k/v tensor (count 1, bias [hidden + 2 * kv_dim]); MHA models three tensors
 *                 and three biases.  tmac_b200_debug_last_launch reports what gemv_rmsnorm reports.
 * R may equal C (each element is read and written by the same thread). */
TMAC_B200_API int tmac_b200_gemv_rmsnorm(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                                         void *const *C);
TMAC_B200_API int tmac_b200_gemv_rmsnorm_bias(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w,
                                              float eps, const float *const *bias, void *const *C);
TMAC_B200_API int tmac_b200_gemv_glu(int64_t handle, int N, int dtype, const void *G, const void *U, const void *R, void *C);
TMAC_B200_API int tmac_b200_gemv_residual(int64_t handle, int N, int dtype, const void *B, const void *R, void *C);
TMAC_B200_API int tmac_b200_gemv_subnorm(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps,
                                         const void *R, void *C);
TMAC_B200_API int tmac_b200_gemv_subnorm_relu2(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps,
                                               const void *R, void *C);
/* The transformed-input calls at prefill sizes (a prompt): exactly the arguments and output layouts of gemv_rmsnorm /
 * gemv_rmsnorm_bias / gemv_glu / gemv_residual / gemv_subnorm / gemv_subnorm_relu2, so a caller switches between the two forms by N (DESIGN.md 3.3), but the linears run on the prefill tiles (wgmma),
 * which stream each tensor once per 128 or 256 tokens instead of once per token.  They are the routed-expert tiles of
 * tmac_b200_prefill_experts run as one expert with the identity routing, written on the device: no host sync, graph-capturable.
 *   Input.  The call builds the input a in fp32 exactly as the gemv_* form does (fp16 inputs widened first): prefill_rmsnorm
 *           a[n][k] = fmul_rn(fmul_rn(H[n][k], inv_n), w[k]) with inv_n and its sum of squares in the order of seq_add_gemv_rmsnorm,
 *           prefill_glu a = swiglu(G, U), prefill_residual a = B, prefill_subnorm the a of gemv_subnorm (X = G or swiglu(G, U) in
 *           fp32, then its RMS norm in the order of gemv_rmsnorm), prefill_subnorm_relu2 the a of gemv_subnorm_relu2.  The preprocessor builds the LUT of each of the N rows once, and all
 *           count tensors share it.
 *   Per-row equality.  For every tensor i, row n of C[i] equals, bit for bit, row n of tmac_b200_gemv(handles[i], N, F32, a) on the
 *           same tile kind (a one-scale tensor: that call on its twin, the same codes with per-row scales all equal to its scale,
 *           no zero points, the same group and act group), then y = fadd_rn(that row, R) when there is a residual R (fp16 R widened), rounded once to fp16 when dtype
 *           is F16.  Against the float oracle: the fp16 tile within 5e-4 of max|C|, the int8 tile within 2e-5.
 *   Tile.   One kind per launch: the fp16 tile when the prefill16 knob is on, N >= 64 and the tensor fits it, else the int8 tile -- the
 *           dense calls' own rule, so without knobs the result is tmac_b200_gemv's wherever that call takes a tile.  prefill,
 *           prefill_min_n and pf_streamk do not apply; no stream-K; any N >= 1.  tmac_b200_debug_last_launch reports the tile in its
 *           own format with -N as the last field.
 *   prefill_rmsnorm: C[i] [N][Mout] for count >= 1 tensors of one geometry (q/k/v, gate/up), all in ONE tile launch over
 *                    (row tiles, token tiles, count).  w: fp32 [K], 16-byte aligned; eps finite, >= 0.
 *   prefill_glu:     C = gemv(handle, a) (+ R when R != NULL), G, U [N][K], R and C [N][Mout].
 *   prefill_residual: C = fadd_rn(gemv(handle, B), R), B [N][K], R and C [N][Mout].
 *   prefill_subnorm: C = gemv(handle, a) (+ R when R != NULL), G, U (or NULL) [N][K], R and C [N][Mout]; w and eps as for
 *                    prefill_rmsnorm.  A BitNet b1.58 prompt's linears run as prefill_rmsnorm(q/k/v, x, w1),
 *                    prefill_subnorm(o, att, NULL, w_as, x) -> h, prefill_rmsnorm(gate/up, h, w2), prefill_subnorm(down, gate, up, w_fs, h).
 *   prefill_subnorm_relu2: prefill_subnorm with gemv_subnorm_relu2's input; U must not be NULL.  A BitNet b1.58 2B4T prompt's down
 *                    projection: prefill_subnorm_relu2(down, gate, up, w_fs, h).
 *   prefill_rmsnorm_bias: prefill_rmsnorm with gemv_rmsnorm_bias's bias: C[i][n][row] = fadd_rn(y, bias[i][row]), y the fp32 value
 *                    prefill_rmsnorm gives that row on the same tile kind, rounded once to fp16 when dtype is F16.  The tile choice,
 *                    workspaces and rejections are prefill_rmsnorm's, plus the bias checks of gemv_rmsnorm_bias.  A Qwen2 prompt's
 *                    q/k/v: prefill_rmsnorm_bias(q/k/v, x, w1, b).
 * R may equal C.  Tensors: W2/W3/W4 fp-path tensors with the act group inside the chunk: per-row scales with or without zero points,
 * K % 128 == 0, chunk 128/64/32 K; or one scale with act group 128, 64 or 32 K < K and K % 128 == 0 (chunk 128 K) or K % 128 == 64
 * (chunk 64 K, e.g. BitNet-3B's down projection, K = 8640: the int8 tile at every N, whatever the prefill16 knob).  One geometry
 * for all.  -1 with a message, nothing launched: tensors the tiles do not take (the message
 * names the gemv_* form to use), mixed geometry, host pointers, the gemv_* forms' own rejections (w, eps, a null R for
 * prefill_residual), more than 65535 token tiles, an armed tmac_b200_peer_outputs (disarmed).  Workspaces are library buffers that grow
 * with N, K and Mout: make one eager call at the largest of them before capturing a call in a CUDA graph. */
TMAC_B200_API int tmac_b200_prefill_rmsnorm(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w, float eps,
                                            void *const *C);
TMAC_B200_API int tmac_b200_prefill_rmsnorm_bias(const int64_t *handles, int count, int N, int dtype, const void *H, const float *w,
                                                 float eps, const float *const *bias, void *const *C);
TMAC_B200_API int tmac_b200_prefill_glu(int64_t handle, int N, int dtype, const void *G, const void *U, const void *R, void *C);
TMAC_B200_API int tmac_b200_prefill_residual(int64_t handle, int N, int dtype, const void *B, const void *R, void *C);
TMAC_B200_API int tmac_b200_prefill_subnorm(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w, float eps,
                                            const void *R, void *C);
TMAC_B200_API int tmac_b200_prefill_subnorm_relu2(int64_t handle, int N, int dtype, const void *G, const void *U, const float *w,
                                                  float eps, const void *R, void *C);
/* Routed MoE experts: the router's top-k choice stays on the device, so a MoE FFN is two launches with no host sync and the token step
 * stays graph-capturable: gemv_experts([gate, up], h2, ids) -> G, U, then gemv_experts_glu(down, G, U, ids, weights, h) -> y.
 *   gemv_experts:     handles [count][n_experts] (host), entry i * n_experts + e = tensor i of expert e (e.g. i = 0 gate, 1 up).
 *                     B [N][K]; ids: device int32 [N][topk], read only by the kernel; C[i] [N][topk][Mout] with
 *                     C[i][n][j] = gemv(handles[i * n_experts + ids[n][j]], B[n]).
 *   gemv_experts_glu: handles [n_experts], K the FFN width.  G, U [N][topk][K] (C[0], C[1] of the call above); weights: device fp32
 *                     [N][topk]; R [N][Mout] or NULL, may equal C; C [N][Mout].  y_j = gemv(handles[ids[n][j]], a_j) with
 *                     a_j = swiglu(G[n][j], U[n][j]) as for gemv_glu, and
 *                     C[n] = fadd_rn(...fadd_rn(fmul_rn(w_0, y_0), fmul_rn(w_1, y_1))..., fmul_rn(w_{topk-1}, y_{topk-1})) (+ R[n]),
 *                     j ascending, no fma contraction, fp16 R widened, rounded once to fp16 when dtype is F16; the result does not
 *                     depend on which slot finishes first.
 * Each slot's row sums are those of tmac_b200_gemv_grouped over the N * count * topk selected tensors at N = 1, fed row n (the same
 * decomposition).  The rules of gemv_grouped apply: device pointers of dtype unless said otherwise, one geometry for all tensors,
 * the GEMV kernel at every N, an armed tmac_b200_peer_outputs makes the call fail; fp-path tensors with the activation group inside a
 * chunk only.  1 <= topk <= 8.  Repeated ids are allowed; each slot is computed on its own.  An id outside [0, n_experts) is never read
 * out of bounds: in gemv_experts that slot's Mout outputs are quiet NaN, in gemv_experts_glu every output of that token is; other
 * slots and tokens are unaffected.  gemv_experts_glu keeps a library workspace and arrival counters that return to zero by the end of
 * each launch: make one eager call at the largest N * topk and Mout before capturing it in a CUDA graph. */
TMAC_B200_API int tmac_b200_gemv_experts(const int64_t *handles, int count, int n_experts, int N, int dtype, const void *B,
                                         const int32_t *ids, int topk, void *const *C);
TMAC_B200_API int tmac_b200_gemv_experts_glu(const int64_t *handles, int n_experts, int N, int dtype, const void *G, const void *U,
                                             const int32_t *ids, const float *weights, int topk, const void *R, void *C);
/* Routed MoE experts at prefill sizes (a prompt, a decode batch of many requests): the arguments and output layouts of
 * gemv_experts / gemv_experts_glu, so a caller switches between the two forms by N (from N * topk of about 16 * n_experts on
 * Mixtral-8x7B's FFN, DESIGN.md 3.3), but each expert's tokens are grouped on the device and run on the prefill tiles (wgmma), which stream each
 * expert's weights once per 128 rows instead of once per slot.  Still no host sync, and the calls are graph-capturable.
 *   Slots.  Slot s = n * topk + j.  The slots of expert e in ascending s are that expert's rows.  The plain form's row of slot s is
 *           B[n]; the GLU form's is a_s = swiglu(G[n][j], U[n][j]) in fp32, rounded as for seq_add_gemv_glu.
 *   Per-slot equality.  Slot s's output row equals, bit for bit, row r of tmac_b200_gemv(handle_e, n_e, dtype, rows_e, .) on the same
 *           tile kind, where rows_e are expert e's n_e rows in order and s is the r-th of them: the preprocessor builds each row's LUT
 *           on its own, a token column of either tile depends only on its own column, and an expert's token tiles start at its first
 *           row, so each row sits at the tile position it has in that dense call.  Against the float oracle: the fp16 tile within
 *           5e-4 of max|C|, the int8 tile within 2e-5.
 *   Tile.   One kind per launch: the fp16 tile when the prefill16 knob is on and N * topk >= 256 * n_experts, else the int8 tile
 *           (prefill, prefill_min_n and pf_streamk do not apply; no stream-K).  tmac_b200_debug_last_launch reports that tile in its
 *           own format with -(N * topk) as the last field.
 *   prefill_experts:     C[i][n][j] = tensor i of expert ids[n][j] applied to B[n]; layouts as tmac_b200_gemv_experts.
 *   prefill_experts_glu: C[n] = fadd_rn(...fadd_rn(fmul_rn(w_0, y_0), fmul_rn(w_1, y_1))..., fmul_rn(w_{topk-1}, y_{topk-1}))
 *                        (+ R[n]), y_j the fp32 row of slot n * topk + j; the expression and layouts of gemv_experts_glu (no fma
 *                        contraction, fp16 R widened, rounded once for F16, R may equal C).
 * Tensors: those of tmac_b200_prefill_rmsnorm (per-row scales with K % 128 == 0, or one scale with act group < K and K % 128 == 0
 * or 64; a one-scale expert's slot equals the same call on its twin), one geometry for all.  An id outside [0, n_experts) is dropped from the grouping and nothing is read out of bounds:
 * prefill_experts stores quiet NaN in that slot's row, prefill_experts_glu in that token's whole output; other slots and tokens are
 * unaffected.  Repeated ids are independent slots.  -1 with a message, nothing launched: W1, integer-path and other tensors the tiles
 * do not take (gemv_experts is the call for them), host pointers, topk outside 1..8, n_experts outside 1..256,
 * count * n_experts > 65535, mixed geometry, an armed tmac_b200_peer_outputs (disarmed).  Workspaces are library buffers that grow
 * with N * topk, K and Mout: make one eager call at the largest of them before capturing a call in a CUDA graph. */
TMAC_B200_API int tmac_b200_prefill_experts(const int64_t *handles, int count, int n_experts, int N, int dtype, const void *B,
                                            const int32_t *ids, int topk, void *const *C);
TMAC_B200_API int tmac_b200_prefill_experts_glu(const int64_t *handles, int n_experts, int N, int dtype, const void *G, const void *U,
                                                const int32_t *ids, const float *weights, int topk, const void *R, void *C);
/* Fused convenience (llama_cpp_init + llama_cpp_compute of the whole tensor in one call,
 * workspaces owned by the library): C [N][M] = qgemm_lut(preprocessor(B)). */
TMAC_B200_API int tmac_b200_gemv(int64_t handle, int N, int dtype, const void *B, void *C);
/* ---- multi-GPU row sharding (SURVEY 8e) without a collective launch ------------------------------------------------
 * The reference spreads a mat-vec over threads by rows: tiles are independent given the replicated activation row
 * (3rdparty/llama.cpp/ggml/src/ggml.c:12636-12691).  Over GPUs the same partition makes the "all-gather" of the output vector
 * every rank storing its finished rows into every rank's vector: tmac_b200_peer_outputs arms the NEXT N = 1 launch
 * (tmac_b200_gemv / tmac_b200_qgemm_lut) to store its rows, besides C, at ptrs[q] + the same index -- device pointers into peer
 * memory, each already offset to this shard's first row.  The stores ride NVLink inside the GEMV's epilogue; a consumer on a
 * peer may read them after the producing launch has completed and the ranks have synchronised.  One-shot, 0..7 peers. */
TMAC_B200_API int tmac_b200_peer_outputs(void *const *ptrs, int count);
/* The flag / barrier per fused group: one tiny launch after which, in stream order, every launch this rank AND its peers
 * enqueued before their matching call has completed (so the peers' rows stored by tmac_b200_peer_outputs are in place).
 * flags: (world + 1) x uint32 inside this rank's ipc allocation, zero-initialised; peer_flags[q]: rank q's array mapped here. */
TMAC_B200_API int tmac_b200_peer_barrier(void *flags, void *const *peer_flags, int rank, int world);
/* Device allocations other processes of the node can map (cudaIpc*): alloc writes a 64-byte handle to send to the peers. */
TMAC_B200_API void *tmac_b200_ipc_alloc(size_t bytes, void *handle64);
TMAC_B200_API void *tmac_b200_ipc_open(const void *handle64);
TMAC_B200_API int tmac_b200_ipc_close(void *peer_ptr);
TMAC_B200_API int tmac_b200_ipc_free(void *ptr);

/* ---- decode sequences: a chain of (dependent) GEMVs in ONE persistent launch ------------------------------------------
 * The reference executes a token step as ggml's graph loop: one mul_mat node after the other on a persistent thread pool
 * (3rdparty/llama.cpp/ggml/src/ggml.c:12562-12706 per node; llama_cpp_init + llama_cpp_compute per node,
 * include/t-mac/tmac_gemm_wrapper.h:173-228).  A sequence is that loop for the quantised linears on the GPU: one CTA per
 * SM stays resident, the weight stream of op i+1, i+2 runs under the arithmetic of op i (weights do not depend on
 * activations), and the data dependency op -> op is carried by {value, epoch} words in HBM instead of a kernel boundary.
 *   seq_add_gemv: C = gemv(handle, input).  input = x (external device fp32 vector [K], 16-byte aligned) when x != NULL,
 *                 else elements [in_offset, in_offset + K) of the output of the earlier op `in_op` (in_offset even).
 *                 C (device, [M] of dtype, optional) receives a plain copy of the output.  Returns the op index.
 *   seq_add_gemv_glu: the down projection of a SwiGLU FFN, C = gemv(handle, a) with a[k] = silu(g[k]) * u[k] for k < K,
 *                 g = elements [gate_offset, gate_offset + K) of op gate_op's output, u = the same of op up_op (offset
 *                 up_offset).  Both ops must be earlier in the sequence (they may be the same op: the halves of a fused
 *                 gate_up tensor); both offsets even.  a is fp32 with exactly this rounding:
 *                 a = fmul_rn(fdiv_rn(g, fadd_rn(1, expf(-g))), u) (expf, not a fast-math exponential), and its LUT is built as
 *                 for any input, so the op equals seq_add_gemv fed with the vector a.  C and the return value as for seq_add_gemv.
 *   seq_add_gemv_rmsnorm: an op behind an RMSNorm (a decoder layer's FFN gate / up), C = gemv(handle, a) with a = the RMS norm of
 *                 the WHOLE output h of the earlier op in_op (K == that op's Mout):
 *                   a[k] = fmul_rn(fmul_rn(h[k], inv), w[k]),  inv = fdiv_rn(1, fsqrt_rn(fadd_rn(fdiv_rn(ss, K), eps)))
 *                 with ss = sum of h[k]^2 in this order: lane l of a warp adds, for the 4-element groups g = l, l + 32, ... in
 *                 ascending order, (h0*h0 + h1*h1) + (h2*h2 + h3*h3) to its sum, which starts at +0; the 32 lane sums are then
 *                 combined by the shfl_xor butterfly over 16, 8, 4, 2, 1; every operation is an fp32 rn multiply or add.  Every
 *                 consumer computes inv itself from the producer's rows, so the op equals seq_add_gemv fed with the vector a.
 *                 w: device fp32 [K], 16-byte aligned; eps finite, >= 0.  C and the return value as for seq_add_gemv.
 *   seq_residual: before seq_build, op `op` outputs y[row] = fadd_rn(gemv[row], r[row]), r an external device fp32 vector [Mout]
 *                 (16-byte aligned; r_op = -1) or the output of an earlier op r_op with the same Mout (r = NULL).  At most one
 *                 residual per op.  y is what C, the consumers' inputs and the peer outputs receive.
 *   seq_set_batch: before the first op, the sequence runs n activation rows (1 <= n <= 4, default 1) per launch -- a step for
 *                 a few tokens (concurrent requests, speculative drafts) that streams and decodes every weight block once for all
 *                 rows.  n = 1 is the one-row sequence.  With n > 1 every vector is n rows:
 *                   external x: fp32 [n][K], row t at x + t * K;
 *                   in_op / in_offset (and the two inputs of a GLU op): token t reads elements [in_offset, in_offset + K) of row t
 *                   of the producer's [n][Mout] output;
 *                   C: [n][Mout] of dtype, as tmac_b200_gemv's C; the library's internal outputs and words are n times as large;
 *                   GLU and norm inputs per row (each row its own inv; the norm weight w [K] is shared by the rows);
 *                   residual per row: r is [n][Mout], or row t of r_op's output.
 *                 Row t of every output equals, bit for bit, the same sequence built with n = 1 and fed row t.  A batch runs in
 *                 the resident chain kernel only: seq_build fails when seq_impl is 0, seq_grid > 0, an op has peer outputs, or the
 *                 sequence does not qualify for the chain (the rules below, and a multiple of 4 as every producer's Mout), which
 *                 includes all of its clusters being resident at once.  The batch kernels take 119-168 registers (3 or 4 CTAs
 *                 per SM), so on a 132-SM H100 the 11008-row W2 ops of Llama-2-7B (86 clusters, 344 CTAs) qualify at every n,
 *                 and 11008-row W3 / W4 ops (172 clusters, 688 CTAs: 6 CTAs per SM) do not -- their batch build fails.
 *   All tensors of a sequence share bits / group_size / act_group_size (one kernel instantiation); fp path
 *   (act_group_size <= 128).  Results equal tmac_b200_gemv up to fp32 re-association (different K split). */
TMAC_B200_API int64_t tmac_b200_seq_create(void);
TMAC_B200_API int tmac_b200_seq_set_batch(int64_t seq, int n);
TMAC_B200_API int tmac_b200_seq_add_gemv(int64_t seq, int64_t handle, const void *x, int in_op, int in_offset, void *C, int dtype);
TMAC_B200_API int tmac_b200_seq_add_gemv_glu(int64_t seq, int64_t handle, int gate_op, int gate_offset, int up_op, int up_offset,
                                             void *C, int dtype);
TMAC_B200_API int tmac_b200_seq_add_gemv_rmsnorm(int64_t seq, int64_t handle, int in_op, const float *w, float eps, void *C, int dtype);
TMAC_B200_API int tmac_b200_seq_residual(int64_t seq, int op, const float *r, int r_op);
/* Row-sharded sequences (multi-GPU): op `op` also stores its finished rows at ptrs[q][row] for q < count <= 7 -- device
 * pointers into peer memory (tmac_b200_ipc_open), each already offset to this shard's first row -- from the same epilogue that
 * stores C; the all-gather of a sharded chain without a collective launch (pair with tmac_b200_peer_barrier after the launch).
 * Call before tmac_b200_seq_build; needs the resident chain kernel (the build fails otherwise). */
TMAC_B200_API int tmac_b200_seq_peer_outputs(int64_t seq, int op, void *const *ptrs, int count);
TMAC_B200_API int tmac_b200_seq_build(int64_t seq);     /* allocates the device tables; no more ops afterwards */
TMAC_B200_API int tmac_b200_seq_launch(int64_t seq);    /* asynchronous, on the current stream; capturable in a CUDA graph */
TMAC_B200_API int tmac_b200_seq_status(int64_t seq);    /* synchronises; 0 = ok, -1 = a bounded wait inside the kernel expired */
/* Two kernels serve a sequence (tmac_b200_debug_set("seq_impl", 0 | 1 | 2), default 2): the resident chain kernel (tmac_chain.cuh: gemv3's
 * decomposition kept resident, an op's inputs arrive as {value, epoch} words written by the producing clusters; needs the fp path, one weight
 * format, fp32 producers, 16-byte aligned external inputs, even in_offset -- for both sources of a GLU op, the producer of a norm op and
 * the source of a residual, and offsets that are multiples of 4 in the grid-barrier form -- and all clusters resident at once) when
 * the sequence qualifies,
 * else the stream-K sequence kernel (tmac_seq.cuh).
 * info[8] = {grid, ring slots (-4 = resident chain, clusters of 4), slot bytes, shared-memory bytes, ops, planes/word, quads/chunk,
 * quads/activation group} */
TMAC_B200_API int tmac_b200_seq_info(int64_t seq, int *out8);
/* Debug (tmac_b200_debug_set("trace", 1) before seq_build): globaltimer stamps [ops][grid][16] of the last launch.  Stream-K kernel:
 * 0 op entered, 1 own LUT work done, 2 first block resident, 3/5/4 lookups done (first / middle / last warp), 6 CTA sums read,
 * 7 rows published, 8/9 producer thread enters / has requested the op.  Resident chain kernel (thread 0 of every CTA): 0 op entered,
 * 1/2 grid barrier seen / passed (barrier form only), 3 LUT slice built, 4 weight block resident, 5 lookups done, 6 CTA sums ready,
 * 7 partial sums sent, 8 rows published (leaders).  Returns grid.  tools/seq_bench.py --trace prints both. */
TMAC_B200_API int tmac_b200_seq_trace(int64_t seq, long long *dst, size_t cap_bytes);
TMAC_B200_API int tmac_b200_seq_free(int64_t seq);
/* Debug / parity gate G2: integer bit-plane sums CBits int32 [N][M*bits] in the reference
 * plane layout ([M/8][bits][8] per tensor), act-group sums folded over K. */
TMAC_B200_API int tmac_b200_cbits(int64_t handle, int N, const void *QLUT, int32_t *CBits);

/* ---- the reference's generated dispatchers (deploy/compile.py:60-67; instance
 *      deploy/tuned/aarch64-llama-2-7b-2bit/kernels.h:21-37).  Identical signature and
 *      argument meaning: m = (rows of this call) * bits, b = bits.  The configuration comes
 *      from the registered kcfg for (k, b); A must lie inside a range registered with
 *      tmac_b200_upload_weights (any tile offset), or be a device pointer returned by it. */
TMAC_B200_API int qgemm_lut_int8(int m, int k, int n, int b, void *A, void *LUT, void *Scales,
                                 void *LUT_Scales, void *LUT_Biases, void *C);
TMAC_B200_API int preprocessor_int8(int m, int k, int n, int b, void *B, void *LUT_Scales,
                                    void *LUT_Biases, void *QLUT);

/* ---- ggml hook (3rdparty/llama.cpp/ggml/include/ggml-tmac.h:25-38).  The four entry points
 *      that take raw buffers keep their exact signatures; the four that take `ggml_tensor *`
 *      are offered ggml-free (shape arguments) -- INTEGRATION.md shows the 6-line shim. */
#ifndef TMAC_B200_NO_GGML_DECLS   /* a translation unit that includes the reference's ggml-tmac.h takes these six from there */
TMAC_B200_API void ggml_tmac_init(void);
TMAC_B200_API void ggml_tmac_free(void);
TMAC_B200_API void ggml_tmac_mul_mat_task_init(void *src1, void *qlut, void *lut_scales,
                                               void *lut_biases, int n, int k, int m, int bits);
TMAC_B200_API void ggml_tmac_mul_mat_task_compute(void *src0, void *scales, void *qlut,
                                                  void *lut_scales, void *lut_biases, void *dst,
                                                  int n, int k, int m, int bits);
TMAC_B200_API void ggml_tmac_set_n_threads(int n_threads);
#ifndef TMAC_B200_NO_GGML_DECLS
/* Caller emulation (measurement / tests): ggml's T-MAC mul_mat branch for one activation row with HOST buffers --
 * task_init once, then task_compute once for the whole tensor (per_tile = 0; ref:ggml.c:12610-12630) or once per weight tile
 * of tile_rows rows from `threads` tile-stealing host threads (per_tile = 1; ref:ggml.c:12632-12703).  wdata: the op's
 * workspace (ggml_tmac_mul_mat_get_wsize bytes). */
TMAC_B200_API int tmac_b200_debug_ggml_mul_mat(void *src0_qweights, void *src0_scales, void *src1_row, void *wdata, void *dst,
                                               int ne01, int ne00, int bits, int tile_rows, int per_tile, int threads);
#endif
TMAC_B200_API int ggml_tmac_get_type_bits(int ggml_type);           /* ggml-tmac.cpp:503-526 */
#endif
/* ggml-free forms of can_mul_mat / get_wsize / get_nbytes / transform_tensor */
TMAC_B200_API int ggml_tmac_b200_can_mul_mat(int src0_type, int src1_is_f32, int dst_is_f32,
                                             const char *src0_name);
TMAC_B200_API size_t ggml_tmac_b200_mul_mat_get_wsize(int ne01, int ne10, int ne11, int bits);
TMAC_B200_API size_t ggml_tmac_b200_get_nbytes(int ne00, int ne01, int bits);
struct tmac_tensor_extra_b200 {  /* mirrors struct tmac_tensor_extra, ggml-tmac.h:17-23 */
    int lut_scales_size;
    int scales_size;
    int n_tile_num;
    uint8_t *qweights;  /* host alias key: pass qweights + tile offset to task_compute */
    float *scales;
};
TMAC_B200_API int ggml_tmac_b200_transform_tensor(void *data, int ne00, int ne01, int bits,
                                                  struct tmac_tensor_extra_b200 *extra);
/* The same for every ggml type the reference transforms (ggml-tmac.cpp:72-96, :290-498): I1..I4 (36..39) as above;
 * Q4_0 (2), TQ1_0 (34), TQ2_0 (35) blocks are decoded like the reference's accessors (:98-236; code w, real value
 * (w - 2^(bits-1)) * d) and re-encoded.  extra->qweights is then an address key (a reserved, unbacked range of the size
 * of the reference's permuted copy) to which ggml.c adds its tile offsets; extra->scales holds the scales in the
 * reference's run-time order.  The kcfg for the shape must have group_size = 32 (Q4_0) / 256 (TQ*), no zero point. */
TMAC_B200_API int ggml_tmac_b200_transform_tensor_typed(void *data, int ggml_type, int ne00, int ne01,
                                                        struct tmac_tensor_extra_b200 *extra);
/* Host-only: the block decode alone (codes [ne01][ne00], scales [ne01][ne00 / block]); returns the block size. */
TMAC_B200_API int tmac_b200_debug_decode_ggml(int ggml_type, const void *data, int ne00, int ne01, uint8_t *w, float *scales);

/* Host-only converter-side quantisers (3rdparty/llama.cpp/convert_hf_to_gguf.py): fp32 weights [rows][cols] -> codes in
 * [0, 2^bits) + scales (+ biased zeros) in the convention of tmac_b200_upload_plain.
 *   bitdistiller: Model._t_mac_quantize_tensor_bitdistiller (:409-452, zero-point branch), bit-identical (fp32, round half even);
 *                 group_size <= 0 = one group per row; scales / zeros [rows][cols / group_size].
 *   bitnet:       BitnetModel.weight_quant (:1884-1893) + the ternary rule (:1909-1917): codes 1, 2, 3 and ONE scale. */
TMAC_B200_API int tmac_b200_quantize_bitdistiller(const float *w, int rows, int cols, int bits, int group_size, uint8_t *codes,
                                                  float *scales, float *zeros);
TMAC_B200_API int tmac_b200_quantize_bitnet(const float *w, int rows, int cols, uint8_t *codes, float *scale);

/* The reference's default tiling for a shape without a tuned kcfg (python/t_mac/ops/qgemm.py:98-115, first candidate of
 * every knob).  0 or -1. */
TMAC_B200_API int tmac_b200_default_kcfg(int M, int K, int bits, int group_size, int act_group_size, int zero_point,
                                         int one_scale, tmac_b200_kcfg *out);

/* ---- GGUF files: what the reference pipeline produces (convert_hf_to_gguf.py:536-588; tensor blob python/t_mac/
 * model_utils.py:271) read without llama.cpp: metadata, tensor directory, tensor data mapped read-only. ---------------- */
struct tmac_b200_gguf_tensor {
    char name[128];
    int ggml_type;         /* ggml.h enum: 0 F32, 1 F16, 2 Q4_0, 34 TQ1_0, 35 TQ2_0, 36..39 I1..I4, ... */
    int n_dims;
    int64_t ne[4];         /* ne[0] = innermost (K for a weight matrix), ne[1] = rows */
    uint64_t offset;       /* from the start of the data section */
    uint64_t nbytes;       /* bytes available up to the next tensor (I-type tensors carry their scales behind the weights) */
    const void *data;      /* mapped, valid until tmac_b200_gguf_close */
};
TMAC_B200_API int64_t tmac_b200_gguf_open(const char *path);                       /* handle > 0 or -1 */
TMAC_B200_API int tmac_b200_gguf_close(int64_t gguf);
TMAC_B200_API int tmac_b200_gguf_tensor_count(int64_t gguf);
TMAC_B200_API int tmac_b200_gguf_tensor_info(int64_t gguf, int index, struct tmac_b200_gguf_tensor *out);
TMAC_B200_API int tmac_b200_gguf_find_tensor(int64_t gguf, const char *name);     /* index or -1 */
TMAC_B200_API int tmac_b200_gguf_meta_number(int64_t gguf, const char *key, double *out);
TMAC_B200_API int tmac_b200_gguf_meta_string(int64_t gguf, const char *key, char *dst, size_t cap);   /* length or -1 */
/* One quantised linear (2-D, I1..I4 / Q4_0 / TQ1_0 / TQ2_0) -> resident weights through the typed transform; the kcfg of
 * the shape must be registered for I-type tensors (their bytes are permuted by that tiling); block types carry their
 * grouping themselves, so without a registered kcfg the reference's default tiling (tmac_b200_default_kcfg) is registered
 * for the shape.  Returns the weight handle; extra as for ggml_tmac_b200_transform_tensor_typed. */
TMAC_B200_API int64_t tmac_b200_gguf_load_tensor(int64_t gguf, int index, struct tmac_tensor_extra_b200 *extra);

#ifdef __cplusplus
}
#endif
#endif /* TMAC_B200_H_ */
