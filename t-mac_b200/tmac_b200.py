"""tmac_b200.py -- ctypes binding of libtmac_b200.so (the C ABI in include/tmac_b200.h) plus a
Python mirror of the reference's host wrapper `TMAC::TMACGeMMWrapper`
(include/t-mac/tmac_gemm_wrapper.h:79-347) for tests and benchmarks.

This module never computes anything itself and has no CPU fallback: if the shared library is
missing it raises, and every compute call goes through the C ABI into the sm_90a kernels.
PyTorch is used by callers only to own device memory / streams; raw pointers cross this boundary.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TMAC_B200_LIB", os.path.join(HERE, "libtmac_b200.so"))

F32, F16 = 0, 1


class KCfg(C.Structure):
    """struct tmac_b200_kcfg (include/tmac_b200.h) == TMACGeMMConfig + compile-time options."""
    _fields_ = [("M", C.c_int), ("K", C.c_int), ("bits", C.c_int), ("bm", C.c_int), ("kfactor", C.c_int),
                ("simd_n_in", C.c_int), ("simd_n_out", C.c_int), ("group_size", C.c_int),
                ("act_group_size", C.c_int), ("zero_point", C.c_int), ("one_scale", C.c_int)]


class TensorExtra(C.Structure):
    """struct tmac_tensor_extra_b200 (mirrors ggml-tmac.h:17-23)."""
    _fields_ = [("lut_scales_size", C.c_int), ("scales_size", C.c_int), ("n_tile_num", C.c_int),
                ("qweights", C.c_void_p), ("scales", C.c_void_p)]


class GgufTensor(C.Structure):
    """struct tmac_b200_gguf_tensor."""
    _fields_ = [("name", C.c_char * 128), ("ggml_type", C.c_int), ("n_dims", C.c_int), ("ne", C.c_int64 * 4),
                ("offset", C.c_uint64), ("nbytes", C.c_uint64), ("data", C.c_void_p)]


EXPORTS = [
    "tmac_b200_init", "tmac_b200_shutdown", "tmac_b200_last_error", "tmac_b200_version", "tmac_b200_set_stream",
    "tmac_b200_set_float_type", "tmac_b200_set_lut_mode", "tmac_b200_register_kcfg", "tmac_b200_load_kcfg_file",
    "tmac_b200_find_kcfg", "tmac_b200_clear_kcfg", "tmac_b200_upload_weights", "tmac_b200_upload_plain",
    "tmac_b200_upload_plain_rows", "tmac_b200_debug_encode", "tmac_b200_free_weights", "tmac_b200_clone_weights", "tmac_b200_hint_next_weights",
    "tmac_b200_graph_begin", "tmac_b200_graph_end", "tmac_b200_graph_launch", "tmac_b200_graph_free", "tmac_b200_sync", "tmac_b200_debug_trace", "tmac_b200_debug_last_launch", "tmac_b200_debug_set", "tmac_b200_weights_nbytes", "tmac_b200_preprocessor",
    "tmac_b200_qgemm_lut", "tmac_b200_qgemm_lut_grouped", "tmac_b200_gemv", "tmac_b200_gemv_grouped", "tmac_b200_gemv_rmsnorm", "tmac_b200_gemv_rmsnorm_bias", "tmac_b200_gemv_glu", "tmac_b200_gemv_residual", "tmac_b200_gemv_subnorm", "tmac_b200_gemv_subnorm_relu2", "tmac_b200_gemv_experts", "tmac_b200_gemv_experts_glu", "tmac_b200_prefill_experts", "tmac_b200_prefill_experts_glu", "tmac_b200_prefill_rmsnorm", "tmac_b200_prefill_rmsnorm_bias", "tmac_b200_prefill_glu", "tmac_b200_prefill_residual", "tmac_b200_prefill_subnorm", "tmac_b200_prefill_subnorm_relu2", "tmac_b200_cbits", "qgemm_lut_int8", "preprocessor_int8",
    "ggml_tmac_init", "ggml_tmac_free", "ggml_tmac_mul_mat_task_init", "ggml_tmac_mul_mat_task_compute",
    "ggml_tmac_set_n_threads", "ggml_tmac_get_type_bits", "ggml_tmac_b200_can_mul_mat",
    "ggml_tmac_b200_mul_mat_get_wsize", "ggml_tmac_b200_get_nbytes", "ggml_tmac_b200_transform_tensor",
    "ggml_tmac_b200_transform_tensor_typed", "tmac_b200_debug_decode_ggml", "tmac_b200_upload_gptq", "tmac_b200_debug_unpack_gptq",
    "tmac_b200_default_kcfg", "tmac_b200_quantize_bitdistiller", "tmac_b200_quantize_bitnet", "tmac_b200_gguf_open", "tmac_b200_gguf_close", "tmac_b200_gguf_tensor_count", "tmac_b200_gguf_tensor_info", "tmac_b200_gguf_find_tensor",
    "tmac_b200_gguf_meta_number", "tmac_b200_gguf_meta_string", "tmac_b200_gguf_load_tensor",
    "tmac_b200_seq_create", "tmac_b200_seq_set_batch", "tmac_b200_seq_add_gemv", "tmac_b200_seq_add_gemv_glu", "tmac_b200_seq_add_gemv_rmsnorm",
    "tmac_b200_seq_residual", "tmac_b200_seq_build", "tmac_b200_seq_launch", "tmac_b200_seq_status",
    "tmac_b200_seq_info", "tmac_b200_seq_trace", "tmac_b200_seq_free", "tmac_b200_seq_peer_outputs",
    "tmac_b200_debug_ggml_mul_mat", "tmac_b200_peer_outputs", "tmac_b200_peer_barrier", "tmac_b200_ipc_alloc", "tmac_b200_ipc_open", "tmac_b200_ipc_close", "tmac_b200_ipc_free",
]

_lib = None


def load() -> C.CDLL:
    """Load the in-tree shared library; fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libtmac_b200.so is not built (run ./build.sh or __graft_entry__.build()); "
                           "there is no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    vp, i, i64, sz = C.c_void_p, C.c_int, C.c_int64, C.c_size_t
    sig = {
        "tmac_b200_init": (i, [i]), "tmac_b200_shutdown": (None, []), "tmac_b200_last_error": (C.c_char_p, []),
        "tmac_b200_version": (i, []), "tmac_b200_set_stream": (i, [vp]), "tmac_b200_set_float_type": (i, [i]),
        "tmac_b200_set_lut_mode": (i, [i]),
        "tmac_b200_register_kcfg": (i, [C.POINTER(KCfg)]), "tmac_b200_load_kcfg_file": (i, [C.c_char_p]),
        "tmac_b200_find_kcfg": (i, [i, i, i, C.POINTER(KCfg)]), "tmac_b200_clear_kcfg": (None, []),
        "tmac_b200_upload_weights": (i64, [C.POINTER(KCfg), vp, vp, i]),
        "tmac_b200_upload_plain": (i64, [C.POINTER(KCfg), vp, vp, vp]),
        "tmac_b200_upload_plain_rows": (i64, [C.POINTER(KCfg), vp, vp, vp, i, i]),
        "tmac_b200_debug_encode": (i64, [C.POINTER(KCfg), vp, vp, vp, sz, C.POINTER(C.c_int)]),
        "tmac_b200_free_weights": (i, [i64]), "tmac_b200_clone_weights": (i64, [i64]), "tmac_b200_hint_next_weights": (i, [i64]),
        "tmac_b200_graph_begin": (i, []), "tmac_b200_graph_end": (i64, []), "tmac_b200_graph_launch": (i, [i64, i]),
        "tmac_b200_graph_free": (i, [i64]), "tmac_b200_sync": (i, []), "tmac_b200_debug_trace": (i, [vp, i]), "tmac_b200_debug_last_launch": (i, [C.POINTER(C.c_int)]), "tmac_b200_debug_set": (i, [C.c_char_p, i]), "tmac_b200_weights_nbytes": (sz, [i64]),
        "tmac_b200_preprocessor": (i, [i, i, i, i, vp, vp, vp, vp]),
        "tmac_b200_qgemm_lut": (i, [i64, i, i, i, i, vp, vp, vp, vp]),
        "tmac_b200_qgemm_lut_grouped": (i, [vp, i, i, i, vp, vp, vp, vp]),
        "tmac_b200_gemv_grouped": (i, [vp, i, i, i, vp, vp]),
        "tmac_b200_gemv_rmsnorm": (i, [vp, i, i, i, vp, vp, C.c_float, vp]),
        "tmac_b200_gemv_rmsnorm_bias": (i, [vp, i, i, i, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_gemv_glu": (i, [i64, i, i, vp, vp, vp, vp]), "tmac_b200_gemv_residual": (i, [i64, i, i, vp, vp, vp]),
        "tmac_b200_gemv_subnorm": (i, [i64, i, i, vp, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_gemv_subnorm_relu2": (i, [i64, i, i, vp, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_gemv_experts": (i, [vp, i, i, i, i, vp, vp, i, vp]),
        "tmac_b200_gemv_experts_glu": (i, [vp, i, i, i, vp, vp, vp, vp, i, vp, vp]),
        "tmac_b200_prefill_experts": (i, [vp, i, i, i, i, vp, vp, i, vp]),
        "tmac_b200_prefill_experts_glu": (i, [vp, i, i, i, vp, vp, vp, vp, i, vp, vp]),
        "tmac_b200_prefill_rmsnorm": (i, [vp, i, i, i, vp, vp, C.c_float, vp]),
        "tmac_b200_prefill_rmsnorm_bias": (i, [vp, i, i, i, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_prefill_glu": (i, [i64, i, i, vp, vp, vp, vp]), "tmac_b200_prefill_residual": (i, [i64, i, i, vp, vp, vp]),
        "tmac_b200_prefill_subnorm": (i, [i64, i, i, vp, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_prefill_subnorm_relu2": (i, [i64, i, i, vp, vp, vp, C.c_float, vp, vp]),
        "tmac_b200_gemv": (i, [i64, i, i, vp, vp]), "tmac_b200_cbits": (i, [i64, i, vp, vp]),
        "qgemm_lut_int8": (i, [i, i, i, i, vp, vp, vp, vp, vp, vp]),
        "preprocessor_int8": (i, [i, i, i, i, vp, vp, vp, vp]),
        "ggml_tmac_init": (None, []), "ggml_tmac_free": (None, []),
        "ggml_tmac_mul_mat_task_init": (None, [vp, vp, vp, vp, i, i, i, i]),
        "ggml_tmac_mul_mat_task_compute": (None, [vp, vp, vp, vp, vp, vp, i, i, i, i]),
        "ggml_tmac_set_n_threads": (None, [i]), "ggml_tmac_get_type_bits": (i, [i]),
        "ggml_tmac_b200_can_mul_mat": (i, [i, i, i, C.c_char_p]),
        "ggml_tmac_b200_mul_mat_get_wsize": (sz, [i, i, i, i]), "ggml_tmac_b200_get_nbytes": (sz, [i, i, i]),
        "ggml_tmac_b200_transform_tensor": (i, [vp, i, i, i, C.POINTER(TensorExtra)]),
        "ggml_tmac_b200_transform_tensor_typed": (i, [vp, i, i, i, C.POINTER(TensorExtra)]),
        "tmac_b200_debug_decode_ggml": (i, [i, vp, i, i, vp, vp]),
        "tmac_b200_upload_gptq": (i64, [C.POINTER(KCfg), vp, vp, vp, i]),
        "tmac_b200_debug_unpack_gptq": (i, [vp, vp, vp, i, i, i, i, i, vp, vp, vp]),
        "tmac_b200_default_kcfg": (i, [i, i, i, i, i, i, i, C.POINTER(KCfg)]),
        "tmac_b200_quantize_bitdistiller": (i, [vp, i, i, i, i, vp, vp, vp]), "tmac_b200_quantize_bitnet": (i, [vp, i, i, vp, vp]),
        "tmac_b200_gguf_open": (i64, [C.c_char_p]), "tmac_b200_gguf_close": (i, [i64]), "tmac_b200_gguf_tensor_count": (i, [i64]),
        "tmac_b200_gguf_tensor_info": (i, [i64, i, C.POINTER(GgufTensor)]), "tmac_b200_gguf_find_tensor": (i, [i64, C.c_char_p]),
        "tmac_b200_gguf_meta_number": (i, [i64, C.c_char_p, C.POINTER(C.c_double)]), "tmac_b200_gguf_meta_string": (i, [i64, C.c_char_p, C.c_char_p, sz]),
        "tmac_b200_gguf_load_tensor": (i64, [i64, i, C.POINTER(TensorExtra)]),
        "tmac_b200_seq_create": (i64, []), "tmac_b200_seq_set_batch": (i, [i64, i]), "tmac_b200_seq_add_gemv": (i, [i64, i64, vp, i, i, vp, i]),
        "tmac_b200_seq_add_gemv_glu": (i, [i64, i64, i, i, i, i, vp, i]),
        "tmac_b200_seq_add_gemv_rmsnorm": (i, [i64, i64, i, vp, C.c_float, vp, i]), "tmac_b200_seq_residual": (i, [i64, i, vp, i]),
        "tmac_b200_seq_build": (i, [i64]), "tmac_b200_seq_launch": (i, [i64]), "tmac_b200_seq_status": (i, [i64]),
        "tmac_b200_debug_ggml_mul_mat": (i, [vp, vp, vp, vp, vp, i, i, i, i, i, i]), "tmac_b200_peer_outputs": (i, [vp, i]), "tmac_b200_peer_barrier": (i, [vp, vp, i, i]), "tmac_b200_ipc_alloc": (vp, [sz, vp]), "tmac_b200_ipc_open": (vp, [vp]),
        "tmac_b200_ipc_close": (i, [vp]), "tmac_b200_ipc_free": (i, [vp]),
        "tmac_b200_seq_peer_outputs": (i, [i64, i, vp, i]),
        "tmac_b200_seq_info": (i, [i64, C.POINTER(C.c_int)]), "tmac_b200_seq_trace": (i, [i64, vp, sz]), "tmac_b200_seq_free": (i, [i64]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class TMACError(RuntimeError):
    pass


def last_error() -> str:
    return load().tmac_b200_last_error().decode()


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        raise TMACError("%s failed: %s" % (what or "tmac_b200 call", last_error()))
    return rc


def ptr(x) -> int:
    """Raw address of a numpy array (host) or torch tensor (host or device)."""
    if x is None:
        return 0
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    return x.ctypes.data


def make_kcfg(M, K, bits, bm, kfactor=16, group_size=128, act_group_size=64, zero_point=False, one_scale=False) -> KCfg:
    return KCfg(M, K, bits, bm, kfactor, 16, 8, group_size, act_group_size, int(zero_point), int(one_scale))


@dataclass
class Weights:
    handle: int
    cfg: KCfg

    @property
    def nbytes(self) -> int:
        return load().tmac_b200_weights_nbytes(self.handle)

    def free(self):
        if self.handle > 0:
            load().tmac_b200_free_weights(self.handle)
            self.handle = -1


def last_launch() -> dict:
    v = (C.c_int * 8)()
    load().tmac_b200_debug_last_launch(v)
    return dict(zip(["cluster", "warps_per_cta", "chunks_per_warp", "min_blocks", "grid_x", "planes_per_word", "sym_lut", "batch"], list(v)))


def debug_set(key: str, value: int) -> None:
    check(load().tmac_b200_debug_set(key.encode(), int(value)), "tmac_b200_debug_set")


def clone(wt: "Weights") -> "Weights":
    h = load().tmac_b200_clone_weights(wt.handle)
    check(h, "tmac_b200_clone_weights")
    return Weights(h, wt.cfg)


def upload_reference_layout(cfg: KCfg, A, scales) -> Weights:
    """A / scales: host numpy arrays in the reference run-time layout (kept alive by the caller:
    the host range of A is the alias key used by qgemm_lut_int8)."""
    h = load().tmac_b200_upload_weights(C.byref(cfg), ptr(A), ptr(scales), F32)
    check(h, "tmac_b200_upload_weights")
    return Weights(h, cfg)


def upload_plain(cfg: KCfg, w, scales, zeros=None, row0: int = 0, rows: Optional[int] = None) -> Weights:
    rows = cfg.M - row0 if rows is None else rows
    h = load().tmac_b200_upload_plain_rows(C.byref(cfg), ptr(w), ptr(scales), ptr(zeros), row0, rows)
    check(h, "tmac_b200_upload_plain_rows")
    return Weights(h, cfg)


def preprocessor(K, N, ags, B, lut_scales, lut_biases, qlut, dtype=F32):
    check(load().tmac_b200_preprocessor(K, N, ags, dtype, ptr(B), ptr(lut_scales), ptr(lut_biases), ptr(qlut)),
          "tmac_b200_preprocessor")


def qgemm_lut(wt: Weights, N, qlut, lut_scales, lut_biases, Cout, row0=0, rows=None, dtype=F32):
    rows = wt.cfg.M - row0 if rows is None else rows
    check(load().tmac_b200_qgemm_lut(wt.handle, row0, rows, N, dtype, ptr(qlut), ptr(lut_scales), ptr(lut_biases), ptr(Cout)),
          "tmac_b200_qgemm_lut")


def _call(fn, *args):
    check(getattr(load(), fn)(*args), fn)


def _handles(wts):
    return (C.c_int64 * len(wts))(*[w.handle for w in wts])


def _ptrs(xs, n):
    """The n-entry host array of the addresses of xs (None: a null array)."""
    return None if xs is None else (C.c_void_p * n)(*[ptr(x) for x in xs])


def _topk(ids):
    return ids.shape[-1] if hasattr(ids, "shape") else 0


def qgemm_lut_grouped(wts, N, qluts, lut_scales, lut_biases, outs, dtype=F32):
    """One launch for len(wts) problems of identical geometry (device tensors)."""
    n = len(wts)
    _call("tmac_b200_qgemm_lut_grouped", _handles(wts), n, N, dtype, _ptrs(qluts, n), _ptrs(lut_scales, n), _ptrs(lut_biases, n),
          _ptrs(outs, n))


def gemv_grouped(wts, N, B, outs, dtype=F32):
    """len(wts) tensors of one geometry applied to the same activation rows B in ONE launch, LUT built inside (device tensors)."""
    _call("tmac_b200_gemv_grouped", _handles(wts), len(wts), N, dtype, ptr(B), _ptrs(outs, len(wts)))


# The bodies each gemv_* call with arrays shares with its prefill_* form, fn the C symbol.
def _rmsnorm(fn, wts, N, H, w, eps, outs, dtype, *bias):
    n = len(wts)
    _call(fn, _handles(wts), n, N, dtype, ptr(H), ptr(w), float(eps), *[_ptrs(b, n) for b in bias], _ptrs(outs, n))


def _experts(fn, tables, N, B, ids, outs, dtype):
    count, n_experts = len(tables), len(tables[0]) if tables else 0
    if any(len(t) != n_experts for t in tables):
        raise ValueError(fn[len("tmac_b200_"):] + ": every tensor needs one entry per expert")
    _call(fn, _handles([w for t in tables for w in t]), count, n_experts, N, dtype, ptr(B), ptr(ids), _topk(ids), _ptrs(outs, count))


def _experts_glu(fn, wts, N, G, U, ids, weights, Cout, R, dtype):
    _call(fn, _handles(wts), len(wts), N, dtype, ptr(G), ptr(U), ptr(ids), ptr(weights), _topk(ids), ptr(R), ptr(Cout))


def gemv_rmsnorm(wts, N, H, w, eps, outs, dtype=F32):
    """gemv_grouped on the RMS norm of H: input (H[n] * inv_n) * w, inv_n = 1 / sqrt(mean(H[n]^2) + eps) with the sum of squares in
    the order tmac_b200_gemv_rmsnorm documents.  w: device fp32 [K], 16-byte aligned."""
    _rmsnorm("tmac_b200_gemv_rmsnorm", wts, N, H, w, eps, outs, dtype)


def gemv_rmsnorm_bias(wts, N, H, w, eps, bias, outs, dtype=F32):
    """gemv_rmsnorm plus a bias on each tensor's outputs, outs[i] = gemv_rmsnorm's row + bias[i] rounded once (Qwen2's q/k/v;
    tmac_b200_gemv_rmsnorm_bias).  bias: len(wts) device fp32 [Mout] vectors, 16-byte aligned."""
    _rmsnorm("tmac_b200_gemv_rmsnorm_bias", wts, N, H, w, eps, outs, dtype, bias)


def gemv_glu(wt: Weights, N, G, U, Cout, R=None, dtype=F32):
    """Cout = gemv(wt, silu(G) * U) (+ R), the down projection of a SwiGLU FFN and its residual add (device tensors)."""
    _call("tmac_b200_gemv_glu", wt.handle, N, dtype, ptr(G), ptr(U), ptr(R), ptr(Cout))


def gemv_residual(wt: Weights, N, B, R, Cout, dtype=F32):
    """Cout = gemv(wt, B) + R (device tensors; R may be Cout)."""
    _call("tmac_b200_gemv_residual", wt.handle, N, dtype, ptr(B), ptr(R), ptr(Cout))


def gemv_subnorm(wt: Weights, N, G, w, eps, Cout, U=None, R=None, dtype=F32):
    """Cout = gemv(wt, rmsnorm(X) * w) (+ R), X = G, or silu(G) * U when U is given: a BitNet layer's o projection behind its
    attn_sub_norm, or its down projection behind its ffn_sub_norm (tmac_b200_gemv_subnorm; device tensors, R may be Cout)."""
    _call("tmac_b200_gemv_subnorm", wt.handle, N, dtype, ptr(G), ptr(U), ptr(w), float(eps), ptr(R), ptr(Cout))


def gemv_subnorm_relu2(wt: Weights, N, G, w, eps, Cout, U=None, R=None, dtype=F32):
    """Cout = gemv(wt, rmsnorm(relu(G)^2 * U) * w) (+ R): the down projection of a squared-ReLU BitNet FFN (b1.58 2B4T) behind its
    ffn_sub_norm (tmac_b200_gemv_subnorm_relu2; gemv_subnorm's argument order, U required; device tensors, R may be Cout)."""
    _call("tmac_b200_gemv_subnorm_relu2", wt.handle, N, dtype, ptr(G), ptr(U), ptr(w), float(eps), ptr(R), ptr(Cout))


def gemv_experts(tables, N, B, ids, outs, dtype=F32):
    """Routed experts: tables[i][e] is tensor i of expert e (e.g. i = 0 gate, 1 up).  outs[i] [N][topk][Mout] gets
    gemv(tables[i][ids[n][j]], B[n]) in row (n, j); ids: device int32 [N][topk], read only on the device."""
    _experts("tmac_b200_gemv_experts", tables, N, B, ids, outs, dtype)


def gemv_experts_glu(wts, N, G, U, ids, weights, Cout, R=None, dtype=F32):
    """Cout[n] = sum_j weights[n][j] * gemv(wts[ids[n][j]], silu(G[n][j]) * U[n][j]) (+ R[n]), the down projection of routed
    experts and their combine in ascending j (device tensors; ids int32 and weights fp32 [N][topk])."""
    _experts_glu("tmac_b200_gemv_experts_glu", wts, N, G, U, ids, weights, Cout, R, dtype)


def prefill_experts(tables, N, B, ids, outs, dtype=F32):
    """gemv_experts' arguments and output, run on the prefill tiles with each expert's tokens grouped on the device (the form for
    large N * topk, tmac_b200_prefill_experts)."""
    _experts("tmac_b200_prefill_experts", tables, N, B, ids, outs, dtype)


def prefill_experts_glu(wts, N, G, U, ids, weights, Cout, R=None, dtype=F32):
    """gemv_experts_glu's arguments and output, run on the prefill tiles (tmac_b200_prefill_experts_glu)."""
    _experts_glu("tmac_b200_prefill_experts_glu", wts, N, G, U, ids, weights, Cout, R, dtype)


def prefill_rmsnorm(wts, N, H, w, eps, outs, dtype=F32):
    """gemv_rmsnorm's arguments and output, run on the prefill tiles with all len(wts) tensors in one launch (the form for a prompt,
    tmac_b200_prefill_rmsnorm)."""
    _rmsnorm("tmac_b200_prefill_rmsnorm", wts, N, H, w, eps, outs, dtype)


def prefill_rmsnorm_bias(wts, N, H, w, eps, bias, outs, dtype=F32):
    """gemv_rmsnorm_bias's arguments and output, run on the prefill tiles (tmac_b200_prefill_rmsnorm_bias)."""
    _rmsnorm("tmac_b200_prefill_rmsnorm_bias", wts, N, H, w, eps, outs, dtype, bias)


def prefill_glu(wt: Weights, N, G, U, Cout, R=None, dtype=F32):
    """gemv_glu's arguments and output, run on the prefill tiles (tmac_b200_prefill_glu)."""
    _call("tmac_b200_prefill_glu", wt.handle, N, dtype, ptr(G), ptr(U), ptr(R), ptr(Cout))


def prefill_residual(wt: Weights, N, B, R, Cout, dtype=F32):
    """gemv_residual's arguments and output, run on the prefill tiles (tmac_b200_prefill_residual)."""
    _call("tmac_b200_prefill_residual", wt.handle, N, dtype, ptr(B), ptr(R), ptr(Cout))


def prefill_subnorm(wt: Weights, N, G, w, eps, Cout, U=None, R=None, dtype=F32):
    """gemv_subnorm's arguments and output, run on the prefill tiles (tmac_b200_prefill_subnorm)."""
    _call("tmac_b200_prefill_subnorm", wt.handle, N, dtype, ptr(G), ptr(U), ptr(w), float(eps), ptr(R), ptr(Cout))


def prefill_subnorm_relu2(wt: Weights, N, G, w, eps, Cout, U=None, R=None, dtype=F32):
    """gemv_subnorm_relu2's arguments and output, run on the prefill tiles (tmac_b200_prefill_subnorm_relu2)."""
    _call("tmac_b200_prefill_subnorm_relu2", wt.handle, N, dtype, ptr(G), ptr(U), ptr(w), float(eps), ptr(R), ptr(Cout))


def gemv(wt: Weights, N, B, Cout, dtype=F32):
    check(load().tmac_b200_gemv(wt.handle, N, dtype, ptr(B), ptr(Cout)), "tmac_b200_gemv")


def cbits(wt: Weights, N, qlut, out):
    check(load().tmac_b200_cbits(wt.handle, N, ptr(qlut), ptr(out)), "tmac_b200_cbits")


def peer_outputs(ptrs) -> None:
    """Arm the next N = 1 launch to store its rows into these peer-memory addresses too (tmac_b200_peer_outputs)."""
    n = len(ptrs)
    arr = (C.c_void_p * max(1, n))(*[int(p) for p in ptrs])
    check(load().tmac_b200_peer_outputs(arr, n), "tmac_b200_peer_outputs")


class _RawCuda:
    """Device memory that is not owned by torch, exposed through __cuda_array_interface__ (torch.as_tensor wraps it)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


class SharedVector:
    """One float32 buffer per rank that every rank of the node can write (cudaIpc): `local` is this rank's buffer as a torch
    tensor, `peer_ptr(q)` the address of rank q's buffer in this process.  Used for the all-gather fused into the GEMV
    epilogue (tmac_b200_peer_outputs).  Collective: every rank must construct it."""

    def __init__(self, nfloats: int, dist, rank: int, world: int):
        import torch
        lib = load()
        nfloats += world + 1                    # + the barrier flags (tmac_b200_peer_barrier)
        self.n, self.rank, self.world = nfloats, rank, world
        h = (C.c_ubyte * 64)()
        self.ptr = lib.tmac_b200_ipc_alloc(nfloats * 4, h)
        if not self.ptr:
            raise TMACError("tmac_b200_ipc_alloc failed: " + last_error())
        handles = [None] * world
        dist.all_gather_object(handles, bytes(h))
        self.peers = {}
        for q in range(world):
            if q == rank:
                continue
            hb = (C.c_ubyte * 64).from_buffer_copy(handles[q])
            pp = lib.tmac_b200_ipc_open(hb)
            if not pp:
                raise TMACError("tmac_b200_ipc_open failed: " + last_error())
            self.peers[q] = pp
        self._raw = _RawCuda(self.ptr, nfloats * 4)
        self.local = torch.as_tensor(self._raw, device="cuda").view(torch.float32)[: nfloats - (world + 1)]
        dist.barrier()

    def peer_ptr(self, q: int) -> int:
        return self.ptr if q == self.rank else self.peers[q]

    def barrier(self):
        """Stream-ordered barrier over the ranks (tmac_b200_peer_barrier); the last world + 1 floats of the buffer are its flags."""
        off = 4 * (self.n - (self.world + 1))
        arr = (C.c_void_p * 8)(*[self.peer_ptr(q) + off for q in range(self.world)] + [0] * (8 - self.world))
        check(load().tmac_b200_peer_barrier(self.ptr + off, arr, self.rank, self.world), "tmac_b200_peer_barrier")

    def close(self, dist=None):
        lib = load()
        if dist is not None:
            dist.barrier()
        for pp in self.peers.values():
            lib.tmac_b200_ipc_close(pp)
        self.peers = {}
        if dist is not None:
            dist.barrier()
        if self.ptr:
            lib.tmac_b200_ipc_free(self.ptr)
            self.ptr = 0


SEQ_WARPS = 19      # kSeqWarps (consumer warps per CTA of the sequence kernel)


class Sequence:
    """A chain of (dependent) GEMVs executed by one persistent launch (tmac_b200_seq_*, include/tmac_b200.h).  batch: activation
    rows per launch (1..4, tmac_b200_seq_set_batch); with batch > 1 every vector (x, out, residual) is [batch][length]."""

    def __init__(self, batch: int = 1):
        self.h = load().tmac_b200_seq_create()
        check(self.h, "tmac_b200_seq_create")
        self.nops = 0
        self.batch = batch
        if batch != 1:
            try:
                check(load().tmac_b200_seq_set_batch(self.h, batch), "tmac_b200_seq_set_batch")
            except TMACError:
                self.free()
                raise

    def add(self, wt: "Weights", x=None, in_op: int = -1, in_offset: int = 0, out=None, dtype=F32) -> int:
        """x: external device fp32 vector, or None -> elements [in_offset, in_offset + K) of op `in_op`'s output."""
        rc = load().tmac_b200_seq_add_gemv(self.h, wt.handle, ptr(x), in_op, in_offset, ptr(out), dtype)
        check(rc, "tmac_b200_seq_add_gemv")
        self.nops += 1
        return rc

    def add_glu(self, wt: "Weights", gate_op: int, gate_offset: int, up_op: int, up_offset: int, out=None, dtype=F32) -> int:
        """The down projection of a SwiGLU FFN: input silu(g) * u, g / u = elements [offset, offset + K) of the outputs of the
        earlier ops gate_op / up_op (tmac_b200_seq_add_gemv_glu)."""
        rc = load().tmac_b200_seq_add_gemv_glu(self.h, wt.handle, gate_op, gate_offset, up_op, up_offset, ptr(out), dtype)
        check(rc, "tmac_b200_seq_add_gemv_glu")
        self.nops += 1
        return rc

    def add_rmsnorm(self, wt: "Weights", in_op: int, w, eps: float, out=None, dtype=F32) -> int:
        """An op behind an RMSNorm: input (h * inv) * w, h = the whole output of the earlier op in_op, inv = 1 / sqrt(mean(h^2) + eps)
        with the sum of squares in the order tmac_b200_seq_add_gemv_rmsnorm documents.  w: device fp32 [K], 16-byte aligned."""
        rc = load().tmac_b200_seq_add_gemv_rmsnorm(self.h, wt.handle, in_op, ptr(w), float(eps), ptr(out), dtype)
        check(rc, "tmac_b200_seq_add_gemv_rmsnorm")
        self.nops += 1
        return rc

    def residual(self, op: int, r=None, r_op: int = -1):
        """Op `op` outputs gemv + r: r an external device fp32 vector [Mout], or the output of the earlier op r_op (r=None)."""
        check(load().tmac_b200_seq_residual(self.h, op, ptr(r), r_op), "tmac_b200_seq_residual")

    def peer_outputs(self, op: int, ptrs):
        """Row sharding: op `op` also stores its rows at these peer addresses (ints, already offset to the shard's first row)."""
        n = len(ptrs)
        arr = (C.c_void_p * max(n, 1))(*ptrs)
        check(load().tmac_b200_seq_peer_outputs(self.h, op, arr, n), "tmac_b200_seq_peer_outputs")

    def build(self):
        check(load().tmac_b200_seq_build(self.h), "tmac_b200_seq_build")
        return self

    def launch(self):
        check(load().tmac_b200_seq_launch(self.h), "tmac_b200_seq_launch")

    def status(self):
        check(load().tmac_b200_seq_status(self.h), "tmac_b200_seq_status")

    def info(self) -> dict:
        v = (C.c_int * 8)()
        check(load().tmac_b200_seq_info(self.h, v), "tmac_b200_seq_info")
        return dict(zip(["grid", "ring_slots", "slot_bytes", "smem_bytes", "ops", "planes_per_word", "quads_per_chunk", "quads_per_act_group"], list(v)))

    def trace(self):
        import numpy as np
        inf = self.info()
        n, g = inf["ops"], inf["grid"]
        buf = np.zeros(n * g * (16 + 16 * SEQ_WARPS), np.int64)
        check(load().tmac_b200_seq_trace(self.h, buf.ctypes.data, buf.nbytes), "tmac_b200_seq_trace")
        self.warp_trace = buf[n * g * 16:].reshape(n, g, SEQ_WARPS, 16)      # per consumer warp: clock64 stamps (tmac_seq.cuh)
        return buf[:n * g * 16].reshape(n, g, 16)

    def free(self):
        if self.h > 0:
            load().tmac_b200_seq_free(self.h)
            self.h = -1


class TMACGeMMWrapper:
    """Python mirror of TMAC::TMACGeMMWrapper<T> (include/t-mac/tmac_gemm_wrapper.h:79-347):
    same method names and argument meaning; kernels are looked up by (M, K, N, bits) in the kcfg
    registry instead of a generated `if` chain."""

    def __init__(self, n_threads: int = 1, act_group_size: int = 32, kcfg_file: str = "", library_file: str = ""):
        self._lib = load()
        check(self._lib.tmac_b200_init(-1), "tmac_b200_init")
        self._act_group_size = act_group_size
        kcfg_file = kcfg_file or os.environ.get("TMAC_KCFG_FILE", "")  # tmac_gemm_wrapper.h:40-56
        if kcfg_file:
            check(self._lib.tmac_b200_load_kcfg_file(kcfg_file.encode()), "load kcfg")

    def set_num_threads(self, n_threads: int):  # :102-112 -- no CPU thread pool on the GPU path
        self._lib.ggml_tmac_set_n_threads(n_threads)

    def get_kcfg(self, M, K, N, bits) -> KCfg:  # :230-255
        out = KCfg()
        check(self._lib.tmac_b200_find_kcfg(M * bits, K, bits, C.byref(out)), "get_kcfg")
        return out

    def llama_cpp_init(self, B, qlut, lut_scales, lut_biases, M, K, N, bits):  # :173-195
        check(self._lib.preprocessor_int8(M * bits, K, N, bits, ptr(B), ptr(lut_scales), ptr(lut_biases), ptr(qlut)),
              "preprocessor_int8")

    def llama_cpp_compute(self, A, scales, qlut, lut_scales, lut_biases, Cout, M, K, N, bits):  # :200-228
        check(self._lib.qgemm_lut_int8(M * bits, K, N, bits, ptr(A), ptr(qlut), ptr(scales), ptr(lut_scales),
                                       ptr(lut_biases), ptr(Cout)), "qgemm_lut_int8")
