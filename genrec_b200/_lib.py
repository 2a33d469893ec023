"""ctypes binding of include/genrec_b200.h - the reference-side stub a genrec maintainer would add (INTEGRATION.md).

There is NO fallback: if the shared library is missing or the device is not sm_90, importing callers get a
RuntimeError that says how to build.  Nothing here touches ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgenrec_b200.so")

c_void_p, c_int, c_float, c_size_t = C.c_void_p, C.c_int, C.c_float, C.c_size_t
c_u64, c_i64, c_u32 = C.c_uint64, C.c_int64, C.c_uint32


class HstuDims(C.Structure):
    _fields_ = [("B", c_int), ("L", c_int), ("D", c_int), ("H", c_int), ("npos", c_int), ("ntime", c_int),
                ("dropout_p", c_float), ("seed", c_u64), ("seed_dev", c_void_p), ("layer_index", c_int)]


class HstuLayerParams(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w",
                                         "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")]


class HstuLayerParamsF32(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("proj_w_split", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w_split",
                                         "ffn1_b", "ffn2_w_split", "ffn2_b", "ln2_g", "ln2_b")]


class HstuLayerGrads(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w",
                                         "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")]


class HstuSeq(C.Structure):
    _fields_ = [("bias_index", c_void_p), ("ld_index", c_int), ("has_time", c_int), ("pos_uniform", c_int), ("pos_bucket0", c_int),
                ("timestamps", c_void_p), ("pad", c_void_p), ("rel32", c_void_p), ("wide", c_void_p), ("time_thr", c_void_p)]


class HstuCache(C.Structure):
    _fields_ = [("B", c_int), ("capacity", c_int), ("num_layers", c_int), ("kv", c_void_p), ("timestamps", c_void_p),
                ("lengths", c_void_p), ("overflow", c_void_p)]


class HstuPool(C.Structure):
    _fields_ = [("max_users", c_int), ("num_layers", c_int), ("page_size", c_int), ("num_pages", c_int), ("max_items", c_int),
                ("kv", c_void_p), ("timestamps", c_void_p), ("page_table", c_void_p), ("lengths", c_void_p), ("overflow", c_void_p),
                ("free_stack", c_void_p), ("free_top", c_void_p), ("errors", c_void_p), ("row_of", c_void_p)]


class SasrecDims(C.Structure):
    _fields_ = [("B", c_int), ("L", c_int), ("D", c_int), ("H", c_int), ("dropout_p", c_float), ("seed", c_u64),
                ("seed_dev", c_void_p), ("layer_index", c_int)]


# name -> (restype, argtypes) ; must list EVERY symbol declared in include/genrec_b200.h (tests/test_abi.py checks)
P = C.POINTER
SIGNATURES = {
    "grb_last_error": (C.c_char_p, []),
    "grb_version": (c_int, []),
    "grb_launch_count": (c_u64, []),
    "grb_check_device": (c_int, [c_int]),
    "grb_set_defer_weight_grads": (c_int, [c_int]),
    "grb_join_deferred": (c_int, [c_void_p]),
    "grb_hstu_layer_saved_bytes": (c_size_t, [P(HstuDims)]),
    "grb_hstu_layer_workspace_bytes": (c_size_t, [P(HstuDims)]),
    "grb_hstu_layer_forward": (c_int, [P(HstuDims), P(HstuLayerParams), P(HstuSeq), c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_layer_backward": (c_int, [P(HstuDims), P(HstuLayerParams), P(HstuSeq), c_void_p, c_void_p, c_void_p,
                                        P(HstuLayerGrads), c_void_p, c_void_p]),
    "grb_hstu_bias_index": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "grb_hstu_seq_prepare": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_bucket_bytes_debug": (c_int, [P(HstuSeq), c_int, c_int, c_int, c_void_p, c_void_p]),
    "grb_hstu_attention_scratch_bytes": (c_size_t, [P(HstuDims)]),
    "grb_hstu_attention_forward": (c_int, [P(HstuDims), c_void_p, c_void_p, P(HstuSeq), c_void_p, c_void_p, c_void_p]),
    "grb_hstu_attention_backward": (c_int, [P(HstuDims), c_void_p, c_void_p, P(HstuSeq), c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_cache_append": (c_int, [P(HstuCache), c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_layer_extend_workspace_bytes": (c_size_t, [P(HstuDims), c_int]),
    "grb_hstu_layer_extend": (c_int, [P(HstuDims), P(HstuLayerParams), P(HstuCache), c_int, c_void_p, c_void_p, c_int, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_pool_append": (c_int, [P(HstuPool), c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_hstu_pool_release": (c_int, [P(HstuPool), c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "grb_hstu_layer_extend_paged_workspace_bytes": (c_size_t, [P(HstuDims), P(HstuPool)]),
    "grb_hstu_layer_extend_paged": (c_int, [P(HstuDims), P(HstuLayerParams), P(HstuPool), c_int, c_void_p, c_void_p, c_void_p, c_int,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_collate_jagged": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_embed_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_int,
                                  c_float, c_u64, c_void_p, c_void_p]),
    "grb_embed_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_int, c_float,
                                   c_u64, c_void_p, c_void_p, c_void_p]),
    "grb_head_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "grb_head_loss_forward_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_int, c_int,
                                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_head_logits": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                c_void_p]),
    "grb_eval_rank_metrics": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "grb_sasrec_attention_forward": (c_int, [P(SasrecDims), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p]),
    "grb_sasrec_attention_backward": (c_int, [P(SasrecDims), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_linear_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float,
                                   c_u64, c_void_p, c_u32, c_void_p]),
    "grb_linear_residual_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                            c_float, c_u64, c_void_p, c_u32, c_void_p]),
    "grb_linear_backward_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "grb_linear_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    "grb_linear_dact_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_u64, c_void_p, c_u32,
                                         c_void_p, c_void_p]),
    "grb_cast_rows_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_float, c_u64, c_void_p, c_u32, c_void_p]),
    "grb_layernorm_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    "grb_layernorm_backward_workspace_bytes": (c_size_t, [c_int, c_int]),
    "grb_layernorm_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    "grb_split3_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "grb_linear_f32x3_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "grb_linear_f32x3_bias_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "grb_hstu_layer_f32_workspace_bytes": (c_size_t, [P(HstuDims)]),
    "grb_hstu_layer_forward_f32": (c_int, [P(HstuDims), P(HstuLayerParamsF32), P(HstuSeq), c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_layernorm_f32_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p, c_void_p]),
    "grb_t5_attention_forward": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 8 + [c_void_p, c_void_p, c_int, c_void_p, c_int, c_float, c_float,
                                         c_u64, c_void_p, C.c_uint32, c_void_p, c_int, c_void_p, c_void_p]),
    "grb_t5_attention_backward": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 8 + [c_void_p, c_void_p, c_int, c_void_p, c_int, c_float, c_float,
                                          c_u64, c_void_p, C.c_uint32, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                          c_void_p, c_void_p, c_void_p]),
    "grb_trie_log_softmax": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                     c_void_p, c_void_p]),
    "grb_beam_select": (c_int, [c_void_p] * 8 + [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_cast_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "grb_adam_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_float, c_float,
                              c_float, c_float, c_float, c_float, c_int, c_void_p]),
    "grb_assert_unit_scalar": (c_int, [c_void_p, c_void_p]),
    "grb_dp_adam_step": (c_int, [c_void_p] * 14 + [c_size_t, c_int, c_int, c_void_p, c_float, c_float, c_float, c_float, c_float, c_float,
                                 c_void_p]),
    "grb_rq_residual_argmin": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_rq_sinkhorn_workspace_bytes": (c_size_t, [c_i64, c_int]),
    "grb_rq_sinkhorn": (c_int, [c_void_p, c_i64, c_int, C.c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "grb_kmeans_update": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
}

_lib: Optional[C.CDLL] = None
_loaded_count = {"launches": 0}


def load() -> C.CDLL:
    """dlopen the in-tree library and bind signatures.  Raises RuntimeError (never falls back)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"genrec_b200: {LIB_PATH} is missing.  Build it with `python -m genrec_b200.build` "
            "(nvcc, sm_90a).  There is no CPU or PyTorch fallback for this path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class GrbError(RuntimeError):
    pass


def check(rc: int) -> None:
    if rc != 0:
        raise GrbError(f"genrec_b200 error {rc}: {load().grb_last_error().decode()}")


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(*tensors: Optional[torch.Tensor]) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("genrec_b200 ops run on CUDA (sm_90a) tensors only - there is no CPU fallback; "
                               f"got a tensor on {t.device}")


_device_ok = set()


def ensure_device(device: torch.device) -> None:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx in _device_ok:
        return
    check(load().grb_check_device(idx))
    _device_ok.add(idx)


def launches() -> int:
    """CUDA kernels launched by libgenrec_b200.so in this process (counted inside its single launch helper)."""
    return int(load().grb_launch_count()) if _lib is not None or os.path.exists(LIB_PATH) else 0
