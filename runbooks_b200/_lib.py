"""ctypes binding of include/b200w.h — the only way Python reaches the CUDA path.

There is deliberately no fallback: if libb200w.so is missing or a call fails, an exception is
raised (the product path must fail loudly when the CUDA extension is missing).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200w.so")

c_ctx = C.c_void_p
i32p = C.POINTER(C.c_int32)
f32p = C.POINTER(C.c_float)
i64p = C.POINTER(C.c_int64)
vp = C.c_void_p

BF16, F32, I32 = 0, 1, 2
ABI_VERSION = 2  # include/b200w.h B200W_ABI_VERSION


class Arch(C.Structure):
    _fields_ = [
        ("vocab_size", C.c_int32), ("hidden_size", C.c_int32), ("intermediate_size", C.c_int32),
        ("num_layers", C.c_int32), ("num_heads", C.c_int32), ("num_kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("max_seq_len", C.c_int32), ("rms_norm_eps", C.c_float),
        ("rope_theta", C.c_float), ("family", C.c_int32), ("pad_token_id", C.c_int32),
        ("max_positions", C.c_int32), ("reserved", C.c_int32 * 3),
    ]


class InferArch(C.Structure):
    """b200w_infer_arch; reserved[1] is parallel_norms (Falcon's ln_attn + ln_mlp)."""
    _fields_ = [
        ("family", C.c_int32), ("vocab_size", C.c_int32), ("hidden_size", C.c_int32),
        ("intermediate_size", C.c_int32), ("num_layers", C.c_int32), ("num_heads", C.c_int32),
        ("num_kv_heads", C.c_int32), ("head_dim", C.c_int32), ("max_ctx", C.c_int32),
        ("norm_eps", C.c_float), ("rope_theta", C.c_float), ("tie_embeddings", C.c_int32),
        ("max_positions", C.c_int32), ("weight_dtype", C.c_int32), ("reserved", C.c_int32 * 2),
    ]


MAX_TOP_LOGPROBS = 5  # include/b200w.h B200W_MAX_TOP_LOGPROBS


class Logprobs(C.Structure):
    """b200w_logprobs: HOST output arrays of the token log-probability calls."""
    _fields_ = [("top_k", C.c_int32), ("reserved", C.c_int32), ("lse", vp), ("token_lp", vp), ("top_ids", vp),
                ("top_lp", vp)]


class Sampling(C.Structure):
    """b200w_sampling: HOST per-row parameter arrays of b200w_infer_sample / b200w_op_sample."""
    _fields_ = [("reserved", C.c_int32), ("temperature", vp), ("top_p", vp), ("top_k", vp), ("seed", vp),
                ("draw", vp)]


class Penalties(C.Structure):
    """b200w_penalties: HOST per-row penalties and CSR entry arrays of b200w_infer_sample_penalized /
    b200w_op_penalize."""
    _fields_ = [("reserved", C.c_int32), ("presence", vp), ("frequency", vp), ("repetition", vp), ("offsets", vp),
                ("ids", vp), ("out_count", vp), ("in_prompt", vp), ("bias", vp)]


class HParams(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("max_grad_norm", C.c_float)]


# name -> (restype, argtypes); mirrors include/b200w.h one to one (tests check the symbol list)
PROTOTYPES = {
    "b200w_abi_version": (C.c_int, []),
    "b200w_debug_gemm_raster": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
    "b200w_create": (C.c_int, [C.c_int, C.POINTER(c_ctx)]),
    "b200w_destroy": (None, [c_ctx]),
    "b200w_last_error": (C.c_char_p, [c_ctx]),
    "b200w_sync": (C.c_int, [c_ctx]),
    "b200w_default_hparams": (None, [C.POINTER(HParams)]),
    "b200w_model_init": (C.c_int, [c_ctx, C.POINTER(Arch), C.POINTER(HParams), C.c_int, C.c_int]),
    "b200w_param_count": (C.c_int, [c_ctx, i64p, i64p]),
    "b200w_param_info": (C.c_int, [c_ctx, C.c_int64, C.c_char_p, C.c_size_t, i64p, i64p]),
    "b200w_load_tensor": (C.c_int, [c_ctx, C.c_char_p, vp, C.c_int, C.c_int64]),
    "b200w_read_tensor": (C.c_int, [c_ctx, C.c_char_p, vp, C.c_int, C.c_int64]),
    "b200w_read_state": (C.c_int, [c_ctx, C.c_char_p, C.c_int, vp, C.c_int64]),
    "b200w_init_random": (C.c_int, [c_ctx, C.c_uint64, C.c_float]),
    "b200w_comm_unique_id": (C.c_int, [vp]),
    "b200w_comm_init": (C.c_int, [c_ctx, C.c_int, C.c_int, vp]),
    "b200w_train_step": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_float, f32p, f32p]),
    "b200w_train_step_resident": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int64, C.c_float]),
    "b200w_read_scalars": (C.c_int, [c_ctx, f32p, f32p]),
    "b200w_timer_start": (C.c_int, [c_ctx]),
    "b200w_timer_stop": (C.c_int, [c_ctx, f32p]),
    "b200w_profile_gemm": (C.c_int, [c_ctx, C.c_int]),
    "b200w_profile_read": (C.c_int, [c_ctx, C.POINTER(C.c_double), C.POINTER(C.c_double), i64p]),
    "b200w_forward_backward": (C.c_int, [c_ctx, vp, vp, C.c_int, f32p]),
    "b200w_forward": (C.c_int, [c_ctx, vp, vp, C.c_int, vp, vp, f32p]),
    "b200w_train_step_docs": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, C.c_float, f32p, f32p]),
    "b200w_forward_backward_docs": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, f32p]),
    "b200w_forward_docs": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, vp, vp, f32p]),
    "b200w_launch_count": (C.c_int64, [c_ctx]),
    "b200w_device_bytes": (C.c_int64, [c_ctx]),
    "b200w_infer_init": (C.c_int, [c_ctx, C.POINTER(InferArch), C.c_int]),
    "b200w_infer_param_count": (C.c_int, [c_ctx, i64p, i64p]),
    "b200w_infer_param_info": (C.c_int, [c_ctx, C.c_int64, C.c_char_p, C.c_size_t, i64p, i64p]),
    "b200w_infer_load_tensor": (C.c_int, [c_ctx, C.c_char_p, vp, C.c_int, C.c_int64]),
    "b200w_infer_init_random": (C.c_int, [c_ctx, C.c_uint64, C.c_float]),
    "b200w_infer_read_weight": (C.c_int, [c_ctx, C.c_char_p, vp, C.c_int64]),
    "b200w_infer_step": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, vp, vp]),
    "b200w_infer_prefill": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, C.c_int, vp, vp]),
    "b200w_infer_device_bytes": (C.c_int64, [c_ctx]),
    "b200w_infer_weight_bytes": (C.c_int64, [c_ctx]),
    "b200w_infer_init_paged": (C.c_int, [c_ctx, C.POINTER(InferArch), C.c_int, C.c_int, C.c_int64]),
    "b200w_infer_init_paged_kv": (C.c_int, [c_ctx, C.POINTER(InferArch), C.c_int, C.c_int, C.c_int64, C.c_int]),
    "b200w_infer_kv_read": (C.c_int, [c_ctx, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]),
    "b200w_infer_reserve": (C.c_int, [c_ctx, C.c_int, C.c_int]),
    "b200w_infer_release": (C.c_int, [c_ctx, C.c_int]),
    "b200w_infer_kv_pages": (C.c_int, [c_ctx, i64p, i64p]),
    "b200w_infer_slot_pages": (C.c_int, [c_ctx, C.c_int, vp, C.c_int]),
    "b200w_infer_reserve_shared": (C.c_int, [c_ctx, C.c_int, C.c_int, vp, C.c_int]),
    "b200w_infer_retain_pages": (C.c_int, [c_ctx, vp, C.c_int, C.c_int]),
    "b200w_infer_prefill_cached": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp]),
    "b200w_infer_step_logprobs": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, vp, vp, vp]),
    "b200w_infer_prefill_logprobs": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]),
    "b200w_infer_sample": (C.c_int, [c_ctx, C.c_int, vp, vp, vp]),
    "b200w_infer_sample_penalized": (C.c_int, [c_ctx, C.c_int, vp, vp, vp, vp]),
    "b200w_infer_set_step_rows": (C.c_int, [c_ctx, C.c_int]),
    "b200w_op_gemm": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, C.c_int,
                                C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_op_gemm_bias": (C.c_int, [c_ctx, vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp,
                                     C.c_int, C.c_int]),
    "b200w_op_gemm_wire": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_int, vp]),
    "b200w_op_gemm_reserve": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_int,
                                        C.c_int, C.c_int, C.c_int, vp, C.c_int]),
    "b200w_op_gemm_group": (C.c_int, [c_ctx, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int]),
    "b200w_op_gemm_decode": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_w4_image_bytes": (C.c_int64, [C.c_int, C.c_int]),
    "b200w_op_quantize_w4": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int]),
    "b200w_op_dequantize_w4": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int]),
    "b200w_op_gemm_decode_w4": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_w8_image_bytes": (C.c_int64, [C.c_int, C.c_int]),
    "b200w_op_quantize_w8": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int]),
    "b200w_op_dequantize_w8": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int]),
    "b200w_op_gemm_decode_w8": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_op_gemm_decode_window": (C.c_int, [c_ctx, C.c_int, vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int]),
    "b200w_op_embed_fwd": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_op_embed_bwd": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int]),
    "b200w_op_layernorm_fwd": (C.c_int, [c_ctx, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_float]),
    "b200w_op_layernorm_bwd": (C.c_int, [c_ctx, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int]),
    "b200w_op_bias_act": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200w_op_relu_bwd": (C.c_int, [c_ctx, vp, vp, vp, C.c_int64]),
    "b200w_op_gelu_fwd": (C.c_int, [c_ctx, vp, vp, C.c_int64]),
    "b200w_op_gelu_bwd": (C.c_int, [c_ctx, vp, vp, vp, C.c_int64]),
    "b200w_op_colsum": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int, C.c_int]),
    "b200w_op_rmsnorm_fwd": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, C.c_int, C.c_float]),
    "b200w_op_rmsnorm_bwd": (C.c_int, [c_ctx, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int]),
    "b200w_op_rope": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                C.c_int]),
    "b200w_op_rope_positions": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                          C.c_int, vp]),
    "b200w_op_swiglu_fwd": (C.c_int, [c_ctx, vp, vp, C.c_int, C.c_int]),
    "b200w_op_swiglu_bwd": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, C.c_int]),
    "b200w_op_ce": (C.c_int, [c_ctx, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_float]),
    "b200w_op_attention_fwd": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp,
                                         C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "b200w_op_attention_fwd_cached": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, vp, vp, C.c_int64, vp, C.c_int, vp, vp,
                                                vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                C.c_float]),
    "b200w_op_attention_fwd_cached_fp8": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int64, vp,
                                                    C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.c_int, C.c_int, C.c_float]),
    "b200w_op_decode_attention": (C.c_int, [c_ctx, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int64, vp, C.c_int, vp,
                                            vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            vp, vp, C.c_float]),
    "b200w_op_logprobs": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp]),
    "b200w_op_sample": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]),
    "b200w_op_penalize": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, vp]),
    "b200w_op_attention_bwd": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp,
                                         vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "b200w_op_attention_fwd_docs": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp,
                                              C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "b200w_op_attention_bwd_docs": (C.c_int, [c_ctx, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp,
                                              vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "b200w_op_adamw": (C.c_int, [c_ctx, vp, vp, vp, vp, C.c_int, vp, C.c_int64, C.c_float, C.c_float,
                                 C.c_float, C.c_float, C.c_float, C.c_int, C.c_float]),
    "b200w_op_grad_norm": (C.c_int, [c_ctx, vp, C.c_int, C.c_int64, f32p]),
    "b200w_op_poison_onchip": (C.c_int, [c_ctx, C.c_uint32]),
}

_lib: Optional[C.CDLL] = None


class B200WError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"b200w status {status}: {msg}")
        self.status = status


def load() -> C.CDLL:
    """Loads libb200w.so (built in-tree by runbooks_b200/build.py). No fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(needs nvcc). runbooks_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.b200w_abi_version() != ABI_VERSION:
        raise ImportError("libb200w.so ABI version mismatch")
    _lib = lib
    return lib


def ptr(t) -> int:
    """Device / host address of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data
