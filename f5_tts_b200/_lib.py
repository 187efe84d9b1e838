"""ctypes binding of libf5tts_b200.so (C ABI declared in include/f5tts_b200.h).

There is NO fallback: if the shared library is missing or the device is not sm_90 the import of any
operator raises.  Build with ``python -c "import __graft_entry__ as g; g.build()"`` or
``make -C f5_tts_b200/csrc``.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("F5_LIB") or os.path.join(_HERE, "libf5tts_b200.so")  # F5_LIB: diagnostic (TRACE=1) build

c_void_p, c_int, c_float, c_size_t, c_ll = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_longlong

ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_MISH = 0, 1, 2, 3
EPI_F16, EPI_F32, EPI_RESID, EPI_QKV_ROPE, EPI_QKV_NORM_ROPE = 0, 1, 2, 3, 4


class GemmArgs(C.Structure):
    _fields_ = [
        ("rows", c_int), ("batches", c_int), ("n_out", c_int), ("k", c_int), ("lda", c_int), ("ldw", c_int),
        ("bn", c_int), ("epi", c_int), ("act", c_int), ("conv_taps", c_int), ("cta_pair", c_int),
        ("bias", c_void_p), ("out", c_void_p), ("out16b", c_void_p), ("resid", c_void_p), ("ldo", c_int),
        ("gate", c_void_p), ("step_ptr", c_void_p), ("gate_step_stride", c_ll), ("row_len", c_void_p),
        ("seq", c_int), ("rope_cos", c_void_p), ("rope_sin", c_void_p), ("inner", c_int), ("pe_heads", c_int),
        ("weights_static", c_int),
        ("skip_padded_tiles", c_int), ("q_norm", c_void_p), ("k_norm", c_void_p), ("dim_head", c_int),
    ]


class VocosWeights(C.Structure):
    _fields_ = [
        ("embed_w", c_void_p), ("embed_b", c_void_p), ("norm_w", c_void_p), ("norm_b", c_void_p),
        ("dw_w", c_void_p * 8), ("dw_b", c_void_p * 8), ("ln_w", c_void_p * 8), ("ln_b", c_void_p * 8),
        ("pw1_w", c_void_p * 8), ("pw1_b", c_void_p * 8), ("pw2_w", c_void_p * 8), ("pw2_b", c_void_p * 8),
        ("gamma", c_void_p * 8), ("final_w", c_void_p), ("final_b", c_void_p), ("head_w", c_void_p),
        ("head_b", c_void_p), ("dim", c_int), ("inter", c_int), ("layers", c_int), ("n_mels", c_int),
    ]


class Arch(C.Structure):
    _fields_ = [(n, c_int) for n in ("backbone", "dim", "depth", "heads", "dim_head", "ff_inner", "mel_dim", "text_dim",
                                     "text_num_embeds", "conv_layers", "text_mask_padding", "pe_attn_head",
                                     "attn_mask_enabled", "qk_norm", "long_skip", "text_avg_upsample", "skip_type")]


class LayerWeights(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("w_qkv", "b_qkv", "w_out", "b_out", "w_ff1", "b_ff1", "w_ff2", "b_ff2",
                                        "w_skip", "g_attn", "g_ff", "q_norm_w", "k_norm_w")]


class CtxLayerWeights(C.Structure):  # f5_ctx_layer_weights: MMDiT text stream of one block
    _fields_ = [(n, c_void_p) for n in ("w_qkv_c", "b_qkv_c", "w_out_c", "b_out_c", "w_ff1_c", "b_ff1_c", "w_ff2_c",
                                        "b_ff2_c", "q_norm_c", "k_norm_c")]


class TextBlock(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("dw_w", "dw_b", "ln_w", "ln_b", "pw1_w", "pw1_b", "grn_gamma", "grn_beta",
                                        "pw2_w", "pw2_b")]


class Weights(C.Structure):
    _fields_ = [
        ("time_w0", c_void_p), ("time_b0", c_void_p), ("time_w1", c_void_p), ("time_b1", c_void_p),
        ("text_table", c_void_p), ("text_blocks", TextBlock * 8),
        ("proj_w", c_void_p), ("proj_b", c_void_p), ("proj_kpad", c_int),
        ("conv_w", c_void_p * 2), ("conv_b", c_void_p * 2),
        ("mod_w", c_void_p), ("mod_b", c_void_p),
        ("layers", C.POINTER(LayerWeights)), ("g_out", c_void_p), ("out_w", c_void_p), ("out_b", c_void_p),
        ("long_skip_w", c_void_p), ("ctx_layers", C.POINTER(CtxLayerWeights)),
    ]


class SampleArgs(C.Structure):
    _fields_ = [
        ("B", c_int), ("N", c_int), ("nt", c_int), ("steps", c_int),
        ("text", c_void_p), ("step_cond", c_void_p), ("y", c_void_p), ("duration", c_void_p),
        ("t", C.POINTER(c_float)), ("cfg_strength", c_float), ("trajectory", c_void_p), ("use_graph", c_int),
        ("v_out", c_void_p), ("exact_varlen", c_int), ("method", c_int),
    ]


class ForwardArgs(C.Structure):  # f5_forward_args: one backbone evaluation (the reference's transformer operator)
    _fields_ = [
        ("B", c_int), ("N", c_int), ("nt", c_int),
        ("x", c_void_p), ("step_cond", c_void_p), ("text", c_void_p), ("duration", c_void_p), ("time", c_void_p),
        ("mode", c_int), ("v_out", c_void_p), ("use_graph", c_int), ("reuse_text", c_int),
    ]


# ForwardArgs.mode: the conditional flow, cond | uncond packed (cfg_infer), the unconditional flow (joint drop)
FORWARD_COND, FORWARD_CFG, FORWARD_UNCOND = 0, 1, 2

ODE_METHODS = {"euler": 0, "midpoint": 1}
BACKBONES = {"DiT": 0, "UNetT": 1, "MMDiT": 2}  # Arch.backbone  # SampleArgs.method; backbone evaluations per grid interval: 1 and 2
SKIP_TYPES = {"concat": 0, "add": 1, "none": 2}  # Arch.skip_type: UNetT skip_connect_type


def sample_args(y, step_cond, text, duration, tg, steps, cfg_strength, trajectory, use_graph, exact_varlen, method,
                v_out=None) -> SampleArgs:
    """The f5_sample argument block of one call over these tensors.  `tg` is the ctypes float array of the time grid;
    the block points into it, so it must outlive the call."""
    a = SampleArgs()
    B, N, _ = y.shape
    a.B, a.N, a.nt, a.steps = B, N, text.shape[1], steps
    a.text, a.step_cond, a.y = text.data_ptr(), step_cond.data_ptr(), y.data_ptr()
    a.duration = duration.data_ptr() if duration is not None else None
    a.t = tg
    a.cfg_strength = float(cfg_strength)
    a.trajectory = trajectory.data_ptr() if trajectory is not None else None
    a.use_graph = 1 if use_graph else 0
    a.v_out = v_out.data_ptr() if v_out is not None else None
    a.exact_varlen = 1 if (exact_varlen and duration is not None) else 0
    a.method = ODE_METHODS[method]
    return a


_lock = threading.Lock()
_lib = None


class F5LibraryError(RuntimeError):
    pass


def lib():
    """Load the shared library once; raise loudly when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise F5LibraryError(
                f"{LIB_PATH} not found: the H100 CUDA library is not built (run __graft_entry__.build()). "
                "There is no CPU / PyTorch fallback for this path.")
        L = C.CDLL(LIB_PATH)
        L.f5_version.restype = c_int
        L.f5_last_error.restype = C.c_char_p
        L.f5_launch_count.restype = C.c_ulonglong
        L.f5_gemm.argtypes = [c_void_p, c_void_p, C.POINTER(GemmArgs), c_void_p]
        L.f5_gemm_tile.argtypes = [C.POINTER(GemmArgs), C.POINTER(c_int), C.POINTER(c_int)]
        L.f5_attention.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_float, c_void_p]
        L.f5_attention_dh.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_void_p]
        L.f5_attention_joint.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                         c_void_p, c_void_p, c_int, c_float, c_void_p]
        L.f5_attention_qwg.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_int,
                                       c_void_p]
        L.f5_attention_joint_qwg.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                             c_void_p, c_void_p, c_int, c_float, c_int, c_void_p]
        L.f5_attention_qwg_choice.argtypes = [c_int, c_int, c_int, c_int]
        L.f5_row_norm.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]
        L.f5_mel_spectrogram.argtypes = [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p]
        L.f5_vocos_workspace_bytes.argtypes = [c_int, c_int]
        L.f5_vocos_workspace_bytes.restype = c_size_t
        L.f5_vocos_decode.argtypes = [C.POINTER(VocosWeights), c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p,
                                      c_void_p]
        L.f5_vocos_decode_varlen.argtypes = [C.POINTER(VocosWeights), c_void_p, c_int, c_int, C.POINTER(c_int),
                                             c_void_p, c_size_t, c_void_p, c_void_p]
        L.f5_engine_create.argtypes = [C.POINTER(Arch), C.POINTER(Weights), C.POINTER(c_void_p)]
        L.f5_engine_destroy.argtypes = [c_void_p]
        L.f5_engine_destroy.restype = None
        L.f5_sample_workspace_bytes.argtypes = [c_void_p, c_int, c_int, c_int, c_float]
        L.f5_sample_workspace_bytes.restype = c_size_t
        L.f5_sample.argtypes = [c_void_p, C.POINTER(SampleArgs), c_void_p, c_size_t, c_void_p]
        L.f5_sample_flops.argtypes = [c_void_p, c_int, c_int, c_int, c_float]
        L.f5_sample_flops.restype = C.c_double
        L.f5_sample_workspace_bytes_nt.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_float]
        L.f5_sample_workspace_bytes_nt.restype = c_size_t
        L.f5_sample_flops_nt.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_float]
        L.f5_sample_flops_nt.restype = C.c_double
        L.f5_sample_cfg_split.argtypes = [c_void_p, C.POINTER(SampleArgs), c_void_p, c_size_t, c_void_p,
                                          c_void_p, C.POINTER(SampleArgs), c_void_p, c_size_t, c_void_p]
        L.f5_sample_cfg_split_workspace_bytes.argtypes = [c_void_p, c_int, c_int, c_int, c_int]
        L.f5_sample_cfg_split_workspace_bytes.restype = c_size_t
        L.f5_forward.argtypes = [c_void_p, C.POINTER(ForwardArgs), c_void_p, c_size_t, c_void_p]
        L.f5_forward_workspace_bytes.argtypes = [c_void_p, c_int, c_int, c_int, c_int]
        L.f5_forward_workspace_bytes.restype = c_size_t
        L.f5_engine_graph_count.argtypes = [c_void_p]
        L.f5_engine_graph_count.restype = c_int
        for name in ("f5_gemm", "f5_gemm_tile", "f5_attention", "f5_attention_dh", "f5_attention_joint", "f5_attention_qwg", "f5_attention_joint_qwg",
                     "f5_row_norm", "f5_mel_spectrogram",
                     "f5_vocos_decode",
                     "f5_vocos_decode_varlen", "f5_engine_create", "f5_sample", "f5_sample_cfg_split", "f5_forward"):
            getattr(L, name).restype = c_int
        _lib = L
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().f5_last_error().decode("utf-8", "replace")
        raise F5LibraryError(f"{what} failed (rc={rc}): {msg}")


def launch_count() -> int:
    return int(lib().f5_launch_count())


EXPORTED_SYMBOLS = [
    "f5_version", "f5_last_error", "f5_launch_count", "f5_gemm", "f5_gemm_tile", "f5_attention", "f5_attention_dh",
    "f5_row_norm", "f5_mel_spectrogram",
    "f5_vocos_workspace_bytes", "f5_vocos_decode", "f5_vocos_decode_varlen", "f5_engine_create", "f5_engine_destroy",
    "f5_sample_workspace_bytes", "f5_sample", "f5_sample_flops", "f5_attention_joint", "f5_sample_workspace_bytes_nt",
    "f5_sample_flops_nt", "f5_sample_cfg_split", "f5_sample_cfg_split_workspace_bytes", "f5_forward",
    "f5_forward_workspace_bytes", "f5_engine_graph_count", "f5_attention_qwg", "f5_attention_joint_qwg",
    "f5_attention_qwg_choice",
]

# Test-only library: the same objects plus one extern "C" wrapper per kernel launcher (csrc/kernel_hooks.cu), used by
# tests/test_gpu_small_kernels.py and tests/test_gpu_engine_kernels_f64.py.  Nothing in the package loads it.
KERNELS_LIB_PATH = os.path.join(_HERE, "libf5tts_b200_kernels.so")
KERNEL_HOOK_SYMBOLS = [
    "f5k_last_error", "f5k_row_norm", "f5k_dwconv7_ln", "f5k_text_gather", "f5k_mask_rows", "f5k_mask_rows_len",
    "f5k_grn_rows", "f5k_grn", "f5k_pack_input", "f5k_cfg_euler", "f5k_small_linear", "f5k_time_features",
    "f5k_silu_to_half", "f5k_rope_table", "f5k_prepend_time_token", "f5k_concat_half", "f5k_vocos_im2col",
    "f5k_ln_affine_f32", "f5k_istft", "f5k_row_norm_add_skip", "f5k_gemm_resid_sample",
    "f5k_mmdit_text_embed", "f5k_text_avg_upsample", "f5k_row_norm_sample", "f5k_prepend_time_token_sample",
    "f5k_dwconv7_ln_len", "f5k_vocos_im2col_len", "f5k_istft_len",
]
