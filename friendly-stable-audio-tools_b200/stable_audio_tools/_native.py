"""ctypes binding of libsatb200.so (the C ABI declared in include/satb200.h).

The library is the only compute path of this package: if it is missing, or if a
tensor is not on a CUDA device, the calls below raise - there is no CPU or eager
PyTorch fallback (the oracle under ``oracle/`` is test infrastructure and is never
imported from here).
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libsatb200.so")

_lib = None


class NativeError(RuntimeError):
    pass


class SatbDitConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in (
        "io_channels", "embed_dim", "depth", "num_heads", "cond_token_dim", "global_cond_dim",
        "project_cond_tokens", "project_global_cond", "global_cond_type", "patch_size", "operand_dtype", "qk_norm",
        "input_concat_dim", "prepend_cond_dim")]


SATB_MAX_STAGES = 8


class SatbT5Config(ctypes.Structure):
    _fields_ = ([(n, ctypes.c_int) for n in (
        "vocab_size", "d_model", "d_kv", "num_heads", "d_ff", "num_layers", "relative_attention_num_buckets",
        "relative_attention_max_distance", "feed_forward_proj")]
        + [("layer_norm_epsilon", ctypes.c_float), ("operand_dtype", ctypes.c_int)])


# SatbT5Config.feed_forward_proj
T5_FF_RELU, T5_FF_GATED_GELU = 0, 1


class SatbRobertaConfig(ctypes.Structure):
    _fields_ = ([(n, ctypes.c_int) for n in (
        "vocab_size", "hidden_size", "num_heads", "intermediate_size", "num_layers", "max_position_embeddings",
        "type_vocab_size", "pad_token_id")]
        + [("layer_norm_eps", ctypes.c_float), ("operand_dtype", ctypes.c_int)])


class SatbOobleckConfig(ctypes.Structure):
    _fields_ = [("in_channels", ctypes.c_int), ("channels", ctypes.c_int), ("latent_dim", ctypes.c_int),
                ("n_stages", ctypes.c_int), ("c_mults", ctypes.c_int * SATB_MAX_STAGES),
                ("strides", ctypes.c_int * SATB_MAX_STAGES), ("final_tanh", ctypes.c_int),
                ("is_decoder", ctypes.c_int), ("operand_dtype", ctypes.c_int)]


# name -> (restype, argtypes); must list every symbol of include/satb200.h
_VP, _I, _LL, _F = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float

# satb_gemm_probe (tests only): epilogue kinds and the parameter block, in the order of include/satb200.h
EPI_STORE32, EPI_STORE16, EPI_HEAD_NORM16, EPI_QKV_ROPE, EPI_SWIGLU, EPI_RESIDUAL = range(6)
EPI_RESIDUAL_LN = 6   # retired (the LayerNorm-fold residual epilogue): refused, and the number is not reused
EPI_STORE32_POS = 7   # store32 plus a [seq_len, N] position-table row (project_in with a positional embedding)
# satb_gemm_probe_qk8 only: the e4m3 QKV epilogues of FP8 self-attention
EPI_QKV_ROPE_E4M3, EPI_HEAD_NORM_E4M3 = 8, 9
# satb_gemm_probe_ff8 only: the GEMMs of the FP8 FF-out option
EPI_SWIGLU_E4M3, EPI_SILU_E4M3, EPI_RESIDUAL_A8 = 13, 14, 15
# satb_t5_gemm_probe only: the T5 encoder's FF-in epilogues
EPI_RELU16, EPI_GEGLU16 = 10, 11
# satb_roberta_linear_probe only: the RoBERTa encoder's FF-in epilogue
EPI_BIAS_GELU16 = 12


class SatbQkE4m3(ctypes.Structure):
    _fields_ = [(n, _VP) for n in ("q8", "k8", "sq", "sk")] + [("heads", _I), ("scale_ld", _I)]


class SatbGemmProbe(ctypes.Structure):
    _fields_ = ([(n, _I) for n in ("epi", "bn", "bf16", "b_static")] + [("out", _VP), ("ld", _I), ("bias", _VP),
                ("act", _I), ("h", _VP), ("gate", _VP)]
                + [(n, _I) for n in ("rows_per_item", "gate_ld", "n_items", "rope_cols", "seq_len", "head_dim", "nf")]
                + [("cos_tab", _VP), ("sin_tab", _VP), ("norm_cols", _I), ("pos_tab", _VP)])


SATB_SAMPLER_STEP_BUFS = 4


# satb_sampler_step: the parameter block of include/satb200.h
class SatbSamplerStep(ctypes.Structure):
    _fields_ = ([("x", _VP), ("y", _VP), ("buf", _VP * SATB_SAMPLER_STEP_BUFS)]
                + [(n, _VP) for n in ("noise", "mask", "init", "renoise", "den", "d", "x_next", "x_in_next")]
                + [("n", _LL), ("L", _I)]
                + [(n, _F) for n in ("c_skip", "c_out", "inv_sigma", "a", "b", "g")] + [("c", _F * SATB_SAMPLER_STEP_BUFS)]
                + [(n, _F) for n in ("s", "c_in_next", "blend_sigma", "blend_thr")])


# satb_attention_probe (tests only): the parameter block of include/satb200.h
class SatbAttentionProbe(ctypes.Structure):
    _fields_ = ([(n, _I) for n in ("B", "H", "Hkv", "Nq", "Nk", "head_dim", "bf16")]
                + [(n, _VP) for n in ("q", "k", "v", "o")]
                + [(n, _LL) for n in ("ldq", "ldk", "ldv", "ldo", "q_bs", "k_bs", "v_bs", "o_bs")]
                + [(n, _I) for n in ("q_cols", "k_cols", "v_cols", "q_col", "k_col", "v_col")])


# satb_oobleck_probe / satb_oobleck_weights (tests only): steps, route bits and the parameter block of include/satb200.h
OOB_DEC_IN, OOB_DEC_UP, OOB_DEC_RES, OOB_DEC_OUT, OOB_ENC_IN, OOB_ENC_RES, OOB_ENC_DOWN, OOB_ENC_OUT = range(8)
OOB_ROUTES = {1: "gemm", 2: "gemm_lean", 4: "fused", 8: "fused_lean", 16: "halo_ncl", 32: "gemm_ncl", 64: "cuda_core"}
# satb_oobleck_create_variant: the blocks' activation
OOB_ACT_SNAKE, OOB_ACT_ELU = 0, 1


class SatbOobleckProbe(ctypes.Structure):
    _fields_ = ([(n, _I) for n in ("step", "block", "unit", "B", "L")]
                + [(n, _VP) for n in ("in_", "raw_in", "raw_out", "out16", "scratch", "out32")]
                + [("lo_off", _LL)] + [(n, _I) for n in ("result_in_scratch", "wrote_raw", "routes")])


SIGNATURES = {
    "satb_last_error": (ctypes.c_char_p, []),
    "satb_abi_version": (_I, []),
    "satb_launch_count": (ctypes.c_ulonglong, []),
    "satb_reset_launch_count": (None, []),
    "satb_add_launch_count": (None, [ctypes.c_ulonglong]),
    "satb_dit_create": (_I, [ctypes.POINTER(SatbDitConfig), ctypes.POINTER(_VP)]),
    "satb_dit_destroy": (None, [_VP]),
    "satb_dit_set_conformer": (_I, [_VP, _I]),
    "satb_dit_set_feedforward": (_I, [_VP, _I, _I, _I, _I]),
    "satb_dit_set_positions": (_I, [_VP, _I, _I, _I]),
    "satb_dit_set_attention_fp8": (_I, [_VP, _I]),
    "satb_dit_set_ff_out_fp8": (_I, [_VP, _I]),
    "satb_dit_load_weight": (_I, [_VP, ctypes.c_char_p, _VP, _LL, _VP]),
    "satb_dit_finalize": (_I, [_VP, _VP]),
    "satb_dit_reserve": (_I, [_VP, _I, _I]),
    "satb_dit_set_prepend_cond": (_I, [_VP, _VP, _I, _I, _VP]),
    "satb_dit_prepare_cond": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "satb_dit_forward": (_I, [_VP, _VP, _VP, _VP, _I, _I, _F, _F, _VP]),
    "satb_dit_forward_debug": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _F, _F, _VP]),
    "satb_dit_group_plan": (_I, [_I, _I, _I, _VP]),
    "satb_dit_group_create": (_I, [_VP, _VP, _I, ctypes.POINTER(_VP)]),
    "satb_dit_group_create_cfg": (_I, [_VP, _VP, _I, ctypes.POINTER(_VP)]),
    "satb_dit_group_destroy": (None, [_VP]),
    "satb_dit_group_forward": (_I, [_VP, _VP, _VP, _VP, _I, _I, _F, _F, _VP]),
    "satb_dit_group_graph_forward": (_I, [_VP, _VP, _VP, _VP, _I, _I, _F, _F, _VP, _VP]),
    "satb_dit_group_graph_reset": (_I, [_VP]),
    "satb_dit_group_graph_stats": (_I, [_VP, ctypes.POINTER(_LL), ctypes.POINTER(_LL), ctypes.POINTER(ctypes.c_ulonglong)]),
    "satb_kv_gather": (_I, [_VP, _VP, _I, _VP, _I, _I, _VP]),
    "satb_dit_profile": (_I, [_VP, _I]),
    "satb_dit_profile_read": (_I, [_VP, _VP, _VP]),
    "satb_snake_beta": (_I, [_VP, _VP, _VP, _VP, _I, _I, _LL, _I, _VP]),
    "satb_sampler_update": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _LL] + [_F] * 8 + [_VP]),
    "satb_vdiffusion_update": (_I, [_VP, _VP, _VP, _VP, _VP, _LL] + [_F] * 5 + [_VP]),
    "satb_sampler_step": (_I, [ctypes.POINTER(SatbSamplerStep), _VP]),
    "satb_layernorm": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "satb_layernorm_fp8": (_I, [_VP, _VP, _VP, _VP, _VP, _LL, _I, _I, _VP, _VP, _I, _I, _VP]),
    "satb_linear_f32out": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "satb_gemm_probe": (_I, [_VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
    "satb_gemm_probe_fp8": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
    "satb_token_conv_probe": (_I, [_VP, _LL, _VP, _I, _I, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
    "satb_dit_pre_probe": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "satb_layernorm_mod": (_I, [_VP, _VP, _VP, _VP, _VP, _LL, _I, _I, _VP, _I, _I, _I, _VP]),
    "satb_fourier_probe": (_I, [_VP, _VP, _VP, _I, _I, _VP]),
    "satb_skinny_linear_probe": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "satb_write_prepend_probe": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "satb_gate_sigmoid_probe": (_I, [_VP, _I, _I, _I, _VP]),
    "satb_dit_post_probe": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _I, _I, _F, _F, _VP]),
    "satb_cast_rows_probe": (_I, [_VP, _VP, _VP, _I, _I, _LL, _LL, _I, _VP]),
    "satb_quant_rows_fp8_probe": (_I, [_VP, _VP, _VP, _VP, _I, _I, _VP]),
    "satb_matmul_f64_probe": (_I, [_VP, _VP, _VP, _I, _I, _I, _VP]),
    "satb_attention": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP]),
    "satb_attention_hd": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "satb_attention_probe": (_I, [ctypes.POINTER(SatbAttentionProbe), _VP]),
    "satb_attention_fp8_vt": (_I, [_VP] * 3 + [_I, _I, _I, _I, _VP]),
    "satb_gemm_probe_qk8": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), ctypes.POINTER(SatbQkE4m3),
                                 _VP]),
    "satb_gemm_probe_ff8": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP, _VP, _VP]),
    "satb_attention_fp8_core": (_I, [_VP] * 7 + [_I, _I, _I, _I, _I, _VP]),
    "satb_conformer_dwconv": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "satb_oobleck_create": (_I, [ctypes.POINTER(SatbOobleckConfig), ctypes.POINTER(_VP)]),
    "satb_oobleck_create_variant": (_I, [ctypes.POINTER(SatbOobleckConfig), _I, _I, ctypes.POINTER(_VP)]),
    "satb_oobleck_destroy": (None, [_VP]),
    "satb_oobleck_load_weight": (_I, [_VP, ctypes.c_char_p, _VP, _LL, _VP]),
    "satb_oobleck_finalize": (_I, [_VP, _VP]),
    "satb_oobleck_decode": (_I, [_VP, _VP, _VP, _I, _I, _VP]),
    "satb_oobleck_encode": (_I, [_VP, _VP, _VP, _I, _LL, _VP]),
    "satb_oobleck_group_plan": (_I, [_I, _I, ctypes.POINTER(SatbOobleckConfig), _I, _VP, _VP, _VP]),
    "satb_oobleck_group_create": (_I, [_VP, _VP, _I, ctypes.POINTER(_VP)]),
    "satb_oobleck_group_destroy": (None, [_VP]),
    "satb_oobleck_group_decode": (_I, [_VP, _VP, _VP, _I, _I, _VP]),
    "satb_oobleck_group_encode": (_I, [_VP, _VP, _VP, _I, _LL, _VP]),
    "satb_oobleck_probe": (_I, [_VP, ctypes.POINTER(SatbOobleckProbe), _VP]),
    "satb_oobleck_weights": (_I, [_VP, ctypes.c_char_p, _VP, ctypes.POINTER(_LL), _VP]),
    "satb_pqmf_create": (_I, [_I, _I, ctypes.POINTER(_VP)]),
    "satb_pqmf_destroy": (None, [_VP]),
    "satb_pqmf_load_filter": (_I, [_VP, _VP, _VP]),
    "satb_pqmf_analysis": (_I, [_VP, _VP, _VP, _I, _I, _LL, _VP]),
    "satb_pqmf_synthesis": (_I, [_VP, _VP, _VP, _I, _I, _I, _VP]),
    "satb_t5_create": (_I, [ctypes.POINTER(SatbT5Config), ctypes.POINTER(_VP)]),
    "satb_t5_destroy": (None, [_VP]),
    "satb_t5_load_weight": (_I, [_VP, ctypes.c_char_p, _VP, _LL, _VP]),
    "satb_t5_set_buckets": (_I, [_VP, _VP, _I]),
    "satb_t5_set_proj_out": (_I, [_VP, _VP, _VP, _I, _VP]),
    "satb_t5_finalize": (_I, [_VP, _VP]),
    "satb_t5_encode": (_I, [_VP, _VP, _VP, _I, _I, _VP, _VP]),
    "satb_t5_rmsnorm_probe": (_I, [_VP, _VP, _VP, _I, _I, _F, _I, _VP]),
    "satb_t5_attention_probe": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP, _VP]),
    "satb_t5_gemm_probe": (_I, [_VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
    "satb_t5_linear_probe": (_I, [_VP, _I, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
    "satb_t5_bias_table": (_I, [_VP, _VP, _VP]),
    "satb_roberta_create": (_I, [ctypes.POINTER(SatbRobertaConfig), ctypes.POINTER(_VP)]),
    "satb_roberta_destroy": (None, [_VP]),
    "satb_roberta_load_weight": (_I, [_VP, ctypes.c_char_p, _VP, _LL, _VP]),
    "satb_roberta_set_proj_out": (_I, [_VP, _VP, _VP, _I, _VP]),
    "satb_roberta_finalize": (_I, [_VP, _VP]),
    "satb_roberta_encode": (_I, [_VP, _VP, _VP, _I, _I, _VP, _VP]),
    "satb_roberta_embed_probe": (_I, [_VP, _I, _I, _VP, _I, _VP, _I, _VP, _VP, _VP, _I, _I, _F, _VP, _VP, _I, _VP]),
    "satb_roberta_layernorm_probe": (_I, [_VP, _VP, _VP, _I, _I, _F, _VP, _VP, _I, _VP]),
    "satb_roberta_attention_probe": (_I, [_VP, _VP, _I, _I, _I, _I, _VP, _VP]),
    "satb_roberta_linear_probe": (_I, [_VP, _VP, _I, _I, _I, ctypes.POINTER(SatbGemmProbe), _VP]),
}


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError(
                f"{LIB_PATH} not found: build it with `python friendly-stable-audio-tools_b200/build.py` "
                "(or __graft_entry__.build()); this package has no non-CUDA fallback")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc):
    if rc != 0:
        msg = lib().satb_last_error()
        raise NativeError(f"satb200 error {rc}: {msg.decode() if msg else '?'}")


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def dev_f32(t, name="tensor"):
    """Validate a CUDA fp32 contiguous tensor and return its device pointer."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise NativeError(f"{name} must be a CUDA tensor: this package runs on the GPU only (no CPU fallback)")
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise NativeError(f"{name} must be contiguous float32")
    return ctypes.c_void_p(t.data_ptr())


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def group_plan(world, n_prepend, L):
    """The token split of a sharded DiT forward (satb_dit_group_plan): token_begin[world + 1] over the n_prepend + L
    tokens of an item; rank r holds tokens token_begin[r] .. token_begin[r + 1] - 1.  Host only."""
    tb = (ctypes.c_int * (world + 1))()
    check(lib().satb_dit_group_plan(int(world), int(n_prepend), int(L), tb))
    return list(tb)


def oobleck_group_plan(world, L, cfg, nearest_upsample=False):
    """The split of a time-sharded Oobleck decode / encode (satb_oobleck_group_plan) for a handle of SatbOobleckConfig
    cfg: (begin[world + 1], [(lo, hi)] * world extended latent ranges, margin in latents).  Host only."""
    begin, ext, m = (ctypes.c_int * (world + 1))(), (ctypes.c_int * (2 * world))(), ctypes.c_int()
    check(lib().satb_oobleck_group_plan(int(world), int(L), ctypes.byref(cfg), int(bool(nearest_upsample)), begin, ext,
                                        ctypes.byref(m)))
    return list(begin), [(ext[2 * r], ext[2 * r + 1]) for r in range(world)], m.value


def launch_count():
    return int(lib().satb_launch_count())
