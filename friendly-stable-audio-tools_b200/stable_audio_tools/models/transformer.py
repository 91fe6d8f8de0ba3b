"""Parameter containers for the continuous transformer of the DiT.

These classes reproduce the *interface* of reference ``models/transformer.py``
(class names, constructor kwargs, state-dict keys - SURVEY.md 3.3) so reference
checkpoints and JSON configs load unchanged.  They hold ``nn.Parameter``s only:
the arithmetic of ``ContinuousTransformer.forward`` (transformer.py:764-809) is
executed by ``libsatb200.so`` from ``DiffusionTransformer`` (models/dit.py here),
so calling ``forward`` on an inner container raises instead of silently running
eager PyTorch.
"""
import typing as tp

import torch
from torch import nn


# Attention head widths the native attention kernel and RoPE epilogue are built for (csrc/attention_tc.cu, gemm.cuh).
SUPPORTED_HEAD_DIMS = (32, 64, 96, 128)
# Widest model whose conformer branch the native depthwise-convolution kernel runs (csrc/conformer.cu).
CONFORMER_MAX_DIM = 1536


def check_head_dim(dim_heads, qk_norm=False):
    """Raises NotImplementedError for a head dim the native path does not run (before any CUDA call)."""
    if dim_heads not in SUPPORTED_HEAD_DIMS:
        raise NotImplementedError(f"attention head dim {dim_heads} is not on the native hot path "
                                  f"(supported head dims: {', '.join(map(str, SUPPORTED_HEAD_DIMS))})")
    if qk_norm and dim_heads != 64:
        raise NotImplementedError(f"qk_norm is on the native hot path for head dim 64 only (got {dim_heads})")


class _FusedModule(nn.Module):
    """A module whose math is part of a fused native kernel sequence."""

    def forward(self, *args, **kwargs):
        raise RuntimeError(
            f"{type(self).__name__} is a parameter container: its arithmetic is fused into the native "
            "DiffusionTransformer forward (libsatb200.so); call the enclosing DiffusionTransformer instead")


class RotaryEmbedding(_FusedModule):
    """Holds ``inv_freq`` (reference transformer.py:100-128). xpos / interpolation are not supported."""

    def __init__(self, dim, use_xpos=False, scale_base=512, interpolation_factor=1.0, base=10000,
                 base_rescale_factor=1.0):
        super().__init__()
        if use_xpos or interpolation_factor != 1.0:
            raise NotImplementedError("xpos / interpolated rotary embeddings are outside the native hot path")
        base = base * base_rescale_factor ** (dim / (dim - 2))
        self.register_buffer("inv_freq", 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim)))
        self.register_buffer("scale", None)
        self.dim = dim


class ScaledSinusoidalEmbedding(_FusedModule):
    """Reference transformer.py:74-96: ``scale`` (a Parameter [1], dim ** -0.5 at init) and ``inv_freq`` (a
    non-persistent buffer [dim / 2]: not in the state dict, so DiffusionTransformer hands it to the native handle
    itself).  The embedding of position p is cat(sin(p inv_freq), cos(p inv_freq)) * scale."""

    def __init__(self, dim, theta=10000):
        super().__init__()
        assert (dim % 2) == 0, 'dimension must be divisible by 2'
        self.scale = nn.Parameter(torch.ones(1) * dim ** -0.5)
        half = dim // 2
        self.register_buffer("inv_freq", theta ** -(torch.arange(half).float() / half), persistent=False)


class AbsolutePositionalEmbedding(_FusedModule):
    """Reference transformer.py:50-71: ``emb`` = nn.Embedding(max_seq_len, dim); position p adds emb.weight[p] *
    dim ** -0.5.  Sequences longer than max_seq_len (prepended tokens included) fail its assertion."""

    def __init__(self, dim, max_seq_len):
        super().__init__()
        self.scale = dim ** -0.5
        self.max_seq_len = max_seq_len
        self.emb = nn.Embedding(max_seq_len, dim)


class LayerNorm(_FusedModule):
    """gamma (parameter, or buffer when ``fix_scale``) and beta (buffer unless ``bias``)."""

    def __init__(self, dim, bias=False, fix_scale=False):
        super().__init__()
        if fix_scale:
            self.register_buffer("gamma", torch.ones(dim))
        else:
            self.gamma = nn.Parameter(torch.ones(dim))
        if bias:
            self.beta = nn.Parameter(torch.zeros(dim))
        else:
            self.register_buffer("beta", torch.zeros(dim))


class GLU(_FusedModule):
    """``proj``: Linear(dim_in, 2 * dim_out); value = first half, gate = second half (SiLU)."""

    def __init__(self, dim_in, dim_out, activation=None, use_conv=False, conv_kernel_size=3):
        super().__init__()
        if use_conv:
            raise NotImplementedError("convolutional GLU is outside the native hot path")
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(_FusedModule):
    """Reference transformer.py:238-287, every option but ``dim_out != dim``.  Keys: ``ff.0.proj.{weight,bias}`` (GLU,
    the default SwiGLU: Linear(dim, 2 inner), always biased) or ``ff.0.1.{weight,bias}`` (``glu=False``: Linear, or
    Conv1d with ``use_conv``, then SiLU); ``ff.2.{weight,bias}`` (Linear, or Conv1d with ``use_conv``); no biases but the
    GLU's with ``no_bias``.  inner = int(dim * mult).  The ``Rearrange`` modules of the reference have no parameters and
    are ``nn.Identity`` here.  Natively (``satb_dit_set_feedforward``) the convolutions run over each item's tokens as a
    k-tap GEMM, with 16-bit operands in every ``operand_dtype``."""

    def __init__(self, dim, dim_out=None, mult=4, no_bias=False, glu=True, use_conv=False, conv_kernel_size=3,
                 zero_init_output=True):
        super().__init__()
        if dim_out not in (None, dim):
            # the reference builds it, then fails at the residual add (transformer.py:692-700)
            raise NotImplementedError(f"a feed-forward with dim_out {dim_out} != dim {dim} cannot be added to the "
                                      "residual stream")
        if use_conv and (conv_kernel_size < 1 or conv_kernel_size % 2 == 0):
            # padding k // 2 keeps the length only for odd k: an even k gives L + 1 positions
            raise NotImplementedError(f"conv_kernel_size must be odd and positive (got {conv_kernel_size})")
        inner = int(dim * mult)
        if inner < 1:
            raise NotImplementedError(f"feed-forward inner dim int({dim} * {mult}) = {inner} must be >= 1")
        self.inner_dim, self.glu, self.bias = inner, bool(glu), not no_bias
        self.conv_kernel_size = conv_kernel_size if use_conv else 0
        conv = lambda i, o: nn.Conv1d(i, o, conv_kernel_size, padding=conv_kernel_size // 2, bias=not no_bias)
        if glu:
            linear_in = GLU(dim, inner)                 # the reference builds GLU without use_conv (:260)
        else:
            linear_in = nn.Sequential(nn.Identity(), conv(dim, inner) if use_conv else nn.Linear(dim, inner, bias=not no_bias),
                                      nn.Identity(), nn.SiLU())
        linear_out = conv(inner, dim) if use_conv else nn.Linear(inner, dim, bias=not no_bias)
        if zero_init_output:
            nn.init.zeros_(linear_out.weight)
            if not no_bias:
                nn.init.zeros_(linear_out.bias)
        self.ff = nn.Sequential(linear_in, nn.Identity(), linear_out, nn.Identity())

    def native_spec(self):
        """The satb_dit_set_feedforward arguments: (inner_dim, glu, conv_kernel_size, bias)."""
        return (self.inner_dim, int(self.glu), self.conv_kernel_size, int(self.bias))


class Attention(_FusedModule):
    """Fused ``to_qkv`` for self-attention, ``to_q`` + ``to_kv`` when a context dim is given."""

    def __init__(self, dim, dim_heads=64, dim_context=None, causal=False, zero_init_output=True, qk_norm=False,
                 natten_kernel_size=None):
        super().__init__()
        if causal or natten_kernel_size:
            raise NotImplementedError("causal / neighbourhood attention are outside the native hot path")
        check_head_dim(dim_heads, qk_norm)
        self.dim, self.dim_heads = dim, dim_heads
        self.qk_norm = bool(qk_norm)      # cosine-similarity attention (reference transformer.py:433-436)
        dim_kv = dim_context if dim_context else dim
        self.num_heads = dim // dim_heads
        self.kv_heads = dim_kv // dim_heads
        if dim_context:
            self.to_q = nn.Linear(dim, dim, bias=False)
            self.to_kv = nn.Linear(dim_kv, dim_kv * 2, bias=False)
        else:
            self.to_qkv = nn.Linear(dim, dim * 3, bias=False)
        self.to_out = nn.Linear(dim, dim, bias=False)
        if zero_init_output:
            nn.init.zeros_(self.to_out.weight)


class ConformerModule(_FusedModule):
    """Reference transformer.py:557-591: in_norm -> pointwise_conv (1x1) -> GLU (SiLU gate) -> depthwise_conv (17 taps,
    zero padding 8, over the token axis) -> mid_norm -> SiLU -> pointwise_conv_2 (1x1).  Natively, pointwise_conv is
    folded into glu.proj (one GEMM) and the depthwise convolution, mid_norm and SiLU are one kernel
    (csrc/conformer.cu); its GEMMs take 16-bit operands in every operand_dtype, fp16 in the "fp8" mode."""

    def __init__(self, dim, norm_kwargs={}):
        super().__init__()
        if dim > CONFORMER_MAX_DIM:
            raise NotImplementedError(f"conformer blocks are on the native hot path up to dim {CONFORMER_MAX_DIM} "
                                      f"(got {dim})")
        self.dim = dim
        self.in_norm = LayerNorm(dim, **norm_kwargs)
        self.pointwise_conv = nn.Conv1d(dim, dim, kernel_size=1, bias=False)
        self.glu = GLU(dim, dim, nn.SiLU())
        self.depthwise_conv = nn.Conv1d(dim, dim, kernel_size=17, groups=dim, padding=8, bias=False)
        self.mid_norm = LayerNorm(dim, **norm_kwargs)
        self.swish = nn.SiLU()
        self.pointwise_conv_2 = nn.Conv1d(dim, dim, kernel_size=1, bias=False)


class TransformerBlock(_FusedModule):
    def __init__(self, dim, dim_heads=64, cross_attend=False, dim_context=None, global_cond_dim=None, causal=False,
                 zero_init_branch_outputs=True, conformer=False, layer_ix=-1, remove_norms=False, attn_kwargs={},
                 ff_kwargs={}, norm_kwargs={}):
        super().__init__()
        if remove_norms:
            raise NotImplementedError("norm-free blocks are outside the native hot path")
        self.dim, self.dim_heads = dim, dim_heads
        self.cross_attend, self.dim_context = cross_attend, dim_context
        self.global_cond_dim, self.layer_ix = global_cond_dim, layer_ix
        self.pre_norm = LayerNorm(dim, **norm_kwargs)
        self.self_attn = Attention(dim, dim_heads=dim_heads, causal=causal,
                                   zero_init_output=zero_init_branch_outputs, **attn_kwargs)
        if cross_attend:
            self.cross_attend_norm = LayerNorm(dim, **norm_kwargs)
            self.cross_attn = Attention(dim, dim_heads=dim_heads, dim_context=dim_context, causal=causal,
                                        zero_init_output=zero_init_branch_outputs, **attn_kwargs)
        self.ff_norm = LayerNorm(dim, **norm_kwargs)
        self.ff = FeedForward(dim, zero_init_output=zero_init_branch_outputs, **ff_kwargs)
        # x = x + conformer(x) between cross-attention and the feed-forward (reference transformer.py:680-681,697-698)
        self.conformer = ConformerModule(dim, norm_kwargs=norm_kwargs) if conformer else None
        if global_cond_dim:
            self.to_scale_shift_gate = nn.Sequential(nn.SiLU(), nn.Linear(global_cond_dim, dim * 6, bias=False))
            nn.init.zeros_(self.to_scale_shift_gate[1].weight)


class ContinuousTransformer(_FusedModule):
    """Reference transformer.py:705-809 without ``causal``.  Positions: rotary (``rotary_pos_emb``) and / or one
    embedding added to the residual stream (``use_sinusoidal_emb`` or ``use_abs_pos_emb``)."""

    def __init__(self, dim, depth, *, dim_in=None, dim_out=None, dim_heads=64, cross_attend=False,
                 cond_token_dim=None, global_cond_dim=None, causal=False, rotary_pos_emb=True,
                 zero_init_branch_outputs=True, conformer=False, use_sinusoidal_emb=False, use_abs_pos_emb=False,
                 abs_pos_emb_max_length=10000, **kwargs):
        super().__init__()
        assert not (use_sinusoidal_emb and use_abs_pos_emb), \
            "Can't select both of sinusoidal/abs positional embedding type."
        if causal:
            raise NotImplementedError("causal attention is outside the native hot path")
        self.dim, self.depth = dim, depth
        self.project_in = nn.Linear(dim_in, dim, bias=False) if dim_in else nn.Identity()
        self.project_out = nn.Linear(dim, dim_out, bias=False) if dim_out else nn.Identity()
        self.rotary_pos_emb = RotaryEmbedding(max(dim_heads // 2, 32)) if rotary_pos_emb else None
        # added to every row after the prepend concat (transformer.py:770-785); natively in project_in's epilogue
        self.pos_type, self.pos_emb = None, None
        if use_sinusoidal_emb:
            self.pos_type, self.pos_emb = "sinusoidal", ScaledSinusoidalEmbedding(dim)
        elif use_abs_pos_emb:
            self.pos_type, self.pos_emb = "abs", AbsolutePositionalEmbedding(dim, abs_pos_emb_max_length)
        self.layers = nn.ModuleList([
            TransformerBlock(dim, dim_heads=dim_heads, cross_attend=cross_attend, dim_context=cond_token_dim,
                             global_cond_dim=global_cond_dim, causal=causal,
                             zero_init_branch_outputs=zero_init_branch_outputs, conformer=conformer, layer_ix=i,
                             **kwargs)
            for i in range(depth)])
