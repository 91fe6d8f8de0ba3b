"""CPU restatement of the DiT forward with conformer blocks (``conformer=True``).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Builds on ``oracle/dit_oracle.py`` and leaves it unchanged: every
function there is used as it is, and only the TransformerBlock is restated here with the conformer branch added
(reference models/transformer.py:557-591, added at :680-681 / :697-698).  ``dit_forward`` / ``dit_inner_forward``
run dit_oracle's forward with this block in place of its own for the duration of the call (the same module-attribute
swap tests/fp8_ref.py uses), so operand_rounding and fp8_ref.fp8_operands apply to the conformer branch too: its
contractions go through ``dit_oracle._lin16``, its stored 16-bit tensors through ``dit_oracle._rnd``.

Pinned against the real reference by tests/golden/dit_conformer*.npz (oracle/make_golden_conformer.py).
"""
import math

import torch
import torch.nn.functional as F

from . import dit_oracle as do

CONFORMER_KERNEL = 17   # depthwise_conv kernel_size (transformer.py:571), padding 8


def conformer_module(x, sd, pfx):
    """models/transformer.py:557-591: in_norm, pointwise_conv (1x1, no bias), GLU (Linear D -> 2D with bias, value =
    first half, SiLU on the gate, :211-235), depthwise_conv (17 taps, groups = D, zero padding 8 over the token axis of
    each item, no bias), mid_norm, SiLU, pointwise_conv_2 (1x1, no bias).

    Under dit_oracle.operand_rounding the two contractions in front of the GLU run as the native path runs them: one
    Linear with W = W_glu W_pw (folded in fp64, then rounded to the operand type), and the GLU output is rounded to the
    operand type it is stored in."""
    a = do.layer_norm(x, sd[pfx + "in_norm.gamma"], sd.get(pfx + "in_norm.beta"))
    w_pw, w_glu, b_glu = sd[pfx + "pointwise_conv.weight"], sd[pfx + "glu.proj.weight"], sd[pfx + "glu.proj.bias"]
    if do._OPERAND_DTYPE is None:
        u = do._lin(F.conv1d(a.transpose(1, 2), w_pw).transpose(1, 2), w_glu, b_glu)
    else:
        u = do._lin16(a, (w_glu.double() @ w_pw[:, :, 0].double()).to(w_glu.dtype), b_glu)
    val, gate = u.chunk(2, dim=-1)
    g = do._rnd(val * F.silu(gate))
    c = F.conv1d(g.transpose(1, 2), sd[pfx + "depthwise_conv.weight"], padding=CONFORMER_KERNEL // 2,
                 groups=g.shape[-1]).transpose(1, 2)
    c = F.silu(do.layer_norm(c, sd[pfx + "mid_norm.gamma"], sd.get(pfx + "mid_norm.beta")))
    return do._lin16(c, sd[pfx + "pointwise_conv_2.weight"][:, :, 0])


def transformer_block(x, ctx, global_cond, sd, pfx, dim_heads, freqs, qk_norm=False):
    """models/transformer.py:656-702 (dit_oracle.transformer_block) with the conformer branch between cross-attention
    and the feed-forward, in both the adaLN and the plain block, without modulation or gate."""
    ssg_key = pfx + "to_scale_shift_gate.1.weight"
    has_cross = (pfx + "cross_attn.to_q.weight") in sd and ctx is not None
    has_conformer = (pfx + "conformer.pointwise_conv.weight") in sd
    if ssg_key in sd and global_cond is not None:
        # adaLN branch, :665-689
        ssg = do._lin(F.silu(global_cond), sd[ssg_key]).unsqueeze(1)
        scale_self, shift_self, gate_self, scale_ff, shift_ff, gate_ff = ssg.chunk(6, dim=-1)
        res = x
        a = do.layer_norm(x, sd[pfx + "pre_norm.gamma"], sd.get(pfx + "pre_norm.beta"))
        a = a * (1 + scale_self) + shift_self
        a = do.self_attention(a, sd, pfx + "self_attn.", dim_heads, freqs, qk_norm)
        x = a * torch.sigmoid(1 - gate_self) + res
        if has_cross:
            a = do.layer_norm(x, sd[pfx + "cross_attend_norm.gamma"], sd.get(pfx + "cross_attend_norm.beta"))
            x = x + do.cross_attention(a, ctx, sd, pfx + "cross_attn.", dim_heads, qk_norm)
        if has_conformer:                                                        # :680-681
            x = x + conformer_module(x, sd, pfx + "conformer.")
        res = x
        a = do.layer_norm(x, sd[pfx + "ff_norm.gamma"], sd.get(pfx + "ff_norm.beta"))
        a = a * (1 + scale_ff) + shift_ff
        a = do.feed_forward(a, sd, pfx + "ff.")
        x = a * torch.sigmoid(1 - gate_ff) + res
    else:
        # plain branch, :691-700
        a = do.layer_norm(x, sd[pfx + "pre_norm.gamma"], sd.get(pfx + "pre_norm.beta"))
        x = x + do.self_attention(a, sd, pfx + "self_attn.", dim_heads, freqs, qk_norm)
        if has_cross:
            a = do.layer_norm(x, sd[pfx + "cross_attend_norm.gamma"], sd.get(pfx + "cross_attend_norm.beta"))
            x = x + do.cross_attention(a, ctx, sd, pfx + "cross_attn.", dim_heads, qk_norm)
        if has_conformer:                                                        # :697-698
            x = x + conformer_module(x, sd, pfx + "conformer.")
        a = do.layer_norm(x, sd[pfx + "ff_norm.gamma"], sd.get(pfx + "ff_norm.beta"))
        x = x + do.feed_forward(a, sd, pfx + "ff.")
    return x


class conformer_blocks:
    """Within this context dit_oracle's forward runs the block above (identical to its own for layers without
    conformer keys)."""

    def __enter__(self):
        self.prev = do.transformer_block
        do.transformer_block = transformer_block
        return self

    def __exit__(self, *exc):
        do.transformer_block = self.prev


def dit_forward(sd, cfg, *args, **kwargs):
    """dit_oracle.dit_forward (models/dit.py:228-364) with conformer blocks."""
    with conformer_blocks():
        return do.dit_forward(sd, cfg, *args, **kwargs)


def dit_inner_forward(sd, cfg, *args, **kwargs):
    """dit_oracle.dit_inner_forward (models/dit.py:135-226) with conformer blocks."""
    with conformer_blocks():
        return do.dit_inner_forward(sd, cfg, *args, **kwargs)


# ---------------------------------------------------------------------------
# synthetic weights
# ---------------------------------------------------------------------------

def conformer_param_shapes(cfg):
    """The nine state-dict entries of every layer's ConformerModule (transformer.py:557-574,645); empty unless
    ``cfg["conformer"]``."""
    if not cfg.get("conformer", False):
        return {}
    D = cfg["embed_dim"]
    shapes = {}
    for i in range(cfg["depth"]):
        c = f"transformer.layers.{i}.conformer."
        shapes[c + "in_norm.gamma"] = (D,)
        shapes[c + "in_norm.beta"] = (D,)
        shapes[c + "pointwise_conv.weight"] = (D, D, 1)
        shapes[c + "glu.proj.weight"] = (2 * D, D)
        shapes[c + "glu.proj.bias"] = (2 * D,)
        shapes[c + "depthwise_conv.weight"] = (D, 1, CONFORMER_KERNEL)
        shapes[c + "mid_norm.gamma"] = (D,)
        shapes[c + "mid_norm.beta"] = (D,)
        shapes[c + "pointwise_conv_2.weight"] = (D, D, 1)
    return shapes


def dit_param_shapes(cfg):
    """dit_oracle.dit_param_shapes plus the conformer entries."""
    return {**do.dit_param_shapes(cfg), **conformer_param_shapes(cfg)}


def make_dit_weights(cfg, seed=0, std=0.02, dtype=torch.float32):
    """dit_oracle.make_dit_weights(cfg, seed) - for every config, the very tensors it draws - plus, for conformer
    configs, the conformer tensors from a generator of their own (seed + 7919): LN gamma ~ 1 + N(0, 0.1), beta = 0,
    the GLU bias ~ N(0, std); pointwise_conv, glu.proj and depthwise_conv with unit gain (std 1 / sqrt(fan_in)), so that
    mid_norm sees a signal well above its eps; pointwise_conv_2 ~ N(0, std) (the reference does not zero-init it)."""
    sd = do.make_dit_weights(cfg, seed=seed, std=std, dtype=dtype)
    g = torch.Generator().manual_seed(seed + 7919)
    for k, shp in conformer_param_shapes(cfg).items():
        if k.endswith(".gamma"):
            v = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".beta"):
            v = torch.zeros(shp)
        elif k.endswith("bias"):
            v = torch.randn(shp, generator=g) * std
        elif k.endswith("pointwise_conv_2.weight"):
            v = torch.randn(shp, generator=g) * std
        else:
            fan_in = shp[1] * (shp[2] if len(shp) == 3 else 1)
            v = torch.randn(shp, generator=g) / math.sqrt(fan_in)
        sd[k] = v.to(dtype)
    return sd
