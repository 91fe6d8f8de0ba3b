"""CPU restatement of the DiT forward with the reference's positional options (``ContinuousTransformer`` kwargs
``rotary_pos_emb``, ``use_sinusoidal_emb``, ``use_abs_pos_emb`` / ``abs_pos_emb_max_length``).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Builds on ``oracle/dit_oracle.py`` and leaves it unchanged.  Rotary
off needs nothing new: dit_oracle applies RoPE only when the state dict holds ``transformer.rotary_pos_emb.inv_freq``.
The embeddings (reference models/transformer.py:50-96, 784-785) are restated here: after project_in and the prepend
concat, every row of an item gets the embedding of its position (prepended tokens are positions 0 .., and with
patching positions count patched tokens):

    sinusoidal   cat(sin(p inv_freq), cos(p inv_freq)) * scale,  inv_freq = 10000 ** -(arange(D / 2) / (D / 2)) (fp32)
    absolute     emb.weight[p] * D ** -0.5                          (asserts the length is at most max_seq_len)

The state dict says which: ``transformer.pos_emb.scale`` (sinusoidal; inv_freq is a non-persistent buffer of the
reference, so it is recomputed here with the reference's ops) or ``transformer.pos_emb.emb.weight`` (absolute).

``dit_forward`` / ``dit_inner_forward`` run feedforward_oracle's forward (so conformer blocks and the feed-forward
variants compose) with ``continuous_transformer`` swapped for the one below, the module-attribute swap the other
oracles use.  The add is fp32, as the native path adds the fp32 table to project_in's fp32 output, so operand
rounding applies unchanged.

Pinned against the real reference by tests/golden/dit_pos_*.npz (oracle/make_golden_positions.py).
"""
import torch

from . import dit_oracle as do
from . import feedforward_oracle as fo


def sinusoid_inv_freq(dim, theta=10000):
    """ScaledSinusoidalEmbedding.inv_freq (transformer.py:84-87), fp32."""
    half = dim // 2
    return theta ** -(torch.arange(half).float() / half)


def pos_embedding(sd, n, dim):
    """The [n, dim] embedding of positions 0 .. n-1 of the state dict's variant, or None."""
    pfx = "transformer.pos_emb."
    if (pfx + "scale") in sd:
        scale = sd[pfx + "scale"].float()
        f = torch.einsum("i,j->ij", torch.arange(n, device=scale.device).float(), sinusoid_inv_freq(dim).to(scale.device))
        return torch.cat((f.sin(), f.cos()), dim=-1) * scale
    if (pfx + "emb.weight") in sd:
        w = sd[pfx + "emb.weight"]
        assert n <= w.shape[0], f"sequence length {n} exceeds the absolute embedding's max length {w.shape[0]}"
        return w[:n] * dim ** -0.5
    return None


def continuous_transformer(x, prepend, ctx, global_cond, sd, depth, dim_heads, hidden_states=None, qk_norm=False):
    """dit_oracle.continuous_transformer plus the positional embedding after the prepend concat (transformer.py:770-785)."""
    pfx = "transformer."
    x = do._lin16(x, sd[pfx + "project_in.weight"])
    if prepend is not None:
        x = torch.cat((prepend, x), dim=-2)
    freqs = None
    if (pfx + "rotary_pos_emb.inv_freq") in sd:
        freqs = do.rotary_freqs(x.shape[1], sd[pfx + "rotary_pos_emb.inv_freq"])
    e = pos_embedding(sd, x.shape[1], x.shape[-1])
    if e is not None:
        x = x + e.to(x.dtype)
    for i in range(depth):
        x = do.transformer_block(x, ctx, global_cond, sd, f"{pfx}layers.{i}.", dim_heads, freqs, qk_norm)
        if hidden_states is not None:
            hidden_states.append(x)
    return do._lin16(x, sd[pfx + "project_out.weight"])


class positions:
    """Within this context dit_oracle's forward runs the continuous transformer above."""

    def __enter__(self):
        self.prev = do.continuous_transformer
        do.continuous_transformer = continuous_transformer
        return self

    def __exit__(self, *exc):
        do.continuous_transformer = self.prev


def dit_forward(sd, cfg, *args, **kwargs):
    """feedforward_oracle.dit_forward (models/dit.py:228-364) with the positional options."""
    with positions():
        return fo.dit_forward(sd, cfg, *args, **kwargs)


def dit_inner_forward(sd, cfg, *args, **kwargs):
    """feedforward_oracle.dit_inner_forward (models/dit.py:135-226) with the positional options."""
    with positions():
        return fo.dit_inner_forward(sd, cfg, *args, **kwargs)


# ---------------------------------------------------------------------------
# synthetic weights
# ---------------------------------------------------------------------------

def pos_param_shapes(cfg):
    """The positional entries of the state dict (transformer.py:737-752); the sinusoid's inv_freq is not one."""
    D = cfg["embed_dim"]
    if cfg.get("use_sinusoidal_emb", False):
        return {"transformer.pos_emb.scale": (1,)}
    if cfg.get("use_abs_pos_emb", False):
        return {"transformer.pos_emb.emb.weight": (cfg.get("abs_pos_emb_max_length", 10000), D)}
    return {}


def dit_param_shapes(cfg):
    """feedforward_oracle.dit_param_shapes without the rotary key when rotary is off, plus the embedding's entries."""
    shapes = fo.dit_param_shapes(cfg)
    if not cfg.get("rotary_pos_emb", True):
        del shapes["transformer.rotary_pos_emb.inv_freq"]
    return {**shapes, **pos_param_shapes(cfg)}


def make_dit_weights(cfg, seed=0, std=0.02, dtype=torch.float32):
    """feedforward_oracle.make_dit_weights(cfg, seed) - the very tensors it draws - without the rotary inv_freq when
    rotary is off, plus the embedding's entries from a generator of their own (seed + 7919).  They are drawn large
    enough that the embedding moves the output well past the GPU tolerances: scale ~ U(0.75, 1.25) (16 times the
    reference's init at D = 256), emb.weight ~ N(0, 8^2) (an amplitude of 0.5 at D = 256)."""
    sd = fo.make_dit_weights(cfg, seed=seed, std=std, dtype=dtype)
    if not cfg.get("rotary_pos_emb", True):
        del sd["transformer.rotary_pos_emb.inv_freq"]
    g = torch.Generator().manual_seed(seed + 7919)
    for k, shp in pos_param_shapes(cfg).items():
        v = 0.75 + 0.5 * torch.rand(shp, generator=g) if k.endswith("scale") else 8.0 * torch.randn(shp, generator=g)
        sd[k] = v.to(dtype)
    return sd
