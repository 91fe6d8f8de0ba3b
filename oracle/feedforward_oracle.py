"""CPU restatement of the DiT forward with the reference's other feed-forward options (``ff_kwargs``).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Builds on ``oracle/dit_oracle.py`` and leaves it unchanged: only the
feed-forward is restated here (reference models/transformer.py:211-287), for every row of

    glu    use_conv   FF-in                                           FF-out
    True   False      ff.0.proj  Linear(dim, 2 inner), biased, SwiGLU    ff.2  Linear(inner, dim)
    True   True       ff.0.proj  the same Linear GLU (:260)               ff.2  Conv1d(inner, dim, k, padding k // 2)
    False  False      ff.0.1     Linear(dim, inner), then SiLU            ff.2  Linear(inner, dim)
    False  True       ff.0.1     Conv1d(dim, inner, k), then SiLU         ff.2  Conv1d(inner, dim, k)

(biases, other than the GLU's, unless ``no_bias``).  The convolutions run over the token axis of each item, zero-padded
at its ends: prepended tokens are part of the sequence, and every CFG row is its own item.

``dit_forward`` / ``dit_inner_forward`` run dit_oracle's forward with this feed-forward in place of its own (the
module-attribute swap that conformer_oracle.py and tests/fp8_ref.py use), inside ``conformer_oracle.conformer_blocks``
so that conformer models compose.  In fp32 the convolutions follow the reference (F.conv1d); under operand rounding
every contraction goes through ``dit_oracle._lin16`` (a convolution as one Linear over the k shifted copies of its
input) and stored 16-bit tensors through ``dit_oracle._rnd``, so ``operand_rounding`` and ``fp8_ref.fp8_operands``
apply.

Pinned against the real reference by tests/golden/dit_ff_*.npz (oracle/make_golden_feedforward.py).
"""
import torch
import torch.nn.functional as F

from . import conformer_oracle as co
from . import dit_oracle as do

DEFAULT_FF = dict(mult=4, no_bias=False, glu=True, use_conv=False, conv_kernel_size=3)


def ff_options(cfg):
    """The FeedForward kwargs of a DiT config (``ff_kwargs``) with the reference's defaults filled in."""
    return {**DEFAULT_FF, **cfg.get("ff_kwargs", {})}


def inner_dim(cfg):
    """transformer.py:251: Python truncation of the float product."""
    return int(cfg["embed_dim"] * ff_options(cfg)["mult"])


def padded_inner(inner):
    """The stored inner width of the native path: the next multiple of 64 (zero rows / columns; exact)."""
    return (inner + 63) // 64 * 64


def token_conv(x, w, b=None):
    """Conv1d over the token axis of x [B, N, Cin] with w [Cout, Cin, k], padding k // 2 (zeros at each item's ends).
    In fp32 as the reference computes it (F.conv1d); under operand_rounding as one Linear over the k shifted copies of
    x, out[:, l] = sum_t x[:, l + t - k // 2] W[:, :, t]^T (+ b), so that the operand emulation applies."""
    k, n = w.shape[-1], x.shape[1]
    if do._OPERAND_DTYPE is None:
        return F.conv1d(x.transpose(1, 2), w, b, padding=k // 2).transpose(1, 2)
    xp = F.pad(x, (0, 0, k // 2, k // 2))
    xu = torch.cat([xp[:, t:t + n] for t in range(k)], dim=-1)              # [B, N, k Cin], tap-major
    return do._lin16(xu, w.permute(0, 2, 1).reshape(w.shape[0], -1), b)


def _layer(x, sd, key):
    w = sd[key + ".weight"]
    b = sd.get(key + ".bias")
    return token_conv(x, w, b) if w.dim() == 3 else do._lin16(x, w, b)


def feed_forward(x, sd, pfx):
    """transformer.py:238-287 for every option (see the module docstring); the variant is read off the keys."""
    if (pfx + "ff.0.proj.weight") in sd:                                      # GLU (:211-235, :259-260)
        u = do._lin16(x, sd[pfx + "ff.0.proj.weight"], sd[pfx + "ff.0.proj.bias"])
        val, gate = u.chunk(2, dim=-1)
        m = do._rnd(val * F.silu(gate))
    else:                                                                     # :262-268
        m = do._rnd(F.silu(_layer(x, sd, pfx + "ff.0.1")))
    return _layer(m, sd, pfx + "ff.2")


class feedforward_variants:
    """Within this context dit_oracle's forward (and conformer_oracle's block) run the feed-forward above."""

    def __enter__(self):
        self.prev = do.feed_forward
        do.feed_forward = feed_forward
        return self

    def __exit__(self, *exc):
        do.feed_forward = self.prev


def dit_forward(sd, cfg, *args, **kwargs):
    """dit_oracle.dit_forward (models/dit.py:228-364) with any feed-forward variant and conformer blocks."""
    with feedforward_variants(), co.conformer_blocks():
        return do.dit_forward(sd, cfg, *args, **kwargs)


def dit_inner_forward(sd, cfg, *args, **kwargs):
    """dit_oracle.dit_inner_forward (models/dit.py:135-226) with any feed-forward variant and conformer blocks."""
    with feedforward_variants(), co.conformer_blocks():
        return do.dit_inner_forward(sd, cfg, *args, **kwargs)


# ---------------------------------------------------------------------------
# synthetic weights
# ---------------------------------------------------------------------------

def ff_param_shapes(cfg):
    """The feed-forward entries of every layer (transformer.py:258-284)."""
    o, D, inner = ff_options(cfg), cfg["embed_dim"], inner_dim(cfg)
    k = o["conv_kernel_size"]
    tail = (k,) if o["use_conv"] else ()
    shapes = {}
    for i in range(cfg["depth"]):
        p = f"transformer.layers.{i}.ff.ff."
        if o["glu"]:
            shapes[p + "0.proj.weight"] = (2 * inner, D)
            shapes[p + "0.proj.bias"] = (2 * inner,)
        else:
            shapes[p + "0.1.weight"] = (inner, D) + tail
            if not o["no_bias"]:
                shapes[p + "0.1.bias"] = (inner,)
        shapes[p + "2.weight"] = (D, inner) + tail
        if not o["no_bias"]:
            shapes[p + "2.bias"] = (D,)
    return shapes


def _without_ff(shapes):
    return {k: v for k, v in shapes.items() if ".ff.ff." not in k}


def dit_param_shapes(cfg):
    """conformer_oracle.dit_param_shapes with the feed-forward entries of the config's variant."""
    return {**_without_ff(co.dit_param_shapes(cfg)), **ff_param_shapes(cfg)}


def make_dit_weights(cfg, seed=0, std=0.02, dtype=torch.float32):
    """conformer_oracle.make_dit_weights(cfg, seed) - for every config the very tensors it draws - with the
    feed-forward entries of a non-default variant replaced by tensors from a generator of their own (seed + 104729):
    biases and FF-in weights ~ N(0, std), as dit_oracle draws the default's; FF-out weights ~ N(0, std^2 / k) (k taps;
    1 for a Linear), so a convolutional FF-out adds a branch of the Linear's size (re-randomised: the reference
    zero-inits them).  A config without ff_kwargs gets conformer_oracle's weights."""
    sd = co.make_dit_weights(cfg, seed=seed, std=std, dtype=dtype)
    if not cfg.get("ff_kwargs"):
        return sd
    sd = _without_ff(sd)
    g = torch.Generator().manual_seed(seed + 104729)
    for k, shp in ff_param_shapes(cfg).items():
        if k.endswith("bias") or ".ff.ff.0." in k:
            v = torch.randn(shp, generator=g) * std
        else:
            v = torch.randn(shp, generator=g) * (std / (shp[2] if len(shp) == 3 else 1) ** 0.5)
        sd[k] = v.to(dtype)
    return sd
