"""Generate tests/golden/dit_ff_*.npz from the REAL reference DiffusionTransformer: DiTs built with the reference's
other feed-forward options (``ff_kwargs``: mult, no_bias, glu, use_conv, conv_kernel_size; reference
models/transformer.py:211-287).

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_feedforward

Same inputs and keys as ``oracle.make_golden_head_dims`` (x, t, cross, glob, neg; the four guidance cases and the
last hidden state; a checksum of the weights), with the synthetic weights of ``oracle.feedforward_oracle``, plus the
reference model's state-dict key / shape list ("keys", JSON) and, for the prepend-conditioning fixture, the prepend
tokens ("prepend", passed to every call).  The token counts are not multiples of the GEMM row tile (128), so the last
m-tile of every item is partial.
"""
import json
import os

import numpy as np
import torch

from . import feedforward_oracle as fo
from . import ref_shims
from .make_golden import DIT_SMALL, GOLDEN_DIR, _np, weights_checksum

# (file, global_cond_type, DIT_SMALL overrides, seed, latent tokens, prepend-conditioning tokens)
FF_GOLDENS = (
    # SwiGLU, inner int(256 * 8/3) = 682: stored padded to 704                                        201 tokens
    ("dit_ff_mult83_small.npz", "prepend", dict(ff_kwargs=dict(mult=8 / 3)), 60, 200, 0),
    # SwiGLU FF-in, Conv1d k 3 FF-out, no biases but the GLU's; 3 prepend-conditioning tokens         194 tokens
    ("dit_ff_glu_conv3_nobias_small.npz", "prepend",
     dict(prepend_cond_dim=96, ff_kwargs=dict(use_conv=True, conv_kernel_size=3, no_bias=True)), 61, 190, 3),
    # Conv1d k 5 + SiLU, Conv1d k 5; adaLN; head dim 128                                              203 tokens
    ("dit_ff_conv5_adaln_hd128_small.npz", "adaLN",
     dict(embed_dim=256, num_heads=2, cond_token_dim=128, ff_kwargs=dict(glu=False, use_conv=True, conv_kernel_size=5)),
     62, 203, 0),
    # Linear + SiLU, Linear, bias-free, mult 2; head dim 32                                           201 tokens
    ("dit_ff_plain_nobias_hd32_small.npz", "prepend",
     dict(embed_dim=256, num_heads=8, cond_token_dim=128, ff_kwargs=dict(glu=False, no_bias=True, mult=2)), 63, 200, 0),
    # conformer blocks + SwiGLU FF-in, Conv1d k 3 FF-out                                              151 tokens
    ("dit_ff_conformer_conv3_small.npz", "prepend",
     dict(conformer=True, ff_kwargs=dict(use_conv=True, conv_kernel_size=3)), 64, 150, 0),
)


def gen_dit_ff(ref, path, gtype, overrides, seed, L, n_prepend):
    cfg = dict(DIT_SMALL, global_cond_type=gtype, **overrides)
    sd = fo.make_dit_weights(cfg, seed=seed)
    m = ref.dit.DiffusionTransformer(**cfg).eval()
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(100 + seed)
    B, M = 2, 10
    x = torch.randn(B, cfg["io_channels"], L, generator=g)
    t = torch.rand(B, generator=g)
    c = torch.randn(B, M, cfg["cond_token_dim"], generator=g)
    ge = torch.randn(B, cfg["global_cond_dim"], generator=g)
    neg = torch.randn(B, M, cfg["cond_token_dim"], generator=g)
    keys = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    out = {"cfg": json.dumps(cfg), "seed": seed, "wsum": weights_checksum(sd), "keys": json.dumps(keys),
           "x": _np(x), "t": _np(t), "cross": _np(c), "glob": _np(ge), "neg": _np(neg)}
    kw = dict(cross_attn_cond=c, global_embed=ge)
    if n_prepend:
        pc = torch.randn(B, n_prepend, cfg["prepend_cond_dim"], generator=g)
        out["prepend"] = _np(pc)
        kw.update(prepend_cond=pc, prepend_cond_mask=torch.ones(B, n_prepend, dtype=torch.bool))
    with torch.no_grad():
        out["y_nocfg"] = _np(m(x, t, cfg_scale=1.0, **kw))
        out["y_cfg7"] = _np(m(x, t, cfg_scale=7.0, **kw))
        out["y_cfg4_phi"] = _np(m(x, t, cfg_scale=4.0, scale_phi=0.7, **kw))
        out["y_neg3"] = _np(m(x, t, negative_cross_attn_cond=neg, cfg_scale=3.0, **kw))
        y, info = m(x, t, cfg_scale=1.0, return_info=True, **kw)
        out["hidden_last"] = _np(info["hidden_states"][-1])
    np.savez_compressed(path, **out)


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    for name, gtype, overrides, seed, L, n_prepend in FF_GOLDENS:
        path = os.path.join(GOLDEN_DIR, name)
        gen_dit_ff(ref, path, gtype, overrides, seed, L, n_prepend)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
