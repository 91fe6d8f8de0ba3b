"""Generate tests/golden/dit_conformer*.npz from the REAL reference DiffusionTransformer: DiTs built with
``conformer=True``, whose every TransformerBlock adds the ConformerModule branch (reference
models/transformer.py:557-591,680-681,697-698).

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_conformer

Same inputs and keys as ``oracle.make_golden_head_dims`` (x, t, cross, glob, neg; the four guidance cases and the
last hidden state; a checksum of the weights), with the synthetic weights of ``oracle.conformer_oracle``.  The token
counts (latents + prepended token) are multiples of neither the GEMM row tile (128) nor the depthwise-convolution chunk
(12).
"""
import json
import os

import numpy as np
import torch

from . import conformer_oracle as co
from . import ref_shims
from .make_golden import DIT_SMALL, GOLDEN_DIR, _np, weights_checksum

# (file, global_cond_type, DIT_SMALL overrides, seed, latent tokens)
CONFORMER_GOLDENS = (
    ("dit_conformer_small.npz", "prepend", dict(conformer=True), 40, 200),                  # 201 tokens
    ("dit_conformer_adaln_small.npz", "adaLN", dict(conformer=True), 41, 203),              # 203 tokens
    ("dit_conformer_hd128_small.npz", "prepend", dict(conformer=True, embed_dim=256, num_heads=2,
                                                      cond_token_dim=128), 42, 150),        # 151 tokens
)


def gen_dit_conformer(ref, path, gtype, overrides, seed, L):
    cfg = dict(DIT_SMALL, global_cond_type=gtype, **overrides)
    sd = co.make_dit_weights(cfg, seed=seed)
    m = ref.dit.DiffusionTransformer(**cfg).eval()
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(100 + seed)
    B, M = 2, 10
    x = torch.randn(B, cfg["io_channels"], L, generator=g)
    t = torch.rand(B, generator=g)
    c = torch.randn(B, M, cfg["cond_token_dim"], generator=g)
    ge = torch.randn(B, cfg["global_cond_dim"], generator=g)
    neg = torch.randn(B, M, cfg["cond_token_dim"], generator=g)
    out = {"cfg": json.dumps(cfg), "seed": seed, "wsum": weights_checksum(sd),
           "x": _np(x), "t": _np(t), "cross": _np(c), "glob": _np(ge), "neg": _np(neg)}
    with torch.no_grad():
        out["y_nocfg"] = _np(m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=1.0))
        out["y_cfg7"] = _np(m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0))
        out["y_cfg4_phi"] = _np(m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=4.0, scale_phi=0.7))
        out["y_neg3"] = _np(m(x, t, cross_attn_cond=c, global_embed=ge, negative_cross_attn_cond=neg, cfg_scale=3.0))
        y, info = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=1.0, return_info=True)
        out["hidden_last"] = _np(info["hidden_states"][-1])
    np.savez_compressed(path, **out)


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    for name, gtype, overrides, seed, L in CONFORMER_GOLDENS:
        path = os.path.join(GOLDEN_DIR, name)
        gen_dit_conformer(ref, path, gtype, overrides, seed, L)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
