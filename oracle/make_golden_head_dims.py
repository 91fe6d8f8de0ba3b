"""Generate tests/golden/dit_hd*.npz from the REAL reference DiffusionTransformer: DiTs whose attention head dim
(embed_dim / num_heads) is 128, 96 or 32 instead of 64.

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_head_dims

Same recipe, inputs and keys as ``oracle.make_golden.gen_dit`` (synthetic weights re-derived from the seed, a checksum
of them stored; x, t, cross, glob, neg; the four guidance cases and the last hidden state), with the width, head count
and cond_token_dim of each fixture.  Cross-attention kv heads = cond_token_dim / head dim.  The head-dim-96 model is
384 wide, so it runs 150 latent tokens instead of 200 to keep its file (dominated by hidden_last) as small as the
others; 151 tokens still end in a ragged key tile.
"""
import json
import os

import numpy as np
import torch

from . import dit_oracle as do
from . import ref_shims
from .make_golden import DIT_SMALL, GOLDEN_DIR, _np, weights_checksum

# (file, global_cond_type, DIT_SMALL overrides, seed, latent tokens)
HEAD_DIM_GOLDENS = (
    ("dit_hd128_small.npz", "prepend", dict(embed_dim=256, num_heads=2, cond_token_dim=128), 16, 200),   # 1 kv head
    ("dit_hd96_small.npz", "prepend", dict(embed_dim=384, num_heads=4, cond_token_dim=192), 17, 150),    # 2 kv heads
    ("dit_hd32_small.npz", "prepend", dict(embed_dim=256, num_heads=8, cond_token_dim=128), 18, 200),    # 4 kv heads
    ("dit_hd128_adaln_small.npz", "adaLN", dict(embed_dim=256, num_heads=2, cond_token_dim=128), 19, 200),
)


def gen_dit_head_dim(ref, path, gtype, overrides, seed, L):
    cfg = dict(DIT_SMALL, global_cond_type=gtype, **overrides)
    sd = do.make_dit_weights(cfg, seed=seed)
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
    for name, gtype, overrides, seed, L in HEAD_DIM_GOLDENS:
        path = os.path.join(GOLDEN_DIR, name)
        gen_dit_head_dim(ref, path, gtype, overrides, seed, L)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
