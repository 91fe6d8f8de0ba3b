"""Generate tests/golden/dit_width_*.npz from the REAL reference DiffusionTransformer: DiTs whose channel widths are not
multiples of the GEMM alignment (io_channels * patch_size not a multiple of 32, (io + input_concat_dim) * patch_size
not a multiple of 8): an inpainting DiT on 64-channel latents (input_concat_dim 65 = 1 mask channel + 64 masked latent
channels, reference training/diffusion.py:680-755), a 16-channel DiT (PQMF mono x 16 bands), raw stereo-ish audio with
patch_size 4, a single channel, and 40 channels with conformer blocks.

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_widths

Same inputs and keys as ``oracle.make_golden_positions`` (x, t, cross, glob, neg; the four guidance cases and the last
hidden state; a checksum of the weights; the reference's state-dict key / shape list), with the synthetic weights of
``oracle.positions_oracle`` (which composes the conformer and feed-forward oracles), plus "concat" (the input-concat
conditioning, when the model has one) and "y_noconcat": the conditional output with that input zeroed, which shows that
the concat channels move the result.  The token counts are not multiples of the GEMM row tile (128).

With io_channels 1 the reference's CFG rescale takes an unbiased std over one channel, which is NaN: "y_cfg4_phi" of
that fixture is all NaN, and so is what this package returns for it.
"""
import json
import os

import numpy as np
import torch

from . import positions_oracle as po
from . import ref_shims
from .make_golden import DIT_SMALL, GOLDEN_DIR, _np, weights_checksum

# (file, global_cond_type, DIT_SMALL overrides, seed, latent positions, concat kind)
WIDTH_GOLDENS = (
    # inpainting: io 64 + concat 65 (mask, masked latents); Cin 129 -> K 136                              201 tokens
    ("dit_width_inpaint_small.npz", "prepend", dict(input_concat_dim=65), 90, 200, "inpaint"),
    # io 16 (PQMF mono x 16 bands): N 16 -> 32, K 16; adaLN, head dim 128                                  203 tokens
    ("dit_width_io16_adaln_hd128_small.npz", "adaLN",
     dict(io_channels=16, embed_dim=256, num_heads=2, cond_token_dim=128), 91, 203, None),
    # io 2, patch 4, concat 3: native C 8 -> N 32, Cin 20 -> K 24                                          118 tokens
    ("dit_width_io2_patch4_concat3_small.npz", "prepend", dict(io_channels=2, patch_size=4, input_concat_dim=3),
     92, 468, "random"),
    # io 1: N 1 -> 32, K 1 -> 8; scale_phi over one channel                                                251 tokens
    ("dit_width_io1_small.npz", "prepend", dict(io_channels=1), 93, 250, None),
    # io 40 with conformer blocks: N 40 -> 64, K 40 (no K padding)                                        191 tokens
    ("dit_width_io40_conformer_small.npz", "prepend", dict(io_channels=40, conformer=True), 94, 190, None),
)


def make_concat(kind, B, C, L, g):
    """The input-concat conditioning: "inpaint" = a binary mask channel, then latents times that mask (the
    inpaint_mask / inpaint_masked_input pair); "random" = Gaussian channels."""
    if kind == "inpaint":
        mask = (torch.rand(B, 1, L, generator=g) > 0.5).float()
        latents = torch.randn(B, C - 1, L, generator=g)
        return torch.cat([mask, latents * mask], dim=1)
    return torch.randn(B, C, L, generator=g)


def gen_dit_width(ref, path, gtype, overrides, seed, L, concat_kind):
    cfg = dict(DIT_SMALL, global_cond_type=gtype, **overrides)
    sd = po.make_dit_weights(cfg, seed=seed)
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
    if concat_kind:
        ic = make_concat(concat_kind, B, cfg["input_concat_dim"], L, g)
        out["concat"] = _np(ic)
        kw["input_concat_cond"] = ic
    with torch.no_grad():
        out["y_nocfg"] = _np(m(x, t, cfg_scale=1.0, **kw))
        out["y_cfg7"] = _np(m(x, t, cfg_scale=7.0, **kw))
        out["y_cfg4_phi"] = _np(m(x, t, cfg_scale=4.0, scale_phi=0.7, **kw))
        out["y_neg3"] = _np(m(x, t, negative_cross_attn_cond=neg, cfg_scale=3.0, **kw))
        y, info = m(x, t, cfg_scale=1.0, return_info=True, **kw)
        out["hidden_last"] = _np(info["hidden_states"][-1])
        if concat_kind:
            out["y_noconcat"] = _np(m(x, t, cfg_scale=1.0, **dict(kw, input_concat_cond=torch.zeros_like(ic))))
    np.savez_compressed(path, **out)


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    for name, gtype, overrides, seed, L, concat_kind in WIDTH_GOLDENS:
        path = os.path.join(GOLDEN_DIR, name)
        gen_dit_width(ref, path, gtype, overrides, seed, L, concat_kind)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
