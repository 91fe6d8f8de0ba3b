"""Generate tests/golden/dit_pos_*.npz from the REAL reference DiffusionTransformer: DiTs built with the reference's
positional options (``rotary_pos_emb``, ``use_sinusoidal_emb``, ``use_abs_pos_emb``; reference
models/transformer.py:50-96, 705-809).

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_positions

Same inputs and keys as ``oracle.make_golden_feedforward`` (x, t, cross, glob, neg, optional prepend; the four guidance
cases and the last hidden state; a checksum of the weights; the reference's state-dict key / shape list), with the
synthetic weights of ``oracle.positions_oracle``, plus "y_nopos": the conditional output with the embedding zeroed
(scale 0 / weight 0) or, for the fixture without one, with rotary switched back on, which shows that the positional
term matters.  The token counts are not multiples of the GEMM row tile (128).
"""
import json
import os

import numpy as np
import torch

from . import positions_oracle as po
from . import ref_shims
from .make_golden import DIT_SMALL, GOLDEN_DIR, _np, weights_checksum

# (file, global_cond_type, DIT_SMALL overrides, seed, latent positions, prepend-conditioning tokens)
POS_GOLDENS = (
    # sinusoidal embedding + rotary, prepend mode, head dim 64                                           201 tokens
    ("dit_pos_sin_small.npz", "prepend", dict(use_sinusoidal_emb=True), 70, 200, 0),
    # absolute embedding + rotary, 3 prepend-conditioning tokens                                         194 tokens
    ("dit_pos_abs_prepcond_small.npz", "prepend",
     dict(prepend_cond_dim=96, use_abs_pos_emb=True, abs_pos_emb_max_length=300), 71, 190, 3),
    # no rotary, absolute embedding with max_len == the sequence length; adaLN; head dim 128            203 tokens
    ("dit_pos_norope_abs_adaln_hd128_small.npz", "adaLN",
     dict(embed_dim=256, num_heads=2, cond_token_dim=128, rotary_pos_emb=False, use_abs_pos_emb=True,
          abs_pos_emb_max_length=203), 72, 203, 0),
    # no rotary and no embedding; qk_norm                                                                201 tokens
    ("dit_pos_norope_qknorm_small.npz", "prepend", dict(rotary_pos_emb=False, attn_kwargs=dict(qk_norm=True)), 73, 200, 0),
    # sinusoidal + conformer blocks + patch_size 2 + Conv1d k 3 FF-out                                   116 tokens
    ("dit_pos_sin_conformer_patch2_conv3_small.npz", "prepend",
     dict(use_sinusoidal_emb=True, conformer=True, patch_size=2, ff_kwargs=dict(use_conv=True, conv_kernel_size=3)),
     74, 230, 0),
)


def _without_positions(cfg, sd):
    """The config and weights whose output "y_nopos" is: the embedding zeroed, or rotary back on without one."""
    sd = dict(sd)
    if "transformer.pos_emb.scale" in sd:
        sd["transformer.pos_emb.scale"] = torch.zeros_like(sd["transformer.pos_emb.scale"])
    elif "transformer.pos_emb.emb.weight" in sd:
        sd["transformer.pos_emb.emb.weight"] = torch.zeros_like(sd["transformer.pos_emb.emb.weight"])
    else:
        cfg = dict(cfg, rotary_pos_emb=True)
        sd["transformer.rotary_pos_emb.inv_freq"] = po.make_dit_weights(cfg, seed=0)["transformer.rotary_pos_emb.inv_freq"]
    return cfg, sd


def gen_dit_pos(ref, path, gtype, overrides, seed, L, n_prepend):
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
    if cfg.get("use_sinusoidal_emb"):
        out["pos_inv_freq"] = _np(m.transformer.pos_emb.inv_freq)
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
        cfg0, sd0 = _without_positions(cfg, sd)
        m0 = ref.dit.DiffusionTransformer(**cfg0).eval()
        m0.load_state_dict(sd0, strict=True)
        out["y_nopos"] = _np(m0(x, t, cfg_scale=1.0, **kw))
    np.savez_compressed(path, **out)


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    for name, gtype, overrides, seed, L, n_prepend in POS_GOLDENS:
        path = os.path.join(GOLDEN_DIR, name)
        gen_dit_pos(ref, path, gtype, overrides, seed, L, n_prepend)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
