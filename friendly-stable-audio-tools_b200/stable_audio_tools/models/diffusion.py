"""Diffusion model wrappers (interface parity with reference ``models/diffusion.py:90-209,
482-529,585-655``): ``ConditionedDiffusionModelWrapper`` routes conditioner outputs to the
denoiser, ``DiTWrapper`` adapts keyword names, ``create_diffusion_cond_from_config``
assembles the three from a reference JSON config."""
import typing as tp

import numpy as np
import torch
from torch import nn

from .dit import DiffusionTransformer
from .factory import create_pretransform_from_config


class ConditionedDiffusionModel(nn.Module):
    def __init__(self, *args, supports_cross_attention: bool = False, supports_input_concat: bool = False,
                 supports_global_cond: bool = False, supports_prepend_cond: bool = False, **kwargs):
        super().__init__(*args, **kwargs)
        self.supports_cross_attention = supports_cross_attention
        self.supports_input_concat = supports_input_concat
        self.supports_global_cond = supports_global_cond
        self.supports_prepend_cond = supports_prepend_cond

    def forward(self, x, t, **kwargs):
        raise NotImplementedError()


class DiTWrapper(ConditionedDiffusionModel):
    """Holds the DiT as ``.model`` and renames the sampler's kwargs
    (``global_cond -> global_embed``, ``cross_attn_mask -> cross_attn_cond_mask``)."""

    def __init__(self, *args, **kwargs):
        super().__init__(supports_cross_attention=True, supports_global_cond=False, supports_input_concat=False)
        self.model = DiffusionTransformer(*args, **kwargs)
        with torch.no_grad():  # the reference halves every parameter at construction (diffusion.py:487-489)
            for p in self.model.parameters():
                p *= 0.5
        self.model.refresh_native_weights()

    def forward(self, x, t, cross_attn_cond=None, cross_attn_mask=None, negative_cross_attn_cond=None,
                negative_cross_attn_mask=None, input_concat_cond=None, negative_input_concat_cond=None,
                global_cond=None, negative_global_cond=None, prepend_cond=None, prepend_cond_mask=None, cfg_scale=1.0,
                cfg_dropout_prob: float = 0.0, batch_cfg: bool = True, rescale_cfg: bool = False,
                scale_phi: float = 0.0, **kwargs):
        assert batch_cfg, "batch_cfg must be True for DiTWrapper"
        return self.model(x, t, cross_attn_cond=cross_attn_cond, cross_attn_cond_mask=cross_attn_mask,
                          negative_cross_attn_cond=negative_cross_attn_cond,
                          negative_cross_attn_mask=negative_cross_attn_mask, input_concat_cond=input_concat_cond,
                          prepend_cond=prepend_cond, prepend_cond_mask=prepend_cond_mask, cfg_scale=cfg_scale,
                          cfg_dropout_prob=cfg_dropout_prob, scale_phi=scale_phi, global_embed=global_cond, **kwargs)


class ConditionedDiffusionModelWrapper(nn.Module):
    """A denoiser + conditioner + optional pretransform (reference diffusion.py:95-209)."""

    def __init__(self, model, conditioner, io_channels, sample_rate, min_input_length: int,
                 diffusion_objective: str = "v", pretransform=None, cross_attn_cond_ids: tp.List[str] = [],
                 global_cond_ids: tp.List[str] = [], input_concat_ids: tp.List[str] = [],
                 prepend_cond_ids: tp.List[str] = []):
        super().__init__()
        self.model = model
        self.conditioner = conditioner
        self.io_channels = io_channels
        self.sample_rate = sample_rate
        self.diffusion_objective = diffusion_objective
        self.pretransform = pretransform
        self.cross_attn_cond_ids = cross_attn_cond_ids
        self.global_cond_ids = global_cond_ids
        self.input_concat_ids = input_concat_ids
        self.prepend_cond_ids = prepend_cond_ids
        self.min_input_length = min_input_length

    def get_conditioning_inputs(self, conditioning_tensors: tp.Dict[str, tp.Any], negative=False):
        """Concatenate cross-attention conds along the sequence, global conds along channels,
        input-concat conds along channels, prepend conds along the sequence."""
        cross = masks = glob = concat = prepend = prepend_mask = None
        if self.cross_attn_cond_ids:
            xs, ms = [], []
            for key in self.cross_attn_cond_ids:
                c, m = conditioning_tensors[key]
                if c.dim() == 2:
                    c, m = c.unsqueeze(1), m.unsqueeze(1)
                xs.append(c)
                ms.append(m)
            cross, masks = torch.cat(xs, dim=1), torch.cat(ms, dim=1)
        if self.global_cond_ids:
            glob = torch.cat([conditioning_tensors[k][0] for k in self.global_cond_ids], dim=-1)
            if glob.dim() == 3:
                glob = glob.squeeze(1)
        if self.input_concat_ids:
            concat = torch.cat([conditioning_tensors[k][0] for k in self.input_concat_ids], dim=1)
        if self.prepend_cond_ids:
            ps, pm = zip(*[conditioning_tensors[k] for k in self.prepend_cond_ids])
            prepend, prepend_mask = torch.cat(ps, dim=1), torch.cat(pm, dim=1)
        if negative:
            return {"negative_cross_attn_cond": cross, "negative_cross_attn_mask": masks,
                    "negative_global_cond": glob, "negative_input_concat_cond": concat}
        return {"cross_attn_cond": cross, "cross_attn_mask": masks, "global_cond": glob,
                "input_concat_cond": concat, "prepend_cond": prepend, "prepend_cond_mask": prepend_mask}

    def forward(self, x, t, cond, **kwargs):
        return self.model(x, t, **self.get_conditioning_inputs(cond), **kwargs)

    def generate(self, *args, **kwargs):
        from ..inference.generation import generate_diffusion_cond
        return generate_diffusion_cond(self, *args, **kwargs)


def create_diffusion_cond_from_config(config: tp.Dict[str, tp.Any]):
    model_cfg = config["model"]
    model_type = config["model_type"]
    diff_cfg = model_cfg["diffusion"]
    if diff_cfg["type"] != "dit":
        raise NotImplementedError(f"diffusion backbone '{diff_cfg['type']}' is outside the native hot path (DiT only)")
    extra = {}
    if model_type in ("diffusion_cond", "diffusion_cond_inpaint"):
        wrapper_fn = ConditionedDiffusionModelWrapper
        extra["diffusion_objective"] = diff_cfg.get("diffusion_objective", "v")
    elif model_type == "diffusion_prior":
        # reference diffusion.py:636-641: the prior wrapper gets no diffusion_objective, so it keeps the default "v"
        prior_type = model_cfg["prior_type"]
        if prior_type != "mono_stereo":
            raise NotImplementedError(f"prior_type '{prior_type}' is not a diffusion prior of the reference "
                                      "(mono_stereo only)")
        from .diffusion_prior import MonoToStereoDiffusionPrior
        wrapper_fn = MonoToStereoDiffusionPrior
    else:
        raise NotImplementedError(f"model_type '{model_type}' is outside the native hot path")
    denoiser = DiTWrapper(**diff_cfg["config"])
    conditioner = None
    if model_cfg.get("conditioning"):
        from .conditioners import create_multi_conditioner_from_conditioning_config
        conditioner = create_multi_conditioner_from_conditioning_config(model_cfg["conditioning"])
    pretransform = model_cfg.get("pretransform")
    min_len = 1
    if pretransform:
        pretransform = create_pretransform_from_config(pretransform, config["sample_rate"])
        min_len = pretransform.downsampling_ratio
    min_len *= denoiser.model.patch_size
    return wrapper_fn(
        denoiser, conditioner, min_input_length=min_len, sample_rate=config["sample_rate"],
        cross_attn_cond_ids=diff_cfg.get("cross_attention_cond_ids", []),
        global_cond_ids=diff_cfg.get("global_cond_ids", []), input_concat_ids=diff_cfg.get("input_concat_ids", []),
        prepend_cond_ids=diff_cfg.get("prepend_cond_ids", []), pretransform=pretransform,
        io_channels=model_cfg["io_channels"], **extra)
