"""Diffusion priors (interface parity with reference ``models/diffusion_prior.py``): a conditioned DiT wrapper with a
task-specific entry point.  ``MonoToStereoDiffusionPrior`` generates stereo audio conditioned on an input-concat
"source": the dual-mono mix of the input, encoded by the pretransform when the model has one."""
import typing as tp
from enum import Enum

import torch
from torch.nn import functional as F

from .diffusion import ConditionedDiffusionModelWrapper


class PriorType(Enum):
    MonoToStereo = 1


class DiffusionPrior(ConditionedDiffusionModelWrapper):
    def __init__(self, *args, prior_type: PriorType = None, **kwargs):
        super().__init__(*args, **kwargs)
        self.prior_type = prior_type


class MonoToStereoDiffusionPrior(DiffusionPrior):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, prior_type=PriorType.MonoToStereo, **kwargs)

    def stereoize(self, audio: torch.Tensor, in_sr: int, steps: int, sampler_kwargs: tp.Optional[dict] = None):
        """Stereo audio [B, 2, T'] from audio [B, C, T] at ``in_sr`` (reference diffusion_prior.py:28-82): resample to
        the model's rate, zero-pad on the right to a multiple of ``min_input_length``, mix down to dual mono, encode
        it with the pretransform (if any) and sample with it as the "source" input-concat conditioning.  T' is the
        padded length.  ``sampler_kwargs`` go to ``generate_diffusion_cond`` (e.g. ``cfg_scale``, ``seed``,
        ``sampler_type``, ``noise``)."""
        from ..inference.generation import generate_diffusion_cond
        device = audio.device
        if in_sr != self.sample_rate:
            from torchaudio.transforms import Resample        # the call inference/utils.prepare_audio makes
            audio = Resample(in_sr, self.sample_rate).to(device)(audio)
        length = audio.shape[-1]
        m = self.min_input_length
        padded = length + (m - length % m) % m
        if padded > length:
            audio = F.pad(audio, (0, padded - length))
        dual_mono = audio.mean(1, keepdim=True).repeat(1, 2, 1)
        if self.pretransform:
            dual_mono = self.pretransform.encode(dual_mono)
        # (the reference also passes sample_rate, a deprecated argument that generate_diffusion_cond ignores)
        return generate_diffusion_cond(self, conditioning_tensors={"source": [dual_mono]}, steps=steps,
                                       sample_size=padded, device=device, **(sampler_kwargs or {}))
