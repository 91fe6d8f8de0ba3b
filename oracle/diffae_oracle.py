"""CPU restatement of the reference's v-diffusion sampler (inference/sampling.py:10-13,64-118) and of the diffusion
autoencoder around it (models/autoencoders.py:268-304 encode, :648-690 DiffusionAutoencoder).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Composes ``positions_oracle`` (the DiT, over dit_oracle),
``oobleck_variants_oracle`` (the encoder, over oobleck_oracle) and ``pqmf_oracle`` and leaves them unchanged.  The
state dict is the reference DiffusionAutoencoder's, flat: ``encoder.*``, ``diffusion.model.*`` (the DiT),
``pretransform.pqmf.*`` or ``pretransform.model.{encoder,decoder}.*``.  ``cfg`` is the whole model config
(``model_type: "diffusion_autoencoder"``).  Random draws are explicit arguments: the decode's start noise, the VAE
bottleneck's noise, the Wasserstein bottleneck's noise channels and the sampler's per-step noise for eta > 0.

Supported, as the package supports them: an optional Oobleck encoder; bottleneck none, vae, tanh, l2_norm or
wasserstein; pretransform none, pqmf, or an Oobleck autoencoder without a bottleneck.

Pinned against the real reference by tests/golden/diffae_*.npz (oracle/make_golden_diffae.py).
"""
import math

import torch
import torch.nn.functional as F

from . import oobleck_oracle as oo
from . import oobleck_variants_oracle as ov
from . import positions_oracle as po
from . import pqmf_oracle as pq


def get_alphas_sigmas(t):
    """sampling.py:10-13."""
    return torch.cos(t * math.pi / 2), torch.sin(t * math.pi / 2)


def sample(model_fn, x, steps, eta, noises=None, **extra_args):
    """sampling.py:64-118 without the timing branch and autocast (a no-op on CPU tensors).  noises[i] is the draw of
    step i (i < steps - 1) when eta != 0; None draws torch.randn_like(x) as the reference does."""
    ts = x.new_ones([x.shape[0]])
    t = torch.linspace(1, 0, steps + 1)[:-1]
    alphas, sigmas = get_alphas_sigmas(t)
    for i in range(steps):
        v = model_fn(x, ts * t[i], **extra_args).float()
        pred = x * alphas[i] - v * sigmas[i]
        eps = x * sigmas[i] + v * alphas[i]
        if i < steps - 1:
            ddim_sigma = eta * (sigmas[i + 1] ** 2 / sigmas[i] ** 2).sqrt() * (1 - alphas[i] ** 2 / alphas[i + 1] ** 2).sqrt()
            adjusted_sigma = (sigmas[i + 1] ** 2 - ddim_sigma ** 2).sqrt()
            x = pred * alphas[i + 1] + eps * adjusted_sigma
            if eta:
                x += (torch.randn_like(x) if noises is None else noises[i]) * ddim_sigma
    return pred


def _sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def dit_config(cfg):
    return cfg["model"]["diffusion"]["config"]


def dit_fn(sd, cfg):
    """The DiT as the sampler's model: v = DiT(x, t, input_concat_cond=...), no guidance."""
    dsd, dcfg = _sub(sd, "diffusion.model."), dit_config(cfg)
    return lambda x, t, input_concat_cond=None: po.dit_forward(dsd, dcfg, x, t, input_concat_cond=input_concat_cond)


def pretransform_encode(x, sd, cfg):
    p = cfg["model"].get("pretransform")
    if not p:
        return x
    if p["type"] == "pqmf":
        return pq.analysis(x, sd["pretransform.pqmf.filter_bank"]).to(x.dtype)
    inner = p["config"]                                          # AutoencoderPretransform: encode_audio(x) / scale
    h = ov.oobleck_encoder(x, _sub(sd, "pretransform.model.encoder."), inner["encoder"]["config"])
    return h / p.get("scale", 1.0)


def pretransform_decode(z, sd, cfg):
    p = cfg["model"].get("pretransform")
    if not p:
        return z
    if p["type"] == "pqmf":
        return pq.synthesis(z, sd["pretransform.pqmf.filter_bank"]).to(z.dtype)
    inner = p["config"]                                          # decode_audio(z * scale)
    return ov.oobleck_decoder(z * p.get("scale", 1.0), _sub(sd, "pretransform.model.decoder."),
                              inner["decoder"]["config"])


def bottleneck_encode(h, cfg, noise=None):
    kind = (cfg["model"].get("bottleneck") or {}).get("type")
    if kind == "vae":
        return oo.vae_encode(h, noise)
    if kind == "tanh":
        return torch.tanh(h)
    if kind == "l2_norm":
        return F.normalize(h, dim=1)
    return h                                                     # none, wasserstein (identity in eval)


def bottleneck_decode(z, cfg, noise=None):
    """noise: the Wasserstein bottleneck's [B, noise_augment_dim, n] channels."""
    b = cfg["model"].get("bottleneck") or {}
    if b.get("type") == "l2_norm":
        return F.normalize(z, dim=1)
    if b.get("type") == "wasserstein" and b.get("config", {}).get("noise_augment_dim", 0) > 0:
        return torch.cat([z, noise.to(z.dtype)], dim=1)
    return z


def encode_pre_bottleneck(audio, sd, cfg):
    """AudioAutoencoder.encode up to the bottleneck: pretransform encode, then the Oobleck encoder (if any)."""
    x = pretransform_encode(audio, sd, cfg)
    enc = cfg["model"].get("encoder")
    return ov.oobleck_encoder(x, _sub(sd, "encoder."), enc["config"]) if enc else x


def encode(audio, sd, cfg, noise=None):
    return bottleneck_encode(encode_pre_bottleneck(audio, sd, cfg), cfg, noise)


def upsampled_concat(latents, cfg, bottleneck_noise=None):
    """decode steps 1-2: bottleneck decode and the nearest upsample to n * downsampling_ratio (autoencoders.py:667-678)."""
    n = latents.shape[2] * cfg["model"]["downsampling_ratio"]
    latents = bottleneck_decode(latents, cfg, bottleneck_noise)
    if latents.shape[2] != n:
        latents = F.interpolate(latents, size=n, mode="nearest")
    return latents


def decode(latents, sd, cfg, steps, noise, bottleneck_noise=None):
    """DiffusionAutoencoder.decode (autoencoders.py:667-690) with the start noise [B, io_channels, n * ratio] given."""
    c = upsampled_concat(latents, cfg, bottleneck_noise)
    return pretransform_decode(sample(dit_fn(sd, cfg), noise, steps, 0, input_concat_cond=c), sd, cfg)


def make_state_dict(cfg, seed, pqmf_buffers=None):
    """Seeded synthetic weights under the reference's keys: the encoder from oobleck_variants_oracle (seed), the DiT
    from positions_oracle (seed + 1), an autoencoder pretransform's encoder / decoder (seed + 2, seed + 3).  A pqmf
    pretransform's buffers are given ({"filter_bank", "prototype"}: the reference designs them, not a seed)."""
    m = cfg["model"]
    sd = {}
    if m.get("encoder"):
        sd.update({"encoder." + k: v for k, v in ov.make_encoder_weights(m["encoder"]["config"], seed=seed).items()})
    sd.update({"diffusion.model." + k: v for k, v in po.make_dit_weights(dit_config(cfg), seed=seed + 1).items()})
    p = m.get("pretransform")
    if p and p["type"] == "pqmf":
        sd.update({"pretransform.pqmf." + k: torch.as_tensor(v) for k, v in pqmf_buffers.items()})
    elif p:
        inner = p["config"]
        sd.update({"pretransform.model.encoder." + k: v
                   for k, v in ov.make_encoder_weights(inner["encoder"]["config"], seed=seed + 2).items()})
        sd.update({"pretransform.model.decoder." + k: v
                   for k, v in ov.make_decoder_weights(inner["decoder"]["config"], seed=seed + 3).items()})
    return sd
