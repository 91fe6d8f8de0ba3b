"""Generate tests/golden/diffae_*.npz from the REAL reference: diffusion autoencoders built by the reference's
``create_model_from_config`` (``model_type: "diffusion_autoencoder"``, models/autoencoders.py:790-847) and its
v-diffusion sampler ``inference.sampling.sample`` (:64-118), plus its Wasserstein and L2 bottlenecks
(models/bottleneck.py:85-115).

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_diffae

The reference's ``sample`` is called with ``verbose=False`` (its verbose branch records CUDA events); its decode calls
it with the default, so the decode runs with ``sample`` rebound to the non-verbose call.  Every random draw is made
from a seeded global torch RNG and stored: the decode's start noise, the VAE bottleneck's noise, and the per-step noise
of the eta > 0 case (the seed is re-applied and the same draws repeated; the DiT draws nothing in eval mode).

Each file: "config" (JSON), "seed" (diffae_oracle.make_state_dict), "keys" (the reference state dict's keys and
shapes), audio "a", its pre-bottleneck latents "h", latents "z" and the decode "y" of "z" from "noise" in "steps"
steps.  diffae_raw_small.npz also holds the eta > 0 case ("eta", "x0", "concat", "step_noise", "y_eta") and the
bottleneck cases ("bn_*").  PQMF files hold the reference's "filter_bank" / "prototype".
"""
import json
import os

import numpy as np
import torch

from . import diffae_oracle, pqmf_oracle, ref_shims
from .make_golden import GOLDEN_DIR, _np

DIT = dict(embed_dim=256, depth=2, num_heads=4, cond_token_dim=0, global_cond_dim=0, project_cond_tokens=False,
           transformer_type="continuous_transformer")
ENC = dict(channels=32, c_mults=[1, 2], strides=[2, 2], use_snake=True)


def _config(io, latent, ratio, encoder_in, bottleneck=None, pretransform=None, enc_latent=None):
    m = {"io_channels": io, "latent_dim": latent, "downsampling_ratio": ratio,
         "encoder": {"type": "oobleck", "config": dict(ENC, in_channels=encoder_in, latent_dim=enc_latent or latent)},
         "diffusion": {"type": "dit", "config": dict(DIT, io_channels=io, input_concat_dim=latent)}}
    if bottleneck:
        m["bottleneck"] = bottleneck
    if pretransform:
        m["pretransform"] = pretransform
    return {"model_type": "diffusion_autoencoder", "sample_rate": 44100, "model": m}


INNER_AE = {"io_channels": 2, "latent_dim": 8, "downsampling_ratio": 4,
            "encoder": {"type": "oobleck", "config": dict(ENC, in_channels=2, latent_dim=8)},
            "decoder": {"type": "oobleck", "config": dict(ENC, out_channels=2, latent_dim=8, final_tanh=False)}}

# (file, config, seed, audio samples, steps)
GOLDENS = (
    # raw stereo audio: Oobleck encoder (x4) + VAE, DiT at io 2 with 8 concat channels; 96 tokens
    ("diffae_raw_small.npz", _config(2, 8, 4, 2, bottleneck={"type": "vae"}, enc_latent=16), 110, 96, 8),
    # 16-band PQMF: the DiT diffuses 2 x 16 sub-bands; L2 bottleneck; 48 tokens of 768 samples
    ("diffae_pqmf16_small.npz", _config(32, 8, 4, 32, bottleneck={"type": "l2_norm"},
                                        pretransform={"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}}),
     120, 768, 6),
    # an Oobleck autoencoder pretransform: the DiT diffuses its 8 latent channels; no bottleneck; 160 tokens
    ("diffae_aepre_small.npz", _config(8, 8, 4, 8, pretransform={"type": "autoencoder", "scale": 1.5,
                                                                  "config": INNER_AE}), 130, 640, 5),
)


def _sample(ref):
    return lambda *a, **k: ref.sampling.sample(*a, verbose=False, **k)


def gen(ref, name, cfg, seed, T, steps):
    with ref_shims.reference_modules(ref):
        model = ref.factory.create_model_from_config(json.loads(json.dumps(cfg))).eval()
    bufs = None
    if cfg["model"].get("pretransform", {}).get("type") == "pqmf":
        bufs = {k: model.pretransform.pqmf.state_dict()[k] for k in ("filter_bank", "prototype")}
    sd = diffae_oracle.make_state_dict(cfg, seed, bufs)
    model.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(1000 + seed)
    a = (0.5 * torch.randn(2, 2, T, generator=g)).clamp(-1, 1)
    out = {"config": json.dumps(cfg), "seed": seed, "steps": steps, "a": _np(a),
           "keys": json.dumps({k: list(v.shape) for k, v in model.state_dict().items()})}
    if bufs:
        out.update({k: _np(v) for k, v in bufs.items()})
    ref.autoencoders.sample = _sample(ref)
    with torch.no_grad():
        pre = model.pretransform.encode(a) if model.pretransform is not None else a
        out["h"] = _np(model.encoder(pre))
        torch.manual_seed(seed)
        z = model.encode(a)
        torch.manual_seed(seed)
        if cfg["model"].get("bottleneck", {}).get("type") == "vae":
            out["enc_noise"] = _np(torch.randn(z.shape))
        out["z"] = _np(z)
        torch.manual_seed(seed + 1)
        y = model.decode(z, steps=steps)
        torch.manual_seed(seed + 1)
        out["noise"] = _np(torch.randn(z.shape[0], cfg["model"]["io_channels"], z.shape[2] * model.downsampling_ratio))
        out["y"] = _np(y)
    return model, out


def eta_case(ref, model, cfg, seed, eta=0.6, steps=7):
    """sample(model.diffusion, x0, steps, eta, verbose=False, input_concat_cond=concat) with the per-step draws stored."""
    g = torch.Generator().manual_seed(2000 + seed)
    L = 64
    x0 = torch.randn(2, cfg["model"]["io_channels"], L, generator=g)
    concat = torch.randn(2, cfg["model"]["latent_dim"], L, generator=g)
    torch.manual_seed(seed + 2)
    with torch.no_grad():
        y = ref.sampling.sample(model.diffusion, x0, steps, eta, verbose=False, input_concat_cond=concat)
    torch.manual_seed(seed + 2)
    noise = torch.stack([torch.randn_like(x0) for _ in range(steps - 1)])
    return {"eta": eta, "eta_steps": steps, "x0": _np(x0), "concat": _np(concat), "step_noise": _np(noise),
            "y_eta": _np(y)}


def bottleneck_cases(ref):
    g = torch.Generator().manual_seed(77)
    x = torch.randn(2, 6, 11, generator=g)
    l2 = ref.bottleneck.L2Bottleneck()
    w = ref.bottleneck.WassersteinBottleneck(noise_augment_dim=3).eval()
    torch.manual_seed(78)
    w_dec = w.decode(x)
    w_enc, info = w.encode(x, return_info=True)
    assert not info and torch.equal(w_enc, x)
    return {"bn_x": _np(x), "bn_l2_enc": _np(l2.encode(x)), "bn_l2_dec": _np(l2.decode(x)), "bn_w_dec": _np(w_dec),
            "bn_w_seed": 78}


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    pqmf_oracle.patch_reference_firwin(ref)
    for name, cfg, seed, T, steps in GOLDENS:
        model, out = gen(ref, name, cfg, seed, T, steps)
        if name == "diffae_raw_small.npz":
            out.update(eta_case(ref, model, cfg, seed))
            out.update(bottleneck_cases(ref))
        path = os.path.join(GOLDEN_DIR, name)
        np.savez_compressed(path, **out)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
