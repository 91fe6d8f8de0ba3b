"""Generate tests/golden/pqmf_small.npz and tests/golden/oobleck_pqmf_small.npz from the REAL reference PQMF
(models/pqmf.py) and an Oobleck autoencoder built with a nested ``pqmf`` pretransform through the reference's
``create_autoencoder_from_config`` (models/autoencoders.py:750-787).

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_pqmf

pqmf_small.npz, per (attenuation, bands) in BANKS, keys prefixed "a{att}_n{n}_":
  filter_bank, prototype    the reference PQMF's buffers
  x_long, y_long            stereo [2, 2, T] with T not a multiple of n, and its PQMF.forward as [B, C * n, T / n]
  x_short, y_short          the same for a signal shorter than the filter
  z, s                      seeded bands [2, 2 * n, t] and PQMF.inverse of them, [2, 2, t * n]
oobleck_pqmf_small.npz: the config (JSON) and the weight seed (pqmf_oracle.autoencoder_state_dict rebuilds the state
dict from it and the (100, 16) bank above), audio a and its pre-bottleneck latents h = encoder(pretransform(a)),
latents z and their decode audio y, and the reference state dict's keys and shapes.
"""
import json
import os

import numpy as np
import torch

from . import pqmf_oracle, ref_shims
from .make_golden import GOLDEN_DIR, _np

BANKS = [(100, 16), (100, 32), (80, 64)]

# stereo x 16 bands -> a 32-channel Oobleck; downsampling 16 (PQMF) x 4 (strides)
AE_CONFIG = {
    "sample_rate": 44100,
    "model_type": "autoencoder",
    "model": {
        "io_channels": 2,
        "latent_dim": 8,
        "downsampling_ratio": 64,
        "pretransform": {"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}},
        "encoder": {"type": "oobleck", "config": {"in_channels": 32, "channels": 32, "c_mults": [1, 2],
                                                  "strides": [2, 2], "latent_dim": 8, "use_snake": True}},
        "decoder": {"type": "oobleck", "config": {"out_channels": 32, "channels": 32, "c_mults": [1, 2],
                                                  "strides": [2, 2], "latent_dim": 8, "use_snake": True,
                                                  "final_tanh": False}},
    },
}
AE_SEED = 90


def _banks(ref, g):
    out = {}
    for att, n in BANKS:
        pq = pqmf_oracle.reference_pqmf(ref, att, n)
        F_ = pq.filter_bank.shape[-1]
        p = f"a{att}_n{n}_"
        out[p + "filter_bank"] = _np(pq.filter_bank)
        out[p + "prototype"] = _np(pq.prototype)
        for name, T in (("long", 3 * F_ + n // 2 + 3), ("short", F_ // 2 - 5)):
            x = torch.randn(2, 2, T, generator=g)
            with torch.no_grad():
                y = pq(x).flatten(1, 2)
            out[p + "x_" + name], out[p + "y_" + name] = _np(x), _np(y)
        z = torch.randn(2, 2 * n, 2 * (F_ // n) + 7, generator=g)
        with torch.no_grad():
            s = pq.inverse(z.unflatten(1, (2, n)))
        out[p + "z"], out[p + "s"] = _np(z), _np(s)
    return out


def _autoencoder(ref, g):
    pq = pqmf_oracle.reference_pqmf(ref, 100, 16)
    sd = pqmf_oracle.autoencoder_state_dict(AE_CONFIG, pq.filter_bank, pq.prototype, AE_SEED)
    with ref_shims.reference_modules(ref):
        model = ref.factory.create_model_from_config(AE_CONFIG).eval()
    model.load_state_dict(sd, strict=True)
    a = (0.5 * torch.randn(2, 2, 64 * 20, generator=g)).clamp(-1, 1)
    z = torch.randn(2, 8, 13, generator=g)
    with torch.no_grad():
        h = model.encode(a)
        y = model.decode(z)
    return {"config": json.dumps(AE_CONFIG), "seed": AE_SEED, "a": _np(a), "h": _np(h), "z": _np(z), "y": _np(y),
            "keys": json.dumps({k: list(v.shape) for k, v in model.state_dict().items()})}


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    pqmf_oracle.patch_reference_firwin(ref)
    g = torch.Generator().manual_seed(88)
    files = {"pqmf_small.npz": _banks(ref, g), "oobleck_pqmf_small.npz": _autoencoder(ref, g)}
    for name, out in files.items():
        path = os.path.join(GOLDEN_DIR, name)
        np.savez_compressed(path, **out)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
