"""Generate tests/golden/oobleck_{elu,nearest,elu_nearest}_small.npz from the REAL reference OobleckEncoder /
OobleckDecoder built with the block options other than SnakeBeta + transposed conv: ELU activations
(``use_snake=False``, the reference's default) and nearest-neighbour upsampling (``use_nearest_upsample=True``),
reference models/autoencoders.py:29-194.

TEST INFRASTRUCTURE.  Run in the build container only (needs /root/reference):

    python -m oracle.make_golden_oobleck_variants

Synthetic weights from ``oracle.oobleck_variants_oracle`` (seeded; a checksum is stored), 32 / 64 channels and a few
hundred audio samples, so the files stay small.  Keys: the configs as JSON, the seeds and checksums, the inputs and the
reference outputs, and the reference modules' state-dict keys and shapes.
"""
import json
import os

import numpy as np
import torch

from . import oobleck_variants_oracle as ov
from . import ref_shims
from .make_golden import GOLDEN_DIR, _np, weights_checksum

# ELU encoder + decoder with the reference's defaults (use_snake=False, final_tanh=True)
ELU_DEC = dict(out_channels=2, channels=32, c_mults=[1, 2], strides=[2, 4], latent_dim=8)
ELU_ENC = dict(in_channels=2, channels=32, c_mults=[1, 2], strides=[2, 4], latent_dim=16)
# Snake decoder with nearest upsampling at odd strides (3, 5) and an even one
NEAREST_DEC = dict(out_channels=2, channels=32, c_mults=[1, 2, 2], strides=[2, 3, 5], latent_dim=8, use_snake=True,
                   use_nearest_upsample=True, final_tanh=False)
# ELU decoder with nearest upsampling
ELU_NEAREST_DEC = dict(out_channels=2, channels=32, c_mults=[1, 2], strides=[3, 4], latent_dim=8,
                       use_nearest_upsample=True)


def _keys(m):
    """The reference module's state-dict keys and shapes, as JSON."""
    return json.dumps({k: list(v.shape) for k, v in m.state_dict().items()})


def _dec(ref, cfg, seed, L, g):
    sd = ov.make_decoder_weights(cfg, seed=seed)
    m = ref.autoencoders.OobleckDecoder(**cfg).eval()
    m.load_state_dict(sd, strict=True)
    z = torch.randn(2, cfg["latent_dim"], L, generator=g)
    with torch.no_grad():
        y = m(z)
    return {"dec_cfg": json.dumps(cfg), "dec_seed": seed, "dec_wsum": weights_checksum(sd), "z": _np(z), "audio": _np(y),
            "dec_keys": _keys(m)}


def _enc(ref, cfg, seed, T, g):
    sd = ov.make_encoder_weights(cfg, seed=seed)
    m = ref.autoencoders.OobleckEncoder(**cfg).eval()
    m.load_state_dict(sd, strict=True)
    a = (0.5 * torch.randn(2, cfg["in_channels"], T, generator=g)).clamp(-1, 1)
    with torch.no_grad():
        h = m(a)
    return {"enc_cfg": json.dumps(cfg), "enc_seed": seed, "enc_wsum": weights_checksum(sd), "a": _np(a), "h": _np(h),
            "enc_keys": _keys(m)}


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = ref_shims.import_reference()
    g = torch.Generator().manual_seed(60)
    files = {
        "oobleck_elu_small.npz": {**_dec(ref, ELU_DEC, 61, 37, g), **_enc(ref, ELU_ENC, 62, 8 * 41, g)},
        "oobleck_nearest_small.npz": _dec(ref, NEAREST_DEC, 63, 13, g),
        "oobleck_elu_nearest_small.npz": _dec(ref, ELU_NEAREST_DEC, 64, 23, g),
    }
    for name, out in files.items():
        path = os.path.join(GOLDEN_DIR, name)
        np.savez_compressed(path, **out)
        print(name, os.path.getsize(path))


if __name__ == "__main__":
    main()
