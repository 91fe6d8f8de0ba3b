"""Float64 CPU restatement of the reference's PQMF filterbank (models/pqmf.py) and of an Oobleck autoencoder with a
nested ``pqmf`` pretransform (models/autoencoders.py:268-343, models/pretransforms.py:114-133).

TEST INFRASTRUCTURE (see oracle/__init__.py).  With n bands, a [n, F] bank h and m = F / n taps per polyphase row:

* analysis: the signal zero-padded to a multiple of n is split into its n polyphase rows x_p[t] = x[t n + p]; band k
  is sum_p conv1d(x_p, h_k[p::n], padding m // 2) with the last frame dropped; then every even frame of every odd band
  changes sign (alias cancellation).  Output [B, C * n, ceil(T / n)], band k of channel c at row c n + k.
* synthesis: the same sign change on the bands; output phase q is conv1d over the bands with the flipped bank's
  polyphase rows, padding m // 2 + 1, last frame dropped, times n; phases are flipped, interleaved, and the first
  2 n samples dropped.  Output [B, C, t n].

``reference_pqmf(ref)`` builds the real reference's PQMF module with scipy >= 1.14, which dropped firwin's ``nyq``:
``nyq=x`` is the same filter as ``fs=2x``.
"""
import torch
import torch.nn.functional as F

from . import oobleck_variants_oracle as ov


def _alias_signs(n, t, like):
    s = torch.ones(n, t, dtype=like.dtype, device=like.device)
    s[1::2, ::2] = -1
    return s


def analysis(x, bank):
    """x [B, C, T] -> [B, C * n, ceil(T / n)], float64."""
    x = x.double()
    bank = bank.double()
    n, Fl = bank.shape
    m = Fl // n
    B, C, T = x.shape
    x = F.pad(x, (0, (-T) % n))
    poly = x.reshape(B * C, -1, n).transpose(1, 2)                  # [(B C), n, t]: row p = x[t n + p]
    w = bank.reshape(n, m, n).transpose(1, 2)                        # [k, p, j] = h_k[j n + p]
    y = F.conv1d(poly, w, padding=m // 2)[..., :-1]
    y = y * _alias_signs(n, y.shape[-1], y)
    return y.reshape(B, C * n, -1)


def synthesis(z, bank):
    """z [B, C * n, t] -> [B, C, t * n], float64."""
    z = z.double()
    bank = bank.double()
    n, Fl = bank.shape
    m = Fl // n
    B, CN, t = z.shape
    C = CN // n
    z = z.reshape(B * C, n, t) * _alias_signs(n, t, z)
    w = bank.flip(-1).reshape(n, m, n).permute(2, 0, 1)              # [q, k, j] = flip(h_k)[j n + q]
    r = F.conv1d(z, w, padding=m // 2 + 1)[..., :-1] * n
    r = r.flip(1)                                                     # [(B C), n, t']
    out = r.transpose(1, 2).reshape(B, C, -1)                         # sample t n + q
    return out[..., 2 * n:]


def patch_reference_firwin(ref):
    """Map the reference pqmf module's firwin(..., nyq=x) to firwin(..., fs=2x); returns the module."""
    import importlib

    from . import ref_shims
    with ref_shims.reference_modules(ref):
        mod = importlib.import_module("stable_audio_tools.models.pqmf")
    if not getattr(mod, "_satb_firwin_compat", False):
        firwin = mod.firwin

        def firwin_nyq(*a, nyq=None, **k):
            if nyq is not None:
                k["fs"] = 2 * nyq
            return firwin(*a, **k)

        mod.firwin = firwin_nyq
        mod._satb_firwin_compat = True
    return mod


def reference_pqmf(ref, attenuation, num_bands):
    """The real reference PQMF(attenuation, num_bands)."""
    return patch_reference_firwin(ref).PQMF(attenuation, num_bands)


# ----------------------------------------------------------------------------- the autoencoder around the bank
def autoencoder_state_dict(cfg, bank, prototype, seed):
    """State dict of an Oobleck autoencoder config with a pqmf pretransform and no bottleneck: oobleck_variants_oracle's
    seeded encoder (seed) and decoder (seed + 1) weights and the given PQMF buffers."""
    m = cfg["model"]
    sd = {"encoder." + k: v for k, v in ov.make_encoder_weights(m["encoder"]["config"], seed=seed).items()}
    sd.update({"decoder." + k: v for k, v in ov.make_decoder_weights(m["decoder"]["config"], seed=seed + 1).items()})
    sd["pretransform.pqmf.filter_bank"] = torch.as_tensor(bank)
    sd["pretransform.pqmf.prototype"] = torch.as_tensor(prototype)
    return sd


def encode(audio, sd, cfg, bank):
    """cfg: the model config (model_type "autoencoder").  Pre-bottleneck latents of AudioAutoencoder.encode: analysis, then the Oobleck encoder (any block option)."""
    esd = {k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}
    x = analysis(audio, bank).to(audio.dtype)
    return ov.oobleck_encoder(x, esd, cfg["model"]["encoder"]["config"])


def decode(z, sd, cfg, bank):
    """AudioAutoencoder.decode without a bottleneck: the Oobleck decoder, then synthesis."""
    dsd = {k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")}
    y = ov.oobleck_decoder(z, dsd, cfg["model"]["decoder"]["config"])
    return synthesis(y, bank).to(z.dtype)
