"""Windowed float64 reference of the Oobleck decoder and encoder, and where a whole-batch pass leaves 32-bit range.

The decoder and encoder are convolutional: an output latent's samples (an encoder latent) depend on the latents
(audio samples) within the receptive field ``margin`` on either side, the value ``satb_oobleck_group_plan`` returns
and ``tests/test_oobleck_group.py`` pins against brute force.  So the samples of latents [a, b) of a long item are
the oracle's output over latents [a - margin, b + margin), clipped to the item, cut back to [a, b): an exact float64
check of any window of a 12.6-million-sample decode costs a few dozen latents of oracle work.  A window that touches
the item's first or last latent keeps the real zero padding on that side.

``crossing_latents`` names the latents whose samples sit at element index 2^31 and 2^32 and at byte offset 2^31,
2^32 and 2^33 of some activation buffer of a whole-batch decode or encode, with the element counts and element sizes
of ``decode_impl`` / ``encode_impl`` (csrc/oobleck.cu); ``workspace_bytes`` is the workspace those functions allocate.
"""
import math

import torch

from oracle import oobleck_variants_oracle as ov

OPERAND_DTYPES = ("fp16", "bf16", "fp16x3")


def ratio(cfg):
    """Samples per latent: the product of the strides."""
    return math.prod(cfg["strides"])


def _chans(cfg):
    """c_mults[i] * channels, i = 0 .. n, c_mults prepended with 1 (SatbOobleck::chans)."""
    return [cfg["channels"] * m for m in [1] + list(cfg["c_mults"])]


def native_config(cfg, mode):
    """The SatbOobleckConfig of the oracle config cfg for mode "decode" or "encode" (fp16 operands)."""
    from stable_audio_tools import _native
    assert mode in ("decode", "encode"), mode
    c = _native.SatbOobleckConfig()
    c.in_channels = cfg["out_channels"] if mode == "decode" else cfg["in_channels"]
    c.channels, c.latent_dim, c.n_stages = cfg["channels"], cfg["latent_dim"], len(cfg["c_mults"])
    for i, (m, s) in enumerate(zip(cfg["c_mults"], cfg["strides"])):
        c.c_mults[i], c.strides[i] = m, s
    c.final_tanh = int(cfg.get("final_tanh", True)) if mode == "decode" else 0
    c.is_decoder = int(mode == "decode")
    c.operand_dtype = 0
    return c


def receptive_margin(cfg, mode):
    """The recompute margin of a one-rank plan: the receptive field of one latent, in latents, on either side."""
    from stable_audio_tools import _native
    nearest = mode == "decode" and cfg.get("use_nearest_upsample", False)
    return _native.oobleck_group_plan(1, 1, native_config(cfg, mode), nearest)[2]


def decode_window(z, sd, cfg, a, b, margin, dtype=torch.float64):
    """The samples of latents [a, b) of the one item z [1, latent_dim, L]: the oracle decoder in dtype over latents
    [max(a - margin, 0), min(b + margin, L)).  sd is converted to dtype (pass it converted to skip the copy)."""
    assert z.dim() == 3 and z.shape[0] == 1 and 0 <= a < b <= z.shape[-1], (tuple(z.shape), a, b)
    R = ratio(cfg)
    lo, hi = max(a - margin, 0), min(b + margin, z.shape[-1])
    sd = {k: v.to(dtype) for k, v in sd.items()}
    y = ov.oobleck_decoder(z[..., lo:hi].to(dtype), sd, cfg)
    return y[..., (a - lo) * R:(b - lo) * R]


def encode_window(audio, sd, cfg, a, b, margin, dtype=torch.float64):
    """Latents [a, b) of the one item audio [1, in_channels, L * R]: the oracle encoder in dtype over samples
    [(a - m) R, (b + m) R), clipped to the item."""
    R = ratio(cfg)
    L = audio.shape[-1] // R
    assert audio.dim() == 3 and audio.shape[0] == 1 and audio.shape[-1] == L * R and 0 <= a < b <= L
    lo, hi = max(a - margin, 0), min(b + margin, L)
    sd = {k: v.to(dtype) for k, v in sd.items()}
    y = ov.oobleck_encoder(audio[..., lo * R:hi * R].to(dtype), sd, cfg)
    return y[..., a - lo:b - lo]


def _buffers(cfg, mode, operand_dtype):
    """(name, samples per latent, channels, bytes per element) of every activation buffer a decode / encode writes,
    channels-last [B, L * samples per latent, channels]: the 16-bit activations, their "lo" halves (fp16x3) and the
    raw skip stream (fp32; 16-bit with fp16 operands)."""
    assert mode in ("decode", "encode") and operand_dtype in OPERAND_DTYPES, (mode, operand_dtype)
    n, ch, R = len(cfg["strides"]), _chans(cfg), ratio(cfg)
    split3 = operand_dtype == "fp16x3"
    raw_bytes = 2 if operand_dtype == "fp16" else 4
    out = []

    def act(name, r, C):
        out.append((name, r, C, 2))
        if split3:
            out.append((name + " lo", r, C, 2))

    if mode == "decode":
        r = 1
        act("input 16-bit", r, cfg["latent_dim"])
        act("input conv", r, ch[n])
        for b in range(1, n + 1):
            r *= cfg["strides"][n - b]
            act(f"block {b}", r, ch[n - b])
            out.append((f"block {b} raw", r, ch[n - b], raw_bytes))
    else:
        if cfg["in_channels"] > 2:                     # the wide input conv's 16-bit copy of the audio
            act("input 16-bit", R, cfg["in_channels"])
        r = R
        for i in range(n + 1):
            act(f"level {i}", r, ch[i])
            if i < n:                                  # the last level has no residual units: no skip stream
                out.append((f"level {i} raw", r, ch[i], raw_bytes))
                r //= cfg["strides"][i]
    return out


def crossings(cfg, B, L, mode, operand_dtype):
    """{(item, latent): [what crosses there]} for element index 2^31, 2^32 and byte offset 2^31, 2^32, 2^33 of every
    buffer of ``_buffers`` in a batch of B items of L latents."""
    found = {}
    for name, r, C, nbytes in _buffers(cfg, mode, operand_dtype):
        per_item = L * r * C
        offsets = [(1 << k, f"elem 2^{k}") for k in (31, 32)]
        offsets += [((1 << k) // nbytes, f"byte 2^{k}") for k in (31, 32, 33)]
        for e, what in offsets:
            if e < B * per_item:
                item, rest = divmod(e, per_item)
                found.setdefault((item, rest // (r * C)), []).append(f"{name} {what}")
    return found


def crossing_latents(cfg, B, L, mode, operand_dtype):
    """Sorted (item, latent) whose samples hold one of the offsets of ``crossings``."""
    return sorted(crossings(cfg, B, L, mode, operand_dtype))


def workspace_bytes(cfg, B, L, mode, operand_dtype):
    """The raw stream and the two 16-bit activation buffers (each [hi | lo] in fp16x3) that decode_impl /
    encode_impl allocate for B items of L latents."""
    n, ch, R = len(cfg["strides"]), _chans(cfg), ratio(cfg)
    if mode == "decode":
        elems, l = B * L * max(cfg["latent_dim"], ch[n]), L
        for b in range(1, n + 1):
            l *= cfg["strides"][n - b]
            elems = max(elems, B * l * ch[n - b])
    else:
        elems, l = B * L * R * cfg["in_channels"], L * R
        for i in range(n + 1):
            elems = max(elems, B * l * ch[i])
            if i < n:
                l //= cfg["strides"][i]
    lo_off = (elems * 2 + 255) & ~255 if operand_dtype == "fp16x3" else 0
    return elems * 4 + 2 * (elems * 2 + lo_off)
