"""CPU: the windowed float64 Oobleck reference (oobleck_window_ref) against the whole-item oracle, its sharpness, and
the latents where a whole-batch pass at the Stable Audio 2.0 length leaves 32-bit range.  Nothing here touches a GPU.

A window's float64 result must equal the slice of the full float64 oracle (the margin is the whole receptive field),
and each way of taking the wrong window (a margin one latent short, a window one latent off, the neighbouring item's
window) must miss the gates tests/test_gpu_oobleck_long.py applies: 1.35 x the fp16-operand floor for 16-bit
operands, 68 dB SNR for fp16x3."""
import pytest
import torch

from helpers import rel_l2
from oobleck_window_ref import (crossing_latents, crossings, decode_window, encode_window, receptive_margin,
                                workspace_bytes)

FLOOR_GATE = 1.35          # the GPU test's gates
SNR_GATE_DB = 68.0

SMALL = dict(channels=32, c_mults=[1, 2, 4], strides=[2, 4, 8])
SAO_NARROW = dict(channels=8, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8])   # the SA-Open layer list
SAO = dict(channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8])
WIDTHS = {"small": (SMALL, 200), "sao_narrow": (SAO_NARROW, 64)}   # name -> (widths, latents)

# (mode, use_snake, use_nearest_upsample)
VARIANTS = [("decode", True, False), ("decode", False, False), ("decode", True, True), ("decode", False, True),
            ("encode", True, False), ("encode", False, False)]

_CACHE = {}


def _setup(widths, mode, snake, nearest, B=1):
    """cfg, float64 weights, a batch of B float64 inputs and the full float64 oracle output of each item."""
    key = (widths, mode, snake, nearest, B)
    if key not in _CACHE:
        w, L = WIDTHS[widths]
        if mode == "decode":
            cfg = dict(w, latent_dim=8, out_channels=2, final_tanh=False, use_snake=snake, use_nearest_upsample=nearest)
            sd = ov_weights(cfg, mode, seed=3)
            x = torch.randn(B, 8, L, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
            full = ov_run(cfg, sd, x, mode)
        else:
            cfg = dict(w, latent_dim=16, in_channels=2, use_snake=snake)
            sd = ov_weights(cfg, mode, seed=5)
            R = 1
            for s in w["strides"]:
                R *= s
            x = (0.5 * torch.randn(B, 2, L * R, generator=torch.Generator().manual_seed(6),
                                   dtype=torch.float64)).clamp(-1, 1)
            full = ov_run(cfg, sd, x, mode)
        _CACHE[key] = (cfg, sd, x, full, L)
    return _CACHE[key]


def ov_weights(cfg, mode, seed):
    from oracle import oobleck_variants_oracle as ov
    make = ov.make_decoder_weights if mode == "decode" else ov.make_encoder_weights
    return {k: v.double() for k, v in make(cfg, seed=seed).items()}


def ov_run(cfg, sd, x, mode):
    from oracle import oobleck_variants_oracle as ov
    return (ov.oobleck_decoder if mode == "decode" else ov.oobleck_encoder)(x, sd, cfg)


def _window(cfg, sd, x, a, b, margin, mode, item=0):
    fn = decode_window if mode == "decode" else encode_window
    return fn(x[item:item + 1], sd, cfg, a, b, margin)


def _slice(full, cfg, a, b, mode, item=0):
    if mode == "encode":
        return full[item:item + 1, :, a:b]
    R = 1
    for s in cfg["strides"]:
        R *= s
    return full[item:item + 1, :, a * R:b * R]


def _windows(L):
    """At the item's start, in its interior, at its end, and the whole item."""
    return [(0, 16), (L // 2 - 8, L // 2 + 8), (L - 16, L), (0, L)]


@pytest.mark.parametrize("mode,snake,nearest", VARIANTS)
@pytest.mark.parametrize("widths", sorted(WIDTHS))
def test_window_equals_the_slice_of_the_full_oracle(widths, mode, snake, nearest):
    cfg, sd, x, full, L = _setup(widths, mode, snake, nearest)
    m = receptive_margin(cfg, mode)
    assert m >= 8
    for a, b in _windows(L):
        got = _window(cfg, sd, x, a, b, m, mode)
        want = _slice(full, cfg, a, b, mode)
        assert got.dtype == torch.float64 and got.shape == want.shape
        assert rel_l2(got, want) <= 1e-12, (a, b, rel_l2(got, want))


def _fp16_floor(cfg, sd, x, a, b, m, mode, want):
    from oracle import oobleck_oracle as oo
    with oo.operand_rounding(torch.float16):
        return rel_l2(_window(cfg, sd, x, a, b, m, mode), want)


def _misses_every_gate(err, floor):
    """err is far above the 16-bit gate at this window's fp16 floor, and far below 68 dB of SNR."""
    return err > 10 * FLOOR_GATE * floor and err > 10 * 10 ** (-SNR_GATE_DB / 20)


@pytest.mark.parametrize("mode,snake,nearest", VARIANTS)
@pytest.mark.parametrize("widths", sorted(WIDTHS))
def test_a_margin_one_latent_short_is_visible(widths, mode, snake, nearest):
    """The margin is the whole receptive field: one latent less changes an interior window's first or last latent
    (the only ones it reaches) by far more than the 1e-12 the full margin is held to.  Above 1e-6 with Snake; ELU
    saturates below zero and passes less through the field's outermost taps (measured 2.1e-7 .. 3.7e-6 at these
    seeds), so its bar is 1e-7."""
    cfg, sd, x, full, L = _setup(widths, mode, snake, nearest)
    m = receptive_margin(cfg, mode)
    a, b = L // 2 - 8, L // 2 + 8
    got, want = _window(cfg, sd, x, a, b, m - 1, mode), _slice(full, cfg, a, b, mode)
    r = got.shape[-1] // (b - a)                                    # outputs per latent
    err = max(rel_l2(got[..., :r], want[..., :r]), rel_l2(got[..., -r:], want[..., -r:]))
    print(f"[short margin] {widths} {mode} snake={snake} nearest={nearest} margin {m - 1}: edge rel-L2 {err:.3e}")
    assert err > (1e-6 if snake else 1e-7), err


@pytest.mark.parametrize("mode,snake,nearest", VARIANTS)
@pytest.mark.parametrize("widths", sorted(WIDTHS))
def test_a_window_one_latent_off_or_from_the_neighbouring_item_fails_the_gates(widths, mode, snake, nearest):
    cfg, sd, x, full, L = _setup(widths, mode, snake, nearest, B=2)
    m = receptive_margin(cfg, mode)
    for a, b in _windows(L)[:3]:
        want = _slice(full, cfg, a, b, mode, item=0)
        floor = _fp16_floor(cfg, sd, x, a, b, m, mode, want)
        assert floor > 0
        d = 1 if b < L else -1
        off = rel_l2(_window(cfg, sd, x, a + d, b + d, m, mode), want)
        other = rel_l2(_window(cfg, sd, x, a, b, m, mode, item=1), want)
        assert _misses_every_gate(off, floor), (a, off, floor)
        assert _misses_every_gate(other, floor), (a, other, floor)


# ------------------------------------------------------------------------- where 32-bit range ends
SAO_DEC = dict(SAO, latent_dim=64, out_channels=2)
SAO_ENC = dict(SAO, latent_dim=128, in_channels=2)


@pytest.mark.parametrize("mode", ["decode", "encode"])
def test_crossing_latents_of_the_sa_open_widths_at_the_sa2_length(mode):
    """Hand count.  The last decoder block (first encoder level) holds 2048 samples x 128 channels = 2^18 elements
    per latent, block 4 (level 1) 2^17, block 3 (level 2) 2^16, and an item is 6144 = 3 * 2^11 latents.  An offset of
    2^k elements lands at global latent 2^(k - 18) (2^(k - 17), 2^(k - 16)), i.e. at item 2^(k-18) // 6144 and latent
    2^(k-18) % 6144, which is 2048 or 4096 for every k >= 29."""
    cfg = SAO_DEC if mode == "decode" else SAO_ENC
    # fp16: 16-bit activations and a 16-bit raw stream: elements 2^30 (byte 2^31), 2^31, 2^32 (byte 2^33)
    assert crossing_latents(cfg, 1, 6144, mode, "fp16") == [(0, 4096)]
    assert crossing_latents(cfg, 2, 6144, mode, "fp16") == [(0, 4096), (1, 2048)]
    assert crossing_latents(cfg, 3, 6144, mode, "fp16") == [(0, 4096), (1, 2048), (2, 4096)]
    # an fp32 raw stream adds element 2^29 (byte 2^31): latent 2048 of item 0
    for dt in ("bf16", "fp16x3"):
        assert crossing_latents(cfg, 2, 6144, mode, dt) == [(0, 2048), (0, 4096), (1, 2048)]
        assert crossing_latents(cfg, 3, 6144, mode, dt) == [(0, 2048), (0, 4096), (1, 2048), (2, 4096)]
    last = "block 5" if mode == "decode" else "level 0"
    c = crossings(cfg, 3, 6144, mode, "fp16")
    assert f"{last} elem 2^31" in c[(1, 2048)] and f"{last} elem 2^32" in c[(2, 4096)]
    assert f"{last} raw byte 2^31" in c[(0, 4096)]


def test_no_crossing_below_the_sa2_length():
    for mode, cfg in (("decode", SAO_DEC), ("encode", SAO_ENC)):
        for dt in ("fp16", "bf16", "fp16x3"):
            assert crossing_latents(cfg, 1, 1024, mode, dt) == []


def test_workspace_bytes_follow_the_native_sizing():
    """max_elems = B * L * 2048 * 128 (the last decoder block / first encoder level); the raw stream is allocated at 4
    bytes per element, each 16-bit buffer at 2 (4 with its lo half in fp16x3)."""
    e = 6144 * 2048 * 128
    for mode, cfg in (("decode", SAO_DEC), ("encode", SAO_ENC)):
        assert workspace_bytes(cfg, 3, 6144, mode, "fp16") == 3 * e * 8
        assert workspace_bytes(cfg, 2, 6144, mode, "fp16x3") == 2 * e * 12
        assert workspace_bytes(cfg, 1, 6144, mode, "bf16") == e * 8
    assert 38e9 < workspace_bytes(SAO_DEC, 3, 6144, "decode", "fp16") < 39e9
