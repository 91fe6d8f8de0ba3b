"""GPU: whole-batch Oobleck decode and encode at the Stable Audio 2.0 length (6144 latents, 12 582 912 samples per
item) with the SA-Open widths, where a batch of two or three items leaves 32-bit index range.

``generate_diffusion_cond`` decodes the whole sampled batch in one call, so B prompts at this length reach the
decoder as one [B, 64, 6144] call.  Its last block (the encoder's first) holds [B * 12 582 912, 128] elements:
past 2^31 at B = 2, past 2^32 at B = 3, and past 2^31 bytes at B = 1.  Each case checks

* every element exactly: item b of the batch call equals the call on item b alone, bit for bit.  The one-item call
  keeps every offset of item b below the batch call's, and no convolution route depends on where a position falls in a
  tile (see test_gpu_oobleck_group.py), so this covers every output sample past 2^31 and 2^32;
* windows of 16 latents against float64 (oobleck_window_ref: the oracle over the window and its receptive field):
  each item's first and last 16 latents, a window around every latent ``crossing_latents`` names, and four seeded
  interior positions per item.  16-bit operands: rel-L2 <= 1.35 x the window's own fp16 / bf16 operand-rounding floor
  (as test_gpu_oobleck_group's full-length check); fp16x3: >= 68 dB SNR (as test_gpu_oobleck's fp16x3 test);
* that the windows are sharp on the device: the float64 window one latent off, and the neighbouring item's window,
  both fail the gate against the native window.

A case whose workspace (decode_impl / encode_impl sizing, about 39 GB for B = 3 in fp16 and B = 2 in fp16x3) plus 4 GB
does not fit in the free device memory is skipped with the number in the reason.  Each case's module and workspace
are released before the next."""
import gc
import math
import time

import pytest
import torch

from helpers import rel_l2
from oobleck_window_ref import crossings, decode_window, encode_window, ratio, receptive_margin, workspace_bytes

pytestmark = pytest.mark.gpu

SAO = dict(channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8])
L = 6144
W = 16                         # latents per window
HEADROOM = 4 << 30             # free memory kept beyond the workspace: the machines are shared
FLOOR_GATE = 1.35
SNR_GATE_DB = 68.0
MODELS = {"sao_snake": (True, False), "sao_elu_nearest": (False, True)}   # name -> (use_snake, use_nearest_upsample)

CASES = ([("sao_snake", "decode", B, "fp16") for B in (1, 2, 3)]
         + [("sao_snake", "decode", 2, dt) for dt in ("bf16", "fp16x3")]
         + [("sao_elu_nearest", "decode", 2, "fp16")]
         + [("sao_snake", "encode", B, "fp16") for B in (1, 2, 3)]
         + [("sao_snake", "encode", 2, "fp16x3")])

# four interior window starts per item, the same for every case
_g = torch.Generator().manual_seed(6144)
INTERIOR = [sorted(int(v) for v in torch.randint(W, L - 2 * W, (4,), generator=_g)) for _ in range(3)]

_CACHE = {}                    # oracle weights, items and float64 windows, shared by the cases of one model


@pytest.fixture(autouse=True, scope="module")
def _release():
    yield
    _CACHE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _cfg(name, mode):
    snake, nearest = MODELS[name]
    if mode == "decode":
        return dict(SAO, latent_dim=64, out_channels=2, final_tanh=False, use_snake=snake, use_nearest_upsample=nearest)
    return dict(SAO, latent_dim=128, in_channels=2, use_snake=snake)


def _weights(name, mode):
    """The oracle's synthetic weights (fp32, CPU) and their float64 copy on the device."""
    key = ("sd", name, mode)
    if key not in _CACHE:
        from oracle import oobleck_variants_oracle as ov
        make = ov.make_decoder_weights if mode == "decode" else ov.make_encoder_weights
        sd = make(_cfg(name, mode), seed=17 if mode == "decode" else 19)
        _CACHE[key] = sd, {k: v.to("cuda", torch.float64) for k, v in sd.items()}
    return _CACHE[key]


def _item(mode, b):
    """Item b's input, the same in every case: latents, or audio in [-1, 1]."""
    g = torch.Generator().manual_seed(100 * (mode == "decode") + b)
    if mode == "decode":
        return torch.randn(1, 64, L, generator=g)
    return (0.5 * torch.randn(1, 2, L * ratio(SAO), generator=g)).clamp(-1, 1)


def _module(name, mode, dt):
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    m = (OobleckDecoder if mode == "decode" else OobleckEncoder)(**_cfg(name, mode), operand_dtype=dt)
    m.load_state_dict(_weights(name, mode)[0], strict=True)
    return m.cuda().eval()


def _windows(cfg, B, mode, dt):
    """(item, first latent, crossings it holds) of every window of a case."""
    cross = crossings(cfg, B, L, mode, dt)
    out = []
    for b in range(B):
        for a in [0, L - W] + INTERIOR[b]:
            out.append((b, a, []))
    for (b, lat), what in sorted(cross.items()):
        out.append((b, min(max(lat - W // 2, 0), L - W), what))
    return out


def _reference(name, mode, b, a, x_item, rounding=None):
    """The float64 oracle over latents [a - 1, a + W + 1) of item b, clipped to the item (so that the windows one
    latent either side come with it), or under fp16 / bf16 operand rounding over [a, a + W) only; cached."""
    key = ("ref", name, mode, b, a, rounding)
    if key not in _CACHE:
        from oracle import oobleck_oracle as oo
        cfg = _cfg(name, mode)
        sd64 = _weights(name, mode)[1]
        fn = decode_window if mode == "decode" else encode_window
        margin = receptive_margin(cfg, mode)
        xg = x_item.cuda()
        if rounding is None:
            lo, hi = max(a - 1, 0), min(a + W + 1, L)
            _CACHE[key] = lo, fn(xg, sd64, cfg, lo, hi, margin)
        else:
            with oo.operand_rounding(rounding):
                _CACHE[key] = a, fn(xg, sd64, cfg, a, a + W, margin)
    return _CACHE[key]


def _cut(ref, a, r):
    """Latents [a, a + W) of a reference window (lo, out); r outputs per latent."""
    lo, out = ref
    return out[..., (a - lo) * r:(a - lo + W) * r]


def _holds(err, floor, dt):
    if dt == "fp16x3":
        return err > 0 and -20.0 * math.log10(err) >= SNR_GATE_DB
    return err <= FLOOR_GATE * floor


def _free_or_skip(need, what):
    free = torch.cuda.mem_get_info()[0]
    if free < need + HEADROOM:
        pytest.skip(f"{what}: needs {need / 1e9:.1f} GB of workspace + {HEADROOM / 1e9:.1f} GB, "
                    f"{free / 1e9:.1f} GB free on the device")


def _release_device():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name,mode,B,dt", CASES)
def test_whole_batch_at_sa2_length(name, mode, B, dt):
    cfg = _cfg(name, mode)
    case = f"{name} {mode} B={B} {dt}"
    _weights(name, mode)
    _free_or_skip(workspace_bytes(cfg, B, L, mode, dt), case)
    rounding = {"fp16": torch.float16, "bf16": torch.bfloat16}.get(dt)
    r = ratio(cfg) if mode == "decode" else 1          # outputs per latent
    items = [_item(mode, b) for b in range(B)]
    m = _module(name, mode, dt)
    try:
        x = torch.cat(items).cuda()
        with torch.no_grad():
            y = m(x)                                   # allocates the workspace and uploads the weights
            assert bool(torch.isfinite(y).all())
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            y2 = m(x)
            end.record()
            torch.cuda.synchronize()
            t_batch = start.elapsed_time(end)
            assert torch.equal(y2, y)
            del y2
            for b in range(B):
                yb = m(x[b:b + 1])
                assert torch.equal(y[b], yb[0]), f"{case}: item {b} of the batch call differs from the call on it alone"
                del yb
            y = y.cpu()
        del x
    finally:
        del m
        _release_device()

    t0 = time.perf_counter()
    worst = 0.0
    for b, a, what in _windows(cfg, B, mode, dt):
        ext = _reference(name, mode, b, a, items[b])
        ref = _cut(ext, a, r).cpu()
        got = y[b:b + 1, :, a * r:(a + W) * r]
        err = rel_l2(got, ref)
        floor = rel_l2(_reference(name, mode, b, a, items[b], rounding)[1].cpu(), ref) if rounding else 0.0
        d = 1 if a + W < L else -1
        off = rel_l2(got, _cut(ext, a + d, r).cpu())
        ratio_or_snr = (f"ratio {err / floor:.3f}" if rounding else f"snr {-20 * math.log10(err):.1f} dB")
        print(f"[window] {case} item {b} latents {a}..{a + W - 1} err {err:.3e} floor {floor:.3e} {ratio_or_snr} "
              f"off-by-one {off:.2e} crossing {'; '.join(what) if what else '-'}")
        worst = max(worst, err / floor if rounding else err)
        assert _holds(err, floor, dt), (case, b, a, err, floor)
        assert not _holds(off, floor, dt), (case, b, a, off, floor)
    if B > 1:
        for b in range(B):                   # the first and last windows exist for every item at the same latents
            for a in (0, L - W):
                got = y[b:b + 1, :, a * r:(a + W) * r]
                other = _cut(_reference(name, mode, (b + 1) % B, a, items[(b + 1) % B]), a, r).cpu()
                floor = (rel_l2(_reference(name, mode, b, a, items[b], rounding)[1].cpu(),
                                _cut(_reference(name, mode, b, a, items[b]), a, r).cpu()) if rounding else 0.0)
                assert not _holds(rel_l2(got, other), floor, dt), (case, b, a)
    print(f"[case] {case}: batch call {t_batch:.1f} ms, windows {time.perf_counter() - t0:.1f} s, worst "
          + (f"err/floor {worst:.3f}" if rounding else f"SNR {-20 * math.log10(worst):.1f} dB"))


def test_pretransform_decode_of_a_batch_equals_its_items():
    """The user-facing path: an AudioAutoencoder with a VAE bottleneck and the SA-Open decoder, as the pretransform of
    a create_model_from_config diffusion model; decode at B = 2, L = 6144 equals the items decoded one at a time."""
    from oracle import oobleck_variants_oracle as ov
    from stable_audio_tools.models.factory import create_model_from_config
    dec = dict(SAO, out_channels=2, latent_dim=64, use_snake=True, final_tanh=False)
    enc = dict(SAO, in_channels=2, latent_dim=128, use_snake=True)
    config = {"model_type": "diffusion_cond", "sample_rate": 44100, "model": {
        "io_channels": 64,
        "pretransform": {"type": "autoencoder", "config": {
            "encoder": {"type": "oobleck", "config": enc}, "decoder": {"type": "oobleck", "config": dec},
            "bottleneck": {"type": "vae"}, "latent_dim": 64, "downsampling_ratio": 2048, "io_channels": 2}},
        "diffusion": {"type": "dit", "config": dict(io_channels=64, embed_dim=256, depth=1, num_heads=4,
                                                    transformer_type="continuous_transformer")}}}
    _free_or_skip(workspace_bytes(dec, 2, L, "decode", "fp16"), "pretransform decode B=2")
    model = create_model_from_config(config)
    model.pretransform.model.decoder.load_state_dict(ov.make_decoder_weights(dec, seed=23), strict=True)
    model = model.cuda().eval()
    try:
        z = torch.randn(2, 64, L, generator=torch.Generator().manual_seed(29)).cuda()
        with torch.no_grad():
            y = model.pretransform.decode(z)
            assert y.shape == (2, 2, L * 2048) and bool(torch.isfinite(y).all())
            for b in range(2):
                assert torch.equal(y[b], model.pretransform.decode(z[b:b + 1])[0]), b
    finally:
        del model
        _release_device()
