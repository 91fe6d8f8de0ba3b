"""GPU: the time-sharded Oobleck decode and encode (AudioAutoencoder.shard_time, satb_oobleck_group_*).

On one device the ranks are virtual (every rank a handle and a stream of its own on cuda:0), which runs the same split,
input copies, gather and event schedule as ranks on distinct GPUs; those add only the peer-to-peer reads, tested at
the end when at least two devices are visible.  Every sharded output must be bit-identical to the single-device call:
the plan's recompute margin covers the receptive field, and no convolution route depends on where a position falls in
a tile.  Where the plan refuses a length (a rank range shorter than the margin, more ranks than latents), the refusal
and its message are checked instead."""
import gc
import json
import zlib

import pytest
import torch

from helpers import load_golden, rel_l2

pytestmark = pytest.mark.gpu

SAO = dict(channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8])
SMALL = dict(channels=32, c_mults=[1, 2, 4], strides=[2, 4, 8])

# name -> (widths, use_snake, use_nearest_upsample)
MODELS = {
    "sao_snake": (SAO, True, False),
    "sao_elu": (SAO, False, False),
    "sao_snake_nearest": (SAO, True, True),
    "sao_elu_nearest": (SAO, False, True),
    "small_snake": (SMALL, True, False),
}
WORLDS = [2, 3, 4, 8]

_CACHE = {}


@pytest.fixture(autouse=True, scope="module")
def _release_models():
    """The cached models, their native handles and workspaces (13 GB each at 6144 latents) go with this module: the
    later test modules of a session need the device memory."""
    yield
    _CACHE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def report(**kw):
    print("OOBGROUP", json.dumps(kw))


def _module(kind, name, dtype="fp16", keep=True):
    """A decoder or encoder of MODELS[name] with the oracle's synthetic weights, on cuda:0; cached unless keep is false
    (the caller unshards it again)."""
    key = (kind, name, dtype)
    seed = 11 + zlib.crc32(repr(key).encode()) % 1000
    if key not in _CACHE or not keep:
        from oracle import oobleck_variants_oracle as ov
        from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
        widths, snake, nearest = MODELS[name]
        latent = 64 if widths is SAO else 8
        if kind == "dec":
            cfg = dict(widths, latent_dim=latent, out_channels=2, final_tanh=False, use_snake=snake,
                       use_nearest_upsample=nearest)
            sd = ov.make_decoder_weights(cfg, seed=seed)
            m = OobleckDecoder(**cfg, operand_dtype=dtype)
        else:
            cfg = dict(widths, latent_dim=2 * latent, in_channels=2, use_snake=snake)
            sd = ov.make_encoder_weights(cfg, seed=seed)
            m = OobleckEncoder(**cfg, operand_dtype=dtype)
        m.load_state_dict(sd, strict=True)
        if not keep:
            return m.cuda().eval()
        _CACHE[key] = m.cuda().eval()
    return _CACHE[key]


def _input(kind, m, B, L, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "dec":
        return torch.randn(B, m.__dict__["_ncfg"]["latent_dim"], L, generator=g).cuda()
    return (0.5 * torch.randn(B, 2, L * m.downsampling_ratio, generator=g)).clamp(-1, 1).cuda()


def _plan_refusal(m, world, L):
    """The message the plan refuses (world, L) with, or None."""
    from stable_audio_tools import _native
    try:
        _native.oobleck_group_plan(world, L, m.native_config(), m.__dict__["_ncfg"]["use_nearest_upsample"])
    except _native.NativeError as e:
        return str(e)
    return None


def _check_sharded(kind, name, world, L, dtype="fp16", B=None):
    from stable_audio_tools import _native
    m = _module(kind, name, dtype, keep=L < 6144)   # a 6144-latent workspace is released after its test
    B = B or (2 if L <= 64 else 1)
    x = _input(kind, m, B, L, seed=1000 * world + L)
    with torch.no_grad():
        y1 = m(x)
        why = _plan_refusal(m, world, L)
        m.shard_time(["cuda:0"] * world)
        try:
            if why is not None:
                with pytest.raises(_native.NativeError) as err:
                    m(x)
                assert str(err.value) == why
                report(kind=kind, model=name, dtype=dtype, world=world, L=L, refused=why)
                return
            yw = m(x)
            yw2 = m(x)                       # a second call reuses the group's slices and the ranks' workspaces
        finally:
            m.shard_time(None)
    report(kind=kind, model=name, dtype=dtype, world=world, L=L, B=B, bit_identical=bool(torch.equal(yw, y1)))
    assert yw.shape == y1.shape and bool(torch.isfinite(y1).all())
    assert torch.equal(yw, y1) and torch.equal(yw2, y1)


DEC_CASES = ([(name, L, "fp16") for name in sorted(MODELS) for L in (7, 33, 1024)] + [("sao_snake", 6144, "fp16")]
             + [("sao_snake", 1024, dt) for dt in ("bf16", "fp16x3")] + [("sao_elu_nearest", 33, dt) for dt in ("bf16", "fp16x3")])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name,L,dtype", DEC_CASES)
def test_sharded_decode_is_bit_identical(name, L, dtype, world):
    _check_sharded("dec", name, world, L, dtype)


ENC_CASES = ([(name, L, "fp16") for name in ("sao_snake", "sao_elu", "small_snake") for L in (7, 33, 1024)]
             + [("sao_snake", 6144, "fp16")] + [("sao_snake", 1024, dt) for dt in ("bf16", "fp16x3")])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name,L,dtype", ENC_CASES)
def test_sharded_encode_is_bit_identical(name, L, dtype, world):
    _check_sharded("enc", name, world, L, dtype)


@pytest.mark.parametrize("kind", ["dec", "enc"])
def test_repeated_calls_new_inputs_and_reloaded_weights_stay_exact(kind):
    from oracle import oobleck_variants_oracle as ov
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    widths, snake, _ = MODELS["sao_snake"]
    cfg = (dict(widths, latent_dim=64, out_channels=2, final_tanh=True, use_snake=True) if kind == "dec"
           else dict(widths, latent_dim=128, in_channels=2, use_snake=True))
    make = ov.make_decoder_weights if kind == "dec" else ov.make_encoder_weights
    m = (OobleckDecoder if kind == "dec" else OobleckEncoder)(**cfg)
    m.load_state_dict(make(cfg, seed=31))
    m = m.cuda().eval()
    xs = [_input(kind, m, 2, L, seed=40 + L) for L in (100, 100, 57)]
    with torch.no_grad():
        ref = [m(x) for x in xs]
        m.shard_time(["cuda:0"] * 3)
        for x, r in zip(xs + xs, ref + ref):          # new inputs, a new length, and the same ones again
            assert torch.equal(m(x), r)
        m.load_state_dict(make(cfg, seed=32))         # refreshes the ranks' handles as well as the module's own
        yw = m(xs[0])
        m.shard_time(None)
        y1 = m(xs[0])
    assert not torch.equal(y1, ref[0])
    assert torch.equal(yw, y1)


def _pqmf_autoencoder():
    from oracle import pqmf_oracle as po
    from stable_audio_tools.models.factory import create_model_from_config
    g = load_golden("oobleck_pqmf_small.npz")
    cfg = json.loads(str(g["config"]))
    gb = load_golden("pqmf_small.npz")
    sd = po.autoencoder_state_dict(cfg, gb["a100_n16_filter_bank"], gb["a100_n16_prototype"], int(g["seed"]))
    model = create_model_from_config(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda().eval()


@pytest.mark.parametrize("world", [2, 3])
def test_pqmf_autoencoder_sharded_paths(world):
    """A PQMF pretransform runs on the home device around the sharded Oobleck: encode, decode, iterate_batch and the
    unchunked *_audio calls are bit-identical to one device; the chunked ones run their chunks unsharded."""
    from stable_audio_tools import _native
    ae = _pqmf_autoencoder()
    m = _native.oobleck_group_plan(world, 10 ** 6, ae.decoder.native_config())[2]
    L = max(96, world * m)
    g = torch.Generator().manual_seed(7)
    z = torch.randn(2, ae.latent_dim, L, generator=g).cuda()
    a = (0.5 * torch.randn(2, 2, L * ae.downsampling_ratio, generator=g)).clamp(-1, 1).cuda()

    def run():
        with torch.no_grad():
            return (ae.decode(z), ae.encode(a), ae.decode(z, iterate_batch=1), ae.encode(a, iterate_batch=1),
                    ae.decode_audio(z), ae.encode_audio(a),
                    ae.decode_audio(z, chunked=True, chunk_size=32, overlap=8),
                    ae.encode_audio(a, chunked=True, chunk_size=32, overlap=8))

    ref = run()
    ae.shard_time(["cuda:0"] * world)
    out = run()
    ae.shard_time(None)
    for r, o in zip(ref, out):
        assert torch.equal(o, r)


def test_generate_with_sharded_dit_and_sharded_vae_matches_unsharded():
    """generate_diffusion_cond (dpmpp-3m-sde, CFG 5, 6 steps) with shard_tokens on the DiT and shard_time on the
    pretransform, against the same run on one device: latents and audio bit for bit."""
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    from test_gpu_generate import _build
    model = _build()[0]
    dit = model.model.model
    B, L, steps = 2, 300, 6
    g = torch.Generator().manual_seed(96)
    cond = {"prompt": (torch.randn(B, 10, 128, generator=g).cuda(), torch.ones(B, 10).cuda()),
            "seconds_start": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda()),
            "seconds_total": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda())}
    sde_noise = [torch.randn(B, 64, L, generator=g).cuda() for _ in range(steps)]

    def run():
        it = iter(sde_noise)
        lat = generate_diffusion_cond(model, steps=steps, cfg_scale=5.0, conditioning_tensors=cond, sample_size=L * 64,
                                      seed=97, device="cuda", return_latents=True, sampler_type="dpmpp-3m-sde",
                                      sigma_min=0.3, sigma_max=50.0, noise_sampler=lambda s, sn: next(it))
        return lat.cpu(), model.pretransform.decode(lat).cpu()

    lat1, audio1 = run()
    dit.shard_tokens(["cuda:0"] * 3)
    lat_dit, audio_dit = run()                        # the VAE stays unsharded unless shard_time is called
    assert model.pretransform.model.decoder.__dict__["_shard"] is None
    model.pretransform.shard_time(["cuda:0"] * 2)
    latw, audiow = run()
    dit.shard_tokens(None)
    model.pretransform.shard_time(None)
    report(case="generate_dpmpp_3m_sde", dit_world=3, vae_world=2, latents_bit_identical=bool(torch.equal(latw, lat1)),
           audio_bit_identical=bool(torch.equal(audiow, audio1)), rel_l2_audio=rel_l2(audiow, audio1))
    assert torch.equal(latw, lat_dit) and torch.equal(audiow, audio_dit)
    assert torch.equal(latw, lat1) and torch.equal(audiow, audio1)


def _real_devices(n):
    if torch.cuda.device_count() < 2:
        pytest.skip(f"{torch.cuda.device_count()} CUDA device(s) visible: ranks on distinct GPUs need at least 2")
    return [f"cuda:{i}" for i in range(n)]


def _sa2_length_vs_oracle(devices):
    from oracle import oobleck_oracle as oo
    from oracle import oobleck_variants_oracle as ov
    dec = _module("dec", "sao_snake", keep=False)
    cfg = dict(SAO, latent_dim=64, out_channels=2, final_tanh=False, use_snake=True)
    sd = {k: v.detach().clone() for k, v in dec.state_dict().items()}
    z = torch.randn(1, 64, 6144, generator=torch.Generator().manual_seed(5)).cuda()
    with torch.no_grad():
        y1 = dec(z)
        dec.shard_time(devices)
        try:
            yw = dec(z)
        finally:
            dec.shard_time(None)
        ref = ov.oobleck_decoder(z, sd, cfg)
        with oo.operand_rounding(torch.float16):
            floor = rel_l2(ov.oobleck_decoder(z, sd, cfg), ref)
    err = rel_l2(yw, ref)
    report(case="sa2_length_decode", devices=devices, rel_l2=err, floor=floor, bit_identical=bool(torch.equal(yw, y1)))
    assert torch.equal(yw, y1)
    assert err <= 1.35 * floor, (err, floor)


def test_sa2_length_decode_sharded_over_2_devices_vs_oracle():
    _sa2_length_vs_oracle(_real_devices(2))


def test_sa2_length_decode_sharded_over_every_device_vs_oracle():
    _sa2_length_vs_oracle(_real_devices(min(torch.cuda.device_count(), 8)))
