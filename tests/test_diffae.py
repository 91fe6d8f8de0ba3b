"""CPU: diffusion autoencoders (model_type "diffusion_autoencoder", reference models/autoencoders.py:648-690,790-847),
the v-diffusion sampler ``inference.sampling.sample`` (reference inference/sampling.py:64-118) and the Wasserstein / L2
bottlenecks (reference models/bottleneck.py:85-115).

The oracle (oracle/diffae_oracle.py) against golden outputs of the real reference (tests/golden/diffae_*.npz,
oracle/make_golden_diffae.py); the package's torch path of ``sample`` against the oracle bit for bit; the config route,
the reference's state-dict layout, the parameter halving and the refusals; the bottlenecks against the reference."""
import json

import pytest
import torch

from helpers import load_golden, max_abs
from oracle import diffae_oracle as dao
from oracle import ref_shims

GOLDENS = ["diffae_raw_small.npz", "diffae_pqmf16_small.npz", "diffae_aepre_small.npz"]


def _golden(name):
    g = load_golden(name)
    cfg = json.loads(str(g["config"]))
    bufs = {k: torch.from_numpy(g[k]) for k in ("filter_bank", "prototype") if k in g}
    sd = dao.make_state_dict(cfg, int(g["seed"]), bufs or None)
    return g, cfg, sd, lambda k: torch.from_numpy(g[k])


# ------------------------------------------------------------------------------------------------ oracle vs goldens
@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_encode_matches_the_reference_golden(name):
    g, cfg, sd, T = _golden(name)
    h = dao.encode_pre_bottleneck(T("a"), sd, cfg)
    assert h.shape == T("h").shape and max_abs(h, T("h")) <= 1e-5
    noise = T("enc_noise") if "enc_noise" in g else None
    z = dao.bottleneck_encode(T("h"), cfg, noise)
    assert max_abs(z, T("z")) <= 1e-5


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_decode_matches_the_reference_golden(name):
    g, cfg, sd, T = _golden(name)
    y = dao.decode(T("z"), sd, cfg, int(g["steps"]), T("noise"))
    assert y.shape == T("y").shape and max_abs(y, T("y")) <= 1e-5, max_abs(y, T("y"))


def test_oracle_sampler_with_eta_replays_the_reference_noise():
    g, cfg, sd, T = _golden("diffae_raw_small.npz")
    y = dao.sample(dao.dit_fn(sd, cfg), T("x0"), int(g["eta_steps"]), float(g["eta"]), noises=T("step_noise"),
                   input_concat_cond=T("concat"))
    assert max_abs(y, T("y_eta")) <= 1e-5
    # the noise term is not vacuous: without it the result moves far past the gate
    y0 = dao.sample(dao.dit_fn(sd, cfg), T("x0"), int(g["eta_steps"]), float(g["eta"]),
                    noises=torch.zeros_like(T("step_noise")), input_concat_cond=T("concat"))
    assert max_abs(y0, T("y_eta")) > 1e-2


def test_the_decode_goldens_depend_on_the_latents():
    """The input-concat conditioning moves the decode: the reference's output is not the unconditioned sample."""
    g, cfg, sd, T = _golden("diffae_raw_small.npz")
    y = dao.decode(torch.zeros_like(T("z")), sd, cfg, int(g["steps"]), T("noise"))
    assert max_abs(y, T("y")) > 1e-2


# ------------------------------------------------------------------------------------------------ the package's sampler
def test_package_sample_torch_path_equals_the_oracle_bit_for_bit():
    """On CPU tensors ``sample`` runs the torch expressions with host-side floats; they round as the reference's fp32
    0-d tensors do, so the result equals the oracle's restatement exactly, with and without noise."""
    from stable_audio_tools.inference.sampling import sample
    g, cfg, sd, T = _golden("diffae_raw_small.npz")
    fn = dao.dit_fn(sd, cfg)
    steps, eta, noise = int(g["eta_steps"]), float(g["eta"]), T("step_noise")
    got = sample(fn, T("x0"), steps, eta, verbose=False, noise_sampler=lambda i: noise[i], input_concat_cond=T("concat"))
    assert torch.equal(got, dao.sample(fn, T("x0"), steps, eta, noises=noise, input_concat_cond=T("concat")))
    got0 = sample(fn, T("x0"), steps, 0, input_concat_cond=T("concat"))
    assert torch.equal(got0, dao.sample(fn, T("x0"), steps, 0, input_concat_cond=T("concat")))


@pytest.mark.parametrize("steps", [1, 2, 100])
@pytest.mark.parametrize("eta", [0, 0.3, 1.0])
def test_schedule_floats_are_the_reference_fp32_values(steps, eta):
    from stable_audio_tools.inference.sampling import vdiffusion_schedule
    sched = vdiffusion_schedule(steps, eta)
    t = torch.linspace(1, 0, steps + 1)[:-1]
    a, s = torch.cos(t * torch.pi / 2), torch.sin(t * torch.pi / 2)
    assert len(sched) == steps and sched[-1][3:] == (None, None, None)
    for i, (ti, ai, si, an, adj, dd) in enumerate(sched):
        assert (ti, ai, si) == (float(t[i]), float(a[i]), float(s[i]))
        for v in (ti, ai, si) + ((an, adj, dd) if an is not None else ()):
            assert torch.tensor(v, dtype=torch.float32).item() == v       # every scalar is an fp32 value
    if steps > 1:
        assert (sched[0][5] == 0.0) == (eta == 0)


def test_sample_refuses_zero_steps():
    from stable_audio_tools.inference.sampling import sample
    with pytest.raises(ValueError, match="steps >= 1"):
        sample(lambda x, t: x, torch.zeros(1, 2, 4), 0, 0)


def test_sample_draws_noise_only_when_eta_is_set():
    from stable_audio_tools.inference.sampling import sample
    calls = []
    sample(lambda x, t: -x, torch.ones(1, 2, 4), 4, 0, noise_sampler=lambda i: calls.append(i))
    assert calls == []
    sample(lambda x, t: -x, torch.ones(1, 2, 4), 4, 0.5, noise_sampler=lambda i: calls.append(i) or torch.zeros(1, 2, 4))
    assert calls == [0, 1, 2]


# ------------------------------------------------------------------------------------------------ the model
@pytest.mark.parametrize("name", GOLDENS)
def test_config_builds_with_the_reference_state_dict_layout(name):
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.autoencoders import DiffusionAutoencoder
    g, cfg, sd, T = _golden(name)
    model = create_model_from_config(json.loads(json.dumps(cfg)))
    assert type(model) is DiffusionAutoencoder
    theirs = {k: tuple(v) for k, v in json.loads(str(g["keys"])).items()}
    mine = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert mine == theirs, sorted(set(mine.items()) ^ set(theirs.items()))[:10]
    model.load_state_dict(sd, strict=True)
    assert model.min_length == cfg["model"]["downsampling_ratio"] and model.decoder is None
    assert model.diffusion.model.input_concat_dim == cfg["model"]["latent_dim"]


def test_construction_halves_the_encoder_and_dit_parameters():
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.autoencoders import OobleckEncoder
    from stable_audio_tools.models.dit import DiffusionTransformer
    g, cfg, sd, T = _golden("diffae_raw_small.npz")
    m = cfg["model"]
    torch.manual_seed(0)
    model = create_model_from_config(cfg)
    torch.manual_seed(0)
    enc = OobleckEncoder(**m["encoder"]["config"])
    dit = DiffusionTransformer(**m["diffusion"]["config"])
    for k, v in enc.state_dict().items():
        assert torch.equal(model.encoder.state_dict()[k], 0.5 * v), k
    for k, v in dit.state_dict().items():
        want = v if k.endswith("inv_freq") else 0.5 * v
        assert torch.equal(model.diffusion.model.state_dict()[k], want), k


def test_decode_runs_the_reference_steps_in_order(monkeypatch):
    """decode = bottleneck decode, nearest upsample to n * ratio, sample(diffusion, noise, steps, 0,
    input_concat_cond=...), pretransform decode; the start noise is a torch.randn draw unless given."""
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.inference import sampling
    g, cfg, sd, T = _golden("diffae_pqmf16_small.npz")
    model = create_model_from_config(cfg)
    seen = {}

    def fake_sample(model_, x, steps, eta, **kw):
        seen.update(model=model_, x=x, steps=steps, eta=eta, **kw)
        return torch.ones(x.shape)
    monkeypatch.setattr(sampling, "sample", fake_sample)
    monkeypatch.setattr(model.pretransform, "decode", lambda x: ("decoded", x))
    z = torch.randn(2, 8, 5)
    torch.manual_seed(3)
    out = model.decode(z, steps=9)
    torch.manual_seed(3)
    assert torch.equal(seen["x"], torch.randn(2, 32, 20))
    assert seen["model"] is model.diffusion and seen["steps"] == 9 and seen["eta"] == 0
    want = torch.nn.functional.interpolate(torch.nn.functional.normalize(z, dim=1), size=20, mode="nearest")
    assert torch.equal(seen["input_concat_cond"], want)
    assert out[0] == "decoded" and torch.equal(out[1], torch.ones(2, 32, 20))
    noise = torch.randn(2, 32, 20)
    model.decode(z, steps=2, noise=noise)
    assert seen["x"] is noise
    with pytest.raises(ValueError, match="noise has shape"):
        model.decode(z, steps=2, noise=torch.randn(2, 32, 21))


# ------------------------------------------------------------------------------------------------ refusals
def _raw_config():
    return json.loads(str(load_golden("diffae_raw_small.npz")["config"]))


def test_a_diffae_with_a_decoder_is_refused():
    from stable_audio_tools import create_model_from_config
    cfg = _raw_config()
    cfg["model"]["decoder"] = {"type": "oobleck", "config": {"out_channels": 2, "channels": 32, "c_mults": [1, 2],
                                                            "strides": [2, 2], "latent_dim": 8}}
    with pytest.raises(NotImplementedError, match="recurses without end"):
        create_model_from_config(cfg)


@pytest.mark.parametrize("kind", ["DAU1d", "adp_1d"])
def test_adp_unet_diffusion_blocks_are_refused(kind):
    from stable_audio_tools import create_model_from_config
    cfg = _raw_config()
    cfg["model"]["diffusion"] = {"type": kind, "config": {"strides": [2, 2], "factors": [2, 2]}}
    with pytest.raises(NotImplementedError, match="ADP U-Nets"):
        create_model_from_config(cfg)


def test_a_dit_of_the_wrong_width_is_refused():
    from stable_audio_tools import create_model_from_config
    cfg = _raw_config()
    cfg["model"]["diffusion"]["config"]["input_concat_dim"] = 7
    with pytest.raises(ValueError, match="input_concat_dim"):
        create_model_from_config(cfg)


def test_the_autoencoder_nested_pretransform_refusal_is_unchanged():
    from stable_audio_tools.models.autoencoders import AudioAutoencoder
    from stable_audio_tools.models.pretransforms import AutoencoderPretransform
    inner = AudioAutoencoder(None, None, latent_dim=8, downsampling_ratio=4, sample_rate=44100)
    with pytest.raises(NotImplementedError, match="nested pretransforms"):
        AudioAutoencoder(None, None, latent_dim=8, downsampling_ratio=4, sample_rate=44100,
                         pretransform=AutoencoderPretransform(inner))


# ------------------------------------------------------------------------------------------------ bottlenecks
def test_new_bottlenecks_equal_the_reference_golden():
    from stable_audio_tools.models.factory import create_bottleneck_from_config
    g = load_golden("diffae_raw_small.npz")
    x = torch.from_numpy(g["bn_x"])
    l2 = create_bottleneck_from_config({"type": "l2_norm"})
    assert torch.equal(l2.encode(x), torch.from_numpy(g["bn_l2_enc"]))
    assert torch.equal(l2.decode(x), torch.from_numpy(g["bn_l2_dec"]))
    z, info = l2.encode(x, return_info=True)
    assert info == {}
    w = create_bottleneck_from_config({"type": "wasserstein", "config": {"noise_augment_dim": 3}}).eval()
    torch.manual_seed(int(g["bn_w_seed"]))
    assert torch.equal(w.decode(x), torch.from_numpy(g["bn_w_dec"]))
    z, info = w.encode(x, return_info=True)
    assert z is x and info == {}
    w.train()
    z, info = w.encode(x, return_info=True)
    assert z is x and info["mmd"].shape == ()
    assert torch.equal(create_bottleneck_from_config({"type": "wasserstein"}).decode(x), x)


@pytest.mark.reference
def test_new_bottlenecks_equal_the_reference_modules():
    from stable_audio_tools.models.bottleneck import L2Bottleneck, WassersteinBottleneck
    ref = ref_shims.import_reference()
    x = torch.randn(3, 5, 17)
    assert torch.equal(L2Bottleneck().decode(x), ref.bottleneck.L2Bottleneck().decode(x))
    torch.manual_seed(5)
    theirs = ref.bottleneck.WassersteinBottleneck(noise_augment_dim=4).train().encode(x, return_info=True)[1]["mmd"]
    torch.manual_seed(5)
    mine = WassersteinBottleneck(noise_augment_dim=4).train().encode(x, return_info=True)[1]["mmd"]
    assert torch.equal(mine, theirs)


@pytest.mark.reference
@pytest.mark.parametrize("name", GOLDENS)
def test_a_state_dict_saved_by_the_reference_loads_unchanged(name):
    from stable_audio_tools import create_model_from_config
    from oracle import pqmf_oracle
    g, cfg, sd, T = _golden(name)
    ref = ref_shims.import_reference()
    pqmf_oracle.patch_reference_firwin(ref)
    with ref_shims.reference_modules(ref):
        theirs = ref.factory.create_model_from_config(json.loads(json.dumps(cfg)))
    saved = theirs.state_dict()
    mine = create_model_from_config(cfg)
    mine.load_state_dict(saved, strict=True)
    for k, v in mine.state_dict().items():
        assert torch.equal(v, saved[k]), k
