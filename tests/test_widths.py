"""CPU: DiTs of any channel width - inpainting DiTs (input_concat_dim = latent + 1 mask channel), narrow latents, raw
audio with patching, PQMF sub-bands - and the mono-to-stereo diffusion prior (reference models/diffusion_prior.py,
models/diffusion.py:636-641).

The oracle against golden outputs of the real reference (tests/golden/dit_width_*.npz, oracle/make_golden_widths.py),
the package's parameter containers against the reference's state-dict layout, the C ABI's width checks, the host
refusals, the JSON-config routes and the prior's input preparation (with the sampler stubbed out)."""
import ctypes
import json

import numpy as np
import pytest
import torch

from helpers import load_golden, max_abs, rel_l2
from oracle import positions_oracle as po

WIDTH_GOLDENS = ["dit_width_inpaint_small.npz", "dit_width_io16_adaln_hd128_small.npz",
                 "dit_width_io2_patch4_concat3_small.npz", "dit_width_io1_small.npz",
                 "dit_width_io40_conformer_small.npz"]
SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer")


def _golden(name):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = po.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), f"{name}: synthetic weight RNG drifted from the golden run"
    T = lambda k: torch.from_numpy(g[k])
    kw = dict(cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "concat" in g:
        kw["input_concat_cond"] = T("concat")
    return g, cfg, sd, T, kw


def _same(a, b, tol=1e-5):
    """max-abs within tol, with NaN exactly where the golden has NaN."""
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan)
    return nan.all() or max_abs(a[~nan], b[~nan]) <= tol


@pytest.mark.parametrize("name", WIDTH_GOLDENS)
def test_oracle_matches_reference_width_golden(name):
    g, cfg, sd, T, kw = _golden(name)
    x, t = T("x"), T("t")
    assert _same(po.dit_forward(sd, cfg, x, t, cfg_scale=1.0, **kw), T("y_nocfg"))
    assert _same(po.dit_forward(sd, cfg, x, t, cfg_scale=7.0, **kw), T("y_cfg7"))
    assert _same(po.dit_forward(sd, cfg, x, t, cfg_scale=4.0, scale_phi=0.7, **kw), T("y_cfg4_phi"))
    assert _same(po.dit_forward(sd, cfg, x, t, negative_cross_attn_cond=T("neg"), cfg_scale=3.0, **kw), T("y_neg3"))
    hs = []
    po.dit_inner_forward(sd, cfg, x, t, kw["cross_attn_cond"], kw["global_embed"], hidden_states=hs,
                         input_concat_cond=kw.get("input_concat_cond"))
    assert max_abs(hs[-1], T("hidden_last")) <= 1e-5
    assert g["y_nocfg"].shape == (2, cfg["io_channels"], g["x"].shape[2])


@pytest.mark.parametrize("name", WIDTH_GOLDENS)
def test_state_dict_keys_and_shapes_equal_the_stored_reference_list(name):
    from stable_audio_tools.models.dit import DiffusionTransformer
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    theirs = {k: tuple(s) for k, s in json.loads(str(g["keys"]))}
    mine = {k: tuple(v.shape) for k, v in DiffusionTransformer(**cfg).state_dict().items()}
    assert mine == theirs, sorted(set(mine.items()) ^ set(theirs.items()))[:10]
    want = {k: tuple(v) for k, v in po.dit_param_shapes(cfg).items()}
    assert {k: v for k, v in mine.items() if not k.endswith("rotary_pos_emb.scale")} == want


@pytest.mark.parametrize("name", ["dit_width_inpaint_small.npz", "dit_width_io2_patch4_concat3_small.npz"])
def test_the_concat_input_moves_the_golden(name):
    """Zeroing the input-concat conditioning moves the reference output far past the GPU tolerances."""
    g = load_golden(name)
    move = rel_l2(torch.from_numpy(g["y_noconcat"]), torch.from_numpy(g["y_nocfg"]))
    assert move > 0.05, move


def test_inpaint_golden_concat_is_a_binary_mask_then_masked_latents():
    g = load_golden("dit_width_inpaint_small.npz")
    c = g["concat"]
    assert c.shape[1] == 65
    mask = c[:, :1]
    assert set(np.unique(mask)) == {0.0, 1.0}
    assert np.all(c[:, 1:][np.broadcast_to(mask == 0, c[:, 1:].shape)] == 0)


def test_cfg_rescale_over_one_channel_is_nan_in_the_reference():
    """The reference's scale_phi rescale takes torch.std (unbiased) over the channel dim (dit.py:342-345); over one
    channel that is 0 / 0 = NaN, so every output of that guidance case is NaN.  The native dit_post kernel divides the
    same way, and the patch-size path rescales with torch.std: both reproduce it rather than invent a value."""
    g = load_golden("dit_width_io1_small.npz")
    assert np.isnan(g["y_cfg4_phi"]).all()
    assert np.isfinite(g["y_cfg7"]).all() and np.isfinite(g["y_nocfg"]).all()
    one = torch.randn(2, 1, 5)
    assert torch.isnan(one.std(dim=1, keepdim=True)).all()


# ------------------------------------------------------------------------------------------------ C ABI and host
def _config(io, concat, patch=1):
    from stable_audio_tools import _native
    return _native.SatbDitConfig(io_channels=io, embed_dim=256, depth=1, num_heads=4, cond_token_dim=0,
                                 global_cond_dim=0, project_cond_tokens=0, project_global_cond=1, global_cond_type=0,
                                 patch_size=patch, operand_dtype=0, input_concat_dim=concat)


@pytest.mark.parametrize("io,concat", [(1, 0), (2, 2), (8, 12), (16, 0), (24, 0), (40, 0), (48, 0), (64, 65),
                                       (64, 1), (1, 1), (3, 5), (64, 0), (64, 8)])
def test_native_create_accepts_any_width(io, concat):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _config(io, concat)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0, lib.satb_last_error()
    lib.satb_dit_destroy(h)


@pytest.mark.parametrize("io,concat,match", [(0, 0, b"io_channels must be >= 1"), (-3, 0, b"io_channels must be >= 1"),
                                             (64, -1, b"input_concat_dim must be >= 0"),
                                             (32768, 1, b"at most 32768")])
def test_native_create_refuses_bad_widths_with_a_message(io, concat, match):
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(_config(io, concat)), ctypes.byref(h)) != 0
    assert match in lib.satb_last_error()


def test_native_pre_probe_validates_before_any_cuda_call():
    from stable_audio_tools import _native
    lib = _native.lib()
    fake = 1 << 20
    assert lib.satb_dit_pre_probe(fake, fake, 1, 1, 65, 65, 10, 1, 0, None) != 0
    assert b"lda % 8 == 0" in lib.satb_last_error()
    assert lib.satb_dit_pre_probe(fake, fake, 1, 1, 65, 64, 10, 1, 0, None) != 0
    assert b"lda >= C" in lib.satb_last_error()


@pytest.mark.parametrize("kw,match", [(dict(io_channels=0), "io_channels must be >= 1"),
                                      (dict(io_channels=-1), "io_channels must be >= 1"),
                                      (dict(input_concat_dim=-2), "input_concat_dim must be >= 0")])
def test_constructor_refuses_what_the_library_refuses(kw, match):
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(ValueError, match=match):
        DiffusionTransformer(**dict(SMALL, **kw))


@pytest.mark.parametrize("io,concat,patch", [(1, 0, 1), (16, 0, 1), (2, 3, 4), (64, 65, 1), (40, 0, 2)])
def test_native_config_carries_the_patched_widths(io, concat, patch):
    from stable_audio_tools.models.dit import DiffusionTransformer
    m = DiffusionTransformer(**dict(SMALL, io_channels=io, input_concat_dim=concat, patch_size=patch))
    c = m.native_config()
    assert (c.io_channels, c.input_concat_dim, c.patch_size) == (io * patch, concat * patch, 1)
    assert m.transformer.project_in.weight.shape == (256, (io + concat) * patch)
    assert m.transformer.project_out.weight.shape == (io * patch, 256)


# ------------------------------------------------------------------------------------------------ config routes
def _model_config(model_type, io, concat, **model_extra):
    diff = dict(SMALL, io_channels=io, input_concat_dim=concat)
    return {"model_type": model_type, "sample_rate": 44100,
            "model": dict({"io_channels": io, "diffusion": {"type": "dit", "config": diff}}, **model_extra)}


def test_inpaint_model_type_builds_at_width_65():
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.diffusion import ConditionedDiffusionModelWrapper
    cfg = _model_config("diffusion_cond_inpaint", 64, 65)
    cfg["model"]["diffusion"]["input_concat_ids"] = ["inpaint_mask", "inpaint_masked_input"]
    model = create_model_from_config(json.loads(json.dumps(cfg)))
    assert type(model) is ConditionedDiffusionModelWrapper
    assert model.input_concat_ids == ["inpaint_mask", "inpaint_masked_input"] and model.diffusion_objective == "v"
    dit = model.model.model
    assert dit.transformer.project_in.weight.shape == (256, 129) and dit.preprocess_conv.weight.shape == (129, 129, 1)
    mask, masked = torch.ones(1, 1, 7), torch.randn(1, 64, 7)
    inputs = model.get_conditioning_inputs({"inpaint_mask": [mask], "inpaint_masked_input": [masked]})
    assert torch.equal(inputs["input_concat_cond"], torch.cat([mask, masked], dim=1))


def test_mono_stereo_prior_route_halves_the_parameters_and_keeps_the_default_objective():
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.diffusion_prior import MonoToStereoDiffusionPrior, PriorType
    from stable_audio_tools.models.dit import DiffusionTransformer
    cfg = _model_config("diffusion_prior", 2, 2, prior_type="mono_stereo")
    cfg["model"]["diffusion"]["input_concat_ids"] = ["source"]
    cfg["model"]["diffusion"]["diffusion_objective"] = "rectified_flow"   # the reference passes none to the prior
    torch.manual_seed(0)
    model = create_model_from_config(json.loads(json.dumps(cfg)))
    assert isinstance(model, MonoToStereoDiffusionPrior) and model.prior_type == PriorType.MonoToStereo
    assert model.diffusion_objective == "v" and model.input_concat_ids == ["source"]
    assert model.io_channels == 2 and model.min_input_length == 1 and model.sample_rate == 44100
    torch.manual_seed(0)
    fresh = DiffusionTransformer(**cfg["model"]["diffusion"]["config"])
    mine = model.model.model.state_dict()
    for k, v in fresh.state_dict().items():
        if k.endswith("inv_freq"):
            assert torch.equal(mine[k], v), k
        else:
            assert torch.equal(mine[k], 0.5 * v), k


@pytest.mark.parametrize("prior_type", ["source_separation", "stereo_mono", None])
def test_an_unknown_prior_type_is_refused(prior_type):
    from stable_audio_tools import create_model_from_config
    cfg = _model_config("diffusion_prior", 2, 2, prior_type=prior_type)
    with pytest.raises(NotImplementedError, match="prior_type"):
        create_model_from_config(cfg)


def test_stereoize_mixes_down_pads_and_conditions_on_the_source(monkeypatch):
    """stereoize's preparation (reference diffusion_prior.py:45-80) with generate_diffusion_cond stubbed out: the
    input is resampled, zero-padded to min_input_length, mixed to dual mono and passed as the "source" tensor."""
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.inference import generation
    cfg = _model_config("diffusion_prior", 2, 2, prior_type="mono_stereo")
    cfg["model"]["diffusion"]["input_concat_ids"] = ["source"]
    cfg["model"]["diffusion"]["config"]["patch_size"] = 4                # min_input_length 4
    model = create_model_from_config(cfg)
    seen = {}

    def fake_generate(m, **kw):
        seen.update(kw, model=m)
        return "out"
    monkeypatch.setattr(generation, "generate_diffusion_cond", fake_generate)
    audio = torch.randn(3, 2, 50)
    assert model.stereoize(audio, 44100, steps=7, sampler_kwargs=dict(cfg_scale=1.0, seed=5)) == "out"
    assert seen["model"] is model and seen["steps"] == 7 and seen["sample_size"] == 52
    assert seen["cfg_scale"] == 1.0 and seen["seed"] == 5
    (src,) = seen["conditioning_tensors"]["source"]
    want = torch.nn.functional.pad(audio, (0, 2)).mean(1, keepdim=True).repeat(1, 2, 1)
    assert src.shape == (3, 2, 52) and torch.equal(src, want)
    # another input rate goes through torchaudio's Resample first (the call inference/utils.prepare_audio makes)
    torchaudio = pytest.importorskip("torchaudio")
    model.stereoize(audio[:, :1], 22050, steps=2)
    res = torchaudio.transforms.Resample(22050, 44100)(audio[:, :1])
    n = res.shape[-1] + (-res.shape[-1]) % 4
    (src,) = seen["conditioning_tensors"]["source"]
    assert seen["sample_size"] == n
    assert torch.equal(src, torch.nn.functional.pad(res, (0, n - res.shape[-1])).repeat(1, 2, 1))
