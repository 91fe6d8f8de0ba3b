"""The oracle restatements and the drop-in modules against stored outputs of the reference modules
(tests/golden/reference_checks.npz, written by oracle/make_golden.py from the reference itself) on fresh
random cases beyond the other golden vectors, and state-dict key parity of the drop-in modules with the
reference's."""
import functools
import json
import os

import numpy as np
import pytest
import torch

from helpers import max_abs, rel_l2
from oracle import dit_oracle as do
from oracle import make_golden as mg


@pytest.fixture(scope="module")
def gold(golden_dir):
    z = np.load(os.path.join(golden_dir, "reference_checks.npz"))
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def ref_keys(gold):
    return json.loads(str(gold["keys"]))


def _shapes(sd):
    return {k: list(v.shape) for k, v in sd.items()}


@pytest.mark.parametrize("gtype", ["prepend", "adaLN"])
@pytest.mark.parametrize("seed", [0, 1])
def test_dit_oracle_vs_live_reference(gold, gtype, seed):
    cfg, sd, (x, t, c, ge) = mg.check_dit_case(gtype, seed)
    with torch.no_grad():
        for i, kw in enumerate(mg.CHECK_DIT_KW):
            assert max_abs(do.dit_forward(sd, cfg, x, t, c, ge, **kw),
                           torch.from_numpy(gold[f"dit_{gtype}_{seed}_{i}"])) <= 1e-5


def test_dropin_state_dict_keys_match_reference(ref_keys):
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    from stable_audio_tools.models.dit import DiffusionTransformer
    for gtype in ("prepend", "adaLN"):
        cfg = dict(mg.CHECK_DIT, depth=2, project_cond_tokens=False, global_cond_type=gtype)
        theirs = ref_keys[f"dit_{gtype}"]
        assert _shapes(DiffusionTransformer(**cfg).state_dict()) == theirs
        assert set(do.dit_param_shapes(cfg)) == set(theirs)
    assert _shapes(OobleckDecoder(**mg.DEC_SMALL).state_dict()) == ref_keys["decoder"]
    assert _shapes(OobleckEncoder(**mg.ENC_SMALL).state_dict()) == ref_keys["encoder"]


def test_reference_json_configs_build_with_the_dropin_factory(gold, ref_keys):
    """The reference's shipped autoencoder config builds through the drop-in create_model_from_config
    with the reference's state-dict keys."""
    from stable_audio_tools import create_model_from_config
    mine = create_model_from_config(json.loads(str(gold["vae_2_0_cfg"])))
    assert set(mine.state_dict()) == set(ref_keys["vae_2_0"])
    assert mine.downsampling_ratio == int(gold["vae_2_0_ratio"]) == 2048


def test_sampler_wiring_vs_reference_sample_k(gold):
    """The reference's own sample_k (driving the restated k-diffusion shims) and the drop-in sample_k
    produce the same trajectory for the same toy denoiser and injected noise."""
    from stable_audio_tools.inference import sampling as mine
    toy = mg.toy_denoiser()
    noise = torch.randn(2, 4, 16)
    seq = [torch.randn(2, 4, 16) for _ in range(8)]

    def make_ns():
        it = iter(seq)
        return lambda s, sn: next(it)

    for st in ("dpmpp-2m-sde", "dpmpp-3m-sde"):
        b = mine.sample_k(toy, noise.clone(), steps=8, sampler_type=st, sigma_min=0.3, sigma_max=50, device="cpu",
                          noise_sampler=make_ns())
        assert rel_l2(b, torch.from_numpy(gold[f"sample_k_{st}"])) < 1e-5


def test_number_conditioner_and_multiconditioner_match_reference(gold):
    """The 'next' row conditioners (SURVEY 8f): same state-dict keys and outputs as the reference's."""
    from stable_audio_tools.models import conditioners as mine
    sd = {k[len("numcond_sd."):]: torch.from_numpy(gold[k]) for k in gold if k.startswith("numcond_sd.")}
    b = mine.NumberConditioner(64, min_val=0, max_val=512)
    assert set(b.state_dict()) == set(sd)
    b.load_state_dict(sd)
    xb, mb = b([0.0, 12.5, 600.0])
    assert torch.equal(torch.from_numpy(gold["numcond_x"]), xb) and torch.equal(torch.from_numpy(gold["numcond_m"]), mb)
    assert xb.shape == (3, 1, 64)
    mc = mine.MultiConditioner({"seconds_start": b, "seconds_total": mine.NumberConditioner(64, 0, 512)})
    out = mc([{"seconds_start": 0, "seconds_total": [30]}, {"seconds_start": 1, "seconds_total": 47}])
    assert out["seconds_total"][0].shape == (2, 1, 64)


def test_oracle_sample_k_inpainting_and_mask_vs_live_reference(gold):
    """oracle.sampler_oracle.sample_k / build_mask / cut_paste (used by the GPU init-audio test as the checker)
    against the reference's own sample_k (inference/sampling.py:144-228) and build_mask (generation.py:270-292):
    same toy denoiser, every random draw (SDE noise and the inpainting callback's re-noising) from one seeded
    stream via a patched torch.randn_like."""
    from oracle import sampler_oracle as so
    L = 48
    assert torch.equal(so.build_mask(L, mg.CHECK_MASK_ARGS), torch.from_numpy(gold["mask"]))
    toy = mg.toy_denoiser()
    noise, init = torch.randn(2, 4, L), torch.randn(2, 4, L)
    mask = so.build_mask(L, mg.CHECK_MASK_ARGS)
    for st in ("dpmpp-2m-sde", "dpmpp-3m-sde"):
        for mi, m in enumerate((mask, None)):
            with mg.seeded_randn_like(5):
                b = so.sample_k(toy, noise.clone(), init.clone(), m, steps=7, sampler_type=st, sigma_min=0.3, sigma_max=20)
            assert rel_l2(b, torch.from_numpy(gold[f"inpaint_{st}_{mi}"])) < 1e-6


@pytest.fixture
def fake_t5(monkeypatch):
    import transformers
    monkeypatch.setattr(transformers.AutoTokenizer, "from_pretrained", classmethod(lambda cls, *a, **k: mg.FakeTokenizer()))
    monkeypatch.setattr(transformers.T5EncoderModel, "from_pretrained", classmethod(lambda cls, *a, **k: mg.FakeT5()))


@pytest.mark.parametrize("cfg_name", ["stable_audio_open_1_0.json", "stable_audio_2_0.json"])
def test_shipped_txt2audio_configs_build_and_load_reference_state_dict(gold, ref_keys, fake_t5, cfg_name):
    """SURVEY 8(f)2 / 8(b): create_model_from_config on the reference's SHIPPED text-to-audio configs (T5 stubbed: no
    HF files offline).  (1) at full size on the meta device: same state-dict keys and shapes as the reference's own
    factory; (2) with depth cut to 2 and real tensors: same keys and shapes again, and with the same (seeded)
    conditioner weights the conditioner (stub T5 + NumberConditioners through MultiConditioner) and
    get_conditioning_inputs give the same tensors as the reference's."""
    from stable_audio_tools import create_model_from_config
    name = cfg_name[:-len(".json")]
    cfg = json.loads(str(gold[f"{name}_cfg"]))
    with torch.device("meta"):
        mine = create_model_from_config(json.loads(json.dumps(cfg)))
    b = _shapes(mine.state_dict())
    assert set(b) == set(ref_keys[name]), sorted(set(b) ^ set(ref_keys[name]))[:10]
    assert b == ref_keys[name]
    attrs = json.loads(str(gold[f"{name}_attrs"]))
    assert mine.min_input_length == attrs["min_input_length"] and mine.io_channels == attrs["io_channels"] == 64
    assert mine.cross_attn_cond_ids == attrs["cross_attn_cond_ids"] and mine.global_cond_ids == attrs["global_cond_ids"]
    torch.manual_seed(0)
    mine = create_model_from_config(mg.small_txt2audio(cfg)).eval()
    assert _shapes(mine.state_dict()) == ref_keys[name + "_small"]
    mine.load_state_dict(mg.seeded_conditioner_params(mine.state_dict()), strict=False)
    with torch.no_grad():
        ct_m = mine.conditioner(mg.CHECK_META)
    assert set(ct_m) == {"prompt", "seconds_start", "seconds_total"}
    n = mg.CHECK_TOKENS
    for k in ct_m:
        assert max_abs(ct_m[k][0].float()[:, :n], torch.from_numpy(gold[f"{name}_ct.{k}"])) <= 1e-5
        assert torch.equal(ct_m[k][1].to(torch.float32), torch.from_numpy(gold[f"{name}_ctmask.{k}"]))
    assert ct_m["prompt"][0].shape == (2, 128, 768) and float(ct_m["prompt"][0][0, 6:].abs().max()) == 0.0   # padding = zeros
    ci_m = mine.get_conditioning_inputs(ct_m)
    assert ci_m["cross_attn_cond"].shape == (2, 130, 768) and ci_m["global_cond"].shape == (2, 1536)
    cross = torch.cat([ci_m["cross_attn_cond"][:, :n], ci_m["cross_attn_cond"][:, -2:]], 1)
    assert max_abs(cross.float(), torch.from_numpy(gold[f"{name}_ci.cross_attn_cond"])) <= 1e-5
    for k in ("cross_attn_mask", "global_cond"):
        assert max_abs(ci_m[k].float(), torch.from_numpy(gold[f"{name}_ci.{k}"])) <= 1e-5
