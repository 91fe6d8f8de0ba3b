"""CPU: the RoBERTa oracle (oracle/clap_oracle.py) against the goldens (transformers' RobertaModel in fp32, and the
reference's own CLAPTextConditioner) and live against RobertaModel; the shipped Stable Audio 2.0 conditioning block
built through the drop-in's factory; the refusals of the conditioner and of the native encoder (no CUDA call)."""
import ctypes
import json
import os

import pytest
import torch

from helpers import load_golden, max_abs, rel_l2
from oracle import clap_oracle as co
from oracle import make_golden as mg
from oracle.make_golden import GOLDEN_DIR

GOLDENS = ["clap_d128_l2.npz", "clap_d256_l3.npz"]


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_matches_transformers_golden(name):
    g = load_golden(name)
    cfg = json.loads(str(g["config"]))
    sd = co.make_roberta_weights(cfg, int(g["seed"]))
    ids, mask = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
    hs = co.roberta_hidden_states(sd, cfg, ids, mask)
    gold = torch.from_numpy(g["hidden_states"])
    assert len(hs) == gold.shape[0] == cfg["num_hidden_layers"] + 1
    for i, h in enumerate(hs):   # every position, padded ones included
        assert max_abs(h, gold[i]) <= 2e-5, i


def test_goldens_cover_lengths_and_pad_ids_inside_prompts():
    for n in GOLDENS:
        g = load_golden(n)
        ids, m = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
        lengths = set(m.sum(1).tolist())
        assert 1 in lengths and m.shape[1] in lengths and len(lengths) >= 3
        assert ((ids == 1) & (m == 1)).any()          # a pad id inside a prompt: its position id is the pad's
        assert (co.position_ids(ids, 1)[m == 1] == 1).any()


@pytest.mark.parametrize("feature_layer_ix", [-1, -2, 0])
def test_oracle_matches_robertamodel_live(feature_layer_ix):
    cfg = dict(co.ROBERTA_BASE, vocab_size=1001, hidden_size=256, num_attention_heads=4, intermediate_size=512,
               num_hidden_layers=3)
    sd = co.make_roberta_weights(cfg, 71)
    from oracle.make_golden_clap import ids_and_mask
    ids, mask = ids_and_mask([1, 30, 77, 12], 77, cfg["vocab_size"], 72)
    with torch.no_grad():
        hs = co.hf_model(cfg, sd)(input_ids=ids, attention_mask=mask, output_hidden_states=True)["hidden_states"]
    ref = hs[feature_layer_ix]
    w, b = torch.randn(128, 256) * 256 ** -0.5, torch.randn(128) * 0.1
    got = co.clap_features(sd, cfg, ids, mask, feature_layer_ix)
    assert max_abs(got, ref) <= 2e-5
    got = co.clap_features(sd, cfg, ids, mask, feature_layer_ix, w, b)
    assert max_abs(got, ref.double() @ w.double().T + b.double()) <= 2e-5


def test_oracle_matches_the_reference_conditioner_golden():
    """The reference's CLAPTextConditioner (fp32 RobertaModel on the CPU, hidden_states[-2], no mask multiply)."""
    g = load_golden("clap_conditioner.npz")
    cfg = json.loads(str(g["config"]))
    assert cfg == co.ROBERTA_BASE and int(g["feature_layer_ix"]) == -2
    sd = co.make_roberta_weights(cfg, int(g["seed"]))
    ids, mask = torch.from_numpy(g["input_ids"]), torch.from_numpy(g["attention_mask"])
    assert torch.equal(torch.from_numpy(g["mask"]), mask)
    assert mask.sum(1).tolist()[1] == 1 and mask.sum(1).tolist()[2] == 77   # a one-token and a full prompt
    feats = torch.from_numpy(g["features"])
    ref = co.clap_features(sd, cfg, ids, mask, -2)
    assert rel_l2(feats, ref) < 1e-5 and rel_l2(feats[~mask.bool()], ref[~mask.bool()]) < 1e-5   # padded rows too
    assert torch.equal(torch.from_numpy(g["single_mask"]), mask[:1])
    assert float(g["single_max_abs"]) <= 1e-4                  # the "" pad does not change the first prompt


def _tmp_checkpoint(tmp_path, cfg, seed, prefix="module."):
    sd = co.make_roberta_weights(cfg, seed)
    path = tmp_path / "clap.pt"
    torch.save({"state_dict": {prefix + "text_branch." + k: v for k, v in sd.items()}}, str(path))
    return str(path), sd


@pytest.fixture
def stub_tokenizer(monkeypatch):
    import transformers
    monkeypatch.setattr(transformers.RobertaTokenizer, "from_pretrained",
                        classmethod(lambda cls, *a, **k: mg.FakeTokenizer()))


SMALL_768 = dict(co.ROBERTA_BASE, vocab_size=1001, num_hidden_layers=2, intermediate_size=256)


def test_stable_audio_2_0_conditioning_builds(tmp_path, stub_tokenizer):
    from stable_audio_tools.models.conditioners import CLAPTextConditioner, create_multi_conditioner_from_conditioning_config
    path, sd = _tmp_checkpoint(tmp_path, SMALL_768, 81)
    cond_cfg = json.load(open(os.path.join(GOLDEN_DIR, "clap_sa20_conditioning.json")))
    clap = [c for c in cond_cfg["configs"] if c["type"] == "clap_text"]
    assert len(clap) == 1 and clap[0]["config"]["feature_layer_ix"] == -2 and clap[0]["config"]["use_text_features"]
    clap[0]["config"]["clap_ckpt_path"] = path
    mc = create_multi_conditioner_from_conditioning_config(cond_cfg)
    prompt = mc.conditioners["prompt"]
    assert isinstance(prompt, CLAPTextConditioner) and prompt.dim == 768
    # the text branch stays out of the state dict; proj_out is an Identity at cond_dim 768 (no keys)
    assert not [k for k in mc.state_dict() if k.startswith("conditioners.prompt.")]
    enc = prompt.__dict__["native_encoder"]
    assert enc.n_layers == 1 and enc.num_hidden_layers == 2 and enc.intermediate_size == 256
    assert set(prompt.__dict__["text_branch_state"]) == set(sd)
    from stable_audio_tools._native import NativeError
    with pytest.raises(NativeError):
        mc.set_device("cpu")


def test_checkpoint_reading_follows_laion_clap(tmp_path):
    from stable_audio_tools.models.conditioners import _clap_text_branch
    for prefix in ("module.", ""):
        path, sd = _tmp_checkpoint(tmp_path, dict(SMALL_768, num_hidden_layers=1), 82, prefix)
        got = _clap_text_branch(path)
        assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
        ref = {k[len("text_branch."):]: v for k, v in co.clap_load_state_dict(path).items()}
        assert set(ref) == set(got)


def test_conditioner_refusals(tmp_path, stub_tokenizer):
    from stable_audio_tools.models.conditioners import CLAPTextConditioner
    path, _ = _tmp_checkpoint(tmp_path, dict(SMALL_768, num_hidden_layers=1), 83)
    with pytest.raises(NotImplementedError, match="text_projection"):
        CLAPTextConditioner(768, clap_ckpt_path=path, use_text_features=False)
    with pytest.raises(NotImplementedError, match="inference only"):
        CLAPTextConditioner(768, clap_ckpt_path=path, use_text_features=True, finetune=True)
    # accepted and ignored: they only shape the audio branch
    c = CLAPTextConditioner(512, clap_ckpt_path=path, use_text_features=True, feature_layer_ix=-1,
                            audio_model_type="HTSAT-tiny", enable_fusion=False)
    assert isinstance(c.proj_out, torch.nn.Linear) and set(c.state_dict()) == {"proj_out.weight", "proj_out.bias"}
    with pytest.raises(ValueError):
        CLAPTextConditioner(768, clap_ckpt_path=path, use_text_features=True, feature_layer_ix=-3)


def test_encoder_refusals_before_any_cuda_call():
    from stable_audio_tools._native import NativeError
    from stable_audio_tools.models.roberta import RobertaEncoder, layers_to_run, prompt_lengths
    ok = dict(vocab_size=100, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512)
    RobertaEncoder(**ok)
    for bad in (dict(num_attention_heads=8), dict(hidden_size=192, num_attention_heads=3),
                dict(hidden_size=1152, num_attention_heads=18), dict(intermediate_size=48), dict(hidden_act="gelu_new"),
                dict(position_embedding_type="relative_key")):
        with pytest.raises(NotImplementedError):
            RobertaEncoder(**dict(ok, **bad))
    with pytest.raises(ValueError):
        RobertaEncoder(**ok, operand_dtype="fp8")
    assert [layers_to_run(12, i) for i in (-1, -2, 0, 12, -13)] == [12, 11, 0, 12, 0]
    for bad in (13, -14):
        with pytest.raises(ValueError):
            layers_to_run(12, bad)
    ids = torch.tensor([[5, 6, 7, 1], [9, 1, 1, 1]])
    mask = torch.tensor([[1, 1, 1, 0], [1, 0, 0, 0]])
    assert prompt_lengths(ids, mask, 10).tolist() == [3, 1]
    with pytest.raises(NotImplementedError):     # an empty prompt
        prompt_lengths(ids, torch.tensor([[1, 1, 1, 0], [0, 0, 0, 0]]), 10)
    with pytest.raises(NotImplementedError):     # left padding
        prompt_lengths(ids, torch.tensor([[0, 1, 1, 1], [1, 0, 0, 0]]), 10)
    with pytest.raises(NotImplementedError):
        prompt_lengths(torch.ones(1, 513, dtype=torch.long), torch.ones(1, 513, dtype=torch.long), 10)
    for bad in (-1, 10):
        b = ids.clone()
        b[0, 0] = bad
        with pytest.raises(ValueError):
            prompt_lengths(b, mask, 10)
    enc = RobertaEncoder(**ok)
    with pytest.raises(NativeError):
        enc(torch.zeros(1, 4, dtype=torch.long), torch.ones(1, 4, dtype=torch.long))
    with pytest.raises(NativeError):
        enc.load_state_dict({}, device="cpu")


def test_c_abi_refuses_bad_configs_and_foreign_probe_ids():
    from stable_audio_tools import _native
    lib = _native.lib()
    h = ctypes.c_void_p()
    good = dict(vocab_size=100, hidden_size=256, num_heads=4, intermediate_size=512, num_layers=1,
                max_position_embeddings=514, type_vocab_size=1, pad_token_id=1, layer_norm_eps=1e-5, operand_dtype=0)
    for bad, msg in ((dict(num_heads=2), b"head dim"), (dict(hidden_size=192, num_heads=3), b"hidden_size"),
                     (dict(intermediate_size=40), b"intermediate_size"), (dict(operand_dtype=2), b"operand_dtype"),
                     (dict(max_position_embeddings=2), b"pad_token_id")):
        rc = lib.satb_roberta_create(ctypes.byref(_native.SatbRobertaConfig(**dict(good, **bad))), ctypes.byref(h))
        assert rc != 0 and msg in lib.satb_last_error(), bad
    assert lib.satb_roberta_create(ctypes.byref(_native.SatbRobertaConfig(**good)), ctypes.byref(h)) == 0
    rc = lib.satb_roberta_encode(h, ctypes.c_void_p(1 << 20), (ctypes.c_int * 1)(3), 1, 4, ctypes.c_void_p(1 << 21), None)
    assert rc != 0 and b"finalize" in lib.satb_last_error()
    rc = lib.satb_roberta_finalize(h, None)
    assert rc != 0 and b"missing" in lib.satb_last_error()
    fake = ctypes.c_void_p(1 << 20)
    rc = lib.satb_roberta_load_weight(h, b"encoder.layer.1.output.dense.bias", fake, 256, None)
    assert rc != 0 and b"out of range" in lib.satb_last_error()
    rc = lib.satb_roberta_load_weight(h, b"pooler.dense.weight", fake, 256 * 256, None)
    assert rc != 0 and b"unknown RoBERTa weight key" in lib.satb_last_error()
    lib.satb_roberta_destroy(h)
    p = _native.SatbGemmProbe(epi=_native.EPI_BIAS_GELU16, bn=256, out=1 << 22, ld=256)
    for call in (lambda: lib.satb_gemm_probe(fake, fake, 64, 256, 64, ctypes.byref(p), None),
                 lambda: lib.satb_t5_gemm_probe(fake, fake, 64, 256, 64, ctypes.byref(p), None)):
        assert call() != 0 and b"no such instance" in lib.satb_last_error()
    p.epi = _native.EPI_RELU16
    rc = lib.satb_roberta_linear_probe(fake, fake, 64, 256, 64, ctypes.byref(p), None)
    assert rc != 0 and b"no such instance" in lib.satb_last_error()
    rc = lib.satb_roberta_attention_probe(fake, (ctypes.c_int * 2)(3, 0), 2, 4, 2, 0, fake, None)
    assert rc != 0 and b"[1, L]" in lib.satb_last_error()
