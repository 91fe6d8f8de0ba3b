"""CPU: DiTs built with the reference's positional options (ContinuousTransformer rotary_pos_emb, use_sinusoidal_emb,
use_abs_pos_emb / abs_pos_emb_max_length; reference models/transformer.py:50-96, 705-809).

The oracle against golden outputs of the real reference (tests/golden/dit_pos_*.npz, oracle/make_golden_positions.py),
the package's parameter containers against the reference's stored state-dict layout and buffers, the JSON-config
build, the host refusals and the C ABI's checks that need no GPU."""
import ctypes
import json

import pytest
import torch

from helpers import load_golden, max_abs, rel_l2
from oracle import dit_oracle as do
from oracle import positions_oracle as po

POS_GOLDENS = ["dit_pos_sin_small.npz", "dit_pos_abs_prepcond_small.npz", "dit_pos_norope_abs_adaln_hd128_small.npz",
               "dit_pos_norope_qknorm_small.npz", "dit_pos_sin_conformer_patch2_conv3_small.npz"]
SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer")


def _golden_inputs(g):
    T = lambda k: torch.from_numpy(g[k])
    kw = dict(cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "prepend" in g:
        kw["prepend_cond"] = T("prepend")
    return T, kw


@pytest.mark.parametrize("name", POS_GOLDENS)
def test_oracle_matches_reference_positions_golden(name):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = po.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), f"{name}: synthetic weight RNG drifted from the golden run"
    T, kw = _golden_inputs(g)
    x, t = T("x"), T("t")
    assert max_abs(po.dit_forward(sd, cfg, x, t, cfg_scale=1.0, **kw), T("y_nocfg")) <= 1e-5
    assert max_abs(po.dit_forward(sd, cfg, x, t, cfg_scale=7.0, **kw), T("y_cfg7")) <= 1e-5
    assert max_abs(po.dit_forward(sd, cfg, x, t, cfg_scale=4.0, scale_phi=0.7, **kw), T("y_cfg4_phi")) <= 1e-5
    assert max_abs(po.dit_forward(sd, cfg, x, t, negative_cross_attn_cond=T("neg"), cfg_scale=3.0, **kw), T("y_neg3")) <= 1e-5
    hs = []
    po.dit_inner_forward(sd, cfg, x, t, kw["cross_attn_cond"], kw["global_embed"], hidden_states=hs,
                         prepend_cond=kw.get("prepend_cond"))
    assert max_abs(hs[-1], T("hidden_last")) <= 1e-5


@pytest.mark.parametrize("name", POS_GOLDENS)
def test_state_dict_keys_and_shapes_equal_the_stored_reference_list(name):
    from stable_audio_tools.models.dit import DiffusionTransformer
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    theirs = {k: tuple(s) for k, s in json.loads(str(g["keys"]))}
    mine = {k: tuple(v.shape) for k, v in DiffusionTransformer(**cfg).state_dict().items()}
    assert mine == theirs, sorted(set(mine.items()) ^ set(theirs.items()))[:10]
    want = {k: tuple(v) for k, v in po.dit_param_shapes(cfg).items()}
    assert {k: v for k, v in mine.items() if not k.endswith("rotary_pos_emb.scale")} == want


@pytest.mark.parametrize("name", POS_GOLDENS)
def test_the_positional_term_moves_every_golden(name):
    """The embedding zeroed (or, for the fixture without one, rotary switched back on) moves the reference output.
    With an embedding the move is far beyond the GPU tolerances (fp16 rel-L2 2e-3 x max(1, cfg / 1.5), bf16 1.5e-2).
    In the qk_norm fixture the attention logits are cosines / 8, at most 0.125 in size, so rotation can only move its
    output by a little: there it is above the fp16 gate, and the rotary-off path is pinned far more strongly by the
    head-dim-128 fixture (rotary on moves its output by 25 %)."""
    g = load_golden(name)
    move = rel_l2(torch.from_numpy(g["y_nopos"]), torch.from_numpy(g["y_nocfg"]))
    assert move > (0.15 if "qknorm" not in name else 2e-3), move


@pytest.mark.parametrize("name", ["dit_pos_sin_small.npz", "dit_pos_sin_conformer_patch2_conv3_small.npz"])
def test_sinusoid_inv_freq_is_the_reference_buffer_bit_for_bit(name):
    from stable_audio_tools.models.dit import DiffusionTransformer
    g = load_golden(name)
    m = DiffusionTransformer(**json.loads(str(g["cfg"])))
    pe = m.transformer.pos_emb
    assert torch.equal(pe.inv_freq, torch.from_numpy(g["pos_inv_freq"]))
    assert torch.equal(po.sinusoid_inv_freq(256), pe.inv_freq)
    assert "transformer.pos_emb.inv_freq" not in m.state_dict()
    assert isinstance(pe.scale, torch.nn.Parameter) and pe.scale.shape == (1,)


def test_containers_and_the_native_arguments():
    from stable_audio_tools.models.dit import DiffusionTransformer
    from stable_audio_tools.models.transformer import AbsolutePositionalEmbedding
    assert DiffusionTransformer(**SMALL).pos_spec == (1, 0, 0)
    m = DiffusionTransformer(**dict(SMALL, rotary_pos_emb=False))
    assert m.pos_spec == (0, 0, 0) and m.transformer.rotary_pos_emb is None
    assert not any("rotary" in k for k in m.state_dict())
    assert DiffusionTransformer(**dict(SMALL, use_sinusoidal_emb=True)).pos_spec == (1, 1, 0)
    m = DiffusionTransformer(**dict(SMALL, use_abs_pos_emb=True, rotary_pos_emb=False))
    assert m.pos_spec == (0, 2, 10000)
    assert isinstance(m.transformer.pos_emb, AbsolutePositionalEmbedding)
    assert m.state_dict()["transformer.pos_emb.emb.weight"].shape == (10000, 256)
    assert m.transformer.pos_emb.scale == 256 ** -0.5


def test_create_model_from_config_halves_the_position_parameters():
    """DiTWrapper multiplies every parameter by 0.5 (reference diffusion.py:487-489): pos_emb.scale and emb.weight
    are Parameters, the sinusoid's inv_freq is a buffer and keeps its values."""
    from stable_audio_tools import create_model_from_config
    for extra, key in ((dict(use_sinusoidal_emb=True), "scale"), (dict(use_abs_pos_emb=True, abs_pos_emb_max_length=64),
                                                                    "emb.weight")):
        diff = dict(SMALL, **extra)
        model_config = {"model_type": "diffusion_cond", "sample_rate": 44100,
                        "model": {"io_channels": 64, "diffusion": {"type": "dit", "config": diff}}}
        torch.manual_seed(0)
        dit = create_model_from_config(json.loads(json.dumps(model_config))).model.model
        pe = dit.transformer.pos_emb
        if key == "scale":
            assert torch.equal(pe.scale.detach(), torch.full((1,), 0.5 * 256 ** -0.5))
            assert torch.equal(pe.inv_freq, po.sinusoid_inv_freq(256))
        else:
            torch.manual_seed(0)
            fresh = type(dit)(**diff).transformer.pos_emb.emb.weight.detach()
            assert pe.emb.weight.shape == (64, 256) and torch.equal(pe.emb.weight.detach(), 0.5 * fresh)


def test_both_embeddings_raise_the_reference_assertion():
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(AssertionError, match="Can't select both"):
        DiffusionTransformer(**dict(SMALL, use_sinusoidal_emb=True, use_abs_pos_emb=True))


def test_causal_stays_refused():
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError, match="causal"):
        DiffusionTransformer(**dict(SMALL, causal=True))


@pytest.mark.parametrize("gtype,patch,n_prepend,max_len,L_ok", [
    ("prepend", 1, 0, 40, 39),     # 39 latents + the global token fill 40 positions
    ("prepend", 1, 3, 40, 36),     # + 3 prepend-conditioning tokens
    ("adaLN", 1, 0, 40, 40),       # no prepended token
    ("prepend", 2, 0, 40, 78),     # positions count patched tokens
])
def test_absolute_length_overflow_raises_assertion_before_the_cuda_check(gtype, patch, n_prepend, max_len, L_ok):
    from stable_audio_tools import _native
    from stable_audio_tools.models.dit import DiffusionTransformer
    cfg = dict(SMALL, global_cond_type=gtype, patch_size=patch, use_abs_pos_emb=True, abs_pos_emb_max_length=max_len)
    if n_prepend:
        cfg["prepend_cond_dim"] = 32
    m = DiffusionTransformer(**cfg)
    kw = dict(prepend_cond=torch.randn(1, n_prepend, 32)) if n_prepend else {}
    with pytest.raises(_native.NativeError, match="CUDA"):
        m(torch.randn(1, 64, L_ok), torch.rand(1), **kw)
    with pytest.raises(AssertionError, match="max sequence length of 40"):
        m(torch.randn(1, 64, L_ok + patch), torch.rand(1), **kw)


def test_positions_oracle_leaves_the_dit_oracle_in_place():
    ct = do.continuous_transformer
    with po.positions():
        assert do.continuous_transformer is po.continuous_transformer
    assert do.continuous_transformer is ct
    cfg = dict(SMALL, global_cond_type="prepend")
    base = do.make_dit_weights(cfg, seed=11)
    sd = po.make_dit_weights(cfg, seed=11)
    assert set(sd) == set(base) and all(torch.equal(sd[k], v) for k, v in base.items())


def _create():
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbDitConfig(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128,
                                global_cond_dim=256, project_cond_tokens=0, project_global_cond=1,
                                global_cond_type=0, patch_size=1, operand_dtype=0)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return lib, h


@pytest.mark.parametrize("args,match", [((2, 0, 0), b"rotary must be"), ((1, 3, 0), b"pos_type"),
                                        ((1, -1, 0), b"pos_type"), ((1, 2, 0), b"abs_max_len"),
                                        ((1, 1, 10), b"abs_max_len"), ((0, 0, 5), b"abs_max_len"),
                                        ((1, 2, 1 << 30), b"too large")])
def test_native_set_positions_refuses_bad_values(args, match):
    lib, h = _create()
    try:
        assert lib.satb_dit_set_positions(h, *args) != 0 and match in lib.satb_last_error()
        assert lib.satb_dit_set_positions(h, 0, 2, 40) == 0
    finally:
        lib.satb_dit_destroy(h)


def test_native_set_positions_refuses_a_call_after_a_weight_load():
    lib, h = _create()
    try:
        # a load attempt (refused for its size before any CUDA call) already fixes the handle's key set
        assert lib.satb_dit_load_weight(h, b"transformer.project_in.weight", 1 << 20, 10, None) != 0
        assert lib.satb_dit_set_positions(h, 0, 1, 0) != 0
        assert b"before the first weight" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


@pytest.mark.parametrize("args,missing", [((1, 1, 0), [b"transformer.pos_emb.scale", b"transformer.pos_emb.inv_freq"]),
                                          ((0, 2, 300), [b"transformer.pos_emb.emb.weight"])])
def test_native_finalize_names_the_missing_position_keys(args, missing):
    lib, h = _create()
    try:
        assert lib.satb_dit_set_positions(h, *args) == 0
        assert lib.satb_dit_finalize(h, None) != 0
        msg = lib.satb_last_error()
        assert all(k in msg for k in missing), msg
    finally:
        lib.satb_dit_destroy(h)


def test_native_load_refuses_the_keys_of_another_position_variant():
    lib, h = _create()
    try:
        assert lib.satb_dit_set_positions(h, 0, 2, 300) == 0
        fake = 1 << 20
        for key in (b"transformer.rotary_pos_emb.inv_freq", b"transformer.pos_emb.scale",
                    b"transformer.pos_emb.inv_freq"):
            assert lib.satb_dit_load_weight(h, key, fake, 10, None) == -4
            assert b"unknown DiT weight key" in lib.satb_last_error()
        assert lib.satb_dit_load_weight(h, b"transformer.pos_emb.emb.weight", fake, 10, None) != 0
        assert b"bad size" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


def test_store32_pos_probe_validates_before_any_cuda_call():
    from stable_audio_tools import _native as nat
    lib = nat.lib()
    fake = 1 << 20
    p = nat.SatbGemmProbe(epi=nat.EPI_STORE32_POS, bn=256, out=fake, ld=256, seq_len=0, pos_tab=fake)
    assert lib.satb_gemm_probe(fake, fake, 100, 256, 64, ctypes.byref(p), None) != 0
    assert b"store32_pos" in lib.satb_last_error()
    p = nat.SatbGemmProbe(epi=nat.EPI_STORE32_POS, bn=64, out=fake, ld=256, seq_len=7, pos_tab=fake)
    assert lib.satb_gemm_probe(fake, fake, 100, 256, 64, ctypes.byref(p), None) != 0
    assert b"no such instance" in lib.satb_last_error()
