"""CPU: DiTs built with conformer blocks (reference models/transformer.py:557-591, conformer=True).

The oracle against golden outputs of the real reference (tests/golden/dit_conformer*.npz, oracle/make_golden_conformer.py),
the existing goldens unchanged, the package's parameter containers against the reference's state-dict layout, the
refusals that stay, and the C ABI's checks that need no GPU."""
import ctypes
import json

import pytest
import torch

from helpers import load_golden, max_abs, rel_l2
from oracle import conformer_oracle as co
from oracle import dit_oracle as do

CONFORMER_GOLDENS = ["dit_conformer_small.npz", "dit_conformer_adaln_small.npz", "dit_conformer_hd128_small.npz"]
CONFORMER_KEYS = {"in_norm.gamma": lambda D: (D,), "in_norm.beta": lambda D: (D,),
                  "pointwise_conv.weight": lambda D: (D, D, 1), "glu.proj.weight": lambda D: (2 * D, D),
                  "glu.proj.bias": lambda D: (2 * D,), "depthwise_conv.weight": lambda D: (D, 1, 17),
                  "mid_norm.gamma": lambda D: (D,), "mid_norm.beta": lambda D: (D,),
                  "pointwise_conv_2.weight": lambda D: (D, D, 1)}
SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer", conformer=True)


def _check_golden(name, tol_nocfg=1e-5):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = co.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), f"{name}: synthetic weight RNG drifted from the golden run"
    T = lambda k: torch.from_numpy(g[k])
    x, t, c, ge, neg = T("x"), T("t"), T("cross"), T("glob"), T("neg")
    assert max_abs(co.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=1.0), T("y_nocfg")) <= tol_nocfg
    assert max_abs(co.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=7.0), T("y_cfg7")) <= 1e-5
    assert max_abs(co.dit_forward(sd, cfg, x, t, c, ge, cfg_scale=4.0, scale_phi=0.7), T("y_cfg4_phi")) <= 1e-5
    assert max_abs(co.dit_forward(sd, cfg, x, t, c, ge, negative_cross_attn_cond=neg, cfg_scale=3.0), T("y_neg3")) <= 1e-5
    hs = []
    co.dit_inner_forward(sd, cfg, x, t, c, ge, hidden_states=hs)
    assert max_abs(hs[-1], T("hidden_last")) <= 1e-5
    return cfg, sd


@pytest.mark.parametrize("name", CONFORMER_GOLDENS)
def test_oracle_matches_reference_conformer_golden(name):
    cfg, sd = _check_golden(name)
    assert cfg["conformer"] is True
    assert sum(".conformer." in k for k in sd) == 9 * cfg["depth"]
    assert sd["transformer.layers.0.conformer.pointwise_conv_2.weight"].abs().max() > 0   # branch not zero-initialised


@pytest.mark.parametrize("name", ["dit_prepend_small.npz", "dit_adaln_small.npz", "dit_hd128_small.npz",
                                  "dit_hd96_small.npz", "dit_hd32_small.npz", "dit_hd128_adaln_small.npz"])
def test_oracle_still_matches_the_goldens_without_conformer(name):
    """conformer_oracle draws conformer tensors only when asked and runs dit_oracle's own block where there are none:
    every other config keeps its weights (checksum) and outputs."""
    cfg, sd = _check_golden(name, tol_nocfg=1e-6)
    assert not any(".conformer." in k for k in sd)


def test_conformer_weights_extend_the_dit_oracle_weights_bit_for_bit():
    cfg = dict(SMALL, global_cond_type="adaLN")
    base = do.make_dit_weights(cfg, seed=41)
    sd = co.make_dit_weights(cfg, seed=41)
    assert set(sd) == set(base) | set(co.conformer_param_shapes(cfg)) and len(sd) == len(base) + 9 * cfg["depth"]
    assert all(torch.equal(sd[k], v) for k, v in base.items())
    block = do.transformer_block
    with co.conformer_blocks():
        assert do.transformer_block is co.transformer_block
    assert do.transformer_block is block     # dit_oracle's own block is back after the context


def test_conformer_branch_changes_the_output():
    """The golden is sensitive to the branch: dropping it moves the output far beyond the tolerances."""
    g = load_golden("dit_conformer_small.npz")
    cfg = json.loads(str(g["cfg"]))
    sd = co.make_dit_weights(cfg, seed=int(g["seed"]))
    plain = {k: v for k, v in sd.items() if ".conformer." not in k}
    T = lambda k: torch.from_numpy(g[k])
    y = co.dit_forward(plain, cfg, T("x"), T("t"), T("cross"), T("glob"), cfg_scale=1.0)
    assert rel_l2(y, T("y_nocfg")) > 0.05


def test_operand_rounding_folds_the_pointwise_conv_into_the_glu():
    """Under operand_rounding the oracle runs pointwise_conv and glu.proj as one fp64-folded Linear (as csrc/dit.cu
    does); the fold itself is exact up to fp32 rounding."""
    torch.manual_seed(0)
    D, N = 128, 40
    sd = {k: torch.randn(f(D)) * 0.1 for k, f in CONFORMER_KEYS.items()}
    x = torch.randn(2, N, D)
    ref = co.conformer_module(x.double(), {k: v.double() for k, v in sd.items()}, "")
    with do.operand_rounding(torch.float32):   # the fold with no 16-bit rounding
        folded = co.conformer_module(x, sd, "")
    assert rel_l2(folded, ref) < 1e-5


def test_state_dict_keys_and_shapes_match_the_reference_layout():
    """Key for key what make_dit_weights draws, which the golden generator loads strictly into the reference's
    DiffusionTransformer."""
    from stable_audio_tools.models.dit import DiffusionTransformer
    for gtype in ("prepend", "adaLN"):
        cfg = dict(SMALL, global_cond_type=gtype)
        mine = {k: tuple(v.shape) for k, v in DiffusionTransformer(**cfg).state_dict().items()
                if not k.endswith("rotary_pos_emb.scale")}
        want = {k: tuple(v) for k, v in co.dit_param_shapes(cfg).items()}
        assert mine == want, sorted(set(mine) ^ set(want))[:10]
        for i in range(cfg["depth"]):
            for k, f in CONFORMER_KEYS.items():
                assert mine[f"transformer.layers.{i}.conformer.{k}"] == f(256)


@pytest.mark.reference
def test_state_dict_keys_and_shapes_equal_the_real_reference():
    from oracle import ref_shims
    from stable_audio_tools.models.dit import DiffusionTransformer
    ref = ref_shims.import_reference()
    for gtype in ("prepend", "adaLN"):
        cfg = dict(SMALL, global_cond_type=gtype)
        theirs = {k: tuple(v.shape) for k, v in ref.dit.DiffusionTransformer(**cfg).state_dict().items()}
        mine = {k: tuple(v.shape) for k, v in DiffusionTransformer(**cfg).state_dict().items()}
        assert mine == theirs


def test_create_model_from_config_builds_a_conformer_dit():
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.dit import DiffusionTransformer
    diff = {k: v for k, v in SMALL.items()}
    model_config = {"model_type": "diffusion_cond", "sample_rate": 44100,
                    "model": {"io_channels": 64, "diffusion": {"type": "dit", "config": diff}}}
    m = create_model_from_config(json.loads(json.dumps(model_config)))
    dit = m.model.model
    assert isinstance(dit, DiffusionTransformer) and dit.conformer
    sd = {k[len("model.model."):]: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("model.model.")}
    want = {k: tuple(v) for k, v in co.dit_param_shapes(SMALL).items()}
    assert {k: v for k, v in sd.items() if not k.endswith("rotary_pos_emb.scale")} == want


def test_remove_norms_is_still_refused():
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError, match="norm-free"):
        DiffusionTransformer(**dict(SMALL, remove_norms=True))
    with pytest.raises(NotImplementedError, match="norm-free"):
        DiffusionTransformer(**dict(SMALL, conformer=False, remove_norms=True))


def test_conformer_wider_than_the_kernel_is_refused_on_the_host():
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError, match="conformer"):
        DiffusionTransformer(**dict(SMALL, embed_dim=2048, num_heads=32, global_cond_dim=2048))


def _create(embed_dim=256, num_heads=4):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbDitConfig(io_channels=64, embed_dim=embed_dim, depth=2, num_heads=num_heads, cond_token_dim=128,
                                global_cond_dim=embed_dim, project_cond_tokens=0, project_global_cond=1,
                                global_cond_type=0, patch_size=1, operand_dtype=0)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return lib, h


def test_native_finalize_without_the_conformer_tensors_fails_with_a_message():
    lib, h = _create()
    try:
        assert lib.satb_dit_set_conformer(h, 1) == 0
        rc = lib.satb_dit_finalize(h, None)
        msg = lib.satb_last_error()
        assert rc != 0 and b"conformer weights missing in layer 0" in msg and b"depthwise_conv.weight" in msg
    finally:
        lib.satb_dit_destroy(h)


def test_native_set_conformer_checks_the_width():
    lib, h = _create(2048, 32)
    try:
        assert lib.satb_dit_set_conformer(h, 1) != 0 and b"1536" in lib.satb_last_error()
        assert lib.satb_dit_set_conformer(h, 0) == 0
    finally:
        lib.satb_dit_destroy(h)


def test_conformer_kernel_entry_point_validates_before_any_cuda_call():
    from stable_audio_tools import _native
    lib = _native.lib()
    fake = 1 << 20
    assert lib.satb_conformer_dwconv(fake, fake, fake, fake, fake, 1, 5, 1664, 0, None) != 0
    assert b"1536" in lib.satb_last_error()
    assert lib.satb_conformer_dwconv(fake + 8, fake, fake, fake, fake, 1, 5, 256, 0, None) != 0
    assert b"aligned" in lib.satb_last_error()
    assert lib.satb_conformer_dwconv(fake, fake, fake, fake, fake, 0, 5, 256, 0, None) != 0
    assert b"empty" in lib.satb_last_error()
