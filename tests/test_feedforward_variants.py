"""CPU: DiTs built with the reference's other feed-forward options (ff_kwargs: mult, no_bias, glu, use_conv;
reference models/transformer.py:211-287).

The oracle against golden outputs of the real reference (tests/golden/dit_ff_*.npz, oracle/make_golden_feedforward.py),
the package's parameter containers against the reference's stored state-dict layout, the JSON-config build, the
refusals, the stored inner width, and the C ABI's checks that need no GPU."""
import ctypes
import json

import pytest
import torch

from helpers import load_golden, max_abs, rel_l2
from oracle import dit_oracle as do
from oracle import feedforward_oracle as fo

FF_GOLDENS = ["dit_ff_mult83_small.npz", "dit_ff_glu_conv3_nobias_small.npz", "dit_ff_conv5_adaln_hd128_small.npz",
              "dit_ff_plain_nobias_hd32_small.npz", "dit_ff_conformer_conv3_small.npz"]
SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer")


def _golden_inputs(g):
    T = lambda k: torch.from_numpy(g[k])
    kw = dict(cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "prepend" in g:
        kw["prepend_cond"] = T("prepend")
    return T, kw


@pytest.mark.parametrize("name", FF_GOLDENS)
def test_oracle_matches_reference_feedforward_golden(name):
    """Gates of test_head_dims.py: 1e-6 without CFG, 1e-5 otherwise."""
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = fo.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), f"{name}: synthetic weight RNG drifted from the golden run"
    T, kw = _golden_inputs(g)
    x, t = T("x"), T("t")
    assert max_abs(fo.dit_forward(sd, cfg, x, t, cfg_scale=1.0, **kw), T("y_nocfg")) <= 1e-6
    assert max_abs(fo.dit_forward(sd, cfg, x, t, cfg_scale=7.0, **kw), T("y_cfg7")) <= 1e-5
    assert max_abs(fo.dit_forward(sd, cfg, x, t, cfg_scale=4.0, scale_phi=0.7, **kw), T("y_cfg4_phi")) <= 1e-5
    assert max_abs(fo.dit_forward(sd, cfg, x, t, negative_cross_attn_cond=T("neg"), cfg_scale=3.0, **kw), T("y_neg3")) <= 1e-5
    hs = []
    fo.dit_inner_forward(sd, cfg, x, t, kw["cross_attn_cond"], kw["global_embed"], hidden_states=hs,
                         prepend_cond=kw.get("prepend_cond"))
    assert max_abs(hs[-1], T("hidden_last")) <= 1e-5


@pytest.mark.parametrize("name", FF_GOLDENS)
def test_state_dict_keys_and_shapes_equal_the_stored_reference_list(name):
    from stable_audio_tools.models.dit import DiffusionTransformer
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    theirs = {k: tuple(s) for k, s in json.loads(str(g["keys"]))}
    mine = {k: tuple(v.shape) for k, v in DiffusionTransformer(**cfg).state_dict().items()}
    assert mine == theirs, sorted(set(mine.items()) ^ set(theirs.items()))[:10]
    want = {k: tuple(v) for k, v in fo.dit_param_shapes(cfg).items()}
    assert {k: v for k, v in mine.items() if not k.endswith("rotary_pos_emb.scale")} == want


def test_the_goldens_depend_on_the_feedforward_variant():
    """Running a golden's weights through the default SwiGLU feed-forward is impossible (other keys) and the token
    convolution matters: with its side taps zeroed the output moves far beyond the tolerances."""
    g = load_golden("dit_ff_conv5_adaln_hd128_small.npz")
    cfg = json.loads(str(g["cfg"]))
    sd = fo.make_dit_weights(cfg, seed=int(g["seed"]))
    center = {k: (v * (torch.arange(5) == 2) if v.dim() == 3 and ".ff.ff." in k else v) for k, v in sd.items()}
    T, kw = _golden_inputs(g)
    y = fo.dit_forward(center, cfg, T("x"), T("t"), cfg_scale=1.0, **kw)
    assert rel_l2(y, T("y_nocfg")) > 0.05


def test_default_feedforward_keeps_the_dit_oracle_and_its_weights():
    cfg = dict(SMALL, global_cond_type="prepend")
    sd = fo.make_dit_weights(cfg, seed=11)
    base = do.make_dit_weights(cfg, seed=11)
    assert set(sd) == set(base) and all(torch.equal(sd[k], v) for k, v in base.items())
    g = load_golden("dit_prepend_small.npz")
    T = lambda k: torch.from_numpy(g[k])
    y = fo.dit_forward(sd, cfg, T("x"), T("t"), T("cross"), T("glob"), cfg_scale=7.0)
    assert max_abs(y, T("y_cfg7")) <= 1e-5
    ff = do.feed_forward
    with fo.feedforward_variants():
        assert do.feed_forward is fo.feed_forward
    assert do.feed_forward is ff


def test_token_conv_equals_conv1d():
    torch.manual_seed(0)
    for k in (1, 3, 5, 7):
        x, w, b = torch.randn(3, 11, 16, dtype=torch.float64), torch.randn(24, 16, k, dtype=torch.float64), torch.randn(24, dtype=torch.float64)
        want = torch.nn.functional.conv1d(x.transpose(1, 2), w, b, padding=k // 2).transpose(1, 2)
        with do.operand_rounding(torch.float64):   # the unfolded Linear the operand emulation runs
            assert max_abs(fo.token_conv(x, w, b), want) < 1e-12


@pytest.mark.parametrize("dim,mult,inner,inner_p", [(1536, 8 / 3, 4096, 4096), (1024, 8 / 3, 2730, 2752),
                                                    (256, 8 / 3, 682, 704), (256, 2.5, 640, 640), (1536, 4, 6144, 6144),
                                                    (384, 2, 768, 768), (128, 0.01, 1, 64)])
def test_inner_dim_and_its_padding(dim, mult, inner, inner_p):
    from stable_audio_tools.models.transformer import FeedForward
    assert fo.inner_dim(dict(embed_dim=dim, ff_kwargs=dict(mult=mult))) == inner
    assert fo.padded_inner(inner) == inner_p
    assert FeedForward(dim, mult=mult).native_spec() == (inner, 1, 0, 1)


def test_padding_the_inner_width_is_exact():
    """Zero rows of FF-in (and zero bias entries), zero K-columns of FF-out: padded SwiGLU / plain columns are 0."""
    torch.manual_seed(1)
    D, inner = 64, 42
    ip = fo.padded_inner(inner)
    x = torch.randn(2, 9, D, dtype=torch.float64)
    for glu in (True, False):
        rows = 2 * inner if glu else inner
        w1, b1, w2 = torch.randn(rows, D, dtype=torch.float64), torch.randn(rows, dtype=torch.float64), torch.randn(D, inner, 3, dtype=torch.float64)
        pad = lambda t: torch.cat([t, t.new_zeros((ip - inner,) + t.shape[1:])])
        key = "ff.0.proj" if glu else "ff.0.1"
        sd = {key + ".weight": w1, key + ".bias": b1, "ff.2.weight": w2}
        if glu:
            v, gt = w1.chunk(2)
            bv, bg = b1.chunk(2)
            sdp = {key + ".weight": torch.cat([pad(v), pad(gt)]), key + ".bias": torch.cat([pad(bv), pad(bg)])}
        else:
            sdp = {key + ".weight": pad(w1), key + ".bias": pad(b1)}
        sdp["ff.2.weight"] = torch.cat([w2, w2.new_zeros(D, ip - inner, 3)], dim=1)
        assert max_abs(fo.feed_forward(x, sdp, ""), fo.feed_forward(x, sd, "")) < 1e-12


def test_create_model_from_config_builds_and_loads_a_feedforward_variant():
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.models.dit import DiffusionTransformer
    diff = dict(SMALL, ff_kwargs={"glu": False, "use_conv": True, "conv_kernel_size": 5, "mult": 2.5})
    model_config = {"model_type": "diffusion_cond", "sample_rate": 44100,
                    "model": {"io_channels": 64, "diffusion": {"type": "dit", "config": diff}}}
    m = create_model_from_config(json.loads(json.dumps(model_config)))
    dit = m.model.model
    assert isinstance(dit, DiffusionTransformer) and dit.ff_spec == (640, 0, 5, 1)
    sd = fo.make_dit_weights(diff, seed=5)
    missing, unexpected = dit.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    assert torch.equal(dit.transformer.layers[1].ff.ff[2].weight, sd["transformer.layers.1.ff.ff.2.weight"])
    assert tuple(dit.transformer.layers[0].ff.ff[0][1].weight.shape) == (640, 256, 5)


def test_default_model_does_not_set_a_feedforward_variant():
    from stable_audio_tools.models.dit import DiffusionTransformer
    assert DiffusionTransformer(**SMALL).ff_spec == (4 * 256, 1, 0, 1)
    assert DiffusionTransformer(**dict(SMALL, ff_kwargs={"mult": 4})).ff_spec == (1024, 1, 0, 1)
    assert DiffusionTransformer(**dict(SMALL, ff_kwargs={"no_bias": True})).ff_spec == (1024, 1, 0, 0)


@pytest.mark.parametrize("kw,match", [(dict(dim_out=128), "dim_out"), (dict(use_conv=True, conv_kernel_size=4), "odd"),
                                      (dict(use_conv=True, conv_kernel_size=0), "odd"),
                                      (dict(use_conv=True, conv_kernel_size=-3), "odd"), (dict(mult=0.001), "inner")])
def test_host_refusals(kw, match):
    from stable_audio_tools.models.dit import DiffusionTransformer
    with pytest.raises(NotImplementedError, match=match):
        DiffusionTransformer(**dict(SMALL, ff_kwargs=kw))


def test_even_kernel_size_without_use_conv_is_unused_and_accepted():
    from stable_audio_tools.models.transformer import FeedForward
    assert FeedForward(256, conv_kernel_size=4).native_spec() == (1024, 1, 0, 1)


def _create(embed_dim=256, num_heads=4, operand_dtype=0):
    from stable_audio_tools import _native
    lib = _native.lib()
    cfg = _native.SatbDitConfig(io_channels=64, embed_dim=embed_dim, depth=2, num_heads=num_heads, cond_token_dim=128,
                                global_cond_dim=embed_dim, project_cond_tokens=0, project_global_cond=1,
                                global_cond_type=0, patch_size=1, operand_dtype=operand_dtype)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    return lib, h


@pytest.mark.parametrize("args,match", [((682, 1, 4, 1), b"odd"), ((682, 0, -1, 1), b"conv_kernel_size"),
                                        ((0, 1, 0, 1), b"inner dim"), ((682, 2, 0, 1), b"glu"),
                                        ((682, 1, 0, 3), b"bias"), ((1 << 30, 1, 3, 1), b"too large")])
def test_native_set_feedforward_refuses_bad_values(args, match):
    lib, h = _create()
    try:
        assert lib.satb_dit_set_feedforward(h, *args) != 0 and match in lib.satb_last_error()
        assert lib.satb_dit_set_feedforward(h, 682, 1, 3, 0) == 0
    finally:
        lib.satb_dit_destroy(h)


@pytest.mark.parametrize("args,missing", [
    ((682, 1, 0, 1), [b"ff.ff.0.proj.weight", b"ff.ff.0.proj.bias", b"ff.ff.2.weight", b"ff.ff.2.bias"]),
    ((512, 0, 3, 0), [b"ff.ff.0.1.weight", b"ff.ff.2.weight"]),
    ((512, 0, 0, 1), [b"ff.ff.0.1.weight", b"ff.ff.0.1.bias", b"ff.ff.2.weight", b"ff.ff.2.bias"])])
@pytest.mark.parametrize("operand_dtype", [0, 2])
def test_native_finalize_names_the_missing_feedforward_keys(args, missing, operand_dtype):
    lib, h = _create(operand_dtype=operand_dtype)
    try:
        assert lib.satb_dit_set_feedforward(h, *args) == 0
        assert lib.satb_dit_finalize(h, None) != 0
        msg = lib.satb_last_error()
        assert b"feed-forward weights missing in layer 0" in msg
        for k in missing:
            assert b"transformer.layers.0." + k in msg
        assert (b".bias" in msg) == any(k.endswith(b".bias") for k in missing)
    finally:
        lib.satb_dit_destroy(h)


def test_native_load_refuses_keys_of_another_variant_before_any_cuda_call():
    lib, h = _create()
    try:
        assert lib.satb_dit_set_feedforward(h, 512, 0, 3, 0) == 0
        fake = 1 << 20
        for key in (b"transformer.layers.0.ff.ff.0.proj.weight", b"transformer.layers.0.ff.ff.2.bias",
                    b"transformer.layers.0.ff.ff.0.1.bias"):
            assert lib.satb_dit_load_weight(h, key, fake, 10, None) == -4
            assert b"feed-forward variant" in lib.satb_last_error()
        assert lib.satb_dit_load_weight(h, b"transformer.layers.0.ff.ff.2.weight", fake, 10, None) != 0
        assert b"bad size" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


def test_token_conv_probe_validates_before_any_cuda_call():
    from stable_audio_tools import _native as nat
    lib = nat.lib()
    fake = 1 << 20
    p = nat.SatbGemmProbe(epi=nat.EPI_STORE16, bn=0, out=fake, ld=256)
    call = lambda **kw: lib.satb_token_conv_probe(kw.get("a", fake), kw.get("stride", 40), fake, 2, 33, 256,
                                                   kw.get("N", 256), kw.get("k", 3), ctypes.byref(kw.get("p", p)), None)
    assert call(k=4) != 0 and b"odd" in lib.satb_last_error()
    assert call(stride=32) != 0 and b"item_stride" in lib.satb_last_error()
    assert call(a=fake + 8) != 0 and b"aligned" in lib.satb_last_error()
    assert call(N=48) != 0 and b"N % 32" in lib.satb_last_error()
    assert call(p=nat.SatbGemmProbe(epi=nat.EPI_SWIGLU, bn=256, out=fake, ld=256)) != 0
    assert b"store16 and residual" in lib.satb_last_error()
    assert call(p=nat.SatbGemmProbe(epi=nat.EPI_STORE16, bn=64, out=fake, ld=256)) != 0
    assert b"bn must be" in lib.satb_last_error()
