"""GPU: the token-sharded DiT forward (DiffusionTransformer.shard_tokens, satb_dit_group_*).

On one device the ranks are virtual (every rank a handle and a stream of its own on cuda:0), which runs the same split,
gather and event schedule as ranks on distinct GPUs; those add only the peer-to-peer reads, tested at the end when at
least two devices are visible.  For worlds 2, 3, 4 and 8, small models, two blocks and ragged lengths, across the
model options the sharded forward accepts:
  * the sharded output is within 1.25x of the operand-rounding floor of the fp32 oracle, the gate of the unsharded tests;
  * it matches the unsharded native forward within rel-L2 4e-3, the bound the suite accepts for a prompt against the
    same prompt inside a batch; whether it is bit-identical is reported (`CPGROUP {...}` lines, pytest -s).
A sampler run (dpmpp-3m-sde, CFG) with a sharded DiT matches the unsharded run within the same bound."""
import json

import pytest
import torch

from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, rel_l2

pytestmark = pytest.mark.gpu

SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer")

# name -> (config, operand dtype, forward kwargs beyond x, t, cross_attn_cond, global_embed)
CASES = {
    "prepend_cfg": (SMALL, "fp16", dict(cfg_scale=7.0)),
    "no_cfg": (SMALL, "fp16", dict(cfg_scale=1.0)),
    "adaln": (dict(SMALL, global_cond_type="adaLN"), "fp16", dict(cfg_scale=7.0)),
    "prepend_cond": (dict(SMALL, prepend_cond_dim=64), "fp16", dict(cfg_scale=5.0, prepend_tokens=3)),
    "qk_norm": (dict(SMALL, attn_kwargs=dict(qk_norm=True)), "fp16", dict(cfg_scale=7.0)),
    "hd32": (dict(SMALL, num_heads=8), "fp16", dict(cfg_scale=7.0)),
    "hd96": (dict(SMALL, embed_dim=384, global_cond_dim=384, project_cond_tokens=True), "fp16", dict(cfg_scale=7.0)),
    "hd128": (dict(SMALL, num_heads=2), "fp16", dict(cfg_scale=7.0)),
    "bf16": (SMALL, "bf16", dict(cfg_scale=7.0)),
    "fp8": (SMALL, "fp8", dict(cfg_scale=7.0)),
    "no_rotary": (dict(SMALL, rotary_pos_emb=False), "fp16", dict(cfg_scale=7.0)),
    "sinusoidal": (dict(SMALL, use_sinusoidal_emb=True), "fp16", dict(cfg_scale=7.0)),
    "absolute": (dict(SMALL, use_abs_pos_emb=True, abs_pos_emb_max_length=2048), "fp16", dict(cfg_scale=7.0)),
    "patch2": (dict(SMALL, patch_size=2), "fp16", dict(cfg_scale=7.0)),
    "input_concat": (dict(SMALL, input_concat_dim=1), "fp16", dict(cfg_scale=7.0, concat=True)),
    "negative_phi": (SMALL, "fp16", dict(cfg_scale=4.0, scale_phi=0.7, negative=True)),
}


def report(**kw):
    print("CPGROUP", json.dumps(kw))


def _floor_ctx(dtype):
    from oracle import dit_oracle as do
    if dtype == "fp8":
        return fp8_operands
    return lambda sdd: do.operand_rounding(torch.float16 if dtype == "fp16" else torch.bfloat16)


def _inputs(cfg, extra, L, seed):
    g = torch.Generator().manual_seed(seed)
    x, t = torch.randn(1, cfg["io_channels"], L, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 19, cfg["cond_token_dim"], generator=g), torch.randn(1, cfg["global_cond_dim"], generator=g)
    c[:, 12:] = 0.0
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=extra["cfg_scale"])
    if "scale_phi" in extra:
        kw["scale_phi"] = extra["scale_phi"]
    if extra.get("negative"):
        kw["negative_cross_attn_cond"] = torch.randn(1, 19, cfg["cond_token_dim"], generator=g)
    if extra.get("prepend_tokens"):
        kw["prepend_cond"] = torch.randn(1, extra["prepend_tokens"], cfg["prepend_cond_dim"], generator=g)
    if extra.get("concat"):
        kw["input_concat_cond"] = (torch.rand(1, 1, L, generator=g) > 0.5).float()
    return kw


_ORACLE = {}


def _oracle(case, L):
    """Weights, inputs, the fp32 oracle's output and the operand-rounding floor of one case (shared by the worlds)."""
    if (case, L) not in _ORACLE:
        from oracle import positions_oracle as po
        cfg, dtype, extra = CASES[case]
        sd = po.make_dit_weights(cfg, seed=91)
        kw = _inputs(cfg, extra, L, seed=92 + L)
        ref = po.dit_forward(sd, cfg, **kw)
        with _floor_ctx(dtype)(sd):
            floor = rel_l2(po.dit_forward(sd, cfg, **kw), ref)
        _ORACLE[(case, L)] = (sd, kw, ref, floor)
    return _ORACLE[(case, L)]


def _cuda(kw):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}


@pytest.mark.parametrize("L", [300, 1100])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("case", sorted(CASES))
def test_sharded_forward_vs_oracle_and_unsharded(case, world, L):
    cfg, dtype, extra = CASES[case]
    sd, kw, ref, floor = _oracle(case, L)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    y1 = m(**_cuda(kw)).cpu()
    m.shard_tokens(["cuda:0"] * world)
    yw = m(**_cuda(kw)).cpu()
    yw2 = m(**_cuda(kw)).cpu()           # a second call reuses the group's workspace and conditioning
    m.shard_tokens(None)
    y1b = m(**_cuda(kw)).cpu()           # and the single-device path is as before
    err_w, err_1, vs_1 = rel_l2(yw, ref), rel_l2(y1, ref), rel_l2(yw, y1)
    report(case=case, world=world, L=L, rel_l2_sharded=err_w, rel_l2_unsharded=err_1, floor=floor,
           sharded_vs_unsharded=vs_1, bit_identical=bool(torch.equal(yw, y1)))
    assert torch.equal(yw, yw2) and torch.equal(y1, y1b)
    assert err_w <= 1.25 * floor, (err_w, floor)
    assert vs_1 < 4e-3, vs_1


def test_sharded_generate_diffusion_cond_matches_unsharded():
    """generate_diffusion_cond (dpmpp-3m-sde, CFG 5, 6 steps, then the VAE decode) with a 3-way sharded DiT, against
    the same run unsharded, with the same initial and per-step noise."""
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
    latw, audiow = run()
    dit.shard_tokens(None)
    err, aerr = rel_l2(latw, lat1), rel_l2(audiow, audio1)
    report(case="generate_dpmpp_3m_sde", world=3, rel_l2_latents=err, rel_l2_audio=aerr,
           bit_identical=bool(torch.equal(latw, lat1)))
    assert err < 4e-3, err
    assert aerr < 4e-3, aerr


def _sa2_length_vs_oracle(devices):
    from oracle import dit_oracle as do
    cfg = dict(SAO_DIT, depth=2)
    sd = do.make_dit_weights(cfg, seed=24)
    g = torch.Generator().manual_seed(25)
    x, t = torch.randn(1, 64, 6144, generator=g), torch.tensor([0.3])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    yc = do.dit_inner_forward(sd, cfg, x, t, c, ge)
    yu = do.dit_inner_forward(sd, cfg, x, t, torch.zeros_like(c), ge)
    ref = yu + (yc - yu) * 7.0
    m = build_native_dit(cfg, sd).shard_tokens(devices)
    y = m(x.cuda(), t.cuda(), cross_attn_cond=c.cuda(), global_embed=ge.cuda(), cfg_scale=7.0).cpu()
    err = rel_l2(y, ref)
    report(case="sa2_length_2_blocks_cfg7", devices=[str(d) for d in devices], rel_l2=err)
    assert err < 2e-3 * 7.0 / 1.5, err


def _real_devices(n):
    if torch.cuda.device_count() < 2:
        pytest.skip(f"{torch.cuda.device_count()} CUDA device(s) visible: ranks on distinct GPUs need at least 2")
    return [f"cuda:{i}" for i in range(n)]


def test_sa2_length_dit_sharded_over_2_devices_vs_oracle():
    _sa2_length_vs_oracle(_real_devices(2))


def test_sa2_length_dit_sharded_over_every_device_vs_oracle():
    _sa2_length_vs_oracle(_real_devices(min(torch.cuda.device_count(), 8)))
