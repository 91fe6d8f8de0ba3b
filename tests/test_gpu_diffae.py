"""GPU: diffusion autoencoders and the fused v-diffusion step (satb_vdiffusion_update).

1. The kernel alone against torch fp32 evaluating the reference's expressions on the same device and inputs, bit for
   bit: with and without noise, intermediate and last steps (the last writes pred only), odd element counts, the
   scalars of a real 100-step schedule.  Outputs are pre-filled with NaN.
2. DiffusionAutoencoder.decode / encode through the native path (DiT as CUDA-graph replays, the fused update, PQMF /
   Oobleck pretransforms) against oracle/diffae_oracle.py with the same start noise, on the three golden models and on
   a DiT of SA-Open width over 16-band PQMF sub-bands.  Gate: rel-L2 within 1.25 x of the oracle's own fp16-operand
   floor (dit_oracle / oobleck_oracle operand_rounding) carried through the same steps, as test_gpu_baseline_size.py
   gates the DiT; the encoder within 2 x of its floor, as the Oobleck tests do.
3. Bit checks: a graph-replayed decode equals an eager one; a batch of 2 equals the same items inside a batch of 3.
Measured numbers are printed as `DIFFAE {...}` JSON lines (pytest -s)."""
import json

import pytest
import torch

from helpers import load_golden, rel_l2

pytestmark = pytest.mark.gpu

GOLDENS = ["diffae_raw_small.npz", "diffae_pqmf16_small.npz", "diffae_aepre_small.npz"]


def report(name, **kw):
    print("DIFFAE " + json.dumps(dict(test=name, **kw)), flush=True)


# ------------------------------------------------------------------------------------------------ 1. the kernel
def _torch_step(x, v, nz, a, s, an, adj, dd):
    pred = x * a - v * s
    if an is None:
        return None, pred
    eps = x * s + v * a
    xn = pred * an + eps * adj
    if nz is not None:
        xn += nz * dd
    return xn, None


@pytest.mark.parametrize("n", [1, 3, 1029, 64 * 4099, 2 * 32 * 8192 + 5])
@pytest.mark.parametrize("step", [0, 1, 50, 98, 99])
@pytest.mark.parametrize("with_noise", [False, True])
def test_vdiffusion_update_equals_torch_fp32_bit_for_bit(n, step, with_noise):
    from stable_audio_tools import _native as nat
    from stable_audio_tools.inference.sampling import vdiffusion_schedule
    t, a, s, an, adj, dd = vdiffusion_schedule(100, 0.7 if with_noise else 0)[step]
    g = torch.Generator(device="cuda").manual_seed(n + step)
    x, v, nz = (torch.randn(n, device="cuda", generator=g) * 3 for _ in range(3))
    nz = nz if (with_noise and an is not None) else None
    last = an is None
    x_next = None if last else torch.full_like(x, float("nan"))
    pred = torch.full_like(x, float("nan")) if last else None
    nat.check(nat.lib().satb_vdiffusion_update(nat.ptr(x), nat.ptr(v), nat.ptr(nz), nat.ptr(x_next), nat.ptr(pred), n,
                                               a, s, an or 0.0, adj or 0.0, dd or 0.0, nat.stream_ptr()))
    want_x, want_pred = _torch_step(x, v, nz, a, s, an, adj, dd)
    got = pred if last else x_next
    want = want_pred if last else want_x
    assert torch.equal(got, want), float((got - want).abs().max())


def test_vdiffusion_update_writes_both_outputs_when_asked():
    from stable_audio_tools import _native as nat
    from stable_audio_tools.inference.sampling import vdiffusion_schedule
    _, a, s, an, adj, dd = vdiffusion_schedule(10, 0.5)[3]
    x, v, nz = (torch.randn(777, device="cuda") for _ in range(3))
    x_next, pred = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
    nat.check(nat.lib().satb_vdiffusion_update(nat.ptr(x), nat.ptr(v), nat.ptr(nz), nat.ptr(x_next), nat.ptr(pred), 777,
                                               a, s, an, adj, dd, nat.stream_ptr()))
    assert torch.equal(pred, x * a - v * s)
    assert torch.equal(x_next, _torch_step(x, v, nz, a, s, an, adj, dd)[0])


def test_sample_on_cuda_equals_sample_on_cpu_for_a_torch_model():
    """The fused path (any CUDA fp32 state) and the torch path give the same bits when the model does."""
    from stable_audio_tools.inference.sampling import sample
    g = torch.Generator().manual_seed(9)
    x0, noise = torch.randn(2, 3, 301, generator=g), torch.randn(11, 2, 3, 301, generator=g)

    def model(x, t):
        return torch.tanh(x * 0.5) + t[:, None, None] * 0.25

    cpu = sample(model, x0, 12, 0.4, noise_sampler=lambda i: noise[i])
    gpu = sample(model, x0.cuda(), 12, 0.4, noise_sampler=lambda i: noise[i].cuda())
    # tanh may differ between the CPU and CUDA libraries; the update itself must not add any difference
    v_gap = float((torch.tanh(x0.cuda() * 0.5).cpu() - torch.tanh(x0 * 0.5)).abs().max())
    report("cuda_vs_cpu_torch_model", max_abs=float((gpu.cpu() - cpu).abs().max()), tanh_gap=v_gap)
    if v_gap == 0.0:
        assert torch.equal(gpu.cpu(), cpu)
    else:
        assert float((gpu.cpu() - cpu).abs().max()) < 1e-4


# ------------------------------------------------------------------------------------------------ 2. end to end
def _golden_model(name):
    from oracle import diffae_oracle as dao
    from stable_audio_tools import create_model_from_config
    g = load_golden(name)
    cfg = json.loads(str(g["config"]))
    bufs = {k: torch.from_numpy(g[k]) for k in ("filter_bank", "prototype") if k in g}
    sd = dao.make_state_dict(cfg, int(g["seed"]), bufs or None)
    model = create_model_from_config(cfg)
    model.load_state_dict(sd, strict=True)
    return g, cfg, sd, model.cuda().eval()


def _floors(fn):
    from oracle import dit_oracle as do
    from oracle import oobleck_oracle as oo
    with do.operand_rounding(torch.float16), oo.operand_rounding(torch.float16):
        return fn()


@pytest.mark.parametrize("name", GOLDENS)
def test_golden_models_decode_and_encode_vs_oracle(name):
    from oracle import diffae_oracle as dao
    g, cfg, sd, model = _golden_model(name)
    z, noise, steps = torch.from_numpy(g["z"]), torch.from_numpy(g["noise"]), int(g["steps"])
    y = model.decode(z.cuda(), steps=steps, noise=noise.cuda()).cpu()
    ref = dao.decode(z, sd, cfg, steps, noise)
    floor = rel_l2(_floors(lambda: dao.decode(z, sd, cfg, steps, noise)), ref)
    err = rel_l2(y, ref)
    a = torch.from_numpy(g["a"])
    h = model.encode(a.cuda(), return_info=False) if cfg["model"].get("bottleneck") is None else None
    pre = (model.encoder(model.pretransform.encode(a.cuda())) if model.pretransform is not None
           else model.encoder(a.cuda())).cpu()
    href = dao.encode_pre_bottleneck(a, sd, cfg)
    hfloor = rel_l2(_floors(lambda: dao.encode_pre_bottleneck(a, sd, cfg)), href)
    herr = rel_l2(pre, href)
    report("golden_decode_encode", golden=name, steps=steps, rel_l2=err, fp16_operand_floor=floor, enc_rel_l2=herr,
           enc_floor=hfloor)
    assert y.shape == ref.shape and err <= 1.25 * floor, (err, floor)
    assert herr <= 2.0 * hfloor, (herr, hfloor)
    if h is not None:
        assert torch.equal(h.cpu(), pre)


def test_golden_raw_model_with_eta_vs_oracle():
    from oracle import diffae_oracle as dao
    from stable_audio_tools.inference.sampling import sample
    g, cfg, sd, model = _golden_model("diffae_raw_small.npz")
    x0, c, nz = (torch.from_numpy(g[k]) for k in ("x0", "concat", "step_noise"))
    steps, eta = int(g["eta_steps"]), float(g["eta"])
    y = sample(model.diffusion, x0.cuda(), steps, eta, noise_sampler=lambda i: nz[i].cuda(),
               input_concat_cond=c.cuda()).cpu()
    fn = dao.dit_fn(sd, cfg)
    ref = dao.sample(fn, x0, steps, eta, noises=nz, input_concat_cond=c)
    floor = rel_l2(_floors(lambda: dao.sample(fn, x0, steps, eta, noises=nz, input_concat_cond=c)), ref)
    err = rel_l2(y, ref)
    report("golden_eta", rel_l2=err, fp16_operand_floor=floor)
    assert err <= 1.25 * floor, (err, floor)


def _sao_pqmf_config():
    dit = dict(io_channels=32, input_concat_dim=64, embed_dim=1536, depth=2, num_heads=24, cond_token_dim=0,
               global_cond_dim=0, project_cond_tokens=False, transformer_type="continuous_transformer")
    return {"model_type": "diffusion_autoencoder", "sample_rate": 44100,
            "model": {"io_channels": 32, "latent_dim": 64, "downsampling_ratio": 4,
                      "diffusion": {"type": "dit", "config": dit},
                      "pretransform": {"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}}}}


def test_sa_open_width_dit_over_pqmf_subbands_vs_oracle():
    from oracle import diffae_oracle as dao
    from stable_audio_tools import create_model_from_config
    cfg = _sao_pqmf_config()
    model = create_model_from_config(cfg)
    bufs = {k: v for k, v in model.pretransform.pqmf.state_dict().items()}
    sd = dao.make_state_dict(cfg, 140, bufs)
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(141)
    z = torch.randn(1, 64, 128, generator=g)
    noise = torch.randn(1, 32, 512, generator=g)
    steps = 4
    y = model.decode(z.cuda(), steps=steps, noise=noise.cuda()).cpu()
    ref = dao.decode(z, sd, cfg, steps, noise)
    floor = rel_l2(_floors(lambda: dao.decode(z, sd, cfg, steps, noise)), ref)
    err = rel_l2(y, ref)
    report("sao_width_pqmf16", tokens=512, steps=steps, rel_l2=err, fp16_operand_floor=floor)
    assert y.shape == (1, 2, 512 * 16) and err <= 1.25 * floor, (err, floor)


# ------------------------------------------------------------------------------------------------ 3. bit checks
def test_graph_replayed_decode_equals_an_eager_decode():
    from stable_audio_tools.inference import sampling
    g, cfg, sd, model = _golden_model("diffae_pqmf16_small.npz")
    z, noise, steps = (torch.from_numpy(g["z"]).cuda(), torch.from_numpy(g["noise"]).cuda(), int(g["steps"]))
    graphed = model.decode(z, steps=steps, noise=noise)
    assert model.diffusion.model.__dict__["_graph"] is not None          # the decode did replay a captured graph
    assert model.diffusion.model.cuda_graph is False                     # and put the switch back
    c = torch.nn.functional.interpolate(model.bottleneck.decode(z), size=noise.shape[2], mode="nearest")
    # a plain function is not recognised as a native DiT: every forward runs eagerly
    eager_v = sampling.sample(lambda x, t, **kw: model.diffusion(x, t, **kw), noise, steps, 0, input_concat_cond=c)
    assert torch.equal(graphed, model.pretransform.decode(eager_v))


def test_batch_of_two_equals_the_same_items_inside_a_batch_of_three():
    g, cfg, sd, model = _golden_model("diffae_raw_small.npz")
    gen = torch.Generator().manual_seed(5)
    z = torch.randn(3, 8, 40, generator=gen).cuda()
    noise = torch.randn(3, 2, 160, generator=gen).cuda()
    y3 = model.decode(z, steps=5, noise=noise)
    y2 = model.decode(z[1:].contiguous(), steps=5, noise=noise[1:].contiguous())
    assert torch.equal(y3[1:], y2)
