"""GPU: the token-sharded DiT forward replayed from one multi-device CUDA graph (DiffusionTransformer.shard_tokens with
cuda_graph, satb_dit_group_graph_forward).

The graph holds the same launches as the eager sharded call, with the same event pairs as edges, so its output must be
bit-identical to it, and to the unsharded forward.  On one device the ranks are virtual (a handle and a stream each on
cuda:0); a graph with nodes on distinct GPUs is only tested by the last two tests, which skip when fewer than two
devices are visible.  Every comparison below is torch.equal; `CPGRAPH {...}` lines (pytest -s) record the graph state."""
import json

import pytest
import torch

from helpers import SAO_DIT, build_native_dit, rel_l2
from test_gpu_dit_group import CASES, _cuda, _inputs

pytestmark = pytest.mark.gpu


def report(**kw):
    print("CPGRAPH", json.dumps(kw))


def _model(case, L, seed=91):
    from oracle import positions_oracle as po
    cfg, dtype, extra = CASES[case]
    sd = po.make_dit_weights(cfg, seed=seed)
    return cfg, extra, sd, build_native_dit(cfg, sd, operand_dtype=dtype), _cuda(_inputs(cfg, extra, L, seed=92 + L))


def _call(m, kw, graph):
    m.cuda_graph = graph
    try:
        return m(**kw).clone()
    finally:
        m.cuda_graph = False


@pytest.mark.parametrize("L", [300, 1100])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("case", sorted(CASES))
def test_graph_replay_equals_eager_sharded_and_unsharded(case, world, L):
    cfg, extra, sd, m, kw = _model(case, L)
    y1 = _call(m, kw, False)
    m.shard_tokens(["cuda:0"] * world)
    ye = _call(m, kw, False)
    yg = _call(m, kw, True)                   # warm-up, capture, first launch
    yg2 = _call(m, kw, True)                  # a plain replay
    stats = m.shard_graph_stats()
    # the patch_size > 1 with scale_phi route makes two calls (guided, then conditional) per forward
    calls = 2 if (cfg.get("patch_size", 1) > 1 and extra.get("scale_phi", 0.0) != 0.0) else 1
    report(case=case, world=world, L=L, stats=stats, equal_eager=bool(torch.equal(yg, ye)),
           equal_unsharded=bool(torch.equal(yg, y1)))
    assert stats[1] == 2 * calls and stats[2] > 0
    if calls == 1:
        assert stats[0] == 1                  # captured once, replayed twice
    assert torch.equal(yg, ye) and torch.equal(yg2, ye)
    assert torch.equal(yg, y1)
    m.shard_tokens(None)


def test_replay_with_new_inputs_equals_eager():
    cfg, extra, sd, m, kw = _model("prepend_cfg", 1100)
    m.shard_tokens(["cuda:0"] * 3)
    _call(m, kw, True)
    g = torch.Generator().manual_seed(7)
    for i in range(3):
        kw2 = dict(kw, x=torch.randn(kw["x"].shape, generator=g).cuda(), t=torch.tensor([0.1 + 0.3 * i]).cuda())
        yg = _call(m, kw2, True)
        ye = _call(m, kw2, False)
        assert torch.equal(yg, ye)
    assert m.shard_graph_stats()[0] == 1      # new inputs in the same static buffers: no recapture


def test_every_key_and_state_change_recaptures_and_stays_exact():
    """cfg_scale, scale_phi, B, L, the conditioning tensors, load_state_dict, shard_tokens with other devices and an eager
    call in between: each graph result equals the eager sharded result for the same call."""
    cfg, extra, sd, m, kw = _model("prepend_cfg", 300)
    m.shard_tokens(["cuda:0"] * 2)
    log = []

    def check(name, kw_, recapture=True, new_group=False):
        before = m.shard_graph_stats()
        yg = _call(m, kw_, True)
        after = m.shard_graph_stats()
        ye = _call(m, kw_, False)
        log.append(dict(step=name, stats=after, equal=bool(torch.equal(yg, ye))))
        assert torch.equal(yg, ye), name
        if new_group:                         # weights refreshed or other devices: a new group, captured once
            assert after[:2] == (1, 1), (name, before, after)
        elif recapture:
            assert before is None or after[0] == before[0] + 1, (name, before, after)
        else:
            assert after[0] == before[0], (name, before, after)
        return yg

    check("first", kw)
    check("same", kw, recapture=False)
    check("cfg_scale", dict(kw, cfg_scale=3.0))
    check("scale_phi", dict(kw, cfg_scale=3.0, scale_phi=0.5))
    g = torch.Generator().manual_seed(8)
    kw_b = dict(kw, x=torch.randn(2, 64, 300, generator=g).cuda(), t=torch.tensor([0.2, 0.7]).cuda(),
                cross_attn_cond=torch.randn(2, 19, 128, generator=g).cuda(),
                global_embed=torch.randn(2, 256, generator=g).cuda())
    check("B", kw_b)
    check("L", dict(kw, x=torch.randn(1, 64, 700, generator=g).cuda()))
    check("cond", dict(kw, cross_attn_cond=torch.randn_like(kw["cross_attn_cond"])))
    check("cond_in_place", kw)
    kw["global_embed"].mul_(0.5)              # same tensor, new version: the conditioning is prepared again
    check("cond_mutated", kw)
    m.load_state_dict({k: v * 1.01 if v.dtype.is_floating_point else v for k, v in sd.items()})
    check("load_state_dict", kw, new_group=True)
    m.shard_tokens(["cuda:0"] * 3)
    check("shard_tokens", kw, new_group=True)
    yg = _call(m, kw, True)
    _call(m, dict(kw, x=torch.randn_like(kw["x"])), False)  # an eager call between two replays
    assert torch.equal(_call(m, kw, True), yg)
    _call(m, dict(kw, x=torch.randn(1, 64, 500, generator=g).cuda()), False)  # one that reserves another shape
    check("eager_reserve", kw)
    report(case="recapture", log=log)


def test_generate_diffusion_cond_graph_sharded_equals_eager_sharded_and_unsharded():
    """dpmpp-3m-sde, CFG 5: the sampler switches cuda_graph on, which now reaches the sharded path."""
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
    latg, audiog = run()
    stats = dit.shard_graph_stats()
    dit.__dict__["_sharded_graph_forward"] = dit._sharded_forward    # the same run with every sharded call eager
    try:
        late, audioe = run()
    finally:
        del dit.__dict__["_sharded_graph_forward"]
    assert dit.shard_graph_stats() == stats                          # the eager run launched no graph
    dit.shard_tokens(None)
    report(case="generate_dpmpp_3m_sde", world=3, stats=stats, rel_l2_latents=rel_l2(latg, lat1))
    assert stats[0] >= 1 and stats[1] >= steps - 1, stats           # the sampler's calls were graph launches
    assert torch.equal(latg, late) and torch.equal(audiog, audioe)
    assert torch.equal(latg, lat1) and torch.equal(audiog, audio1)


def test_diffusion_autoencoder_decode_with_a_sharded_dit_decoder():
    """The v-diffusion sample switches cuda_graph on as well: graph-sharded = eager-sharded = unsharded decode."""
    from stable_audio_tools.inference import sampling
    from test_gpu_diffae import _golden_model
    g, cfg, sd, model = _golden_model("diffae_pqmf16_small.npz")
    z, noise, steps = (torch.from_numpy(g["z"]).cuda(), torch.from_numpy(g["noise"]).cuda(), int(g["steps"]))
    dit = model.diffusion.model
    y1 = model.decode(z, steps=steps, noise=noise).clone()
    dit.shard_tokens(["cuda:0"] * 3)
    yg = model.decode(z, steps=steps, noise=noise).clone()
    stats = dit.shard_graph_stats()
    c = torch.nn.functional.interpolate(model.bottleneck.decode(z), size=noise.shape[2], mode="nearest")
    # a plain function is not recognised as a native DiT: every sharded forward runs eagerly
    eager_v = sampling.sample(lambda x, t, **kw: model.diffusion(x, t, **kw), noise, steps, 0, input_concat_cond=c)
    ye = model.pretransform.decode(eager_v)
    assert dit.shard_graph_stats() == stats
    dit.shard_tokens(None)
    report(case="diffae_decode", world=3, stats=stats)
    assert stats[0] >= 1 and stats[1] >= steps - 1, stats
    assert torch.equal(yg, ye) and torch.equal(yg, y1)


def _sa2_length_graph_vs_eager_and_oracle(devices):
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
    kw = dict(x=x.cuda(), t=t.cuda(), cross_attn_cond=c.cuda(), global_embed=ge.cuda(), cfg_scale=7.0)
    ye = _call(m, kw, False)
    yg = _call(m, kw, True)
    yg2 = _call(m, kw, True)
    err = rel_l2(yg.cpu(), ref)
    report(case="sa2_length_2_blocks_cfg7_graph", devices=[str(d) for d in devices], rel_l2=err,
           stats=m.shard_graph_stats())
    assert torch.equal(yg, ye) and torch.equal(yg2, ye)
    assert err < 2e-3 * 7.0 / 1.5, err


def _real_devices(n):
    if torch.cuda.device_count() < 2:
        pytest.skip(f"{torch.cuda.device_count()} CUDA device(s) visible: a graph over distinct GPUs needs at least 2")
    return [f"cuda:{i}" for i in range(n)]


def test_sa2_length_graph_over_2_devices_vs_eager_and_oracle():
    _sa2_length_graph_vs_eager_and_oracle(_real_devices(2))


def test_sa2_length_graph_over_every_device_vs_eager_and_oracle():
    _sa2_length_graph_vs_eager_and_oracle(_real_devices(min(torch.cuda.device_count(), 8)))
