"""GPU: the native step path of the samplers (satb_sampler_step, include/satb200.h).

- the kernel element by element against its torch restatement, blend included;
- a smooth toy model: every sampler type, rectified flow, and the SDE samplers with inpainting and a user callback give
  the torch path's result (gate closed, same device, so the same random draws) within 1e-4 max|x|, with the same
  callback i / sigma sequence and matching denoised;
- the native DiT: after the first call every model call is one graph replay, captured once, and each call adds the
  graph's launches plus exactly one update launch;
- generate_diffusion_cond with each newly fused sampler, rectified flow, and inpainting plus a callback against the
  oracle DiT driven by the same package sampler on the CPU (rel-L2 < 3e-2, the bar of test_gpu_generate.py);
- the inpainting run with a 3-way token-sharded DiT (virtual ranks) equals the unsharded run bit for bit."""
import pytest
import torch

from helpers import rel_l2
from sampler_step_ref import sampler_step_ref

pytestmark = pytest.mark.gpu

FIXED = ["k-heun", "k-dpm-2", "k-lms", "k-dpmpp-2s-ancestral"]


def _s():
    from stable_audio_tools.inference import sampling
    return sampling


def model_fn(x, t, gain=1.0, **kw):
    return torch.tanh(x * gain) * (0.5 + t.view(-1, 1, 1)) - 0.1 * x


class Recorder:
    def __init__(self):
        self.seen = []

    def __call__(self, args):
        self.seen.append((args["i"], float(args["sigma"] if "sigma" in args else args["t"]), args["denoised"].clone()))


@pytest.mark.parametrize("n,L", [(4 * 3 * 40, 40), (2 * 64 * 1024, 1024), (2 * 5 * 36, 36)])
@pytest.mark.parametrize("with_blend", [False, True])
def test_kernel_matches_its_restatement(n, L, with_blend):
    s = _s()
    g = torch.Generator(device="cuda").manual_seed(n)
    r = lambda: torch.randn(n // L, L, device="cuda", generator=g)
    x, y, bufs, nz = r(), r(), [r() for _ in range(4)], r()
    inp = s.InpaintingCallback(r(), torch.rand(L, device="cuda", generator=g), 7) if with_blend else None
    kw = dict(c_skip=0.3, c_out=-0.9, inv_sigma=0.25, a=0.7, b=-0.4, g=1.3, bufs=list(zip([0.5, -0.25, 0.125, 2.0], bufs)),
              noise=nz, s=0.6, den=True, d=True, c_in_next=0.2,
              blend=(inp, 3, r(), 2.5) if with_blend else None)
    xr = x.clone()
    got = s._step(x, y, **kw)
    saved = s._launch_step
    try:
        s._launch_step = lambda p: sampler_step_ref(p, torch.float64)
        ref = s._step(xr, y, **kw)
    finally:
        s._launch_step = saved
    if with_blend:
        assert torch.equal(x, xr)          # the blend itself is exact
    for a, b in zip(got, ref):
        assert float((a.double() - b.double()).abs().max()) <= 4e-6 * float(b.abs().max())


def _toy(name, kind, device, native, monkeypatch, steps=9):
    s = _s()
    g = torch.Generator().manual_seed(7)
    noise = torch.randn(2, 8, 64, generator=g)
    seq = [torch.randn(2, 8, 64, generator=g) for _ in range(steps)]
    it = iter(seq)
    ns = lambda a, b: next(it).to(device)
    init = torch.randn(2, 8, 64, generator=g).to(device) if "inpaint" in kind else None
    mask = torch.rand(64, generator=g).to(device) if "inpaint" in kind else None
    rec = Recorder()
    with monkeypatch.context() as m:
        if not native:
            m.setattr(s, "_fusable", lambda x: False)
        torch.manual_seed(5)
        if name == "rf":
            out = s.sample_rf(model_fn, noise.to(device), steps=steps, device=device,
                              callback=rec if "user" in kind else None, gain=0.7)
        else:
            out = s.sample_k(model_fn, noise.to(device), init, mask, steps=steps, sampler_type=name, sigma_min=0.3,
                             sigma_max=50.0, device=device, callback=rec if "user" in kind else None, noise_sampler=ns,
                             gain=0.7)
    return out.cpu(), rec.seen


@pytest.mark.parametrize("name,kind", [(n, k) for n in FIXED for k in ("none", "user", "inpaint", "inpaint+user")]
                         + [(n, k) for n in ("dpmpp-2m-sde", "dpmpp-3m-sde") for k in ("user", "inpaint", "inpaint+user")]
                         + [("rf", "none"), ("rf", "user"), ("k-dpm-fast", "inpaint"), ("k-dpm-adaptive", "user")])
def test_toy_model_native_equals_torch_path(name, kind, monkeypatch):
    ref, ref_seen = _toy(name, kind, "cuda", False, monkeypatch)
    got, seen = _toy(name, kind, "cuda", True, monkeypatch)
    scale = max(1.0, float(ref.abs().max()))
    assert float((got - ref).abs().max()) <= 1e-4 * scale
    assert [(i, sg) for i, sg, _ in seen] == [(i, sg) for i, sg, _ in ref_seen]
    for (_, _, d), (_, _, rd) in zip(seen, ref_seen):
        assert float((d - rd).abs().max()) <= 1e-4 * max(1.0, float(rd.abs().max()))
    if kind in ("none", "user") and name not in ("k-dpm-fast", "k-dpm-adaptive"):
        # no draws but the injected noise: the package's CPU torch path gives the same result
        cpu, cpu_seen = _toy(name, kind, "cpu", False, monkeypatch)
        assert float((got - cpu).abs().max()) <= 1e-4 * scale
        assert [i for i, _, _ in seen] == [i for i, _, _ in cpu_seen]


# ------------------------------------------------------------------ the native DiT
DIT = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
           project_cond_tokens=False, transformer_type="continuous_transformer")


def _dit():
    from oracle import dit_oracle as do
    from stable_audio_tools.models.diffusion import DiTWrapper
    sd = do.make_dit_weights(DIT, seed=1)
    w = DiTWrapper(**DIT)
    w.model.load_state_dict(sd)
    return w.cuda().eval(), sd


@pytest.mark.parametrize("name,kind", [(n, "none") for n in FIXED] + [(n, "inpaint") for n in FIXED + ["dpmpp-3m-sde"]]
                         + [("rf", "none")])
def test_every_call_after_the_first_is_one_graph_replay(name, kind, monkeypatch):
    from stable_audio_tools import _native
    s = _s()
    w, _ = _dit()
    dit = w.model
    g = torch.Generator().manual_seed(2)
    B, L, steps = 2, 48, 5
    kw = dict(cross_attn_cond=torch.randn(B, 12, 128, generator=g).cuda(),
              global_cond=torch.randn(B, 256, generator=g).cuda(), cfg_scale=4.0)
    noise = torch.randn(B, 64, L, generator=g).cuda()
    init = torch.randn(B, 64, L, generator=g).cuda() if kind == "inpaint" else None
    mask = torch.rand(L, generator=g).cuda() if kind == "inpaint" else None
    calls, captures = [], []
    orig_fwd, orig_graph = dit._graph_forward, torch.cuda.graph
    monkeypatch.setattr(dit, "_graph_forward", lambda *a, **k: (calls.append(1), orig_fwd(*a, **k))[1], raising=False)

    def counting_graph(*a, **k):
        captures.append(1)
        return orig_graph(*a, **k)
    monkeypatch.setattr(torch.cuda, "graph", counting_graph)

    def run():
        if name == "rf":
            return s.sample_rf(w, noise, steps=steps, device="cuda", **kw)
        return s.sample_k(w, noise, init, mask, steps=steps, sampler_type=name, sigma_min=0.3, sigma_max=50.0,
                          device="cuda", **kw)
    run()
    assert len(captures) == 1 and dit.cuda_graph is False
    replayed = dit.__dict__["_graph"]["launches"]
    calls.clear()
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    run()
    torch.cuda.synchronize()
    assert len(captures) == 1, "the graph was captured again"
    n_calls = len(calls)
    assert n_calls == {"k-heun": 2 * steps - 1, "k-dpm-2": 2 * steps - 1,
                       "k-dpmpp-2s-ancestral": 2 * steps - 1}.get(name, steps)
    assert _native.launch_count() - n0 == n_calls * (replayed + 1)


# ------------------------------------------------------------------ end to end
def _generate_vs_oracle(sampler, objective="v", inpaint=False, monkeypatch=None, shard=None, oracle=True):
    from oracle import dit_oracle as do
    from stable_audio_tools.inference import generation
    from test_gpu_generate import _build
    s = _s()
    model, cfg, dit_sd, _, _ = _build()
    model.diffusion_objective = objective
    B, L, steps, seed, cfg_scale = 2, 48, 6, 321, 5.0
    g = torch.Generator().manual_seed(5)
    cond = {"prompt": (torch.randn(B, 10, 128, generator=g).cuda(), torch.ones(B, 10).cuda()),
            "seconds_start": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda()),
            "seconds_total": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda())}
    draws = [torch.randn(B, 64, L, generator=g) for _ in range(4 * steps)]

    def draw_seq(dev):
        it = iter(draws)
        return lambda *a: next(it).to(dev)
    seen, rec = {}, Recorder()
    orig_sample_k = generation.sample_k

    def spy(model_fn, noise, init_data=None, mask=None, *a, **k):
        seen.update(init=None if init_data is None else init_data.cpu(), mask=None if mask is None else mask.cpu())
        return orig_sample_k(model_fn, noise, init_data, mask, *a, **k)
    monkeypatch.setattr(generation, "sample_k", spy)
    orig_randn_like = torch.randn_like

    def renoise(dev):                      # the inpainting re-noise; other draws (the VAE's) stay random
        rl = draw_seq(dev)
        return lambda t, *a, **k: rl().to(t.dtype) if tuple(t.shape) == (B, 64, L) else orig_randn_like(t, *a, **k)
    monkeypatch.setattr(torch, "randn_like", renoise("cuda"))
    if shard:
        model.model.model.shard_tokens(["cuda:0"] * shard)
    kw = dict(sampler_type=sampler, sigma_min=0.3, sigma_max=50.0) if objective == "v" else dict(sigma_max=1.0)
    ns = dict(noise_sampler=draw_seq("cuda")) if objective == "v" else {}
    extra = {}
    if inpaint:
        audio = torch.randn(2, L * 64, generator=g) * 0.3
        extra = dict(init_audio=(16000, audio), callback=rec,
                     mask_args=dict(cropfrom=0, pastefrom=0, pasteto=100, maskstart=20, maskend=60, softnessL=10,
                                    softnessR=10, marination=0))
    lat = generation.generate_diffusion_cond(model, steps=steps, cfg_scale=cfg_scale, conditioning_tensors=cond,
                                             sample_size=L * 64, seed=seed, device="cuda", return_latents=True,
                                             **ns, **kw, **extra)
    if not oracle:
        return lat.cpu(), None
    torch.manual_seed(seed)
    noise = torch.randn([B, 64, L], device="cuda").cpu()
    cross = torch.cat([cond[k][0] for k in ("prompt", "seconds_start", "seconds_total")], dim=1).cpu()
    glob = torch.cat([cond[k][0] for k in ("seconds_start", "seconds_total")], dim=-1).squeeze(1).cpu()

    def oracle_fn(x, t, **k):
        return do.dit_forward(dit_sd, cfg, x, t, cross_attn_cond=cross, global_embed=glob, cfg_scale=cfg_scale)
    monkeypatch.setattr(torch, "randn_like", renoise("cpu"))
    ref_rec = Recorder()
    if objective == "v":
        ref = s.sample_k(oracle_fn, noise, seen.get("init"), seen.get("mask"), steps, device="cpu",
                         noise_sampler=draw_seq("cpu"), callback=ref_rec if inpaint else None, **kw)
    else:
        ref = s.sample_rf(oracle_fn, noise, steps=steps, device="cpu", **kw)
    if inpaint:
        assert [i for i, _, _ in rec.seen] == [i for i, _, _ in ref_rec.seen] == list(range(steps))
    return lat.cpu(), ref


@pytest.mark.parametrize("sampler,objective,inpaint", [(n, "v", False) for n in FIXED] + [("rf", "rectified_flow", False)]
                         + [("dpmpp-3m-sde", "v", True), ("k-heun", "v", True), ("k-dpm-fast", "v", False)])
def test_generate_matches_oracle_pipeline(sampler, objective, inpaint, monkeypatch):
    lat, ref = _generate_vs_oracle(sampler, objective, inpaint, monkeypatch)
    assert rel_l2(lat, ref) < 3e-2


def test_sharded_inpainting_equals_unsharded(monkeypatch):
    with monkeypatch.context() as m:
        one, _ = _generate_vs_oracle("dpmpp-3m-sde", inpaint=True, monkeypatch=m, oracle=False)
    with monkeypatch.context() as m:
        three, _ = _generate_vs_oracle("dpmpp-3m-sde", inpaint=True, monkeypatch=m, shard=3, oracle=False)
    assert torch.equal(one, three)
