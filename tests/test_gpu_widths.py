"""GPU: DiTs of any channel width (inpainting DiTs with input_concat_dim = latent + 1, narrow latents, raw audio with
patching, PQMF sub-bands) and the mono-to-stereo diffusion prior.

1. project_in with a padded K and project_out with a padded N, through the kernels the forward launches: the token-row
   kernel (satb_dit_pre_probe) writes the A operand at the padded pitch into a buffer whose pad columns were poisoned
   with NaN, and satb_gemm_probe runs the forward's GEMM instances (store32 BN 256 / BN 64) on it with the folded
   weights built as satb_dit_finalize builds them (fp64 fold, fp32, 16-bit, zero pad columns / rows).  Element by
   element against float64 with the bound of tests/gemm_epilogue_ref.py.
2. The DiT against the reference goldens (tests/golden/dit_width_*.npz) at the gates of test_gpu_positions.py: rel-L2
   2e-3 (x max(1, cfg / 1.5) with CFG) in fp16, 1.5e-2 in bf16; FP8 within 1.25 x its emulated floor.  The io-1
   fixture's CFG rescale is NaN in the reference and must be NaN here.
3. SA-Open width (1536 wide, 24 heads, 2 blocks) as an inpainting model (Cin = 129) at 1025 and 6145 tokens against
   the oracle's fp16-operand floor.
4. Bit checks: the CUDA-graph call equals the eager call; a batch of 4 equals the same prompts inside a batch of 5;
   reloading preprocess_conv.weight takes effect, eagerly and through the graph.
5. End to end: generate_diffusion_cond with an inpainting DiT and an Oobleck decode, and stereoize on a prior whose DiT
   has 2 io + 2 concat channels, against the oracle pipeline with injected noise at the gates of test_gpu_generate.py.
Measured numbers are printed as `WIDTHS {...}` JSON lines (pytest -s)."""
import ctypes
import json

import pytest
import torch

import gemm_epilogue_ref as ger
from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu

GOLDENS = ["dit_width_inpaint_small.npz", "dit_width_io16_adaln_hd128_small.npz",
           "dit_width_io2_patch4_concat3_small.npz", "dit_width_io1_small.npz", "dit_width_io40_conformer_small.npz"]
TOL = {"fp16": 2e-3, "bf16": 1.5e-2}


def report(name, **kw):
    print("WIDTHS " + json.dumps(dict(test=name, **kw)), flush=True)


def _round_up(v, m):
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ 1. the probes
def _fold_in(cin, D, g):
    """(W_in (I + W_pre)) in fp64 -> fp32 at pitch round_up(cin, 8) with zero pad columns (satb_dit_finalize)."""
    w_in = torch.randn(D, cin, generator=g, dtype=torch.float64) * cin ** -0.5
    w_pre = torch.randn(cin, cin, generator=g, dtype=torch.float64) * 0.04
    fold = (w_in + w_in @ w_pre).float()
    out = torch.zeros(D, _round_up(cin, 8))
    out[:, :cin] = fold
    return out


@pytest.mark.parametrize("cin", [1, 3, 65, 129, 136])
@pytest.mark.parametrize("bf16", [0, 1])
def test_project_in_with_a_padded_k_vs_fp64(cin, bf16):
    from stable_audio_tools import _native as nat
    dt = torch.bfloat16 if bf16 else torch.float16
    D, B, P, L = 1536, 2, 1, 1024          # R = 4 rows of 1025 tokens (CFG), the source batch 2
    R, K = 2 * B, _round_up(cin, 8)
    g = torch.Generator().manual_seed(cin + 10 * bf16)
    x = torch.randn(B, cin, L, generator=g).cuda()
    a = torch.full((R * (P + L), K), float("nan"), device="cuda").to(dt)   # NaN in every column, pads included
    nat.check(nat.lib().satb_dit_pre_probe(x.data_ptr(), a.data_ptr(), R, B, cin, K, L, P, bf16, nat.stream_ptr()))
    w = _fold_in(cin, D, g).to(dt).cuda()
    out = torch.full((R * (P + L), D), float("nan"), device="cuda")
    p = nat.SatbGemmProbe(epi=nat.EPI_STORE32, bn=256, bf16=bf16, b_static=1, out=out.data_ptr(), ld=D)
    nat.check(nat.lib().satb_gemm_probe(a.data_ptr(), w.data_ptr(), R * (P + L), D, K, ctypes.byref(p),
                                        nat.stream_ptr()))
    torch.cuda.synchronize()
    a_c = a.cpu()
    assert torch.isfinite(a_c.float()).all() and not a_c[:, cin:].any()             # pad columns are zeros
    rows = a_c.view(R, P + L, K)
    assert not rows[:, :P].any()                                                     # prepend slots are zeros
    want = torch.cat([x.cpu(), x.cpu()], dim=0).transpose(1, 2).to(dt)
    assert torch.equal(rows[:, P:, :cin], want)
    acc, S = ger.accumulate(a_c, w.cpu())
    rep = ger.check(out.cpu(), ger.epi_store(acc, S), K, "fp32")
    report("project_in_probe", cin=cin, K=K, bf16=bf16, max_err_over_bound=rep.ratio)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("c", [1, 2, 16, 40])
@pytest.mark.parametrize("bf16", [0, 1])
def test_project_out_with_a_padded_n_vs_fp64(c, bf16):
    from stable_audio_tools import _native as nat
    dt = torch.bfloat16 if bf16 else torch.float16
    D, M = 1536, 4 * 1025
    N = _round_up(c, 32)
    g = torch.Generator().manual_seed(100 + c + bf16)
    a = torch.randn(M, D, generator=g).to(dt).cuda()
    w_out = torch.randn(c, D, generator=g, dtype=torch.float64) * D ** -0.5
    w_post = torch.randn(c, c, generator=g, dtype=torch.float64) * 0.04
    w = torch.zeros(N, D)
    w[:c] = (w_out + w_post @ w_out).float()                                         # (I + W_post) W_out, zero rows
    w = w.to(dt).cuda()
    out = torch.full((M, N), float("nan"), device="cuda")
    p = nat.SatbGemmProbe(epi=nat.EPI_STORE32, bn=64, bf16=bf16, b_static=1, out=out.data_ptr(), ld=N)
    nat.check(nat.lib().satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, N, D, ctypes.byref(p), nat.stream_ptr()))
    torch.cuda.synchronize()
    acc, S = ger.accumulate(a.cpu(), w.cpu())
    rep = ger.check(out.cpu(), ger.epi_store(acc, S), D, "fp32", bn=64)
    report("project_out_probe", c=c, N=N, bf16=bf16, max_err_over_bound=rep.ratio)
    assert rep.ok, str(rep)
    assert not out[:, c:].cpu().any()


# ------------------------------------------------------------------------------------------------ 2. the goldens
def _golden_case(name):
    from oracle import positions_oracle as po
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = po.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), "synthetic weight RNG drifted from the golden run"
    return g, cfg, sd


def _golden_kw(g, dev):
    T = lambda k: torch.from_numpy(g[k]).to(dev)
    kw = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "concat" in g:
        kw["input_concat_cond"] = T("concat")
    return kw


@pytest.mark.parametrize("name", GOLDENS)
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_dit_widths_vs_reference_golden(name, dtype):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    kw = _golden_kw(g, "cuda")
    neg = torch.from_numpy(g["neg"]).cuda()
    cases = {"y_nocfg": dict(cfg_scale=1.0), "y_cfg7": dict(cfg_scale=7.0),
             "y_cfg4_phi": dict(cfg_scale=4.0, scale_phi=0.7),
             "y_neg3": dict(cfg_scale=3.0, negative_cross_attn_cond=neg)}
    for key, ck in cases.items():
        y = m(**kw, **ck).cpu()
        want = torch.from_numpy(g[key])
        assert y.shape == want.shape
        if torch.isnan(want).all():            # io 1: the reference's std over one channel
            report("dit_golden", config=name, dtype=dtype, case=key, all_nan=bool(torch.isnan(y).all()))
            assert torch.isnan(y).all()
            continue
        err = rel_l2(y, want)
        report("dit_golden", config=name, dtype=dtype, case=key, rel_l2=err)
        if key == "y_cfg4_phi" and cfg["io_channels"] == 2:
            # the rescale's std over 2 channels is |c0 - c1| / sqrt(2): where the CFG output's two channels nearly
            # agree, cond_std / cfg_std reaches ~60 and magnifies any rounding without bound (16-bit operands in the
            # oracle alone land 0.54 rel-L2 from the fp32 reference, the native fp16 result 2.8 on an H100), so no
            # end-to-end gate exists.  Checked instead: its two inputs against the fp32 oracle at the usual gate, and the rescale of
            # those very native outputs (the patch-size path rescales in torch, dit.py:342-345).
            from oracle import positions_oracle as po
            cpu = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
            cfg_n, cond_n = m(**kw, cfg_scale=4.0).cpu(), m(**kw, cfg_scale=1.0).cpu()
            err4 = rel_l2(cfg_n, po.dit_forward(sd, cfg, **cpu, cfg_scale=4.0))
            assert err4 < TOL[dtype] * 4.0 / 1.5, f"{name} cfg 4 {dtype}: rel l2 {err4}"
            phi = 0.7 * (cfg_n * (cond_n.std(dim=1, keepdim=True) / cfg_n.std(dim=1, keepdim=True))) + 0.3 * cfg_n
            report("dit_golden_phi_inputs", config=name, dtype=dtype, cfg4_rel_l2=err4,
                   rescale_max_abs=float((y - phi).abs().max()))
            assert torch.allclose(y, phi, rtol=1e-6, atol=1e-6)
            continue
        assert err < TOL[dtype] * max(1.0, ck["cfg_scale"] / 1.5), f"{name} {key} {dtype}: rel l2 {err}"
    y, info = m(**kw, cfg_scale=1.0, return_info=True)
    err = rel_l2(info["hidden_states"][-1].cpu(), torch.from_numpy(g["hidden_last"]))
    assert err < TOL[dtype], f"{name} hidden {dtype}: rel l2 {err}"
    if "y_noconcat" in g:                     # the concat channels reach the native result
        kw0 = dict(kw, input_concat_cond=torch.zeros_like(kw["input_concat_cond"]))
        err0 = rel_l2(m(**kw0, cfg_scale=1.0).cpu(), torch.from_numpy(g["y_noconcat"]))
        assert err0 < TOL[dtype], f"{name} y_noconcat {dtype}: rel l2 {err0}"


def _floor_and_native(cfg, sd, m, kw, device, floor_ctx):
    from oracle import positions_oracle as po
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = po.dit_forward(sdd, cfg, **kwd)
    with floor_ctx(sdd):
        emu = po.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDENS)
def test_dit_widths_fp8_vs_fp8_floor(name):
    """project_in / project_out stay 16-bit in the FP8 mode, as the emulation assumes."""
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    base = _golden_kw(g, "cpu")
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", fp8_operands)
        report("dit_fp8", config=name, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
        assert err <= 1.25 * floor, (name, cfg_scale, err, floor)


# ------------------------------------------------------------------------------------------------ 3. SA-Open width
INPAINT = dict(SAO_DIT, depth=2, input_concat_dim=65)


def _inpaint_inputs(seed, B=1, L=1024):
    g = torch.Generator().manual_seed(seed)
    x, t = torch.randn(B, 64, L, generator=g), torch.rand(B, generator=g) * 0.9 + 0.05
    c, ge = torch.randn(B, 130, 768, generator=g), torch.randn(B, 1536, generator=g)
    c[:, 40:] = 0.0
    mask = (torch.rand(B, 1, L, generator=g) > 0.3).float()
    concat = torch.cat([mask, torch.randn(B, 64, L, generator=g) * mask], dim=1)
    return dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, input_concat_cond=concat)


@pytest.mark.parametrize("L,cfg_scale", [(1024, 7.0), (6144, 1.0)])
def test_inpainting_dit_sa_open_width_vs_fp16_floor(L, cfg_scale):
    from oracle import dit_oracle as do
    from oracle import positions_oracle as po
    assert not torch.backends.cuda.matmul.allow_tf32
    sd = po.make_dit_weights(INPAINT, seed=95)
    m = build_native_dit(INPAINT, sd)
    kw = dict(_inpaint_inputs(96, L=L), cfg_scale=cfg_scale)
    floor, err = _floor_and_native(INPAINT, sd, m, kw, "cuda", lambda sdd: do.operand_rounding(torch.float16))
    report("inpaint_sa_open", tokens=L + 1, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
    assert err <= 1.25 * floor, (L, err, floor)


# ------------------------------------------------------------------------------------------------ 4. bit checks
@pytest.mark.parametrize("name", ["dit_width_inpaint_small.npz", "dit_width_io1_small.npz",
                                  "dit_width_io2_patch4_concat3_small.npz"])
def test_widths_cuda_graph_call_equals_the_eager_call(name):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd)
    kw = _golden_kw(g, "cuda")
    x = kw.pop("x")
    eager = lambda xx: m(xx, cfg_scale=7.0, **kw).clone()
    y0 = eager(x)
    m.cuda_graph = True
    y1 = eager(x)
    y2 = eager(x * 0.5 + 0.1)
    m.cuda_graph = False
    assert torch.equal(y0, y1)
    assert torch.equal(y2, eager(x * 0.5 + 0.1))


def test_inpainting_batch_of_4_equals_the_same_prompts_in_a_batch_of_5():
    from oracle import positions_oracle as po
    m = build_native_dit(INPAINT, po.make_dit_weights(INPAINT, seed=97))
    kw = {k: v.cuda() for k, v in _inpaint_inputs(98, B=5).items()}
    y5 = m(**kw, cfg_scale=7.0).clone()
    y4 = m(**{k: v[:4].contiguous() for k, v in kw.items()}, cfg_scale=7.0).clone()
    report("batch_invariance", bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)


@pytest.mark.parametrize("graph", [False, True])
def test_reloading_the_preprocess_conv_changes_the_output(graph):
    """satb_dit_finalize refolds preprocess_conv into the padded project_in weight on every reload."""
    g, cfg, sd = _golden_case("dit_width_inpaint_small.npz")
    m = build_native_dit(cfg, sd)
    m.cuda_graph = graph
    kw = _golden_kw(g, "cuda")
    y0 = m(**kw, cfg_scale=7.0).clone()
    sd2 = dict(sd, **{"preprocess_conv.weight": sd["preprocess_conv.weight"] * 8.0})
    m.load_state_dict(sd2, strict=True)
    y1 = m(**kw, cfg_scale=7.0).clone()
    m.load_state_dict(sd, strict=True)
    y2 = m(**kw, cfg_scale=7.0).clone()
    report("reload", graph=graph, moved=rel_l2(y1.cpu(), y0.cpu()))
    assert rel_l2(y1.cpu(), y0.cpu()) > 0.05
    assert torch.equal(y0, y2)


# ------------------------------------------------------------------------------------------------ 5. end to end
DIT = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
           project_cond_tokens=False, transformer_type="continuous_transformer")
DEC = dict(out_channels=2, channels=32, c_mults=[1, 2, 4], strides=[2, 4, 8], latent_dim=64, use_snake=True,
           final_tanh=False)
ENC = dict(in_channels=2, channels=32, c_mults=[1, 2, 4], strides=[2, 4, 8], latent_dim=128, use_snake=True)


class _StubConditioner(torch.nn.Module):
    def set_device(self, device):
        pass


def _noise_samplers(seq):
    def make(dev):
        it = iter(seq)
        return lambda s, sn: next(it).to(dev)
    return make


def test_generate_with_an_inpainting_dit_matches_the_oracle_pipeline():
    from oracle import dit_oracle as do
    from oracle import oobleck_oracle as oo
    from oracle import sampler_oracle as so
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    from stable_audio_tools.models.autoencoders import AudioAutoencoder, OobleckDecoder, OobleckEncoder
    from stable_audio_tools.models.bottleneck import VAEBottleneck
    from stable_audio_tools.models.diffusion import ConditionedDiffusionModelWrapper, DiTWrapper
    from stable_audio_tools.models.pretransforms import AutoencoderPretransform
    cfg = dict(DIT, input_concat_dim=65)
    dit_sd = do.make_dit_weights(cfg, seed=21)
    wrapper = DiTWrapper(**cfg)
    wrapper.model.load_state_dict(dit_sd)        # after the construction-time halving: the native model holds dit_sd
    dsd = oo.make_oobleck_weights(oo.decoder_param_shapes(DEC), seed=22, transposed=oo.decoder_transposed_prefixes(DEC))
    dec, enc = OobleckDecoder(**DEC), OobleckEncoder(**ENC)
    dec.load_state_dict(dsd)
    enc.load_state_dict(oo.make_oobleck_weights(oo.encoder_param_shapes(ENC), seed=23))
    ae = AudioAutoencoder(enc, dec, latent_dim=64, downsampling_ratio=64, sample_rate=16000, io_channels=2,
                          bottleneck=VAEBottleneck())
    model = ConditionedDiffusionModelWrapper(
        wrapper, _StubConditioner(), io_channels=64, sample_rate=16000, min_input_length=64,
        pretransform=AutoencoderPretransform(ae, scale=1.0, iterate_batch=True), cross_attn_cond_ids=["prompt"],
        global_cond_ids=["seconds_total"], input_concat_ids=["inpaint_mask", "inpaint_masked_input"]).cuda().eval()
    B, L, steps, seed, cfg_scale = 2, 48, 6, 322, 5.0
    g = torch.Generator().manual_seed(24)
    mask = (torch.rand(B, 1, L, generator=g) > 0.5).float()
    masked = torch.randn(B, 64, L, generator=g) * mask
    cond = {"prompt": (torch.randn(B, 10, 128, generator=g).cuda(), torch.ones(B, 10).cuda()),
            "seconds_total": (torch.randn(B, 1, 256, generator=g).cuda(), torch.ones(B, 1).cuda()),
            "inpaint_mask": (mask.cuda(), torch.ones(B, 1).cuda()),
            "inpaint_masked_input": (masked.cuda(), torch.ones(B, 1).cuda())}
    make_ns = _noise_samplers([torch.randn(B, 64, L, generator=g) for _ in range(steps)])
    lat = generate_diffusion_cond(model, steps=steps, cfg_scale=cfg_scale, conditioning_tensors=cond,
                                  sample_size=L * 64, seed=seed, device="cuda", return_latents=True,
                                  sampler_type="dpmpp-2m-sde", sigma_min=0.3, sigma_max=50.0,
                                  noise_sampler=make_ns("cuda"))
    audio = model.pretransform.decode(lat)
    torch.manual_seed(seed)
    noise = torch.randn([B, 64, L], device="cuda").cpu()
    cross, glob = cond["prompt"][0].cpu(), cond["seconds_total"][0].squeeze(1).cpu()
    concat = torch.cat([mask, masked], dim=1)

    def oracle_fn(x, t, **kw):
        return do.dit_forward(dit_sd, cfg, x, t, cross_attn_cond=cross, global_embed=glob, cfg_scale=cfg_scale,
                              input_concat_cond=concat)
    sigmas = so.get_sigmas_polyexponential(steps, 0.3, 50.0, 1.0)
    ref_lat = so.sample_dpmpp_2m_sde(so.VDenoiser(oracle_fn), noise * sigmas[0], sigmas, noise_sampler=make_ns("cpu"))
    ref_audio = oo.oobleck_decoder(ref_lat, dsd, DEC)
    e_lat, e_audio = rel_l2(lat.cpu(), ref_lat), rel_l2(audio.cpu(), ref_audio)
    report("generate_inpaint", rel_l2_latents=e_lat, rel_l2_audio=e_audio)
    assert lat.shape == (B, 64, L) and audio.shape == (B, 2, L * 64)
    assert e_lat < 3e-2 and e_audio < 5e-2


def test_stereoize_matches_the_oracle_pipeline():
    """A mono-to-stereo prior on raw audio: a DiT with 2 io + 2 concat channels (native K 4 -> 8, N 2 -> 32)."""
    from oracle import dit_oracle as do
    from oracle import sampler_oracle as so
    from stable_audio_tools import create_model_from_config
    cfg = dict(DIT, io_channels=2, input_concat_dim=2, cond_token_dim=0, global_cond_dim=0)
    model = create_model_from_config({"model_type": "diffusion_prior", "sample_rate": 16000,
                                      "model": {"io_channels": 2, "prior_type": "mono_stereo",
                                                "diffusion": {"type": "dit", "config": cfg,
                                                              "input_concat_ids": ["source"]}}})
    sd = do.make_dit_weights(cfg, seed=25)
    model.model.model.load_state_dict(sd)
    model = model.cuda().eval()
    B, T, steps, seed = 2, 1000, 6, 323
    g = torch.Generator().manual_seed(26)
    audio = torch.randn(B, 2, T, generator=g) * 0.3
    make_ns = _noise_samplers([torch.randn(B, 2, T, generator=g) for _ in range(steps)])
    out = model.stereoize(audio.cuda(), 16000, steps, sampler_kwargs=dict(
        seed=seed, sampler_type="dpmpp-2m-sde", sigma_min=0.3, sigma_max=50.0, noise_sampler=make_ns("cuda")))
    torch.manual_seed(seed)
    noise = torch.randn([B, 2, T], device="cuda").cpu()
    dual_mono = audio.mean(1, keepdim=True).repeat(1, 2, 1)

    def oracle_fn(x, t, **kw):
        return do.dit_forward(sd, cfg, x, t, input_concat_cond=dual_mono)
    sigmas = so.get_sigmas_polyexponential(steps, 0.3, 50.0, 1.0)
    ref = so.sample_dpmpp_2m_sde(so.VDenoiser(oracle_fn), noise * sigmas[0], sigmas, noise_sampler=make_ns("cpu"))
    err = rel_l2(out.float().cpu(), ref)
    report("stereoize", rel_l2=err)
    assert out.shape == (B, 2, T) and err < 3e-2
