"""GPU: the native PQMF filterbank and the Oobleck autoencoders built around it.

- analysis and synthesis (satb_pqmf_*) against the float64 oracle for 16 / 32 / 64 bands, mono and stereo, B = 2 and
  3, lengths that are not a multiple of the band count and lengths shorter than the filter: rel-L2 <= 1e-5 (fp32 FMA
  over up to 2048 taps), and against the real reference's goldens at the same bound;
- the PQMF autoencoder golden (stereo x 16 bands -> a 32-channel Oobleck, built by the reference's
  create_autoencoder_from_config) in every operand_dtype, at the gates of tests/test_gpu_oobleck_variants.py
  (rel-L2 4e-3 fp16, 2.5e-2 bf16, 70 dB fp16x3), through encode / decode, iterate_batch and the chunked paths;
- wide Oobleck I/O (32 and 128 sub-bands: the encoder's GEMM input conv, the decoder's halo-tile and GEMM output
  routes) against the fp32 oracle within 1.35 x its own fp16-operand floor;
- generate_diffusion_cond with a small DiT whose AutoencoderPretransform wraps a PQMF autoencoder, against the oracle
  pipeline at the gates of tests/test_gpu_generate.py.
"""
import json

import pytest
import torch

from helpers import load_golden, rel_l2

pytestmark = pytest.mark.gpu
BANKS = [(100, 16), (100, 32), (80, 64)]
TOL = {"fp16": 4e-3, "bf16": 2.5e-2, "fp16x3": 10 ** (-70 / 20)}
FLOOR_GATE = 1.35


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _pqmf(att, n):
    from stable_audio_tools.models.pretransforms import PQMFPretransform
    g = load_golden("pqmf_small.npz")
    p = f"a{att}_n{n}_"
    pt = PQMFPretransform(att, n)
    pt.load_state_dict({"pqmf.filter_bank": torch.from_numpy(g[p + "filter_bank"]),
                        "pqmf.prototype": torch.from_numpy(g[p + "prototype"])})
    return pt.cuda(), g, p


@pytest.mark.parametrize("att,n", BANKS)
def test_kernels_match_reference_golden(att, n):
    pt, g, p = _pqmf(att, n)
    for name in ("long", "short"):
        y = pt.encode(torch.from_numpy(g[p + "x_" + name]).cuda()).cpu()
        ref = torch.from_numpy(g[p + "y_" + name])
        assert y.shape == ref.shape
        assert rel_l2(y, ref) <= 1e-5, (name, rel_l2(y, ref))
    s = pt.decode(torch.from_numpy(g[p + "z"]).cuda()).cpu()
    assert s.shape == g[p + "s"].shape
    assert rel_l2(s, torch.from_numpy(g[p + "s"])) <= 1e-5


@pytest.mark.parametrize("att,n", BANKS)
@pytest.mark.parametrize("B,C", [(2, 1), (3, 2)])
@pytest.mark.parametrize("T", [1, 333, 44100 + 7, 5 * 4096])
def test_kernels_match_float64_oracle(att, n, B, C, T):
    from oracle import pqmf_oracle as po
    pt, _, _ = _pqmf(att, n)
    bank = pt.pqmf.filter_bank.cpu()
    gen = torch.Generator().manual_seed(T + 7 * n + C)
    x = torch.randn(B, C, T, generator=gen)
    y = pt.encode(x.cuda())
    ref = po.analysis(x, bank)
    assert y.shape == ref.shape == (B, C * n, -(-T // n))
    err = rel_l2(y.cpu().double(), ref)
    z = torch.randn(B, C * n, max(1, T // n), generator=gen)
    s = pt.decode(z.cuda())
    sref = po.synthesis(z, bank)
    assert s.shape == sref.shape == (B, C, z.shape[-1] * n)
    serr = rel_l2(s.cpu().double(), sref)
    print(f"n={n} B={B} C={C} T={T}: analysis rel-L2 {err:.3g}, synthesis {serr:.3g}")
    assert err <= 1e-5 and serr <= 1e-5


def test_batch_items_are_independent_and_graph_replay_is_bit_identical():
    pt, _, _ = _pqmf(100, 32)
    x = torch.randn(3, 2, 32 * 700 + 5, generator=torch.Generator().manual_seed(1)).cuda()
    y = pt.encode(x)
    assert torch.equal(y[1:2], pt.encode(x[1:2].contiguous()))
    s = pt.decode(y)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y2 = pt.encode(x)
        s2 = pt.decode(y2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y2, y) and torch.equal(s2, s)


def test_reloaded_filter_bank_takes_effect():
    pt, _, _ = _pqmf(100, 16)
    x = torch.randn(1, 1, 4096, generator=torch.Generator().manual_seed(2)).cuda()
    y = pt.encode(x)
    sd = {k: v.clone() for k, v in pt.state_dict().items()}
    sd["pqmf.filter_bank"] *= 2
    pt.load_state_dict(sd)
    assert torch.allclose(pt.encode(x), 2 * y, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------ PQMF autoencoders
def _ae(dtype="fp16"):
    from oracle import pqmf_oracle as po
    from stable_audio_tools.models.factory import create_model_from_config
    g = load_golden("oobleck_pqmf_small.npz")
    cfg = json.loads(str(g["config"]))
    for part in ("encoder", "decoder"):
        cfg["model"][part]["config"]["operand_dtype"] = dtype
    gb = load_golden("pqmf_small.npz")
    sd = po.autoencoder_state_dict(cfg, gb["a100_n16_filter_bank"], gb["a100_n16_prototype"], int(g["seed"]))
    model = create_model_from_config(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda().eval(), g, cfg, sd


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp16x3"])
def test_autoencoder_vs_reference_golden(dtype):
    model, g, _, _ = _ae(dtype)
    a, z = torch.from_numpy(g["a"]).cuda(), torch.from_numpy(g["z"]).cuda()
    with torch.no_grad():
        h = model.encode(a).cpu()
        y = model.decode(z).cpu()
        h_it = model.encode(a, iterate_batch=1).cpu()
        y_it = model.decode(z, iterate_batch=1).cpu()
    eh, ey = rel_l2(h, torch.from_numpy(g["h"])), rel_l2(y, torch.from_numpy(g["y"]))
    print(f"PQMF autoencoder {dtype}: encode rel-L2 {eh:.3g}, decode {ey:.3g}")
    assert h.shape == g["h"].shape and y.shape == g["y"].shape
    assert eh < TOL[dtype] and ey < TOL[dtype]
    assert torch.equal(h_it, h) and torch.equal(y_it, y)


def test_autoencoder_chunked_paths_apply_the_pretransform():
    """encode_audio / decode_audio chunked run the pretransform on each chunk, as the reference's do (they call
    encode / decode): the chunked outputs have the pretransformed shapes and stay near the unchunked ones, which
    match the oracle."""
    from oracle import pqmf_oracle as po
    model, g, cfg, sd = _ae("fp16x3")
    bank = sd["pretransform.pqmf.filter_bank"]
    a = (0.5 * torch.randn(1, 2, 64 * 40, generator=torch.Generator().manual_seed(4))).clamp(-1, 1)
    z = torch.randn(1, 8, 40, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        h = model.encode_audio(a.cuda(), chunked=True, chunk_size=32, overlap=8).cpu()
        y = model.decode_audio(z.cuda(), chunked=True, chunk_size=32, overlap=8).cpu()
        h_full = model.encode_audio(a.cuda()).cpu()
        y_full = model.decode_audio(z.cuda()).cpu()
    assert h.shape == (1, 8, 40) and y.shape == (1, 2, 40 * 64)
    assert rel_l2(h_full, po.encode(a, sd, cfg, bank).float()) < 1e-3
    assert rel_l2(y_full, po.decode(z, sd, cfg, bank).float()) < 1e-3
    assert bool(torch.isfinite(h).all()) and bool(torch.isfinite(y).all())
    assert rel_l2(h[..., 4:-4], h_full[..., 4:-4]) < 0.5 and rel_l2(y, y_full) < 0.5


def _floor_check(fn, cfg, sd, x, y):
    from oracle import oobleck_oracle as oo
    sdc = {k: v.cuda() for k, v in sd.items()}
    xc = x.cuda()
    with torch.no_grad():
        ref = fn(xc, sdc, cfg)
        with oo.operand_rounding(torch.float16):
            floor = rel_l2(fn(xc, sdc, cfg), ref)
    err = rel_l2(y, ref)
    print(f"rel-L2 {err:.4g}, fp16 floor {floor:.4g}, ratio {err / floor:.3f}")
    assert y.shape == ref.shape
    assert err <= FLOOR_GATE * floor, (err, floor)


@pytest.mark.parametrize("width", [32, 128])
@pytest.mark.parametrize("snake", [True, False])
def test_wide_io_oobleck_vs_oracle_floor(width, snake):
    from oracle import oobleck_variants_oracle as ov
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    base = dict(channels=64, c_mults=[1, 2], strides=[2, 4], use_snake=snake)
    ecfg, dcfg = dict(base, in_channels=width, latent_dim=16), dict(base, out_channels=width, latent_dim=8,
                                                                      final_tanh=True)
    esd, dsd = ov.make_encoder_weights(ecfg, seed=width), ov.make_decoder_weights(dcfg, seed=width + 1)
    enc, dec = OobleckEncoder(**ecfg), OobleckDecoder(**dcfg)
    enc.load_state_dict(esd)
    dec.load_state_dict(dsd)
    enc, dec = enc.cuda(), dec.cuda()
    x = torch.randn(2, width, 8 * 300, generator=torch.Generator().manual_seed(6)) * 0.1
    z = torch.randn(2, 8, 300, generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        h = enc(x.cuda())
        y = dec(z.cuda())
    _floor_check(ov.oobleck_encoder, ecfg, esd, x, h)
    _floor_check(ov.oobleck_decoder, dcfg, dsd, z, y)


def test_wide_encoder_input_probe_runs_on_tensor_cores():
    """ENC_IN of a 32-channel encoder runs the implicit GEMM (not the CUDA-core kernel) and matches the float64
    conv + Snake of its input at the operand rounding."""
    import ctypes
    from oracle import oobleck_variants_oracle as ov
    from stable_audio_tools import _native
    from stable_audio_tools.models.autoencoders import OobleckEncoder
    cfg = dict(in_channels=32, channels=64, c_mults=[1], strides=[2], latent_dim=8, use_snake=True)
    sd = ov.make_encoder_weights(cfg, seed=3)
    enc = OobleckEncoder(**cfg)
    enc.load_state_dict(sd)
    enc = enc.cuda()
    B, L = 2, 129
    x = torch.randn(B, 32, L, generator=torch.Generator().manual_seed(8)).cuda()
    raw = torch.empty(B, L, 64, dtype=torch.float16, device="cuda")
    out16 = torch.empty(B, L, 64, dtype=torch.float16, device="cuda")
    scratch = torch.empty(B, L, 32, dtype=torch.float16, device="cuda")
    p = _native.SatbOobleckProbe(step=_native.OOB_ENC_IN, block=0, unit=0, B=B, L=L, in_=x.data_ptr(),
                                 raw_out=raw.data_ptr(), out16=out16.data_ptr(), scratch=scratch.data_ptr())
    h = enc._handle(x.device)
    _native.check(_native.lib().satb_oobleck_probe(h, ctypes.byref(p), _native.stream_ptr(x.device)))
    torch.cuda.synchronize()
    assert p.routes & 3 and not p.routes & 64, p.routes
    from oracle import oobleck_oracle as oo
    sdc = {k: v.cuda().double() for k, v in sd.items()}
    w = oo.fold_weight_norm(sdc["layers.0.weight_g"], sdc["layers.0.weight_v"])
    ref = torch.nn.functional.conv1d(x.half().double(), w.half().double(), sdc["layers.0.bias"], padding=3)
    assert rel_l2(raw.permute(0, 2, 1).double(), ref) < 2e-3
    # without scratch the wide input conv is refused before any launch
    p.scratch = None
    assert _native.lib().satb_oobleck_probe(h, ctypes.byref(p), _native.stream_ptr(x.device)) != 0


# ------------------------------------------------------------------------------------------ generation
class _StubConditioner(torch.nn.Module):
    def set_device(self, device):
        pass


def test_generate_with_a_pqmf_autoencoder_pretransform_matches_oracle_pipeline():
    from oracle import dit_oracle as do
    from oracle import pqmf_oracle as po
    from oracle import sampler_oracle as so
    from stable_audio_tools.inference.generation import generate_diffusion_cond
    from stable_audio_tools.models.diffusion import ConditionedDiffusionModelWrapper, DiTWrapper
    from stable_audio_tools.models.factory import create_model_from_config
    from stable_audio_tools.models.pretransforms import AutoencoderPretransform
    dit_cfg = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
                   project_cond_tokens=False, transformer_type="continuous_transformer")
    dit_sd = do.make_dit_weights(dit_cfg, seed=1)
    wrapper = DiTWrapper(**dit_cfg)
    wrapper.model.load_state_dict(dit_sd)
    oob = dict(channels=32, c_mults=[1, 2], strides=[2, 4], use_snake=True)
    ae_cfg = {"sample_rate": 16000, "model_type": "autoencoder", "model": {
        "io_channels": 2, "latent_dim": 64, "downsampling_ratio": 128, "bottleneck": {"type": "vae"},
        "pretransform": {"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}},
        "encoder": {"type": "oobleck", "config": dict(oob, in_channels=32, latent_dim=128)},
        "decoder": {"type": "oobleck", "config": dict(oob, out_channels=32, latent_dim=64, final_tanh=False)}}}
    ae = create_model_from_config(ae_cfg)
    gb = load_golden("pqmf_small.npz")
    sd = po.autoencoder_state_dict(ae_cfg, gb["a100_n16_filter_bank"], gb["a100_n16_prototype"], 11)
    ae.load_state_dict(sd, strict=True)
    pre = AutoencoderPretransform(ae, scale=1.0, iterate_batch=True)
    model = ConditionedDiffusionModelWrapper(wrapper, _StubConditioner(), io_channels=64, sample_rate=16000,
                                             min_input_length=128, pretransform=pre,
                                             cross_attn_cond_ids=["prompt", "seconds_start", "seconds_total"],
                                             global_cond_ids=["seconds_start", "seconds_total"]).cuda().eval()
    B, L, steps, seed, cfg_scale = 2, 40, 6, 321, 5.0
    g = torch.Generator().manual_seed(5)
    cond = {"prompt": (torch.randn(B, 10, 128, generator=g).cuda(), torch.ones(B, 10).cuda()),
            "seconds_start": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda()),
            "seconds_total": (torch.randn(B, 1, 128, generator=g).cuda(), torch.ones(B, 1).cuda())}
    sde_noise = [torch.randn(B, 64, L, generator=g) for _ in range(steps)]

    def make_ns(dev):
        it = iter(sde_noise)
        return lambda s, sn: next(it).to(dev)

    lat = generate_diffusion_cond(model, steps=steps, cfg_scale=cfg_scale, conditioning_tensors=cond,
                                  sample_size=L * 128, seed=seed, device="cuda", return_latents=True,
                                  sampler_type="dpmpp-3m-sde", sigma_min=0.3, sigma_max=50.0,
                                  noise_sampler=make_ns("cuda"))
    audio = model.pretransform.decode(lat)
    torch.manual_seed(seed)
    noise = torch.randn([B, 64, L], device="cuda").cpu()
    cross = torch.cat([cond[k][0] for k in ("prompt", "seconds_start", "seconds_total")], dim=1).cpu()
    glob = torch.cat([cond[k][0] for k in ("seconds_start", "seconds_total")], dim=-1).squeeze(1).cpu()

    def oracle_fn(x, t, **kw):
        return do.dit_forward(dit_sd, dit_cfg, x, t, cross_attn_cond=cross, global_embed=glob, cfg_scale=cfg_scale)
    sigmas = so.get_sigmas_polyexponential(steps, 0.3, 50.0, 1.0)
    ref_lat = so.sample_dpmpp_3m_sde(so.VDenoiser(oracle_fn), noise * sigmas[0], sigmas, noise_sampler=make_ns("cpu"))
    ref_audio = po.decode(ref_lat, sd, ae_cfg, sd["pretransform.pqmf.filter_bank"]).float()
    assert lat.shape == (B, 64, L) and audio.shape == ref_audio.shape == (B, 2, L * 128)
    lerr, err = rel_l2(lat.cpu(), ref_lat), rel_l2(audio.float().cpu(), ref_audio)
    print(f"generate: latents rel-L2 {lerr:.3g}, PQMF-decoded audio {err:.3g}")
    assert lerr < 3e-2 and err < 5e-2
