"""GPU: Oobleck VAEs with ELU activations and / or nearest-neighbour upsampling through the drop-in modules.

- the real reference's goldens (tests/golden/oobleck_*elu*/nearest*_small.npz) in fp16, bf16 and fp16x3, at the gates
  of tests/test_gpu_oobleck.py (rel-L2 4e-3 fp16, 2.5e-2 bf16) and 70 dB for fp16x3;
- SA-Open width with synthetic weights: ELU and ELU + nearest decoders at 7, 32 and 1024 latents and the ELU encoder,
  within 1.35 x the oracle's own fp16-operand floor (oobleck_oracle.operand_rounding, the nearest fold included).  The
  floor rounds the conv operands only; the fp16 mode also carries the ResidualUnit skip stream in fp16, which costs
  about +23 % on top of it (csrc/oobleck.cu, satb_oobleck_create; measured 1.21-1.25 x here on an H100).  The oracle
  runs on the GPU in fp32 with TF32 off;
- fp16x3 >= 70 dB at SA-Open width;
- a CUDA-graph replay equals the eager decode bit for bit, and batch item 1 equals the same item decoded alone.
"""
import json
import math

import pytest
import torch

from helpers import load_golden, rel_l2

pytestmark = pytest.mark.gpu
TOL = {"fp16": 4e-3, "bf16": 2.5e-2, "fp16x3": 10 ** (-70 / 20)}
FLOOR_GATE = 1.35      # operand floor x the fp16 skip stream's ~1.23 (see the module docstring)
SAO = dict(channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8], latent_dim=64)
GOLDENS = [("oobleck_elu_small.npz", "dec"), ("oobleck_elu_small.npz", "enc"), ("oobleck_nearest_small.npz", "dec"),
           ("oobleck_elu_nearest_small.npz", "dec")]


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _module(kind, cfg, sd, dtype="fp16"):
    from stable_audio_tools.models.autoencoders import OobleckDecoder, OobleckEncoder
    m = (OobleckDecoder if kind == "dec" else OobleckEncoder)(**cfg, operand_dtype=dtype)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp16x3"])
@pytest.mark.parametrize("name,kind", GOLDENS)
def test_vs_reference_golden(name, kind, dtype):
    from oracle import oobleck_variants_oracle as ov
    g = load_golden(name)
    cfg = json.loads(str(g[kind + "_cfg"]))
    sd = (ov.make_decoder_weights if kind == "dec" else ov.make_encoder_weights)(cfg, seed=int(g[kind + "_seed"]))
    m = _module(kind, cfg, sd, dtype)
    x, ref = (g["z"], g["audio"]) if kind == "dec" else (g["a"], g["h"])
    y = m(torch.from_numpy(x).cuda()).cpu()
    assert y.shape == tuple(ref.shape)
    err = rel_l2(y, torch.from_numpy(ref))
    print(f"{name} {kind} {dtype}: rel-L2 {err:.3g}")
    assert err < TOL[dtype], err


def _sao_dec(nearest, seed):
    from oracle import oobleck_variants_oracle as ov
    cfg = dict(SAO, out_channels=2, final_tanh=False, use_nearest_upsample=nearest)
    return cfg, ov.make_decoder_weights(cfg, seed=seed)


def _floor_check(fn, cfg, sd, x, y):
    """y (native, fp16 operands) against the fp32 oracle on the device, gate 1.35 x the oracle's fp16 floor."""
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


@pytest.mark.parametrize("nearest", [False, True])
@pytest.mark.parametrize("L", [7, 32, 1024])
def test_sao_width_elu_decoder_vs_oracle_floor(nearest, L):
    from oracle import oobleck_variants_oracle as ov
    cfg, sd = _sao_dec(nearest, seed=70 + int(nearest))
    dec = _module("dec", cfg, sd)
    z = torch.randn(1, 64, L, generator=torch.Generator().manual_seed(L))
    with torch.no_grad():
        y = dec(z.cuda())
    assert y.shape == (1, 2, L * 2048) and bool(torch.isfinite(y).all())
    _floor_check(ov.oobleck_decoder, cfg, sd, z, y)


def test_sao_width_elu_encoder_vs_oracle_floor():
    from oracle import oobleck_variants_oracle as ov
    cfg = dict(SAO, in_channels=2, latent_dim=128)
    sd = ov.make_encoder_weights(cfg, seed=72)
    enc = _module("enc", cfg, sd)
    a = (0.5 * torch.randn(1, 2, 24 * 2048, generator=torch.Generator().manual_seed(5))).clamp(-1, 1)
    with torch.no_grad():
        h = enc(a.cuda())
    assert h.shape == (1, 128, 24)
    _floor_check(ov.oobleck_encoder, cfg, sd, a, h)


@pytest.mark.parametrize("nearest", [False, True])
def test_sao_width_split_operand_mode_reaches_70_db(nearest):
    from oracle import oobleck_variants_oracle as ov
    cfg, sd = _sao_dec(nearest, seed=74 + int(nearest))
    z = torch.randn(1, 64, 32, generator=torch.Generator().manual_seed(59))
    with torch.no_grad():
        ref = ov.oobleck_decoder(z.cuda(), {k: v.cuda() for k, v in sd.items()}, cfg)
        y = _module("dec", cfg, sd, "fp16x3")(z.cuda())
    snr = -20.0 * math.log10(rel_l2(y, ref))
    print(f"ELU decoder (nearest={nearest}) fp16x3 SNR {snr:.1f} dB")
    assert snr >= 70.0, snr
    if not nearest:
        ecfg = dict(SAO, in_channels=2, latent_dim=128)
        esd = ov.make_encoder_weights(ecfg, seed=72)
        a = (0.5 * torch.randn(1, 2, 8 * 2048, generator=torch.Generator().manual_seed(5))).clamp(-1, 1)
        with torch.no_grad():
            eref = ov.oobleck_encoder(a.cuda(), {k: v.cuda() for k, v in esd.items()}, ecfg)
            h = _module("enc", ecfg, esd, "fp16x3")(a.cuda())
        esnr = -20.0 * math.log10(rel_l2(h, eref))
        print(f"ELU encoder fp16x3 SNR {esnr:.1f} dB")
        assert esnr >= 70.0, esnr


@pytest.mark.parametrize("snake,nearest", [(False, False), (False, True), (True, True)])
def test_graph_replay_and_batch_item_are_bit_identical(snake, nearest):
    from oracle import oobleck_variants_oracle as ov
    cfg = dict(SAO, out_channels=2, final_tanh=True, use_snake=snake, use_nearest_upsample=nearest)
    dec = _module("dec", cfg, ov.make_decoder_weights(cfg, seed=80))
    z = torch.randn(3, 64, 12, generator=torch.Generator().manual_seed(81)).cuda()
    with torch.no_grad():
        eager = dec(z)
        alone = dec(z[1:2].contiguous())
        dec(z)                                          # workspaces sized, tensor maps cached before capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = dec(z)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert torch.equal(eager[1:2], alone)
