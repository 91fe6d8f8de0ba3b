"""Timing driver (not a test): the PQMF filterbank kernels and a PQMF Oobleck autoencoder, CUDA events.

Prints the card, its power limit and max SM clock, then
- per band count (16 / 32 / 64 bands, the banks of tests/golden/pqmf_small.npz), the analysis and synthesis kernel
  time for 47.55 s of stereo (2097152 samples per channel at 44.1 kHz), with the fp32 work (2 * taps FLOP per sample)
  and the time that work takes at the H100 SXM data-sheet fp32 rate (67 TFLOP/s) beside it;
- the encode and decode time per sample (batch 1) of a stereo x 16-band Oobleck autoencoder at SA-Open width
  (channels 128, c_mults [1, 2, 4, 8], strides [2, 4, 4, 8]: 4096 samples per latent, 512 latents), pretransform
  included, with the PQMF kernels' share.
Each number is the median over the rounds (min / max beside it).
usage: python tests/pqmf_time.py [rounds] [reps per round]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
import numpy as np
import torch
from oracle import pqmf_oracle as po
from stable_audio_tools.models.factory import create_model_from_config
from stable_audio_tools.models.pretransforms import PQMFPretransform

T = 2097152
FP32_PEAK = 67e12
BANKS = [(100, 16), (100, 32), (80, 64)]


def _time(fn, rounds, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    out.sort()
    return out[len(out) // 2], out[0], out[-1]


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("gpu:", q or torch.cuda.get_device_name())
    g = np.load(os.path.join(ROOT, "tests", "golden", "pqmf_small.npz"))
    x = torch.randn(1, 2, T, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        for att, n in BANKS:
            pt = PQMFPretransform(att, n)
            pt.load_state_dict({"pqmf.filter_bank": torch.from_numpy(g[f"a{att}_n{n}_filter_bank"]),
                                "pqmf.prototype": torch.from_numpy(g[f"a{att}_n{n}_prototype"])})
            pt = pt.cuda()
            taps = pt.pqmf.filter_bank.shape[-1]
            bands = pt.encode(x)
            flop = 2.0 * taps * 2 * T
            for name, fn in (("analysis", lambda: pt.encode(x)), ("synthesis", lambda: pt.decode(bands))):
                med, lo, hi = _time(fn, rounds, reps)
                print(f"pqmf {n:3d} bands ({taps} taps) {name:9s}: median {med:7.3f} ms  min {lo:7.3f}  max {hi:7.3f}  "
                      f"| {flop / 1e9:.2f} GFLOP fp32, {flop / FP32_PEAK * 1e3:.3f} ms at 67 TFLOP/s, achieved "
                      f"{flop / (med * 1e-3) / 1e12:.1f} TFLOP/s", flush=True)
        oob = dict(channels=128, c_mults=[1, 2, 4, 8], strides=[2, 4, 4, 8], use_snake=True)
        cfg = {"sample_rate": 44100, "model_type": "autoencoder", "model": {
            "io_channels": 2, "latent_dim": 64, "downsampling_ratio": 4096, "bottleneck": {"type": "vae"},
            "pretransform": {"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}},
            "encoder": {"type": "oobleck", "config": dict(oob, in_channels=32, latent_dim=128)},
            "decoder": {"type": "oobleck", "config": dict(oob, out_channels=32, latent_dim=64, final_tanh=False)}}}
        ae = create_model_from_config(cfg)
        ae.load_state_dict(po.autoencoder_state_dict(cfg, g["a100_n16_filter_bank"], g["a100_n16_prototype"], 1))
        ae = ae.cuda().eval()
        z = torch.randn(1, 64, T // 4096, generator=torch.Generator().manual_seed(1)).cuda()
        pre = ae.pretransform
        bands = pre.encode(x)
        for name, fn, pq in (("encode", lambda: ae.encoder(pre.encode(x)), lambda: pre.encode(x)),
                             ("decode", lambda: pre.decode(ae.decoder(z)), lambda: pre.decode(bands))):
            med, lo, hi = _time(fn, rounds, max(1, reps // 5))
            pmed, _, _ = _time(pq, rounds, reps)
            print(f"pqmf-oobleck 16 bands {name}: median {med:7.3f} ms per 47.55 s stereo sample  min {lo:7.3f}  "
                  f"max {hi:7.3f}  (PQMF kernel {pmed:.3f} ms, {pmed / med * 100:.1f} %)", flush=True)


if __name__ == "__main__":
    main()
