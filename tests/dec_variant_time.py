"""Timing driver (not a test): SA-Open-width Oobleck decode of 1024 latents (fp16 operands) for the four block
variants, Snake / ELU activations x transposed / nearest upsampling, alternated in one process, CUDA events.
Prints the card, its power limit and max SM clock, and per variant the median and spread over the rounds.
usage: python tests/dec_variant_time.py [rounds] [reps per round]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
import torch
from oracle import oobleck_variants_oracle as ov
from stable_audio_tools.models.autoencoders import OobleckDecoder

SAO = dict(out_channels=2, channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8], latent_dim=64,
           final_tanh=False)
VARIANTS = {"snake+transposed": (True, False), "elu+transposed": (False, False), "snake+nearest": (True, True),
            "elu+nearest": (False, True)}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("gpu:", q or torch.cuda.get_device_name())
    z = torch.randn(1, 64, 1024, generator=torch.Generator().manual_seed(0)).cuda()
    decs = {}
    for name, (snake, nearest) in VARIANTS.items():
        cfg = dict(SAO, use_snake=snake, use_nearest_upsample=nearest)
        d = OobleckDecoder(**cfg)
        d.load_state_dict(ov.make_decoder_weights(cfg, seed=9))
        decs[name] = d.cuda().eval()
        with torch.no_grad():
            for _ in range(2):
                decs[name](z)
    torch.cuda.synchronize()
    times = {n: [] for n in decs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for _ in range(rounds):
            for name, d in decs.items():
                e0.record()
                for _ in range(reps):
                    d(z)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / reps)
    base = sorted(times["snake+transposed"])[rounds // 2]
    for name, t in times.items():
        t = sorted(t)
        med = t[rounds // 2]
        print(f"decode_ms {name:18s} median {med:8.3f}  min {t[0]:8.3f}  max {t[-1]:8.3f}  vs snake+transposed "
              f"{med / base:.3f}", flush=True)


if __name__ == "__main__":
    main()
