"""Timing driver for the feed-forward variants (not a test): python tests/ff_variant_time.py [calls]

At SA-Open width (D 1536, 24 heads, 24 blocks, a 130 x 768 cross-attention context; batch 4 with CFG = 8 rows of 1025
tokens, M = 8200) it builds four models - the default SwiGLU feed-forward (inner 6144), mult 8/3 (inner 4096), SwiGLU
FF-in + Conv1d k 3 FF-out, and Conv1d k 3 + SiLU FF-in with a Conv1d k 3 FF-out (glu=False, inner 6144) - and, in this one
process:
  - times one CFG forward of each, alternated over two rounds (CUDA events over `calls` calls after a warm-up);
  - reads the FF-in / FF-out GEMM times per block from satb_dit_profile, with their TFLOP/s for the operations the
    layer needs: FF-out 2 M inner D k (154.8 GF per layer for the default's Linear), FF-in 2 M D (2 inner) for SwiGLU,
    2 M D inner k for a plain convolution.
The card's name, power limit and the SM clock (read while timed work is running) are printed in the same run."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from stable_audio_tools import _native as nat

from fp8_time import events_ms, smi
from helpers import SAO_DIT, build_native_dit

ROWS, SEQ, D = 8, 1025, 1536
M = ROWS * SEQ
VARIANTS = {
    "default": {},
    "mult8/3": dict(mult=8 / 3),
    "swiglu+conv3": dict(use_conv=True, conv_kernel_size=3),
    "plain conv3": dict(glu=False, use_conv=True, conv_kernel_size=3),
}


def ff_flops(ffk):
    inner = int(D * ffk.get("mult", 4))
    k = ffk.get("conv_kernel_size", 3) if ffk.get("use_conv") else 1
    glu = ffk.get("glu", True)
    ff_in = 2.0 * M * D * 2 * inner if glu else 2.0 * M * D * inner * k
    return ff_in, 2.0 * M * inner * D * k


def main():
    from oracle import feedforward_oracle as fo
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    c[:, 40:] = 0.0
    call = lambda m: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0)
    models = {}
    for name, ffk in VARIANTS.items():
        cfg = dict(SAO_DIT, ff_kwargs=ffk) if ffk else SAO_DIT
        m = build_native_dit(cfg, fo.make_dit_weights(cfg, seed=10))
        for _ in range(3):
            call(m)
        torch.cuda.synchronize()
        models[name] = m
    lib = nat.lib()
    ms8, cnt8 = (ctypes.c_float * 8)(), (ctypes.c_int * 8)()
    steps, blocks = 5, 5 * SAO_DIT["depth"]
    base_out = None
    for name, m in models.items():
        h = m.__dict__["_h"]
        nat.check(lib.satb_dit_profile(h, 1))
        nat.check(lib.satb_dit_profile_read(h, ms8, cnt8))
        for _ in range(steps):
            call(m)
        nat.check(lib.satb_dit_profile_read(h, ms8, cnt8))
        nat.check(lib.satb_dit_profile(h, 0))
        fin, fout = ff_flops(VARIANTS[name])
        t_in, t_out = ms8[0] / blocks, ms8[1] / blocks
        line = ("profiled per block  %-13s FF-in %7.1f us (%6.1f GF, %5.0f TFLOP/s)  FF-out %7.1f us (%6.1f GF, %5.0f "
                "TFLOP/s)" % (name, t_in * 1e3, fin / 1e9, fin / t_in / 1e9, t_out * 1e3, fout / 1e9, fout / t_out / 1e9))
        if name == "default":
            base_out = fout / t_out
        else:
            line += "  FF-out rate / the default Linear's: %.3f" % (fout / t_out / base_out)
        print(line, flush=True)
    for rnd in range(2):
        for name, m in models.items():
            ms, clock = events_ms(lambda: call(m), calls)
            print("round %d  forward %-13s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)" % (rnd, name, ms, clock),
                  flush=True)


if __name__ == "__main__":
    main()
