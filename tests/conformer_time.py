"""Timing driver for the conformer branch (not a test): python tests/conformer_time.py [reps]

At SA-Open width (D 1536, 24 heads, a 130 x 768 cross-attention context; batch 4 with CFG = 8 rows of 1025 tokens,
M = 8200) it measures, in this one process:
  - conformer_dwconv_ln_silu alone through satb_conformer_dwconv (CUDA events over `reps` launches): time, achieved
    GB/s for the bytes it must move (read and write M x D 16-bit), and that time over the byte floor at the H100 SXM's
    3.35 TB/s data-sheet HBM bandwidth;
  - the forward's per-category timing (satb_dit_profile) of a 24-block conformer model: the conformer branch (in_norm,
    the folded GEMM, the kernel, the pointwise_conv_2 GEMM) against the feed-forward GEMMs, per block;
  - one full 24-block CFG forward of the same model with and without conformer blocks (alternated, CUDA events over 10
    calls after a warm-up).
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

ITEMS, SEQ, D = 8, 1025, 1536
M = ITEMS * SEQ
HBM_PEAK = 3.35e12    # bytes/s, H100 SXM data sheet


def time_kernel(reps):
    lib = nat.lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(M, D, device="cuda", generator=g) * 0.6).half()
    w = torch.randn(D, 1, 17, device="cuda", generator=g) / 17 ** 0.5
    gamma = 1 + 0.1 * torch.randn(D, device="cuda", generator=g)
    beta = 0.1 * torch.randn(D, device="cuda", generator=g)
    out = torch.empty_like(x)
    run = lambda: nat.check(lib.satb_conformer_dwconv(x.data_ptr(), w.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                      out.data_ptr(), ITEMS, SEQ, D, 0, nat.stream_ptr()))
    for _ in range(20):
        run()
    torch.cuda.synchronize()
    nbytes = 2 * M * D * 2
    floor_us = nbytes / HBM_PEAK * 1e6
    for rnd in range(3):
        ms, clock = events_ms(run, reps)
        print("round %d  conformer_dwconv_ln_silu %dx%d fp16: %7.2f us  %6.0f GB/s  %.2f x the byte floor (%.1f us at "
              "3.35 TB/s)  (SM clock: %s)" % (rnd, M, D, ms * 1e3, nbytes / ms / 1e6, ms * 1e3 / floor_us, floor_us, clock),
              flush=True)


def time_forward():
    from oracle import conformer_oracle as co
    cfgs = {"plain": SAO_DIT, "conformer": dict(SAO_DIT, conformer=True)}
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    c[:, 40:] = 0.0
    models = {}
    for name, cfg in cfgs.items():
        models[name] = build_native_dit(cfg, co.make_dit_weights(cfg, seed=10))
    call = lambda m: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0)
    for m in models.values():
        for _ in range(3):
            call(m)
    torch.cuda.synchronize()
    lib = nat.lib()
    h = models["conformer"].__dict__["_h"]
    ms8, cnt8 = (ctypes.c_float * 8)(), (ctypes.c_int * 8)()
    nat.check(lib.satb_dit_profile(h, 1))
    nat.check(lib.satb_dit_profile_read(h, ms8, cnt8))
    steps = 5
    for _ in range(steps):
        call(models["conformer"])
    nat.check(lib.satb_dit_profile_read(h, ms8, cnt8))
    nat.check(lib.satb_dit_profile(h, 0))
    blocks = steps * SAO_DIT["depth"]
    ff = (ms8[0] + ms8[1]) / blocks
    conf = ms8[7] / blocks
    print("profiled per block (24-block conformer model, batch 4 + CFG): conformer branch %.1f us (%d launch groups), "
          "FF-in + FF-out GEMMs %.1f us; branch / FF GEMMs = %.3f" % (conf * 1e3, cnt8[7] // blocks, ff * 1e3, conf / ff),
          flush=True)
    for rnd in range(2):
        for name, m in models.items():
            ms, clock = events_ms(lambda: call(m), 10)
            print("round %d  forward %-9s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)" % (rnd, name, ms, clock),
                  flush=True)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 500
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    time_kernel(reps)
    time_forward()


if __name__ == "__main__":
    main()
