"""Timing driver for the FP8 FF-out option (not a test): python tests/fp8_ff_out_time.py [reps]

At the bench shape (SA-Open width: D 1536, inner 6144, 24 blocks; batch 4 with CFG = 8 rows of 1025 tokens, M = 8200)
it times, alternating the two variants of each pair in this one process, two rounds of:
  - FF-out, 8200 x 1536 x 6144: the fp16 instance the forward runs (EpiResidual, linear_auto's BN, printed) against
    the block-scaled FP8 one (BlockScaledA<EpiResidual>, BN 128), through satb_gemm_probe / satb_gemm_probe_ff8;
  - FF-in, 8200 x 12288 x 1536 on FP8 operands: the 16-bit SwiGLU epilogue against the e4m3 block one;
  - the 24-block CFG forward at batch 4, operand_dtype "fp8" without and with ff_out_dtype "fp8";
with CUDA events over `reps` launches (10 forwards), and the rel-L2 between the two forwards' outputs.  The card's
name, power limit and the SM clock (read while timed work is running) are printed in the same run."""
import ctypes
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from stable_audio_tools import _native as nat

from fp8_ff_out_ref import quantize_fp8_blocks
from fp8_ref import quantize_fp8_rows
from fp8_time import events_ms, smi
from helpers import SAO_DIT, build_native_dit, rel_l2

M, D, FFI = 8200, 1536, 6144


def _fields(p, f):
    for k, v in f.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return p


def _alternate(label, shape, runs, reps, flops):
    for fn in runs.values():
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    for rnd in range(2):
        for mode, fn in runs.items():
            ms, clock = events_ms(fn, reps)
            print("round %d  %-7s %-22s %s: %8.1f us  %6.1f TFLOP/s  (SM clock: %s)"
                  % (rnd, label, mode, shape, ms * 1000, flops / ms / 1e9, clock), flush=True)


def time_ff_out(reps):
    lib = nat.lib()
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(M, FFI, device="cuda", generator=g)
    w = torch.randn(D, FFI, device="cuda", generator=g) * FFI ** -0.5
    h = torch.zeros(M, D, device="cuda")
    bias = torch.randn(D, device="cuda", generator=g)
    a16, w16 = a.half(), w.half()
    qa, sa = quantize_fp8_blocks(a)
    qw, sw = quantize_fp8_rows(w)
    a8, w8 = qa.view(torch.uint8).contiguous(), qw.view(torch.uint8).contiguous()
    sa, sw = sa.contiguous(), sw[:, 0].contiguous()
    # linear_auto's N tile for 65 m-tiles x 1536 columns (csrc/linear.cuh auto_bn)
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def eff(bn):
        waves = 65 * (D // bn) / sms
        return waves / math.ceil(waves)
    bn16 = 128 if eff(128) * 0.9 > eff(256) else 256
    p16 = _fields(nat.SatbGemmProbe(), dict(epi=nat.EPI_RESIDUAL, bn=bn16, b_static=1, h=h, ld=D, bias=bias))
    p8 = _fields(nat.SatbGemmProbe(), dict(epi=nat.EPI_RESIDUAL_A8, bn=128, b_static=1, h=h, ld=D, bias=bias))
    runs = {f"fp16 BN{bn16}": lambda: nat.check(lib.satb_gemm_probe(a16.data_ptr(), w16.data_ptr(), M, D, FFI,
                                                                     ctypes.byref(p16), nat.stream_ptr())),
            "fp8 block-scaled BN128": lambda: nat.check(lib.satb_gemm_probe_ff8(
                a8.data_ptr(), w8.data_ptr(), sa.data_ptr(), sw.data_ptr(), M, D, FFI, ctypes.byref(p8), None, None,
                nat.stream_ptr()))}
    _alternate("FF-out", f"{M}x{D}x{FFI}", runs, reps, 2.0 * M * D * FFI)


def time_ff_in(reps):
    lib = nat.lib()
    g = torch.Generator(device="cuda").manual_seed(2)
    a = torch.randn(M, D, device="cuda", generator=g)
    w = torch.randn(2 * FFI, D, device="cuda", generator=g) * D ** -0.5
    bias = torch.randn(2 * FFI, device="cuda", generator=g) * 0.1
    qa, sa = quantize_fp8_rows(a)
    qw, sw = quantize_fp8_rows(w)
    a8, w8 = qa.view(torch.uint8).contiguous(), qw.view(torch.uint8).contiguous()
    sa, sw = sa[:, 0].contiguous(), sw[:, 0].contiguous()
    out16 = torch.empty(M, FFI, dtype=torch.float16, device="cuda")
    ff8 = torch.empty(M, FFI, dtype=torch.uint8, device="cuda")
    ffs = torch.empty(M, FFI // 128, device="cuda")
    p16 = _fields(nat.SatbGemmProbe(), dict(epi=nat.EPI_SWIGLU, bn=256, b_static=1, out=out16, ld=FFI, bias=bias))
    p8 = _fields(nat.SatbGemmProbe(), dict(epi=nat.EPI_SWIGLU_E4M3, bn=256, b_static=1, ld=FFI, bias=bias))
    args = lambda: (a8.data_ptr(), w8.data_ptr(), sa.data_ptr(), sw.data_ptr(), M, 2 * FFI, D)
    runs = {"16-bit epilogue": lambda: nat.check(lib.satb_gemm_probe_fp8(*args(), ctypes.byref(p16), nat.stream_ptr())),
            "e4m3 block epilogue": lambda: nat.check(lib.satb_gemm_probe_ff8(*args(), ctypes.byref(p8), ff8.data_ptr(),
                                                                             ffs.data_ptr(), nat.stream_ptr()))}
    _alternate("FF-in", f"{M}x{2 * FFI}x{D}", runs, reps, 2.0 * M * 2 * FFI * D)


def time_forward():
    from oracle import dit_oracle as do
    sd = do.make_dit_weights(SAO_DIT, seed=10)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    models = {"fp8": build_native_dit(SAO_DIT, sd, operand_dtype="fp8"),
              "fp8 + ff_out fp8": build_native_dit(dict(SAO_DIT, ff_out_dtype="fp8"), sd, operand_dtype="fp8")}
    outs = {}
    for mode, m in models.items():
        for _ in range(3):
            outs[mode] = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    torch.cuda.synchronize()
    for rnd in range(2):
        for mode, m in models.items():
            ms, clock = events_ms(lambda: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0), 10)
            print("round %d  forward %-16s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)" % (rnd, mode, ms, clock),
                  flush=True)
    print("rel-L2 of the ff_out fp8 output against the fp8 one: %.3e"
          % rel_l2(outs["fp8 + ff_out fp8"].cpu(), outs["fp8"].cpu()), flush=True)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    time_ff_out(reps)
    time_ff_in(reps)
    time_forward()


if __name__ == "__main__":
    main()
