"""Timing driver for the FP8 operand mode (not a test): python tests/fp8_time.py [reps]

At the bench shape (SA-Open width: D 1536, 24 blocks, 24 heads, a 130 x 768 cross-attention context; batch 4 with CFG
= 8 rows of 1025 tokens, M = 8200) it times, with fp16 and FP8 alternated in this one process, two rounds:
  - the three GEMMs the FP8 mode changes (QKV with rotary, FF-in with SwiGLU, the cross-attention q projection), as the
    forward runs them, through satb_gemm_probe / satb_gemm_probe_fp8 (CUDA events over `reps` launches);
  - one full 24-block CFG forward (CUDA events over 10 calls after a warm-up);
and prints the rel-L2 of the FP8 forward output against the fp16 one.  The card's name, power limit and the SM clock
(read while timed work is running) are printed in the same run."""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from stable_audio_tools import _native as nat

from fp8_ref import quantize_fp8_rows
from helpers import SAO_DIT, build_native_dit, rel_l2

M, D, FFI, SEQ = 8200, 1536, 6144, 1025
MC = 4 * SEQ          # rows with a cross-attention context (the conditional half under CFG, no negative prompt)


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unavailable"
    except (OSError, subprocess.SubprocessError):
        return "unavailable"


def events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    clock = smi("clocks.sm")          # the launches above are still running
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, clock


def gemm_cases():
    """name -> (rows, N, K, bn, epilogue fields)"""
    g = torch.Generator(device="cuda").manual_seed(0)
    cos = torch.rand(SEQ, 16, device="cuda", generator=g)
    sin = torch.rand(SEQ, 16, device="cuda", generator=g)
    return {
        "QKV": (M, 3 * D, D, 256, dict(epi=nat.EPI_QKV_ROPE, out=torch.empty(M, 3 * D, dtype=torch.float16, device="cuda"),
                                       ld=3 * D, rope_cols=2 * D, seq_len=SEQ, head_dim=64, nf=16, cos_tab=cos, sin_tab=sin)),
        "FF-in": (M, 2 * FFI, D, 256, dict(epi=nat.EPI_SWIGLU, out=torch.empty(M, FFI, dtype=torch.float16, device="cuda"),
                                           ld=FFI, bias=torch.randn(2 * FFI, device="cuda", generator=g))),
        # linear_auto's choice for 4100 rows x 1536 columns on 132 SMs is BN 256 (printed below)
        "cross-q": (MC, D, D, 256, dict(epi=nat.EPI_STORE16, out=torch.empty(MC, D, dtype=torch.float16, device="cuda"),
                                        ld=D, act=0)),
    }


def time_gemms(reps):
    lib = nat.lib()
    res = {}
    for name, (rows, N, K, bn, f) in gemm_cases().items():
        g = torch.Generator(device="cuda").manual_seed(N + K)
        a = torch.randn(rows, K, device="cuda", generator=g)
        w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
        a16, w16 = a.half(), w.half()
        qa, sa = quantize_fp8_rows(a)
        qw, sw = quantize_fp8_rows(w)
        a8, w8 = qa.view(torch.uint8).contiguous(), qw.view(torch.uint8).contiguous()
        sa, sw = sa[:, 0].contiguous(), sw[:, 0].contiguous()
        p = nat.SatbGemmProbe()
        p.bn, p.bf16, p.b_static = bn, 0, 1
        for k, v in f.items():
            setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
        run16 = lambda: nat.check(lib.satb_gemm_probe(a16.data_ptr(), w16.data_ptr(), rows, N, K, ctypes.byref(p),
                                                      nat.stream_ptr()))
        run8 = lambda: nat.check(lib.satb_gemm_probe_fp8(a8.data_ptr(), w8.data_ptr(), sa.data_ptr(), sw.data_ptr(), rows,
                                                         N, K, ctypes.byref(p), nat.stream_ptr()))
        for fn in (run16, run8):
            for _ in range(10):
                fn()
        torch.cuda.synchronize()
        for rnd in range(2):
            for mode, fn in (("fp16", run16), ("fp8", run8)):
                ms, clock = events_ms(fn, reps)
                print("round %d  %-7s %-4s %dx%dx%d BN%d: %8.1f us  %6.1f TFLOP/s  (SM clock: %s)"
                      % (rnd, name, mode, rows, N, K, bn, ms * 1000, 2.0 * rows * N * K / ms / 1e9, clock), flush=True)
    return res


def time_forward():
    from oracle import dit_oracle as do
    sd = do.make_dit_weights(SAO_DIT, seed=10)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    models = {mode: build_native_dit(SAO_DIT, sd, operand_dtype=mode) for mode in ("fp16", "fp8")}
    outs = {}
    for mode, m in models.items():
        for _ in range(3):
            outs[mode] = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    torch.cuda.synchronize()
    for rnd in range(2):
        for mode, m in models.items():
            ms, clock = events_ms(lambda: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0), 10)
            print("round %d  forward %-4s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)" % (rnd, mode, ms, clock),
                  flush=True)
    print("rel-L2 of the FP8 output against fp16: %.3e" % rel_l2(outs["fp8"].cpu(), outs["fp16"].cpu()), flush=True)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    time_gemms(reps)
    time_forward()


if __name__ == "__main__":
    main()
