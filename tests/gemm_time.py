"""Timing driver for the DiT linears (not a test): python tests/gemm_time.py [reps]

Times the forward's own gemm_wgmma_kernel instances through satb_gemm_probe at the SA-Open bench shapes (8 rows x 1025
tokens, M = 8200, fp16): FF-in (SwiGLU), FF-out (residual), QKV (rotary) and out-proj (residual), with the tile widths
the forward picks.  CUDA events over `reps` launches (default 200) after a warm-up; the SM clock is read while the
timed launches are still running, next to the card's name and power limit.  SATB_LIB points at another build of the
library for side-by-side A/B runs."""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
import torch
from stable_audio_tools import _native as nat

if os.environ.get("SATB_LIB"):          # A/B of kernel variants built side by side (tools only)
    nat.LIB_PATH = os.path.abspath(os.environ["SATB_LIB"])


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unavailable"
    except (OSError, subprocess.SubprocessError):
        return "unavailable"


M, D, FFI = 8200, 1536, 6144
SEQ, HEAD_DIM, NF = 1025, 64, 16


def cases():
    """name -> (N, K, bn, epilogue fields)"""
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.zeros(M, D, device="cuda")
    cos = torch.rand(SEQ, NF, device="cuda", generator=g)
    sin = torch.rand(SEQ, NF, device="cuda", generator=g)
    return {
        "FF-in": (2 * FFI, D, 256, dict(epi=nat.EPI_SWIGLU, out=torch.empty(M, FFI, dtype=torch.float16, device="cuda"),
                                         ld=FFI, bias=torch.randn(2 * FFI, device="cuda", generator=g))),
        "FF-out": (D, FFI, 256, dict(epi=nat.EPI_RESIDUAL, h=h, ld=D, bias=torch.randn(D, device="cuda", generator=g),
                                     rows_per_item=SEQ, n_items=1)),
        "QKV": (3 * D, D, 256, dict(epi=nat.EPI_QKV_ROPE, out=torch.empty(M, 3 * D, dtype=torch.float16, device="cuda"),
                                    ld=3 * D, rope_cols=2 * D, seq_len=SEQ, head_dim=HEAD_DIM, nf=NF, cos_tab=cos,
                                    sin_tab=sin)),
        "out-proj": (D, D, 256, dict(epi=nat.EPI_RESIDUAL, h=h, ld=D, rows_per_item=SEQ, n_items=1)),
    }


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    tag = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("SATB_"))
    lib = nat.lib()
    for name, (N, K, bn, f) in cases().items():
        g = torch.Generator(device="cuda").manual_seed(N + K)
        a = torch.randn(M, K, device="cuda", generator=g).half()
        w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).half()
        p = nat.SatbGemmProbe()
        p.bn, p.bf16, p.b_static = bn, 0, 1
        for k, v in f.items():
            setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)

        def run():
            nat.check(lib.satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, N, K, ctypes.byref(p), nat.stream_ptr()))

        for _ in range(10):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        clock = smi("clocks.sm")          # the launches above are still running
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1000 / reps
        print("%-8s %dx%dx%d BN%d: %8.1f us  %6.1f TFLOP/s  (SM clock during the run: %s)  [%s]"
              % (name, M, N, K, bn, us, 2.0 * M * N * K / us / 1e6, clock, tag), flush=True)


if __name__ == "__main__":
    main()
