"""Timing driver for the FP8 self-attention (not a test): python tests/fp8_attn_time.py [reps]

At the bench shape (batch 4 with CFG = 8 rows of 1025 tokens, 24 heads of 64) it times, alternated in this one process
over two rounds:
  - the self-attention core: the fp16 attn_wgmma_kernel (satb_attention) against the FP8 core alone
    (satb_attention_fp8_core) and the V transpose-quantiser + core (satb_attention_fp8_vt, then the core), CUDA events
    over `reps` calls;
  - the QKV GEMM with rotary (8200 x 4608 x 1536, BN 256, fp16 operands) with its 16-bit epilogue (satb_gemm_probe,
    EPI_QKV_ROPE) and with the e4m3 q / k epilogue (satb_gemm_probe_qk8, EPI_QKV_ROPE_E4M3);
  - one full 24-block SA-Open forward at batch 4 with CFG for operand_dtype fp16 and fp8, each with and without
    attention_dtype "fp8" (CUDA events over 10 calls after a warm-up);
and prints the rel-L2 of each FP8-attention forward against the same operand mode without it.  The card's name, power
limit and the SM clock (read while timed work is running) are printed in the same run."""
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
from helpers import SAO_DIT, build_native_dit, rel_l2

R, H, N = 8, 24, 1025


def time_core(reps):
    lib = nat.lib()
    D, Np = H * 64, (N + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(R, N, D, device="cuda", generator=g).half() for _ in range(3))
    o = torch.empty(R, N, D, dtype=torch.float16, device="cuda")
    q8, k8 = torch.empty(R, N, D, dtype=torch.uint8, device="cuda"), torch.empty(R, N, D, dtype=torch.uint8, device="cuda")
    sq, sk = torch.empty(R * H, Np, device="cuda"), torch.empty(R * H, Np, device="cuda")
    vt, sv = torch.empty(R * H, 64, Np, dtype=torch.uint8, device="cuda"), torch.empty(R * H, 64, device="cuda")
    st = nat.stream_ptr()
    vtq = lambda: nat.check(lib.satb_attention_fp8_vt(v.data_ptr(), vt.data_ptr(), sv.data_ptr(), R, H, N, 0, st))
    core8 = lambda: nat.check(lib.satb_attention_fp8_core(q8.data_ptr(), k8.data_ptr(), sq.data_ptr(), sk.data_ptr(),
                                                          vt.data_ptr(), sv.data_ptr(), o.data_ptr(), R, H, N, N, 0, st))
    cases = {
        "fp16 attn_wgmma_kernel": lambda: nat.check(lib.satb_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                                       o.data_ptr(), R, H, H, N, N, 0, st)),
        "fp8 core": core8,
        "fp8 V quantiser + core": lambda: (vtq(), core8()),
        "fp8 V quantiser alone": vtq,
    }
    # q8 / k8 / scales as the QKV epilogue would write them (any valid e4m3 operands time the same)
    from fp8_ref import quantize_fp8_rows
    for x, x8, sx in ((q, q8, sq), (k, k8, sk)):
        xq, xs = quantize_fp8_rows(x.float().view(R, N, H, 64))
        x8.copy_(xq.view(torch.uint8).view(R, N, D))
        sx.zero_()
        sx[:, :N] = xs[..., 0].permute(0, 2, 1).reshape(R * H, N)
    vtq()
    for fn in cases.values():
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    flops = 4.0 * R * H * N * N * 64
    for rnd in range(2):
        for name, fn in cases.items():
            ms, clock = events_ms(fn, reps)
            print("round %d  core %-26s %dx%dx%d: %8.1f us  %6.1f TFLOP/s  (SM clock: %s)"
                  % (rnd, name, R, H, N, ms * 1000, flops / ms / 1e9, clock), flush=True)


def time_qkv(reps):
    from gemm_epilogue_ref import rope_tables
    lib = nat.lib()
    M, D = R * N, H * 64
    Nn, K = 3 * D, D
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    w = (torch.randn(Nn, K, device="cuda", generator=g) * K ** -0.5).half()
    cos, sin, _ = rope_tables(N, 16)
    cos, sin = cos.cuda(), sin.cuda()
    out = torch.empty(M, Nn, dtype=torch.float16, device="cuda")
    q8, k8 = torch.empty(M, D, dtype=torch.uint8, device="cuda"), torch.empty(M, D, dtype=torch.uint8, device="cuda")
    Np = (N + 127) // 128 * 128
    sq, sk = torch.zeros(R * H, Np, device="cuda"), torch.zeros(R * H, Np, device="cuda")
    p16, p8 = nat.SatbGemmProbe(), nat.SatbGemmProbe()
    for p, epi in ((p16, nat.EPI_QKV_ROPE), (p8, nat.EPI_QKV_ROPE_E4M3)):
        p.epi, p.bn, p.bf16, p.b_static = epi, 256, 0, 1
        p.out, p.ld, p.rope_cols, p.seq_len, p.head_dim, p.nf = out.data_ptr(), Nn, 2 * D, N, 64, 16
        p.cos_tab, p.sin_tab = cos.data_ptr(), sin.data_ptr()
    o = nat.SatbQkE4m3(q8=q8.data_ptr(), k8=k8.data_ptr(), sq=sq.data_ptr(), sk=sk.data_ptr(), heads=H, scale_ld=Np)
    st = nat.stream_ptr()
    cases = {
        "16-bit epilogue": lambda: nat.check(lib.satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, Nn, K, ctypes.byref(p16), st)),
        "e4m3 q / k epilogue": lambda: nat.check(lib.satb_gemm_probe_qk8(a.data_ptr(), w.data_ptr(), None, None, M, Nn, K,
                                                                         ctypes.byref(p8), ctypes.byref(o), st)),
    }
    for fn in cases.values():
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    for rnd in range(2):
        for name, fn in cases.items():
            ms, clock = events_ms(fn, reps)
            print("round %d  QKV + rotary %dx%dx%d, %-20s: %8.1f us  (SM clock: %s)" % (rnd, M, Nn, K, name, ms * 1000, clock),
                  flush=True)


def time_forward():
    from oracle import dit_oracle as do
    sd = do.make_dit_weights(SAO_DIT, seed=10)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    modes = [("fp16", None), ("fp16", "fp8"), ("fp8", None), ("fp8", "fp8")]
    models = {m: build_native_dit(dict(SAO_DIT, attention_dtype=m[1]), sd, operand_dtype=m[0]) for m in modes}
    outs = {}
    for mode, m in models.items():
        for _ in range(3):
            outs[mode] = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    torch.cuda.synchronize()
    for rnd in range(2):
        for mode, m in models.items():
            ms, clock = events_ms(lambda: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0), 10)
            print("round %d  forward operand %-4s attention %-4s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)"
                  % (rnd, mode[0], mode[1] or "16", ms, clock), flush=True)
    for od in ("fp16", "fp8"):
        print("rel-L2 of operand %s + FP8 attention against operand %s: %.3e"
              % (od, od, rel_l2(outs[(od, "fp8")].cpu(), outs[(od, None)].cpu())), flush=True)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    time_core(reps)
    time_qkv(reps)
    time_forward()


if __name__ == "__main__":
    main()
