"""Timing / accuracy driver for the attention kernel (not a test): python tests/attn_time.py [N ...]
SA-Open self-attention shape (8 rows x 24 heads x N tokens), CUDA events, error vs torch fp32 softmax."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
import torch
from stable_audio_tools import _native as nat

if os.environ.get("SATB_LIB"):          # A/B of kernel variants built side by side (tools only)
    nat.LIB_PATH = os.path.abspath(os.environ["SATB_LIB"])

B, H = int(os.environ.get("ATTN_B", "8")), 24
tag = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("SATB_"))
for N in [int(a) for a in sys.argv[1:]] or [1025]:
    torch.manual_seed(0)
    q = (2.0 * torch.randn(B, N, H * 64, device="cuda")).half()
    k = torch.randn(B, N, H * 64, device="cuda").half()
    v = torch.randn(B, N, H * 64, device="cuda").half()
    o = torch.empty_like(q)

    def run():
        nat.check(nat.lib().satb_attention(nat.ptr(q), nat.ptr(k), nat.ptr(v), nat.ptr(o), B, H, H, N, N, 0, nat.stream_ptr()))

    for _ in range(5):
        run()
    torch.cuda.synchronize()
    reps = 50 if N < 3000 else 10
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / reps
    qh, kh, vh = (t[:1].float().view(1, N, H, 64).transpose(1, 2) for t in (q, k, v))
    ref = torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, dim=-1) @ vh
    got = o[:1].float().view(1, N, H, 64).transpose(1, 2)
    err = float((got - ref).norm() / ref.norm())
    print("attention N=%d: %.1f us  (%.0f TF/s)  rel-L2 err %.2e  [%s]" % (N, us, 4.0 * B * H * N * N * 64 / us / 1e6, err, tag), flush=True)
