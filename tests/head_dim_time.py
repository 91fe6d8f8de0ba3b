"""Timing driver for attention head dims other than 64 (not a test):

    python tests/head_dim_time.py attn [D ...]      # self-attention core, default D = 64 128 96
    python tests/head_dim_time.py dit [num_heads ...]  # one CFG denoiser call, default 24 12 16 heads

Both at SA-Open-1.0 width (1536 = heads x head dim, so every head dim does the same FLOPs), 1025 tokens, 8 rows, CUDA
events.  attn: satb_attention_hd with 1536 / D heads (fp16), TFLOP/s and the error vs torch fp32 softmax.  dit: 24
blocks, 130x768 context, 1024 latents + the prepend token, B=4 with CFG 7, synthetic weights.  Each case is timed in
turn, twice over, so the spread shows."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from stable_audio_tools import _native as nat


def time_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attn(dims):
    B, N = 8, 1025
    cases = {}
    for D in dims:
        H = 1536 // D
        torch.manual_seed(0)
        q = (2.0 * torch.randn(B, N, H * D, device="cuda")).half()
        k = torch.randn(B, N, H * D, device="cuda").half()
        v = torch.randn(B, N, H * D, device="cuda").half()
        o = torch.empty_like(q)
        run = lambda q=q, k=k, v=v, o=o, H=H, D=D: nat.check(nat.lib().satb_attention_hd(
            nat.ptr(q), nat.ptr(k), nat.ptr(v), nat.ptr(o), B, H, H, N, N, D, 0, nat.stream_ptr()))
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        qh, kh, vh = (t[:1].float().view(1, N, H, D).transpose(1, 2) for t in (q, k, v))
        ref = torch.softmax(qh @ kh.transpose(-1, -2) / D ** 0.5, dim=-1) @ vh
        err = float((o[:1].float().view(1, N, H, D).transpose(1, 2) - ref).norm() / ref.norm())
        cases[D] = (H, run, err)
    for rnd in range(2):
        for D, (H, run, err) in cases.items():
            us = time_ms(run, 50) * 1000
            print("round %d: attention D=%d H=%d N=%d: %.1f us  (%.0f TF/s)  rel-L2 err %.2e"
                  % (rnd, D, H, N, us, 4.0 * B * H * N * N * D / us / 1e6, err), flush=True)


def dit(heads):
    from helpers import SAO_DIT, build_native_dit
    from oracle import dit_oracle as do
    B = 4
    g = torch.Generator().manual_seed(0)
    x, t = torch.randn(B, 64, 1024, generator=g).cuda(), (torch.rand(B, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(B, 130, 768, generator=g).cuda(), torch.randn(B, 1536, generator=g).cuda()
    models = {}
    for h in heads:
        cfg = dict(SAO_DIT, num_heads=h)
        models[h] = build_native_dit(cfg, do.make_dit_weights(cfg, seed=5))
        for _ in range(3):
            models[h](x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0)
    torch.cuda.synchronize()
    for rnd in range(2):
        for h, m in models.items():
            ms = time_ms(lambda: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0), 20)
            print("round %d: %d heads (head dim %d): %.2f ms per CFG forward" % (rnd, h, 1536 // h, ms), flush=True)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "attn"
    args = [int(a) for a in sys.argv[2:]]
    if what == "attn":
        attn(args or [64, 128, 96])
    else:
        dit(args or [24, 12, 16])
