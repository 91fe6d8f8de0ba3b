"""Timing driver for DiT channel widths (not a test): python tests/width_time.py [calls] [rounds]

At SA-Open width (D 1536, 24 heads, 24 blocks, a 130 x 768 cross-attention context; batch 4 with CFG = 8 rows of 1025
tokens) it builds two models - the default (io 64, no concat: project_in K = 64) and an inpainting one (io 64 + concat
65 = Cin 129: project_in K padded to 136) - and times one CFG forward of each, alternating over `rounds` rounds in this
one process (CUDA events over `calls` calls after a warm-up).  Prints one JSON line per timing with the SM clock read
while the timed work runs, and the card's name and power limit first."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from fp8_time import events_ms, smi
from helpers import SAO_DIT, build_native_dit

VARIANTS = {"cin64": {}, "cin129": dict(input_concat_dim=65)}


def main():
    from oracle import positions_oracle as po
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    print(json.dumps({"card": smi("name,power.limit,clocks.max.sm")}), flush=True)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    c[:, 40:] = 0.0
    mask = (torch.rand(4, 1, 1024, generator=g) > 0.5).float()
    concat = torch.cat([mask, torch.randn(4, 64, 1024, generator=g) * mask], dim=1).cuda()
    models = {}
    for name, kw in VARIANTS.items():
        cfg = dict(SAO_DIT, **kw)
        m = build_native_dit(cfg, po.make_dit_weights(cfg, seed=10))
        extra = dict(input_concat_cond=concat) if kw else {}
        call = (lambda m, extra: lambda: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0, **extra))(m, extra)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        models[name] = call
    for rnd in range(rounds):
        for name, call in models.items():
            ms, clock = events_ms(call, calls)
            print(json.dumps({"round": rnd, "model": name, "forward_ms": round(ms, 3), "calls": calls,
                              "rows": "8 x 1025 (batch 4 + CFG)", "blocks": 24, "sm_clock": clock}), flush=True)


if __name__ == "__main__":
    main()
