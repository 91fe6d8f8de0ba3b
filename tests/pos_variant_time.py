"""Timing driver for the positional options (not a test): python tests/pos_variant_time.py [calls]

At SA-Open width (D 1536, 24 heads, 24 blocks, a 130 x 768 cross-attention context; batch 4 with CFG = 8 rows of 1025
tokens) it builds four models - the default (rotary, no embedding), rotary off, a sinusoidal embedding and an absolute
one (both with rotary) - and times one CFG forward of each, the variants alternating over two rounds in this one
process (CUDA events over `calls` calls after a warm-up).  The card's name, power limit and the SM clock (read while
timed work is running) are printed in the same run."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from fp8_time import events_ms, smi
from helpers import SAO_DIT, build_native_dit

VARIANTS = {
    "default": {},
    "rotary off": dict(rotary_pos_emb=False),
    "sinusoidal": dict(use_sinusoidal_emb=True),
    "absolute": dict(use_abs_pos_emb=True),
}


def main():
    from oracle import positions_oracle as po
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % smi("name,power.limit,clocks.max.sm"), flush=True)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
    c[:, 40:] = 0.0
    call = lambda m: m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0)
    models = {}
    for name, kw in VARIANTS.items():
        cfg = dict(SAO_DIT, **kw)
        m = build_native_dit(cfg, po.make_dit_weights(cfg, seed=10))
        for _ in range(3):
            call(m)
        torch.cuda.synchronize()
        models[name] = m
    for rnd in range(2):
        for name, m in models.items():
            ms, clock = events_ms(lambda: call(m), calls)
            print("round %d  forward %-11s batch 4 + CFG, 24 blocks: %7.2f ms  (SM clock: %s)" % (rnd, name, ms, clock),
                  flush=True)


if __name__ == "__main__":
    main()
