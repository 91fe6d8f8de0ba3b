"""Probe (not a test): where does a batch-of-4 row differ from the same prompt run alone? usage: python tests/batch_vs_single_probe.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from helpers import SAO_DIT, build_native_dit, rel_l2
from oracle import dit_oracle as do
sd = do.make_dit_weights(SAO_DIT, seed=21)
m = build_native_dit(SAO_DIT, sd)
g = torch.Generator().manual_seed(23)
x, t = torch.randn(4, 64, 1024, generator=g).cuda(), (torch.rand(4, generator=g) * 0.9 + 0.05).cuda()
c, ge = torch.randn(4, 130, 768, generator=g).cuda(), torch.randn(4, 1536, generator=g).cuda()
for s in (1.0, 7.0):
    y4 = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=s)
    y1 = m(x[2:3].contiguous(), t[2:3].contiguous(), cross_attn_cond=c[2:3].contiguous(), global_embed=ge[2:3].contiguous(), cfg_scale=s)
    d = (y4[2:3] - y1).float()
    per_pos = d.pow(2).sum(dim=1).sqrt()[0] / y1.float().pow(2).sum(dim=1).sqrt()[0]
    print("cfg %.0f rel_l2 %.3e  per-position err: first %.2e median %.2e last %.2e max %.2e at %d" % (
        s, rel_l2(y4[2:3].cpu(), y1.cpu()), per_pos[0], per_pos.median(), per_pos[-1], per_pos.max(), int(per_pos.argmax())),
          flush=True)
