"""Per-step wall time of each sampler on the torch path (eager DiT, torch update ops) and on the native step path
(graph-replayed DiT, satb_sampler_step), at SA-Open width (24 blocks, 1536 wide), 1024 latents + 1 prepended token =
1025 tokens, classifier-free guidance, batch 1 and 4; inpainting is timed with and without a preview callback.  The
two paths alternate in one process, each timing a whole sampling loop between device synchronises; the native path
is timed on its second loop after each torch loop, once its graph is captured again.

    python tests/sampler_time.py [--steps 8] [--reps 3] [--batches 1 4] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))

SAO_DIT = dict(io_channels=64, embed_dim=1536, depth=24, num_heads=24, cond_token_dim=768, global_cond_dim=1536,
               project_cond_tokens=False, transformer_type="continuous_transformer")
CASES = [("dpmpp-3m-sde", "none"), ("dpmpp-3m-sde", "inpaint"), ("dpmpp-3m-sde", "inpaint+preview"),
         ("dpmpp-2m-sde", "preview"), ("k-heun", "none"), ("k-dpm-2", "none"), ("k-lms", "none"),
         ("k-dpmpp-2s-ancestral", "none"), ("k-dpm-fast", "none"), ("k-dpm-adaptive", "none"), ("rf", "none"),
         ("rf", "preview")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_time.py needs a CUDA device")
    from oracle import dit_oracle as do
    from stable_audio_tools.inference import sampling as s
    from stable_audio_tools.models.diffusion import DiTWrapper
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}", flush=True)
    w = DiTWrapper(**SAO_DIT)
    w.model.load_state_dict(do.make_dit_weights(SAO_DIT, seed=1))
    w = w.cuda().eval()
    fusable = s._fusable
    L = 1024
    rows = []
    for B in args.batches:
        g = torch.Generator().manual_seed(B)
        kw = dict(cross_attn_cond=torch.randn(B, 130, 768, generator=g).cuda(),
                  global_cond=torch.randn(B, 1536, generator=g).cuda(), cfg_scale=7.0)
        noise = torch.randn(B, 64, L, generator=g).cuda()
        init = torch.randn(B, 64, L, generator=g).cuda()
        mask = torch.zeros(L, device="cuda")
        mask[256:768] = 1.0

        def run(name, kind):
            cb = (lambda a: a["denoised"]) if "preview" in kind else None
            if name == "rf":
                return s.sample_rf(w, noise, steps=args.steps, device="cuda", callback=cb, **kw)
            inp = "inpaint" in kind
            return s.sample_k(w, noise, init if inp else None, mask if inp else None, steps=args.steps,
                              sampler_type=name, sigma_min=0.3, sigma_max=50.0, device="cuda", callback=cb, **kw)

        for name, kind in CASES:
            times = {"torch": [], "native": []}
            for rep in range(args.reps + 1):                  # rep 0 warms both paths up (workspaces)
                # an eager DiT call drops the captured graph (it may regrow the workspaces the graph points into), so
                # the native path runs twice after each torch run and the second, steady-state loop is timed
                for path, timed in (("torch", True), ("native", False), ("native", True)):
                    s._fusable = fusable if path == "native" else (lambda x: False)
                    calls = []
                    orig = w.model.forward
                    w.model.forward = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(name, kind)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    del w.model.forward
                    if rep and timed:
                        times[path].append(dt / args.steps * 1e3)
            s._fusable = fusable
            med = {k: statistics.median(v) for k, v in times.items()}
            row = dict(batch=B, sampler=name, callback=kind, calls=len(calls), torch_ms_per_step=round(med["torch"], 3),
                       native_ms_per_step=round(med["native"], 3), speedup=round(med["torch"] / med["native"], 3),
                       spread_torch=[round(v, 3) for v in times["torch"]],
                       spread_native=[round(v, 3) for v in times["native"]])
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sampler_time.json"), "w") as f:
            json.dump(dict(card=card, steps=args.steps, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
