"""Time one CFG denoiser call of one prompt, token-sharded, enqueued eagerly against replayed from the group's CUDA
graph (DiffusionTransformer.cuda_graph, satb_dit_group_graph_forward), at Stable Audio 2.0's length (6145 tokens) and
SA-Open's (1025 tokens), 24 blocks at SA-Open width, seeded random weights, fp16 operands.

Per (shape, mode, world), eager and graph alternated in one process (`--rounds` rounds of `--iters` calls each, medians
over rounds):
  * ms per call from CUDA events on the home device's current stream;
  * host ms per call with the GPU drained first (so the launch queue never blocks): the eager enqueue, or the graph
    call (two small input copies and one graph launch);
  * whether the two outputs are bit-identical.
World 1 is the unsharded model, eager against its single-device graph.  Modes: "devices" (ranks on distinct GPUs, where
that many are visible) and "virtual" (every rank on cuda:0).  The card's name and power limit are read in the same
run.  Worlds beyond the visible devices are printed as "not measured".

    python tests/cp_graph_time.py [--out RESULT.json] [--iters 10] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "friendly-stable-audio-tools_b200"))
sys.path.insert(0, HERE)

from cp_time import SHAPES, WORLDS, call_ms, enqueue_ms, smi  # noqa: E402
from helpers import SAO_DIT  # noqa: E402
from oracle import dit_oracle as do  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from helpers import build_native_dit
    n_dev = torch.cuda.device_count()
    res = dict(gpu=smi("name"), power_limit=smi("power.limit"), max_sm_clock=smi("clocks.max.sm"), devices=n_dev,
               rows=[])
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "max_sm_clock", "devices")}), flush=True)
    runs = {("devices", w): [f"cuda:{r}" for r in range(w)] for w in WORLDS if w <= n_dev}
    runs.update({("virtual", w): ["cuda:0"] * w for w in WORLDS[1:]})
    sd = do.make_dit_weights(SAO_DIT, seed=5)
    m = build_native_dit(SAO_DIT, sd)
    for shape, L in SHAPES.items():
        g = torch.Generator().manual_seed(6)
        kw = dict(x=torch.randn(1, 64, L, generator=g).cuda(), t=torch.tensor([0.5]).cuda(),
                  cross_attn_cond=torch.randn(1, 130, 768, generator=g).cuda(),
                  global_embed=torch.randn(1, 1536, generator=g).cuda(), cfg_scale=7.0)
        for mode in ("devices", "virtual"):
            for w in WORLDS:
                k = (mode, w)
                if mode == "virtual" and w == 1:
                    continue
                if k not in runs:
                    row = dict(shape=shape, tokens=L + 1, mode=mode, world=w, status="not measured",
                               reason=f"{n_dev} device(s) visible")
                    res["rows"].append(row)
                    print(json.dumps(row), flush=True)
                    continue
                m.shard_tokens(None if w == 1 else runs[k])
                times = {False: [], True: []}
                host = {False: [], True: []}
                outs = {}
                for graph in (False, True):                # warm-up: handles, weights, workspaces, the capture
                    m.cuda_graph = graph
                    for _ in range(3):
                        outs[graph] = m(**kw).clone()
                for _ in range(args.rounds):
                    for graph in (False, True):
                        m.cuda_graph = graph
                        m(**kw)      # untimed: an eager unsharded call drops the single-device graph (recaptured here)
                        times[graph].append(call_ms(m, kw, args.iters))
                        host[graph].append(enqueue_ms(m, kw, args.iters))
                m.cuda_graph = False
                stats = m.shard_graph_stats()
                row = dict(shape=shape, tokens=L + 1, mode=mode, world=w,
                           eager_ms_per_call=statistics.median(times[False]),
                           graph_ms_per_call=statistics.median(times[True]),
                           eager_host_ms=statistics.median(host[False]), graph_host_ms=statistics.median(host[True]),
                           eager_rounds=times[False], graph_rounds=times[True],
                           graph_captures=stats[0] if stats else None,
                           graph_kernel_launches=stats[2] if stats else None,
                           bit_identical=bool(torch.equal(outs[False], outs[True])))
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
        m.shard_tokens(None)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
