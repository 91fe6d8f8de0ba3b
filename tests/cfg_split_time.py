"""Time one CFG denoiser call of one prompt split by guidance half (DiffusionTransformer.shard_tokens with two rows,
satb_dit_group_create_cfg) against the unsharded call and plain token sharding, at Stable Audio 2.0's length (6145
tokens) and SA-Open's (1025 tokens), 24 blocks at SA-Open width, CFG 7, seeded random weights, fp16 operands.

Configurations: unsharded; shard_tokens over 2, 4 and 8 ranks; CFG split with rows of 1, 2 and 4 ranks (1x2, 2x2,
4x2).  Every rank is on cuda:0 ("virtual"), and, where enough GPUs are visible, also on distinct GPUs ("devices"); a
layout beyond the visible devices is printed as "not measured".  Per (shape, mode, configuration), the configurations
alternated in one process (`--rounds` rounds of `--iters` calls each, medians over rounds), eager and graph calls:
  * ms per call from CUDA events on the home device's current stream;
  * host ms per call with the GPU drained first (so the launch queue never blocks);
  * combine ms per call: the device time of the dit_post kernels (the CFG combine) of one eager call, from
    torch.profiler;
  * bytes exchanged between ranks per call, computed from the shapes: each rank's K/V gather reads (W - 1) / W of
    R N 2 D 2 bytes per layer from the other ranks of its row (R = 2 rows under plain sharding, 1 per half under the
    CFG split), and the CFG split's combine reads the unconditional half's project_out output, B N C_p 4 bytes;
  * whether the eager and graph outputs are bit-identical, and the rel-L2 of the eager output to the unsharded one.
The card's name, power limit and SM clocks are read in the same run.

    python tests/cfg_split_time.py [--out RESULT.json] [--iters 10] [--rounds 3]
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

from cp_time import SHAPES, call_ms, enqueue_ms, smi  # noqa: E402
from helpers import SAO_DIT, rel_l2  # noqa: E402
from oracle import dit_oracle as do  # noqa: E402

# name -> (ranks per row, CFG split)
CONFIGS = {"unsharded": (1, False), "tokens_2": (2, False), "tokens_4": (4, False), "tokens_8": (8, False),
           "cfg_1x2": (1, True), "cfg_2x2": (2, True), "cfg_4x2": (4, True)}


def layout(name, mode):
    """The shard_tokens argument of a configuration (None: unsharded)."""
    w, split = CONFIGS[name]
    if name == "unsharded":
        return None
    dev = (lambda i: f"cuda:{i}") if mode == "devices" else (lambda i: "cuda:0")
    if split:
        return [[dev(i) for i in range(w)], [dev(w + i) for i in range(w)]]
    return [dev(i) for i in range(w)]


def ranks(name):
    w, split = CONFIGS[name]
    return 2 * w if split else w


def exchanged_bytes(name, N, L):
    """(K/V bytes one rank reads from the other ranks of its row per call, combine bytes per call, all cross-rank bytes
    per call), from the shapes: B = 1 prompt, CFG on."""
    w, split = CONFIGS[name]
    D, depth, Cp = SAO_DIT["embed_dim"], SAO_DIT["depth"], 64
    R = 1 if split else 2
    kv_rank = (w - 1) / w * R * N * 2 * D * 2 * depth if name != "unsharded" else 0.0
    combine = N * Cp * 4 if split else 0.0
    return kv_rank, combine, kv_rank * ranks(name) + combine


def combine_ms(m, kw):
    """Device ms of the dit_post (CFG combine) kernels of one eager call, from torch.profiler."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        m(**kw)
        torch.cuda.synchronize()
    total = 0.0
    for evt in prof.key_averages():
        if "dit_post" in evt.key:
            total += getattr(evt, "device_time_total", getattr(evt, "cuda_time_total", 0.0))
    return total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from helpers import build_native_dit
    n_dev = torch.cuda.device_count()
    res = dict(gpu=smi("name"), power_limit=smi("power.limit"), max_sm_clock=smi("clocks.max.sm"),
               sm_clock_at_start=smi("clocks.sm"), devices=n_dev, rows=[])
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "max_sm_clock", "sm_clock_at_start", "devices")}),
          flush=True)
    runs = [("virtual", c) for c in CONFIGS]
    runs += [("devices", c) for c in CONFIGS if c != "unsharded" and ranks(c) <= n_dev]
    sd = do.make_dit_weights(SAO_DIT, seed=5)
    m = build_native_dit(SAO_DIT, sd)
    for shape, L in SHAPES.items():
        N = L + 1
        g = torch.Generator().manual_seed(6)
        kw = dict(x=torch.randn(1, 64, L, generator=g).cuda(), t=torch.tensor([0.5]).cuda(),
                  cross_attn_cond=torch.randn(1, 130, 768, generator=g).cuda(),
                  global_embed=torch.randn(1, 1536, generator=g).cuda(), cfg_scale=7.0)
        times = {(k, gr): [] for k in runs for gr in (False, True)}
        host = {(k, gr): [] for k in runs for gr in (False, True)}
        outs, comb = {}, {}
        for rnd in range(args.rounds):
            for k in runs:
                m.shard_tokens(layout(k[1], k[0]))        # new rank handles: the warm-up calls load their weights
                for graph in (False, True):
                    m.cuda_graph = graph
                    for _ in range(2):                     # warm-up (workspaces, the capture)
                        outs[(k, graph)] = m(**kw).clone()
                    times[(k, graph)].append(call_ms(m, kw, args.iters))
                    host[(k, graph)].append(enqueue_ms(m, kw, args.iters))
                m.cuda_graph = False
                if rnd == args.rounds - 1:
                    comb[k] = combine_ms(m, kw)
        sm_clock = smi("clocks.sm")
        m.shard_tokens(None)
        ref = outs[(("virtual", "unsharded"), False)]
        for mode in ("virtual", "devices"):
            for c in CONFIGS:
                if mode == "devices" and c == "unsharded":
                    continue
                k = (mode, c)
                if k not in runs:
                    row = dict(shape=shape, tokens=N, mode=mode, config=c, status="not measured",
                               reason=f"{n_dev} device(s) visible, {ranks(c)} needed")
                else:
                    kv_rank, comb_b, total_b = exchanged_bytes(c, N, L)
                    row = dict(shape=shape, tokens=N, mode=mode, config=c,
                               eager_ms_per_call=statistics.median(times[(k, False)]),
                               graph_ms_per_call=statistics.median(times[(k, True)]),
                               eager_host_ms=statistics.median(host[(k, False)]),
                               graph_host_ms=statistics.median(host[(k, True)]),
                               combine_ms_per_call=comb[k],
                               kv_bytes_per_rank_per_call=kv_rank, combine_bytes_per_call=comb_b,
                               exchanged_bytes_per_call=total_b,
                               eager_rounds=times[(k, False)], graph_rounds=times[(k, True)],
                               graph_equals_eager=bool(torch.equal(outs[(k, False)], outs[(k, True)])),
                               rel_l2_vs_unsharded=rel_l2(outs[(k, False)].cpu(), ref.cpu()),
                               bit_identical_to_unsharded=bool(torch.equal(outs[(k, False)], ref)),
                               sm_clock_after=sm_clock)
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
