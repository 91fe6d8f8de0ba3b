"""Time one CFG denoiser call of one prompt, token-sharded over 1, 2, 4 and 8 GPUs (as many as are visible), at two
shapes: Stable Audio 2.0's length (6144 latents + the global token = 6145 tokens, 24 blocks at SA-Open width) and
SA-Open's (1025 tokens).  Seeded random weights, fp16 operands.

Per (shape, world): ms per call from CUDA events on the home device (3 warm-up calls, then `--rounds` rounds that
alternate the worlds, `--iters` calls each; median over rounds), the speedup over world 1, and the host time to enqueue
one call (the GPU drained first, so the launch queue never blocks).  Per shape and world: the K/V gather alone, one
layer's worth (satb_kv_gather on every rank at once, CUDA events), and its rate in GB/s of bytes read from other ranks,
(world - 1) / world of R N 2 D 2 bytes per rank, computed from the shapes.  The card's name and power limit are read
in the same run.  Worlds beyond the visible devices are printed as "not measured".

    python tests/cp_time.py [--out RESULT.json] [--iters 10] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "friendly-stable-audio-tools_b200"))
sys.path.insert(0, HERE)

from helpers import SAO_DIT  # noqa: E402
from oracle import dit_oracle as do  # noqa: E402

SHAPES = {"sa2_6145": 6144, "sa_open_1025": 1024}
WORLDS = [1, 2, 4, 8]


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


def call_ms(m, kw, iters):
    st = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(iters):
        m(**kw)
    b.record(st)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def enqueue_ms(m, kw, iters):
    ts = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m(**kw)
        ts.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    return statistics.median(ts)


def gather_ms(devs, L, D, R, iters):
    """One layer's gather on every rank (each rank's own device and stream), as the group forward runs it."""
    from stable_audio_tools import _native
    lib = _native.lib()
    world = len(devs)
    tb = _native.group_plan(world, 1, L)
    N = tb[-1]
    qkv = [torch.randn(R, tb[r + 1] - tb[r], 3 * D, device=devs[r]).half() for r in range(world)]
    kv = [torch.empty(R, N, 2 * D, device=devs[r], dtype=torch.float16) for r in range(world)]
    srcs = (ctypes.c_void_p * world)(*[q.data_ptr() for q in qkv])
    tba = (ctypes.c_int * (world + 1))(*tb)
    streams = [torch.cuda.Stream(device=dv) for dv in devs]
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(world)]

    def once():
        for r in range(world):
            with torch.cuda.device(devs[r]):
                _native.check(lib.satb_kv_gather(srcs, tba, world, ctypes.c_void_p(kv[r].data_ptr()), R, D,
                                                 ctypes.c_void_p(streams[r].cuda_stream)))
    sync = lambda: [torch.cuda.synchronize(dv) for dv in set(devs)]
    sync()
    once()
    sync()
    for r in range(world):
        with torch.cuda.device(devs[r]):
            ev[r][0].record(streams[r])
    for _ in range(iters):
        once()
    for r in range(world):
        with torch.cuda.device(devs[r]):
            ev[r][1].record(streams[r])
    sync()
    ok = all(torch.equal(kv[r][:, tb[s]:tb[s + 1]].cpu(), qkv[s][:, :, D:].cpu()) for r in range(world) for s in range(world))
    return max(e[0].elapsed_time(e[1]) for e in ev) / iters, N, ok


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
    # (mode, world) -> devices: ranks on distinct GPUs where that many are visible, and virtual ranks on cuda:0 (the
    # same schedule on one GPU: the cost of sharding with no extra hardware)
    runs = {("devices", w): [f"cuda:{r}" for r in range(w)] for w in WORLDS if w <= n_dev}
    runs.update({("virtual", w): ["cuda:0"] * w for w in WORLDS[1:]})
    sd = do.make_dit_weights(SAO_DIT, seed=5)
    m = build_native_dit(SAO_DIT, sd)
    D = SAO_DIT["embed_dim"]
    for shape, L in SHAPES.items():
        g = torch.Generator().manual_seed(6)
        kw = dict(x=torch.randn(1, 64, L, generator=g).cuda(), t=torch.tensor([0.5]).cuda(),
                  cross_attn_cond=torch.randn(1, 130, 768, generator=g).cuda(),
                  global_embed=torch.randn(1, 1536, generator=g).cuda(), cfg_scale=7.0)
        times = {k: [] for k in runs}
        enq = {}
        shard = lambda k: m.shard_tokens(None if k[1] == 1 else runs[k])
        for k in runs:                                     # warm-up: handles, weights, workspaces
            shard(k)
            for _ in range(3):
                m(**kw)
            enq[k] = enqueue_ms(m, kw, args.iters)
        for _ in range(args.rounds):
            for k in runs:
                shard(k)                                   # new rank handles: one untimed call loads their weights
                m(**kw)
                times[k].append(call_ms(m, kw, args.iters))
            m.shard_tokens(None)
        base = statistics.median(times[("devices", 1)])
        for mode in ("devices", "virtual"):
            for w in WORLDS:
                k = (mode, w)
                if mode == "virtual" and w == 1:
                    continue
                if k not in runs:
                    row = dict(shape=shape, tokens=L + 1, mode=mode, world=w, status="not measured",
                               reason=f"{n_dev} device(s) visible")
                else:
                    ms = statistics.median(times[k])
                    gms, N, ok = gather_ms(runs[k], L, D, 2, args.iters)
                    remote = (w - 1) / w * 2 * N * 2 * D * 2
                    row = dict(shape=shape, tokens=L + 1, mode=mode, world=w, ms_per_call=ms, rounds=times[k],
                               speedup=base / ms, host_enqueue_ms=enq[k], gather_ms_per_layer=gms,
                               gather_remote_bytes=remote,
                               gather_remote_gb_s=remote / (gms * 1e-3) / 1e9 if w > 1 else None,
                               gather_total_gb_s=2 * N * 2 * D * 2 / (gms * 1e-3) / 1e9, gather_exact=ok)
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
