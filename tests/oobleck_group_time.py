"""Time the time-sharded Oobleck decode (AudioAutoencoder.shard_time, satb_oobleck_group_*) against the single-device
decode, at SA-Open's length (1024 latents) and Stable Audio 2.0's (6144 latents), batch 1, an SA-Open-width decoder
(SnakeBeta, transposed upsampling, strides 2 4 4 8 8, fp16 operands) with seeded synthetic weights.

Configurations: unsharded; 2, 4 and 8 ranks all on cuda:0 ("virtual"); and 2, 4 and 8 ranks on distinct GPUs where
that many are visible (otherwise printed as not measured).  With virtual ranks the ranks run one after another on one
GPU, so the time measures what sharding adds (the recomputed margins, the input copies and the output gather), not a
speedup.  Per shape, the configurations alternate in one process, `--rounds` rounds of `--iters` calls each:
  * ms per call from CUDA events on the home device's current stream (median and spread over the rounds);
  * the latents every rank decodes, summed, over the clip's latents (the margins' recompute share, from the plan);
  * the gather kernel's device time in one virtual call, from torch.profiler;
  * whether the sharded output is bit-identical to the unsharded one.
The card's name, power limit and SM clocks are read in the same run.

    python tests/oobleck_group_time.py [--out RESULT.json] [--iters 5] [--rounds 2]
"""
import argparse
import gc
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "friendly-stable-audio-tools_b200"))
sys.path.insert(0, HERE)

from cp_time import call_ms, smi  # noqa: E402

CFG = dict(channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8], latent_dim=64, out_channels=2,
           final_tanh=False, use_snake=True)
WORLDS = [2, 4, 8]


def decoder(sd):
    from stable_audio_tools.models.autoencoders import OobleckDecoder
    m = OobleckDecoder(**CFG)
    m.load_state_dict(sd)
    return m.cuda().eval()


def gather_ms(m, z):
    """Device time of the gather kernel(s) in one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(z)
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "time_gather" in e.key) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("oobleck_group_time: no CUDA device; these timings need the GPU")
    from oracle import oobleck_variants_oracle as ov
    from stable_audio_tools import _native
    sd = ov.make_decoder_weights(CFG, seed=5)
    n_dev = torch.cuda.device_count()
    res = dict(gpu=smi("name"), power_limit=smi("power.limit"), clocks_sm=smi("clocks.sm"),
               clocks_max_sm=smi("clocks.max.sm"), devices_visible=n_dev, iters=args.iters, rounds=args.rounds,
               shapes=[])
    for L in (1024, 6144):
        z = torch.randn(1, 64, L, generator=torch.Generator().manual_seed(L)).cuda()
        layouts = {"unsharded": None}
        layouts.update({f"virtual_{w}": ["cuda:0"] * w for w in WORLDS})
        layouts.update({f"devices_{w}": [f"cuda:{i}" for i in range(w)] for w in WORLDS if w <= n_dev})
        mods = {name: decoder(sd).shard_time(lay) for name, lay in layouts.items()}
        with torch.no_grad():
            ref = mods["unsharded"](z)
            exact = {name: bool(torch.equal(m(z), ref)) for name, m in mods.items()}   # also the warm-up
            times = {name: [] for name in mods}
            for _ in range(args.rounds):
                for name, m in mods.items():
                    m(z)
                    times[name].append(call_ms(m, dict(z=z), args.iters))
        shape = dict(latents=L, samples=L * 2048, configs={})
        for name, ts in times.items():
            w = len(layouts[name]) if layouts[name] else 1
            _, ext, margin = _native.oobleck_group_plan(w, L, mods[name].native_config())
            shape["configs"][name] = dict(ms=statistics.median(ts), ms_rounds=ts, bit_identical=exact[name],
                                          margin_latents=margin,
                                          decoded_over_clip=sum(hi - lo for lo, hi in ext) / L)
        for w in WORLDS:
            shape["configs"][f"virtual_{w}"]["gather_ms"] = gather_ms(mods[f"virtual_{w}"], z)
            if w > n_dev:
                shape["configs"][f"devices_{w}"] = f"not measured: {n_dev} device(s) visible"
        res["shapes"].append(shape)
        print(json.dumps(shape), flush=True)
        del mods, ref
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
