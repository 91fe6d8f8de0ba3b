"""Time the native T5 encoder against Hugging Face's T5EncoderModel in fp16 eager (what T5Conditioner runs by
default) on the same GPU and the same weights: t5-base shape (seeded random weights), B in {1, 4, 8, 16} prompts of
8 - 40 tokens padded to max_length 128.  CUDA events around each encode, the two arms alternated, two rounds; the SM
clock and the card's name and power limit are read in the same run.  Then one torch.profiler pass of each arm for the
per-kernel times and the native encode's launch count.

    python tests/t5_time.py [--out RESULT.json] [--iters 30]

The full result goes to --out when given; a summary is printed either way.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "friendly-stable-audio-tools_b200"))

from oracle import t5_oracle as to  # noqa: E402

CFG = dict(vocab_size=32128, d_model=768, d_kv=64, num_heads=12, d_ff=3072, num_layers=12,
           relative_attention_num_buckets=32, relative_attention_max_distance=128, feed_forward_proj="relu",
           layer_norm_epsilon=1e-6)


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


def prompts(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(8, 41, (B,), generator=g).tolist()
    ids = torch.zeros(B, L, dtype=torch.long)
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, n in enumerate(lengths):
        ids[b, :n] = torch.randint(1, CFG["vocab_size"], (n,), generator=g)
        mask[b, :n] = 1
    return ids.cuda(), mask.cuda(), lengths


def time_ms(fn, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "t5_time needs a GPU"
    from transformers import T5Config, T5EncoderModel
    from stable_audio_tools import _native
    from stable_audio_tools.models.t5 import T5Encoder
    torch.set_grad_enabled(False)
    sd = {k: v.half().float() for k, v in to.make_t5_weights(CFG, 61).items()}
    hf = T5EncoderModel(T5Config(**CFG, dropout_rate=0.0, is_encoder_decoder=False, use_cache=False))
    hf.load_state_dict(sd)
    hf = hf.to(torch.float16).cuda().eval()      # as the reference's conditioner holds it
    nat = T5Encoder.from_config(CFG).load_state_dict(sd, device="cuda")
    res = {"gpu": smi("name,power.limit,clocks.max.sm"), "config": "t5-base shape, 12 blocks, fp16", "shapes": []}
    cases = {B: prompts(B, 128, 70 + B) for B in (1, 4, 8, 16)}
    for B, (ids, mask, lengths) in cases.items():   # warm-up of every shape
        for _ in range(3):
            hf(input_ids=ids, attention_mask=mask)
            nat(ids, mask)
    torch.cuda.synchronize()
    for rnd in range(2):
        for B, (ids, mask, lengths) in cases.items():
            t_hf = time_ms(lambda: hf(input_ids=ids, attention_mask=mask), args.iters)
            t_nat = time_ms(lambda: nat(ids, mask), args.iters)
            t_hf2 = time_ms(lambda: hf(input_ids=ids, attention_mask=mask), args.iters)
            t_nat2 = time_ms(lambda: nat(ids, mask), args.iters)
            row = dict(round=rnd, B=B, tokens=sum(lengths), hf_fp16_ms=min(t_hf, t_hf2), native_ms=min(t_nat, t_nat2),
                       sm_clock=smi("clocks.sm"))
            res["shapes"].append(row)
            print(json.dumps(row), flush=True)
    ids, mask, _ = cases[16]
    n0 = _native.launch_count()
    nat(ids, mask)
    torch.cuda.synchronize()
    res["native_launches_per_encode"] = _native.launch_count() - n0
    from torch.profiler import ProfilerActivity, profile
    for name, fn in (("native", lambda: nat(ids, mask)), ("hf_fp16", lambda: hf(input_ids=ids, attention_mask=mask))):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        rows = []
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
                dt = getattr(e, "self_device_time_total", 0) or getattr(e, "self_cuda_time_total", 0)
                if dt > 0:
                    rows.append(dict(kernel=e.key[:90], calls_per_encode=e.count / 5, us_per_encode=dt / 5))
        rows.sort(key=lambda r: -r["us_per_encode"])
        res[f"kernels_{name}_B16"] = rows[:15]
        res[f"kernel_launches_{name}_B16"] = sum(r["calls_per_encode"] for r in rows)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if not k.startswith("kernels_")}, indent=1))


if __name__ == "__main__":
    main()
