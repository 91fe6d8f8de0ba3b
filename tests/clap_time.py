"""Time the native RoBERTa encoder of CLAPTextConditioner against Hugging Face's RobertaModel in fp32 eager (what the
reference's conditioner runs) on the same GPU and the same weights: roberta-base (seeded random weights),
hidden_states[-2] as Stable Audio 2.0 asks (the native encoder runs 11 layers, HF all 12 with output_hidden_states),
B in {1, 2, 4, 8, 16} prompts of 8 - 40 tokens padded to 77.  CUDA events around each encode, the two arms
alternated, two rounds; the SM clock is sampled during the windows, and the card's name and power limit are read in
the same run.

    python tests/clap_time.py [--out RESULT.json] [--iters 30]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "friendly-stable-audio-tools_b200"))

from oracle import clap_oracle as co  # noqa: E402
from oracle.make_golden_clap import ids_and_mask  # noqa: E402


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


class ClockSampler:
    """Reads the SM clock every 0.2 s while a window runs."""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()

    def __enter__(self):
        def run():
            while not self._stop.is_set():
                v = smi("clocks.sm").split()[0]
                if v.isdigit():
                    self.samples.append(int(v))
                self._stop.wait(0.2)
        self._t = threading.Thread(target=run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    from stable_audio_tools import _native
    from stable_audio_tools.models.roberta import RobertaEncoder
    cfg = co.ROBERTA_BASE
    sd = co.make_roberta_weights(cfg, 5)
    hf = co.hf_model(cfg, sd).cuda()
    nat = RobertaEncoder.from_config(cfg, feature_layer_ix=-2).load_state_dict(sd, device="cuda")
    res = dict(gpu=smi("name"), power_limit=smi("power.limit"), max_sm_clock=smi("clocks.max.sm"), rows=[])
    for rnd in range(2):
        for B in (1, 2, 4, 8, 16):
            g = torch.Generator().manual_seed(B)
            ids, mask = ids_and_mask(torch.randint(8, 41, (B,), generator=g).tolist(), 77, cfg["vocab_size"], B)
            ids, mask = ids.cuda(), mask.cuda()
            with torch.no_grad(), ClockSampler() as clk:
                t_hf = time_ms(lambda: hf(input_ids=ids, attention_mask=mask, output_hidden_states=True), args.iters)
                t_nat = time_ms(lambda: nat(ids, mask), args.iters)
            with torch.no_grad():
                ref = hf(input_ids=ids, attention_mask=mask, output_hidden_states=True)["hidden_states"][-2]
            got = nat(ids, mask)
            err = float((got - ref).norm() / ref.norm())
            _native.lib().satb_reset_launch_count()
            nat(ids, mask)
            torch.cuda.synchronize()
            row = dict(round=rnd, B=B, hf_fp32_ms=round(t_hf, 3), native_fp16_ms=round(t_nat, 3),
                       speedup=round(t_hf / t_nat, 2), rel_l2_vs_hf=err, launches=_native.launch_count(),
                       sm_clock_mhz=(min(clk.samples), max(clk.samples)) if clk.samples else None)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "max_sm_clock")}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
