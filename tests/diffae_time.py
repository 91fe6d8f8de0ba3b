"""Timing driver for diffusion-autoencoder decoding (not a test): python tests/diffae_time.py [steps] [rounds] [tokens]

A DiffusionAutoencoder whose DiT has SA-Open width (D 1536, 24 heads, 24 blocks) and diffuses 16-band PQMF sub-bands
of stereo audio (io_channels 32) conditioned on 64 latent channels upsampled x4; batch 1 of `tokens` sub-band frames
(default 4096 = 65 536 samples, 1.49 s at 44.1 kHz).  Per round, in this one process: the bare DiT forward at that
shape as the decode runs it (one CUDA-graph replay, CUDA events over `steps` calls), the fused update kernel alone
(`steps` launches), and whole decodes of `steps` steps (DiT replays + updates + PQMF synthesis).  Prints one JSON line
per round with the decode time per clip and per step, and the loop's overhead over `steps` bare forwards; the card's
name and power limit first."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "friendly-stable-audio-tools_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from fp8_time import events_ms, smi


def main():
    from oracle import diffae_oracle as dao
    from stable_audio_tools import _native as nat
    from stable_audio_tools import create_model_from_config
    from stable_audio_tools.inference.sampling import vdiffusion_schedule
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    tokens = int(sys.argv[3]) if len(sys.argv) > 3 else 4096
    print(json.dumps({"card": smi("name,power.limit,clocks.max.sm")}), flush=True)
    dit = dict(io_channels=32, input_concat_dim=64, embed_dim=1536, depth=24, num_heads=24, cond_token_dim=0,
               global_cond_dim=0, project_cond_tokens=False, transformer_type="continuous_transformer")
    cfg = {"model_type": "diffusion_autoencoder", "sample_rate": 44100,
           "model": {"io_channels": 32, "latent_dim": 64, "downsampling_ratio": 4,
                     "diffusion": {"type": "dit", "config": dit},
                     "pretransform": {"type": "pqmf", "config": {"attenuation": 100, "num_bands": 16}}}}
    model = create_model_from_config(cfg)
    bufs = dict(model.pretransform.pqmf.state_dict())
    model.load_state_dict(dao.make_state_dict(cfg, 7, bufs), strict=True)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(8)
    z = torch.randn(1, 64, tokens // 4, generator=g).cuda()
    noise = torch.randn(1, 32, tokens, generator=g).cuda()
    concat = torch.nn.functional.interpolate(z, size=tokens, mode="nearest")
    t = torch.full((1,), 0.5, device="cuda")
    dit_m = model.diffusion.model
    a, s, an, adj, dd = vdiffusion_schedule(steps, 0)[0][1:]
    x_next = torch.empty_like(noise)

    def forward():
        return model.diffusion(noise, t, input_concat_cond=concat)

    def update():
        nat.check(nat.lib().satb_vdiffusion_update(nat.ptr(noise), nat.ptr(noise), None, nat.ptr(x_next), None,
                                                   noise.numel(), a, s, an, adj, dd, nat.stream_ptr()))

    def decode():
        return model.decode(z, steps=steps, noise=noise)

    dit_m.cuda_graph = True
    for _ in range(3):
        forward()
    dit_m.cuda_graph = False
    decode()
    torch.cuda.synchronize()
    for rnd in range(rounds):
        dit_m.cuda_graph = True
        fwd_ms, fwd_clock = events_ms(forward, steps)
        dit_m.cuda_graph = False
        upd_ms, _ = events_ms(update, steps)
        dec_ms, dec_clock = events_ms(decode, 1)
        print(json.dumps({"round": rnd, "tokens": tokens, "steps": steps, "audio_samples": tokens * 16,
                          "dit_forward_ms": round(fwd_ms, 3), "update_kernel_us": round(upd_ms * 1e3, 2),
                          "decode_ms_per_clip": round(dec_ms, 2), "decode_ms_per_step": round(dec_ms / steps, 3),
                          "loop_overhead_pct": round(100 * (dec_ms / (steps * fwd_ms) - 1), 2),
                          "sm_clock_forward": fwd_clock, "sm_clock_decode": dec_clock}), flush=True)


if __name__ == "__main__":
    main()
