"""Generate tests/golden/t5_*.npz: T5 encoder goldens from transformers.T5EncoderModel in fp32 (loaded with
t5_oracle.make_t5_weights), and one through the reference's own T5Conditioner.forward.

TEST INFRASTRUCTURE.  Run in the build container only (the conditioner golden needs the reference):

    python -m oracle.make_golden_t5

t5_<name>.npz, per config of CONFIGS: the config (JSON) and weight seed, input_ids / attention_mask [B, L] (right-padded
prompts of the listed lengths) and last_hidden_state [B, L, d_model] of T5EncoderModel in fp32.
t5_conditioner.npz: the reference's T5Conditioner (t5-base width: d_model 768, 2 blocks) with T5EncoderModel.from_pretrained
patched to return the seeded random model and the tokenizer stubbed by make_golden.FakeTokenizer; proj_out (768 -> 512)
set from t5_oracle.make_proj_out.  Stores the texts, max_length, the config and seeds, the tokenised ids / mask and the
conditioner's (embeddings, mask) output: the reference's own fp16 model on the CPU, proj_out, masking and padding.
No weights are stored: the tests rebuild them from the seeds.
"""
import json
import os

import numpy as np
import torch

from . import ref_shims, t5_oracle
from .make_golden import GOLDEN_DIR, FakeTokenizer

BASE = dict(vocab_size=1001, relative_attention_num_buckets=32, relative_attention_max_distance=128,
            layer_norm_epsilon=1e-6)
# name -> (config, seed, lengths, max_length)
CONFIGS = {
    "relu_hd64": (dict(BASE, d_model=128, d_kv=64, num_heads=2, d_ff=256, num_layers=2, feed_forward_proj="relu"),
                  11, [1, 48, 17, 33], 48),
    "gelu_hd64_inner": (dict(BASE, d_model=256, d_kv=64, num_heads=3, d_ff=320, num_layers=2,
                             feed_forward_proj="gated-gelu", relative_attention_num_buckets=16,
                             relative_attention_max_distance=40), 12, [70, 3, 1, 66], 70),
    "relu_hd128_inner": (dict(BASE, d_model=256, d_kv=128, num_heads=3, d_ff=512, num_layers=2, feed_forward_proj="relu",
                              relative_attention_num_buckets=8, relative_attention_max_distance=20), 13,
                         [130, 65, 1, 127], 130),
}
COND = dict(cfg=dict(BASE, d_model=768, d_kv=64, num_heads=12, d_ff=1024, num_layers=2, feed_forward_proj="relu"),
            seed=14, proj_seed=15, output_dim=512, max_length=40,
            texts=["a warm analog synth pad with slow attack", "kick", "",
                   " ".join(f"word{i}" for i in range(45))])


def hf_model(cfg, sd):
    from transformers import T5Config, T5EncoderModel
    m = T5EncoderModel(T5Config(**cfg, dropout_rate=0.0, is_encoder_decoder=False, use_cache=False))
    m.load_state_dict(sd, strict=True)
    return m.eval()


def ids_and_mask(lengths, L, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(len(lengths), L, dtype=torch.long)
    mask = torch.zeros(len(lengths), L, dtype=torch.long)
    for b, n in enumerate(lengths):
        ids[b, :n] = torch.randint(1, vocab, (n,), generator=g)
        mask[b, :n] = 1
    return ids, mask


def main():
    torch.set_grad_enabled(False)
    for name, (cfg, seed, lengths, L) in CONFIGS.items():
        sd = t5_oracle.make_t5_weights(cfg, seed)
        ids, mask = ids_and_mask(lengths, L, cfg["vocab_size"], seed + 100)
        out = hf_model(cfg, sd)(input_ids=ids, attention_mask=mask)["last_hidden_state"]
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"t5_{name}.npz"), config=json.dumps(cfg), seed=seed,
                            input_ids=ids.numpy(), attention_mask=mask.numpy(), last_hidden_state=out.float().numpy())
        print("wrote", name, tuple(out.shape))

    import importlib
    import transformers
    ref = ref_shims.import_reference()
    with ref_shims.reference_modules(ref):
        RefT5Conditioner = importlib.import_module("stable_audio_tools.models.conditioners").T5Conditioner
    cfg = COND["cfg"]
    sd = t5_oracle.make_t5_weights(cfg, COND["seed"])
    model = hf_model(cfg, sd)
    transformers.AutoTokenizer.from_pretrained = classmethod(lambda cls, *a, **k: FakeTokenizer())
    transformers.T5EncoderModel.from_pretrained = classmethod(lambda cls, *a, **k: model)
    cond = RefT5Conditioner(output_dim=COND["output_dim"], t5_model_name="t5-base", max_length=COND["max_length"])
    w, b = t5_oracle.make_proj_out(768, COND["output_dim"], COND["proj_seed"])
    cond.proj_out.weight.copy_(w)
    cond.proj_out.bias.copy_(b)
    emb, m = cond(COND["texts"])
    enc = FakeTokenizer()(COND["texts"], max_length=COND["max_length"])
    np.savez_compressed(os.path.join(GOLDEN_DIR, "t5_conditioner.npz"), config=json.dumps(cfg), seed=COND["seed"],
                        proj_seed=COND["proj_seed"], output_dim=COND["output_dim"], max_length=COND["max_length"],
                        texts=np.array(COND["texts"]), input_ids=enc["input_ids"].numpy(),
                        attention_mask=enc["attention_mask"].numpy(), embeddings=emb.float().numpy(),
                        mask=m.numpy())
    print("wrote conditioner", tuple(emb.shape), emb.dtype)


if __name__ == "__main__":
    main()
