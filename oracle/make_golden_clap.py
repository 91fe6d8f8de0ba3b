"""Generate tests/golden/clap_*.npz: RoBERTa encoder goldens from transformers.RobertaModel in fp32 (loaded with
clap_oracle.make_roberta_weights), and one through the reference's own CLAPTextConditioner.forward.

TEST INFRASTRUCTURE.  Run in the build container only (the conditioner golden needs the reference):

    python -m oracle.make_golden_clap

clap_<name>.npz, per config of CONFIGS: the config (JSON) and weight seed, input_ids / attention_mask [B, L] (right-padded
prompts of the listed lengths, with pad ids (1) inside some prompts, which move the position ids) and hidden_states
[n_layers + 1, B, L, hidden] of RobertaModel(output_hidden_states=True) in fp32, padded positions included.
clap_conditioner.npz: the reference's CLAPTextConditioner(use_text_features=True, feature_layer_ix=-2, cond_dim 768 as
in txt2audio/stable_audio_2_0.json) with clap_oracle's laion_clap stand-in: a roberta-base text branch, the checkpoint
written as {"state_dict": {"module.text_branch.<key>": ...}} from the seed, and make_golden.FakeTokenizer for
RobertaTokenizer.  Stores the texts, the seed, the tokenised ids / mask, the conditioner's (features, mask) for the
batch, and for its first text alone (the reference's "" pad) the mask and the largest difference of its features from
the batch's first row.  No weights are stored: the tests rebuild them.
clap_sa20_conditioning.json: the "conditioning" block of the reference's txt2audio/stable_audio_2_0.json, as shipped.
"""
import json
import os
import tempfile

import numpy as np
import torch

from . import clap_oracle as co
from . import ref_shims
from .make_golden import GOLDEN_DIR, FakeTokenizer

SMALL = dict(co.ROBERTA_BASE, vocab_size=1001)
# name -> (config, seed, lengths, L)
CONFIGS = {
    "d128_l2": (dict(SMALL, hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=2), 61,
                [1, 40, 17, 33], 40),
    "d256_l3": (dict(SMALL, hidden_size=256, num_attention_heads=4, intermediate_size=544, num_hidden_layers=3), 62,
                [77, 2, 1, 65, 77], 77),
}
COND = dict(seed=64, feature_layer_ix=-2, output_dim=768,
            texts=["a warm analog synth pad with slow attack", "kick", " ".join(f"word{i}" for i in range(90))])


def ids_and_mask(lengths, L, vocab, seed):
    """Right-padded prompts; padded positions hold the pad id 1, and every third prompt has pad ids inside it too."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.ones(len(lengths), L, dtype=torch.long)
    mask = torch.zeros(len(lengths), L, dtype=torch.long)
    for b, n in enumerate(lengths):
        ids[b, :n] = torch.randint(0, vocab, (n,), generator=g)
        if b % 3 == 0 and n > 4:
            ids[b, 2:n:4] = 1
        mask[b, :n] = 1
    return ids, mask


def write_checkpoint(sd, path):
    torch.save({"state_dict": {"module.text_branch." + k: v for k, v in sd.items()}}, path)


def main():
    torch.set_grad_enabled(False)
    for name, (cfg, seed, lengths, L) in CONFIGS.items():
        sd = co.make_roberta_weights(cfg, seed)
        ids, mask = ids_and_mask(lengths, L, cfg["vocab_size"], seed + 100)
        hs = co.hf_model(cfg, sd)(input_ids=ids, attention_mask=mask, output_hidden_states=True).hidden_states
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"clap_{name}.npz"), config=json.dumps(cfg), seed=seed,
                            input_ids=ids.numpy(), attention_mask=mask.numpy(),
                            hidden_states=torch.stack(hs).float().numpy())
        print("wrote", name, tuple(torch.stack(hs).shape))

    shipped = os.path.join(ref_shims.REFERENCE_ROOT, "stable_audio_tools/configs/model_configs/txt2audio/stable_audio_2_0.json")
    with open(os.path.join(GOLDEN_DIR, "clap_sa20_conditioning.json"), "w") as f:
        json.dump(json.load(open(shipped))["model"]["conditioning"], f, indent=1)
        f.write("\n")

    import importlib
    ref = ref_shims.import_reference()
    co.install_laion_clap_shim(FakeTokenizer)
    try:
        with ref_shims.reference_modules(ref):
            RefCLAP = importlib.import_module("stable_audio_tools.models.conditioners").CLAPTextConditioner
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "clap.pt")
            write_checkpoint(co.make_roberta_weights(co.ROBERTA_BASE, COND["seed"]), path)
            cond = RefCLAP(output_dim=COND["output_dim"], clap_ckpt_path=path, use_text_features=True,
                           feature_layer_ix=COND["feature_layer_ix"], audio_model_type="HTSAT-base",
                           enable_fusion=True)
        feats, m = cond(COND["texts"])
        single, m1 = cond(COND["texts"][:1])
    finally:
        co.remove_laion_clap_shim()
    enc = FakeTokenizer()(COND["texts"], max_length=co.CLAP_MAX_LENGTH)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "clap_conditioner.npz"), config=json.dumps(co.ROBERTA_BASE),
                        seed=COND["seed"], feature_layer_ix=COND["feature_layer_ix"], output_dim=COND["output_dim"],
                        texts=np.array(COND["texts"]), input_ids=enc["input_ids"].numpy(),
                        attention_mask=enc["attention_mask"].numpy(), features=feats.float().numpy(), mask=m.numpy(),
                        single_mask=m1.numpy(), single_max_abs=float((single[0] - feats[0]).abs().max()))
    print("wrote conditioner", tuple(feats.shape), feats.dtype, tuple(single.shape))


if __name__ == "__main__":
    main()
