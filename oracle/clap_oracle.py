"""Torch restatement of Hugging Face's RoBERTa encoder (transformers 5.5, models/roberta/modeling_roberta.py), the text
branch whose hidden states the reference's CLAPTextConditioner returns (reference models/conditioners.py:105-192), as
the checker of the native encoder (csrc/roberta.cu, stable_audio_tools/models/roberta.py), and a `laion_clap` stand-in
that lets the reference's own conditioner run.  TEST INFRASTRUCTURE: never imported by the package.

  RobertaEmbeddings          word + token_type[0], + position, LayerNorm; position ids from the ids
                             (create_position_ids_from_input_ids: cumsum(id != pad) * (id != pad) + pad)
  RobertaSelfAttention       softmax(q k^T / sqrt(64) + mask) v, the mask adding the dtype's minimum at padded keys
  RobertaSelfOutput / Output LayerNorm(dense(x) + bias + residual)  (post-LN)
  RobertaIntermediate        erf GELU (ACT2FN["gelu"])
  hidden_states              the embedding output, then every layer's output

laion_clap itself is not installed; what the reference uses of it is restated from upstream laion_clap (not pinned
here): CLAP_Module.model.text_branch is a RobertaModel with the roberta-base config, CLAP_Module.tokenizer is
RobertaTokenizer("roberta-base")(padding="max_length", truncation=True, max_length=77, return_tensors="pt") followed
by squeeze(0) of every tensor, and clap_module.factory.load_state_dict is torch.load, the "state_dict" entry if there
is one, and the "module." prefix stripped.

operand_rounding (oracle/t5_oracle.py) rounds exactly the tensors the kernels round to 16 bits: the weight matrices,
the LayerNorm outputs that feed a GEMM, q / k / v (after their bias), the unnormalised probabilities P, the attention
output and the FF-in activations.  The embeddings, the residual stream and the biases stay fp32 (fp64 here).
"""
import math
import sys
import types

import torch

MAX_LENGTH = 512
ROBERTA_BASE = dict(vocab_size=50265, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                    intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                    layer_norm_eps=1e-5, hidden_act="gelu")
CLAP_MAX_LENGTH = 77


def make_roberta_weights(cfg, seed):
    """A seeded RobertaModel state dict (HF keys, fp32, no pooler) for cfg (RobertaConfig fields): unit-size
    embeddings, fan-in-scaled matrices, LayerNorm weights near 1 and O(0.1) biases."""
    g = torch.Generator().manual_seed(seed)
    D, F = cfg["hidden_size"], cfg["intermediate_size"]
    rn = lambda *s: torch.randn(*s, generator=g)
    sd = {"embeddings.word_embeddings.weight": rn(cfg["vocab_size"], D),
          "embeddings.position_embeddings.weight": rn(cfg["max_position_embeddings"], D),
          "embeddings.token_type_embeddings.weight": rn(cfg["type_vocab_size"], D),
          "embeddings.LayerNorm.weight": 1 + 0.1 * rn(D), "embeddings.LayerNorm.bias": 0.1 * rn(D)}
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            sd[p + f"attention.self.{n}.weight"] = rn(D, D) * D ** -0.5 * (2.0 if n == "query" else 1.0)
            sd[p + f"attention.self.{n}.bias"] = 0.1 * rn(D)
        sd[p + "attention.output.dense.weight"] = rn(D, D) * D ** -0.5
        sd[p + "attention.output.dense.bias"] = 0.1 * rn(D)
        sd[p + "attention.output.LayerNorm.weight"] = 1 + 0.1 * rn(D)
        sd[p + "attention.output.LayerNorm.bias"] = 0.1 * rn(D)
        sd[p + "intermediate.dense.weight"] = rn(F, D) * D ** -0.5
        sd[p + "intermediate.dense.bias"] = 0.1 * rn(F)
        sd[p + "output.dense.weight"] = rn(D, F) * F ** -0.5
        sd[p + "output.dense.bias"] = 0.1 * rn(D)
        sd[p + "output.LayerNorm.weight"] = 1 + 0.1 * rn(D)
        sd[p + "output.LayerNorm.bias"] = 0.1 * rn(D)
    return sd


def hf_model(cfg, sd):
    """transformers.RobertaModel for cfg with sd loaded (pooler left at its initialisation: unused), eval, eager."""
    from transformers import RobertaConfig, RobertaModel
    m = RobertaModel(RobertaConfig(**cfg, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0))
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("pooler.") for k in missing), (missing, unexpected)
    return m.eval()


def position_ids(input_ids, pad):
    mask = input_ids.ne(pad).int()
    return (torch.cumsum(mask, dim=1).type_as(mask) * mask).long() + pad


def layer_norm(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def roberta_hidden_states(sd, cfg, input_ids, attention_mask, n_layers=None, rounding=None, dtype=torch.float64):
    """hidden_states[0 .. n_layers] of RobertaModel(input_ids, attention_mask, output_hidden_states=True) in `dtype`
    (every position, padded ones included)."""
    r = rounding if rounding is not None else (lambda x: x)
    D, H = cfg["hidden_size"], cfg["num_attention_heads"]
    dk = D // H
    eps, pad = cfg["layer_norm_eps"], cfg["pad_token_id"]
    n_layers = cfg["num_hidden_layers"] if n_layers is None else n_layers
    B, L = input_ids.shape
    f = lambda k: sd[k].to(dtype)
    mat = lambda k: r(f(k))
    pos = position_ids(input_ids, pad)
    x = f("embeddings.word_embeddings.weight")[input_ids] + f("embeddings.token_type_embeddings.weight")[0]
    x = x + f("embeddings.position_embeddings.weight")[pos]
    h = layer_norm(x, f("embeddings.LayerNorm.weight"), f("embeddings.LayerNorm.bias"), eps)
    out = [h]
    mask = attention_mask.to(torch.bool)
    neg = torch.zeros(mask.shape, dtype=dtype, device=mask.device).masked_fill(~mask, torch.finfo(torch.float32).min)
    neg = neg[:, None, None, :]
    heads = lambda t: t.view(B, L, H, dk).transpose(1, 2)
    for i in range(n_layers):
        p = f"encoder.layer.{i}."
        a = r(h)
        q, k, v = (heads(r(a @ mat(p + f"attention.self.{n}.weight").T + f(p + f"attention.self.{n}.bias")))
                   for n in ("query", "key", "value"))
        s = q @ k.transpose(-1, -2) / math.sqrt(dk) + neg
        if rounding is None:
            o = torch.softmax(s, dim=-1) @ v
        else:
            e = torch.exp(s - s.amax(-1, keepdim=True))
            o = (r(e) @ v) / e.sum(-1, keepdim=True)
        o = r(o.transpose(1, 2).reshape(B, L, D))
        h = layer_norm(h + o @ mat(p + "attention.output.dense.weight").T + f(p + "attention.output.dense.bias"),
                       f(p + "attention.output.LayerNorm.weight"), f(p + "attention.output.LayerNorm.bias"), eps)
        a = r(gelu(r(h) @ mat(p + "intermediate.dense.weight").T + f(p + "intermediate.dense.bias")))
        h = layer_norm(h + a @ mat(p + "output.dense.weight").T + f(p + "output.dense.bias"),
                       f(p + "output.LayerNorm.weight"), f(p + "output.LayerNorm.bias"), eps)
        out.append(h)
    return out


def clap_features(sd, cfg, input_ids, attention_mask, feature_layer_ix, proj_w=None, proj_b=None, rounding=None,
                  dtype=torch.float64):
    """CLAPTextConditioner.forward with use_text_features after tokenising (reference conditioners.py:170-181):
    hidden_states[feature_layer_ix], then proj_out if given.  Padded positions are not zeroed."""
    n = feature_layer_ix % (cfg["num_hidden_layers"] + 1)
    e = roberta_hidden_states(sd, cfg, input_ids, attention_mask, n_layers=n, rounding=rounding, dtype=dtype)[n]
    if proj_w is not None:
        w = proj_w.to(dtype)
        if rounding is not None:   # the kernels' proj_out GEMM takes the hidden state and the weight in 16 bits
            e, w = rounding(e), rounding(w)
        e = e @ w.T + proj_b.to(dtype)
    return e


def clap_load_state_dict(checkpoint_path, map_location="cpu"):
    """laion_clap.clap_module.factory.load_state_dict (upstream): torch.load, "state_dict" if present, "module."
    stripped."""
    checkpoint = torch.load(checkpoint_path, map_location=map_location, weights_only=False)
    state_dict = checkpoint["state_dict"] if isinstance(checkpoint, dict) and "state_dict" in checkpoint else checkpoint
    if next(iter(state_dict.items()))[0].startswith("module"):
        state_dict = {k[7:]: v for k, v in state_dict.items()}
    return state_dict


def install_laion_clap_shim(tokenizer_factory, seed=0):
    """sys.modules entries `laion_clap` and `laion_clap.clap_module.factory` for the reference's CLAPTextConditioner:
    CLAP_Module.model.text_branch is a RobertaModel(roberta-base) seeded with make_roberta_weights(ROBERTA_BASE, seed)
    (the checkpoint then overwrites it), an unused audio_branch, and the tokenizer of upstream's CLAP_Module with
    tokenizer_factory() standing for RobertaTokenizer("roberta-base")."""
    from torch import nn

    class _CLAP(nn.Module):
        def __init__(self):
            super().__init__()
            self.text_branch = hf_model(ROBERTA_BASE, make_roberta_weights(ROBERTA_BASE, seed))
            self.audio_branch = nn.Identity()

    class CLAP_Module(nn.Module):
        def __init__(self, enable_fusion=False, device=None, amodel="HTSAT-tiny", tmodel="roberta"):
            super().__init__()
            self.model = _CLAP()
            self.tokenize = tokenizer_factory()

        def tokenizer(self, text):
            result = self.tokenize(text, padding="max_length", truncation=True, max_length=CLAP_MAX_LENGTH,
                                   return_tensors="pt")
            return {k: v.squeeze(0) for k, v in result.items()}

    pkg = types.ModuleType("laion_clap")
    pkg.CLAP_Module = CLAP_Module
    cm = types.ModuleType("laion_clap.clap_module")
    fac = types.ModuleType("laion_clap.clap_module.factory")
    fac.load_state_dict = clap_load_state_dict
    pkg.clap_module, cm.factory = cm, fac
    sys.modules.update({"laion_clap": pkg, "laion_clap.clap_module": cm, "laion_clap.clap_module.factory": fac})


def remove_laion_clap_shim():
    for k in ("laion_clap", "laion_clap.clap_module", "laion_clap.clap_module.factory"):
        sys.modules.pop(k, None)
