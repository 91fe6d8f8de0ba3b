"""Torch restatement of Hugging Face's T5 encoder (transformers 5.5, models/t5/modeling_t5.py), the module the
reference's T5Conditioner wraps (reference models/conditioners.py:261-346), as the checker of the native encoder
(csrc/t5.cu, stable_audio_tools/models/t5.py).  TEST INFRASTRUCTURE: never imported by the package.

Line citations are modeling_t5.py of that version:
  T5LayerNorm                    :46-68    w * (x * rsqrt(mean(x^2) + eps)), statistics in fp32
  T5DenseActDense                :84-103   wo(relu(wi x))
  T5DenseGatedActDense           :106-130  wo(gelu_new(wi_0 x) * wi_1 x)
  _relative_position_bucket      :189-234  (bidirectional in the encoder)
  compute_bias                   :236-251  bias[h, i, j] = rel[bucket(j - i), h]; block 0 only, shared by every block
  T5Attention.forward            :253-340  softmax(q k^T + bias + mask) v, no 1 / sqrt(d) scale
  T5Block / T5Stack              :424-492, 637-780  pre-norm residual blocks, final_layer_norm
The extended attention mask adds the dtype's minimum at masked keys (modeling_utils get_extended_attention_mask).

operand_rounding(dtype) rounds exactly the tensors the kernels round to 16 bits: the weight matrices, the RMSNorm
outputs, q / k / v, the unnormalised probabilities P (exp(s - row max), divided by the fp32 sum of the unrounded
ones), the attention output and the FF-in activations (which saturate at +-65504 in fp16).  The embedding, the
residual stream, the relative-position bias and the final norm stay fp32 (fp64 here).
"""
import math

import torch

MAX_LENGTH = 512


def relative_position_bucket(relative_position, num_buckets=32, max_distance=128):
    """modeling_t5.py:189-234, bidirectional=True, the same torch operations."""
    relative_buckets = 0
    num_buckets //= 2
    relative_buckets += (relative_position > 0).to(torch.long) * num_buckets
    relative_position = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    large = max_exact + (torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return relative_buckets + torch.where(is_small, relative_position, large)


def make_t5_weights(cfg, seed):
    """A seeded T5EncoderModel state dict (HF keys, fp32) for cfg (T5Config fields).  The scales follow HF's
    _init_weights (q by (d_model d_kv)^-1/2, which is where T5 keeps its attention scale; k, v, wi by d_model^-1/2;
    o, wo by their fan-in^-1/2), with unit-size embeddings, norms near 1 and an O(1) position bias, so that activations
    neither vanish nor blow up over 12 blocks."""
    g = torch.Generator().manual_seed(seed)
    D, dk, H, F = cfg["d_model"], cfg["d_kv"], cfg["num_heads"], cfg["d_ff"]
    inner = H * dk
    rn = lambda *s: torch.randn(*s, generator=g)
    sd = {"shared.weight": rn(cfg["vocab_size"], D)}
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer."
        sd[p + "0.layer_norm.weight"] = 1 + 0.1 * rn(D)
        sd[p + "0.SelfAttention.q.weight"] = rn(inner, D) * (D * dk) ** -0.5 * 2.0
        sd[p + "0.SelfAttention.k.weight"] = rn(inner, D) * D ** -0.5
        sd[p + "0.SelfAttention.v.weight"] = rn(inner, D) * D ** -0.5
        sd[p + "0.SelfAttention.o.weight"] = rn(D, inner) * inner ** -0.5
        if i == 0:
            sd[p + "0.SelfAttention.relative_attention_bias.weight"] = rn(cfg["relative_attention_num_buckets"], H)
        sd[p + "1.layer_norm.weight"] = 1 + 0.1 * rn(D)
        if cfg["feed_forward_proj"] == "gated-gelu":
            sd[p + "1.DenseReluDense.wi_0.weight"] = rn(F, D) * D ** -0.5
            sd[p + "1.DenseReluDense.wi_1.weight"] = rn(F, D) * D ** -0.5
        else:
            sd[p + "1.DenseReluDense.wi.weight"] = rn(F, D) * D ** -0.5
        sd[p + "1.DenseReluDense.wo.weight"] = rn(D, F) * F ** -0.5
    sd["encoder.final_layer_norm.weight"] = 1 + 0.1 * rn(D)
    return sd


def make_proj_out(d_in, d_out, seed):
    """Seeded weights of the conditioner's proj_out nn.Linear(d_in, d_out)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(d_out, d_in, generator=g) * d_in ** -0.5, 0.1 * torch.randn(d_out, generator=g)


def operand_rounding(dtype):
    """x -> x rounded to the 16-bit `dtype` (fp16 saturating at +-65504) and back, in x's own dtype."""
    if dtype == torch.float16:
        return lambda x: x.clamp(-65504.0, 65504.0).to(torch.float16).to(x.dtype)
    return lambda x: x.to(dtype).to(x.dtype)


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def rms_norm(x, w, eps):
    """:46-68 (fp32 weight)."""
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def position_bias(rel_weight, L, num_buckets, max_distance):
    """:236-251: [H, L, L] with bias[h, i, j] = rel_weight[bucket(j - i), h]."""
    pos = torch.arange(L, dtype=torch.long)
    buckets = relative_position_bucket(pos[None, :] - pos[:, None], num_buckets, max_distance).to(rel_weight.device)
    return rel_weight[buckets].permute(2, 0, 1)


def t5_encoder(sd, cfg, input_ids, attention_mask, rounding=None, dtype=torch.float64):
    """last_hidden_state [B, L, d_model] of T5EncoderModel(input_ids, attention_mask), computed in `dtype`.  Padded
    positions hold what HF computes there (the conditioner zeroes them)."""
    r = rounding if rounding is not None else (lambda x: x)
    D, dk, H = cfg["d_model"], cfg["d_kv"], cfg["num_heads"]
    eps = cfg.get("layer_norm_epsilon", 1e-6)
    B, L = input_ids.shape
    f = lambda k: sd[k].to(dtype)
    mat = lambda k: r(f(k))
    mask = attention_mask.to(torch.bool)
    h = f("shared.weight")[input_ids]                                                      # :682
    bias = position_bias(f("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"), L,
                         cfg["relative_attention_num_buckets"], cfg["relative_attention_max_distance"])
    neg = torch.zeros(mask.shape, dtype=dtype, device=mask.device).masked_fill(~mask, torch.finfo(torch.float32).min)
    neg = neg[:, None, None, :]
    gated = cfg["feed_forward_proj"] == "gated-gelu"
    heads = lambda t: t.view(B, L, H, dk).transpose(1, 2)
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer."
        x = r(rms_norm(h, f(p + "0.layer_norm.weight"), eps))
        q, k, v = (heads(r(x @ mat(p + f"0.SelfAttention.{n}.weight").T)) for n in "qkv")
        s = q @ k.transpose(-1, -2) + bias + neg                                             # :314-328
        if rounding is None:
            o = torch.softmax(s, dim=-1) @ v                                                   # :331-334
        else:
            e = torch.exp(s - s.amax(-1, keepdim=True))
            o = (r(e) @ v) / e.sum(-1, keepdim=True)
        o = r(o.transpose(1, 2).reshape(B, L, H * dk))
        h = h + o @ mat(p + "0.SelfAttention.o.weight").T                                      # :356-372
        x = r(rms_norm(h, f(p + "1.layer_norm.weight"), eps))
        if gated:
            a = gelu_new(x @ mat(p + "1.DenseReluDense.wi_0.weight").T) * (x @ mat(p + "1.DenseReluDense.wi_1.weight").T)
        else:
            a = torch.relu(x @ mat(p + "1.DenseReluDense.wi.weight").T)
        h = h + r(a) @ mat(p + "1.DenseReluDense.wo.weight").T                                 # :506-515
    return rms_norm(h, f("encoder.final_layer_norm.weight"), eps)                              # :768-770


def t5_conditioner(sd, cfg, input_ids, attention_mask, proj_w=None, proj_b=None, rounding=None, dtype=torch.float64):
    """T5Conditioner.forward after tokenising (reference conditioners.py:324-346): proj_out (if given) on the last
    hidden state, then the rows of padded positions zeroed."""
    e = t5_encoder(sd, cfg, input_ids, attention_mask, rounding=rounding, dtype=dtype)
    if proj_w is not None:
        w = proj_w.to(dtype)
        if rounding is not None:   # the kernels' proj_out GEMM takes the final norm and the weight in 16 bits
            e, w = rounding(e), rounding(w)
        e = e @ w.T + proj_b.to(dtype)
    return e * attention_mask.to(dtype)[..., None]
