"""Reference of the DiT's FP8 self-attention (attention_dtype "fp8", include/satb200.h satb_dit_set_attention_fp8): the
operand quantisers, the stored key order of V^T, and an FP8-attention emulation of the CPU oracle.  No GPU needed.

Definition (DESIGN.md section 5), on the q, k, v the 16-bit path stores (after qk_norm and rotary, rounded to the
operand mode's 16-bit type):
  q, k  e4m3 with one power-of-two scale per (token, head): the FP8 row rule of fp8_ref over the head's 64 values;
  v     e4m3 with one power-of-two scale per (item, head, channel), over the item's N tokens;
  S     (q8 sq)(k8 sk)^T / 8, exact products of the dequantised operands, fp32 accumulation;
  P     e4m3 of exp(S - m), m the row maximum, in [0, 1] with no scale; the row sum l adds the fp32 (unrounded) P;
  O     (P8 (v8 sv)) / l, stored in the mode's 16-bit type.
The kernel rounds P against its running maximum, this emulation against the final one; the floor tolerance of the
forward tests absorbs that difference.

`fp8_attention()` runs the oracle's self-attention this way and leaves cross-attention as it is: the oracle's
self_attention is wrapped so that attention_core is swapped only for the duration of a self-attention call.  Stack it
with fp8_ref.fp8_operands for operand_dtype "fp8", or with dit_oracle.operand_rounding for the 16-bit modes.
"""
import torch

from fp8_ref import quantize_fp8_rows
from oracle import dit_oracle as do


def key_of(j):
    """Key held at stored position j (0 .. 31) of a 32-key group of V^T (the S accumulator's column ownership)."""
    return 16 * (j >> 4) + 8 * ((j & 3) >> 1) + 2 * ((j >> 2) & 3) + (j & 1)


def stored_key_order(n_pad):
    """[n_pad] long: stored position -> key, for a V^T row of n_pad (a multiple of 32) positions."""
    j = torch.arange(n_pad)
    return (j & ~31) + key_of(j & 31)


def quantize_heads(x):
    """q or k [..., n, 64] -> (e4m3 [..., n, 64], scales [..., n, 1]): one scale per (token, head)."""
    return quantize_fp8_rows(x)


def quantize_v(v):
    """v [..., n, 64] -> (e4m3 [..., n, 64], scales [..., 1, 64]): one scale per channel over the n tokens."""
    q, s = quantize_fp8_rows(v.transpose(-1, -2))
    return q.transpose(-1, -2), s.transpose(-1, -2)


def dequant(q, s, dtype=torch.float32):
    return q.to(dtype) * s.to(dtype)


def fp8_attention_core(q, k, v):
    """Self-attention core of the FP8 mode: q, k, v [b, h, n, 64] (one kv head per head)."""
    q, k, v = do._rnd(q), do._rnd(k), do._rnd(v)
    qd, kd, vd = (dequant(*quantize_heads(q)), dequant(*quantize_heads(k)), dequant(*quantize_v(v)))
    s = torch.einsum("bhid,bhjd->bhij", qd, kd) * (1.0 / q.shape[-1] ** 0.5)
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))
    l = p.sum(dim=-1, keepdim=True)
    p8 = p.to(torch.float8_e4m3fn).to(p.dtype)
    return torch.einsum("bhij,bhjd->bhid", p8, vd) / l


class fp8_attention:
    """Run the oracle's self-attention as attention_dtype "fp8" computes it (see the module docstring)."""

    def __enter__(self):
        self.prev = do.self_attention
        prev = self.prev

        def self_attention(*args, **kwargs):
            core = do.attention_core
            do.attention_core = fp8_attention_core
            try:
                return prev(*args, **kwargs)
            finally:
                do.attention_core = core

        do.self_attention = self_attention
        return self

    def __exit__(self, *exc):
        do.self_attention = self.prev
