"""Reference of the DiT's FP8 operand mode (include/satb200.h operand_dtype 2): the e4m3 row quantiser and an FP8
emulation of the CPU oracle.  No GPU needed.

Quantiser.  Each row x (last dim) gets a power-of-two scale s = 2^e, e the smallest integer with amax <= 448 * 2^e
(448: the largest finite e4m3), kept >= -126 so that 2^e and 2^-e are normal fp32 numbers; s = 1 for an all-zero row.
q = e4m3_rn(x * 2^-e).  No value of x * 2^-e exceeds 448, so torch's cast (which turns values above 448 into NaN
instead of saturating) is safe here.  Dequantised values q * s are exact in fp32.

Emulation.  Inside `fp8_operands(sd)` the oracle (oracle/dit_oracle.py) runs its three Linear layers that read a
LayerNorm output - self-attention to_qkv, cross-attention to_q and the feed-forward input ff.0 - on the dequantised
e4m3 operands (one scale per activation row = token, one per weight row), and rounds every other tensor-core operand
to fp16, as operand_rounding(torch.float16) does.  Its error against the fp32 oracle is the floor the FP8 mode sits on.
The oracle itself is not changed: its 16-bit Linear helper is swapped for the duration of the context, and picks the
FP8 path by the identity of the weight tensor.
"""
import torch
import torch.nn.functional as F

from oracle import dit_oracle as do

E4M3_MAX = 448.0
FP8_WEIGHT_SUFFIXES = ("self_attn.to_qkv.weight", "cross_attn.to_q.weight", "ff.ff.0.proj.weight")


def fp8_row_exponent(amax):
    """e of the row scale: with amax = m * 2^E, m in [0.5, 1) (frexp) and 448 = 0.875 * 2^9, e = E - 9 if m <= 0.875,
    else E - 8; at least -126; 0 for amax == 0.  Exact."""
    m, E = torch.frexp(amax)
    e = torch.where(m <= 0.875, E - 9, E - 8).clamp_min(-126)
    return torch.where(amax > 0, e, torch.zeros_like(e))


def quantize_fp8_rows(x):
    """Rows of x -> (q float8_e4m3fn, scale [..., 1] in x's dtype)."""
    e = fp8_row_exponent(x.abs().amax(dim=-1, keepdim=True))
    q = torch.ldexp(x, -e).to(torch.float8_e4m3fn)
    return q, torch.ldexp(torch.ones_like(x[..., :1]), e)


def fp8_roundtrip(x):
    """x through e4m3 with its row scales and back."""
    q, s = quantize_fp8_rows(x)
    return q.to(x.dtype) * s


def fp8_weight_keys(sd):
    return sorted(k for k in sd if k.endswith(FP8_WEIGHT_SUFFIXES))


class fp8_operands:
    """Run the oracle as the FP8 mode computes: see the module docstring.  `roundtrip` replaces fp8_roundtrip (tests
    use it to see which operands go through it)."""

    def __init__(self, sd, roundtrip=None):
        self.ids = {id(sd[k]) for k in fp8_weight_keys(sd)}
        self.roundtrip = roundtrip or fp8_roundtrip
        self.rounding = do.operand_rounding(torch.float16)

    def __enter__(self):
        self.prev = do._lin16
        prev, ids, rt = self.prev, self.ids, self.roundtrip

        def lin(x, w, b=None):
            if id(w) in ids:
                return F.linear(rt(x), rt(w), b)
            return prev(x, w, b)

        do._lin16 = lin
        self.rounding.__enter__()
        return self

    def __exit__(self, *exc):
        self.rounding.__exit__(*exc)
        do._lin16 = self.prev
