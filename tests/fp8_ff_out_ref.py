"""Reference of the DiT's FP8 FF-out option (ff_out_dtype "fp8", include/satb200.h satb_dit_set_ff_out_fp8): the e4m3
block quantiser and an emulation of the oracle that composes with fp8_ref.fp8_operands.  No GPU needed.

Block quantiser.  The last dim of x is cut into blocks of 128 columns (the last one may be shorter: the native inner
width is zero-padded to a multiple of 128, and zeros change no amax); each (row, block) gets the power-of-two scale of
fp8_ref.quantize_fp8_rows, applied to the block's amax.

Emulation.  Inside `fp8_ff_out_operands(sd)` the oracle's FF-out Linear of every layer (ff.ff.2, weight [D, inner])
runs on dequantised e4m3 operands: the activation (the SwiGLU or SiLU output) by (row, 128-column block), the weight by
row.  Every other Linear goes to whatever `dit_oracle._lin16` was on entry, so

    with fp8_operands(sd), fp8_ff_out_operands(sd):

emulates operand_dtype "fp8" with ff_out_dtype "fp8".  Its error against the fp32 oracle is the floor the option sits
on.  A use_conv FF-out (a 3-D weight) is not a Linear and is refused, as the model refuses it.
"""
import torch
import torch.nn.functional as F

from fp8_ref import fp8_roundtrip, quantize_fp8_rows
from oracle import dit_oracle as do

BLOCK = 128
FF_OUT_SUFFIX = "ff.ff.2.weight"


def quantize_fp8_blocks(x, block=BLOCK):
    """x [..., n] -> (q float8_e4m3fn [..., n], scale [..., ceil(n / block)] in x's dtype): one scale per block of
    `block` columns, the last block zero-padded."""
    n = x.shape[-1]
    nb = -(-n // block)
    xp = F.pad(x, (0, nb * block - n)).reshape(*x.shape[:-1], nb, block)
    q, s = quantize_fp8_rows(xp)
    return q.reshape(*x.shape[:-1], nb * block)[..., :n], s[..., 0]


def fp8_block_roundtrip(x, block=BLOCK):
    """x through e4m3 with its (row, block) scales and back."""
    q, s = quantize_fp8_blocks(x, block)
    return q.to(x.dtype) * s.repeat_interleave(block, dim=-1)[..., :x.shape[-1]]


def ff_out_weight_keys(sd):
    return sorted(k for k in sd if k.endswith(FF_OUT_SUFFIX))


class fp8_ff_out_operands:
    """Run the oracle's FF-out Linears as the FP8 FF-out option computes them: see the module docstring.
    `act_roundtrip` / `weight_roundtrip` replace fp8_block_roundtrip / fp8_roundtrip (tests use them to see which
    operands go through them)."""

    def __init__(self, sd, act_roundtrip=None, weight_roundtrip=None):
        keys = ff_out_weight_keys(sd)
        for k in keys:
            if sd[k].dim() != 2:
                raise NotImplementedError(f"{k}: the FP8 FF-out option needs a Linear FF-out (got a convolution)")
        self.ids = {id(sd[k]) for k in keys}
        self.act_rt = act_roundtrip or fp8_block_roundtrip
        self.w_rt = weight_roundtrip or fp8_roundtrip

    def __enter__(self):
        self.prev = do._lin16
        prev, ids, art, wrt = self.prev, self.ids, self.act_rt, self.w_rt

        def lin(x, w, b=None):
            if id(w) in ids:
                return F.linear(art(x), wrt(w), b)
            return prev(x, w, b)

        do._lin16 = lin
        return self

    def __exit__(self, *exc):
        do._lin16 = self.prev
