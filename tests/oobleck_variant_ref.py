"""float64 reference and per-element bound of the Oobleck steps that the ELU and nearest-upsample options add, on top
of tests/conv_ref.py (whose convolution bound, Snake bound, roundings and checker they reuse).

ELU (elu_fast in csrc/gemm.cuh).  For the pre-activation value v with bound dv (conv_ref.Pre), y = v > 0 ? v : e^v - 1:
    dy = dv                                   ELU's slope is <= 1
         + ELU_ABS [v <= -2^-6]               e^v - 1 through the SFU exponential: <= 2^-21.8 absolute
         + ELU_REL |y|                        the cubic polynomial on (-2^-6, 0] (truncation < 2^-22.6 |v|) and the
                                              fp32 roundings of either formula
         + E_OUT16 |y| + TAU16                the 16-bit store
Nearest upsample + conv k = 2s 'same' (nearest_w_prep_kernel, run_conv_gemm kind 3): a 3-tap convolution of the
low-rate input with the stored folded weights [3][s][cout][cin] (oracle.oobleck_variants_oracle.nearest_fold), so
conv_ref's accumulation bound applies with n = 3 * cin products (x 3 in fp16x3)."""
import torch

import conv_ref as C
from gemm_epilogue_ref import E_EPI, e_acc
from oracle.oobleck_variants_oracle import nearest_conv_folded

ELU_ABS = 2.0 ** -21
ELU_REL = 2.0 ** -21


def elu(p, dt):
    """y = ELU(v) rounded to 16 bits: (y, bound)."""
    y = torch.where(p.v > 0, p.v, torch.expm1(p.v))
    dy = p.dv + ELU_ABS * (p.v <= -2.0 ** -6).double() + ELU_REL * y.abs()
    return y, dy + C.E_OUT16[dt] * y.abs() + C.TAU16[dt]


def nearest_stored_to_ref(w, s, cout, cin, tap_shift=0):
    """The kernels' [3 * s * cout, cin] block -> [3, s, cout, cin] (tap o + 1, phase p).  tap_shift restates a kernel
    that reads phase tap o from the block of tap o + tap_shift (checker-sharpness test only)."""
    t = w.view(3, s, cout, cin)
    return torch.roll(t, shifts=tap_shift, dims=0) if tap_shift else t


def conv_nearest(x, wf, dt):
    """v = conv_same(upsample_nearest(x, s), W) through the stored fold wf [3, s, cout, cin] on exact operands
    (x [B, L, cin] float64), and its bound: a conv_ref.Pre over [B, L * s, cout]."""
    xt = x.transpose(1, 2)
    acc = nearest_conv_folded(xt, wf).transpose(1, 2)
    S = nearest_conv_folded(xt.abs(), wf.abs()).transpose(1, 2)
    n = 3 * x.shape[2] * (3 if dt == "fp16x3" else 1)
    dv = e_acc(n) * S + E_EPI * acc.abs() + (C.LO_LO * S if dt == "fp16x3" else 0)
    return C.Pre(acc, dv)
