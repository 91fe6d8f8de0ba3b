"""float64 references of the T5 encoder's own kernels (csrc/t5.cu, the FF-in epilogues of csrc/gemm.cuh) and
per-element error bounds.  No GPU needed: every function runs on the device of its tensors.

RMSNorm:    |got - y| <= (e_out + 2^-20) |y| + tau          y = w (x rsqrt(mean(x^2) + eps)); 2^-20 covers rsqrtf
                                                             (2 ulp) and the fp32 sum of squares
Attention:  |got - o| <= e_out |o| + (e_p + 2^-20) (P |v|) + P (d_s |v - o|)
            o = softmax(q k^T + bias) v on the 16-bit operands; P the float64 probabilities; e_p half an ulp of the
            16-bit type the kernel rounds P to; d_s the fp32 error of a score: (d / 16 + 1) 2^-22 |q| |k| + 2^-22 |s|.
FF-in:      gemm_epilogue_ref.check with the Expect of epi_relu / epi_geglu below (fp16: saturated at +-65504).
"""
import math

import torch

import gemm_epilogue_ref as R

E_OUT = R.E_OUT
BIAS_SPAN = 1023          # relative positions -511 .. 511
GELU_SLOPE_MAX = 1.13     # max |gelu_new'(x)| (at x ~ 1.5)


def _sat(y, out):
    return y.clamp(-65504.0, 65504.0) if out == "fp16" else y


def rmsnorm(x, w, eps):
    x, w = x.double(), w.double()
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def check_rmsnorm(got, y, out):
    """(worst err / bound, number of non-finite outputs)."""
    got = got.double()
    ref = _sat(y, out)
    bound = (E_OUT[out] + 2.0 ** -20) * ref.abs() + R.TAU[out]
    ratio = (got - ref).abs() / bound
    return float(torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf"))).max()), \
        int((~torch.isfinite(got)).sum())


def attention(qkv16, bias_tab, lengths, H, dk, scale=1.0, bias_sign=1):
    """Per-item float64 attention of the packed [M, 3 H dk] operand: (o [M, H dk], P |v| and P (d_s |v - o|) terms).
    scale / bias_sign restate wrong kernels (checker-sharpness test only)."""
    x = qkv16.double()
    inner = H * dk
    o = torch.zeros(x.shape[0], inner, dtype=torch.float64, device=x.device)
    t1, t2 = torch.zeros_like(o), torch.zeros_like(o)
    r0 = 0
    for n in lengths:
        if n == 0:
            continue
        rows = x[r0:r0 + n]
        q = rows[:, :inner].view(n, H, dk).transpose(0, 1)
        k = rows[:, inner:2 * inner].view(n, H, dk).transpose(0, 1)
        v = rows[:, 2 * inner:].view(n, H, dk).transpose(0, 1)
        i = torch.arange(n, device=x.device)
        rel = (bias_sign * (i[None, :] - i[:, None])) + (BIAS_SPAN // 2)
        b = bias_tab.double()[:, rel.clamp(0, BIAS_SPAN - 1)]
        s = scale * (q @ k.transpose(1, 2)) + b
        p = torch.softmax(s, dim=-1)
        oh = p @ v
        ds = (dk / 16 + 1) * 2.0 ** -22 * (q.abs() @ k.abs().transpose(1, 2)) + 2.0 ** -22 * s.abs()
        dv = (v[:, None, :, :] - oh[:, :, None, :]).abs()                     # [H, n, n, dk]
        o[r0:r0 + n] = oh.transpose(0, 1).reshape(n, inner)
        t1[r0:r0 + n] = (p @ v.abs()).transpose(0, 1).reshape(n, inner)
        t2[r0:r0 + n] = ((p * ds)[..., None] * dv).sum(2).transpose(0, 1).reshape(n, inner)
        r0 += n
    return o, t1, t2


def check_attention(got, ref, out):
    """(worst err / bound, number of non-finite outputs) for the tuple `ref` of attention()."""
    o, t1, t2 = ref
    e_p = E_OUT[out]
    bound = E_OUT[out] * o.abs() + (e_p + 2.0 ** -20) * t1 + t2 + R.TAU[out]
    got = got.double()
    ratio = (got - o).abs() / bound
    return float(torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf"))).max()), \
        int((~torch.isfinite(got)).sum())


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def epi_relu(acc, S, out):
    y = acc.clamp_min(0)
    return R.Expect(_sat(y, out), (acc > 0).double() * S, acc.abs())


def epi_geglu(acc, S, out):
    """Reference column order: the first half of the columns is wi_1 x (value), the second wi_0 x (gate)."""
    n = acc.shape[1] // 2
    a, g = acc[:, :n], acc[:, n:]
    gl = gelu_new(g)
    y = a * gl
    sens = gl.abs() * S[:, :n] + a.abs() * GELU_SLOPE_MAX * S[:, n:]
    return R.Expect(_sat(y, out), sens, y.abs() * (g.abs() + 4) + a.abs() + g.abs())
