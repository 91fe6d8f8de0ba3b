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


def attention(qkv16, bias_tab, lengths, H, dk, scale=1.0, bias_sign=1, q_block=64):
    """Per-item float64 attention of the packed [M, 3 H dk] operand: (o [M, H dk], P |v| and P (d_s |v - o|) terms).
    scale / bias_sign restate wrong kernels (checker-sharpness test only).  Evaluated one head at a time and the
    last term in blocks of q_block query rows, so that the largest temporary is [q_block, n, dk] (17 MB at n = 512,
    dk = 128) whatever H is: the whole [H, n, n, dk] difference tensor would be 34 GB at t5-11b's H = 128."""
    x = qkv16.double()
    inner = H * dk
    tab = bias_tab.double()
    o = torch.zeros(x.shape[0], inner, dtype=torch.float64, device=x.device)
    t1, t2 = torch.zeros_like(o), torch.zeros_like(o)
    r0 = 0
    for n in lengths:
        if n == 0:
            continue
        rows = x[r0:r0 + n]
        i = torch.arange(n, device=x.device)
        rel = ((bias_sign * (i[None, :] - i[:, None])) + (BIAS_SPAN // 2)).clamp(0, BIAS_SPAN - 1)
        for h in range(H):
            c = slice(h * dk, (h + 1) * dk)
            q, k, v = rows[:, c], rows[:, inner + h * dk:inner + (h + 1) * dk], rows[:, 2 * inner + h * dk:2 * inner + (h + 1) * dk]
            s = scale * (q @ k.T) + tab[h, rel]
            p = torch.softmax(s, dim=-1)
            oh = p @ v
            ds = (dk / 16 + 1) * 2.0 ** -22 * (q.abs() @ k.abs().T) + 2.0 ** -22 * s.abs()
            w = p * ds
            o[r0:r0 + n, c] = oh
            t1[r0:r0 + n, c] = p @ v.abs()
            for i0 in range(0, n, q_block):
                blk = slice(i0, min(i0 + q_block, n))
                t2[r0 + i0:r0 + blk.stop, c] = (w[blk, :, None] * (v[None, :, :] - oh[blk, None, :]).abs()).sum(1)
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


def gemm_operand(M, K, generator):
    """A GEMM's A operand [M, K] (fp32) in which one 64-wide k-block of every row, block m mod (K / 64) of row m, is
    max(1, K / 1024) times larger than the rest.  gemm_epilogue_ref's bound grows linearly in K, and at K = 65536 it
    is as large as one uniform k-block's share of S = |A| |W|^T, so on uniform data a kernel that dropped a k-block
    would pass.  Here every k-block holds about 1/16 of S in the rows where it is heavy, so a GEMM over all rows
    M >= K / 64 is checked against losing any one of them."""
    a = torch.randn(M, K, generator=generator)
    blocks = K // 64
    if blocks > 1:
        rows = torch.arange(M)
        cols = (rows % blocks)[:, None] * 64 + torch.arange(64)[None, :]
        a[rows[:, None], cols] *= max(1, K // 1024)
    return a


def both_16bit(x):
    """x rounded to bf16 values that fp16 holds exactly too (|x| < 2^-14 flushed to zero), in fp32: one set of
    operands, and so one float64 reference, for the fp16 and the bf16 instances of a GEMM."""
    x = x.to(torch.bfloat16).float()
    return torch.where(x.abs() < 2.0 ** -14, torch.zeros_like(x), x)


def auto_bn(M, N, sms):
    """The N tile t5_linear picks when none is given (csrc/linear.cuh auto_bn): 128 when N is a multiple of 128 and
    its fraction of the last wave of `sms` CTAs beats BN 256's by more than 10 %."""
    tiles = (M + R.BLOCK_M - 1) // R.BLOCK_M

    def eff(bn):
        waves = tiles * ((N + bn - 1) // bn) / sms
        return waves / math.ceil(waves)
    return 128 if N % 128 == 0 and eff(128) * 0.9 > eff(256) else 256


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def epi_relu(acc, S, out):
    """ReLU is 1-Lipschitz: sensitivity S everywhere.  Not (acc > 0) S: where the exact accumulator is a hair below
    zero, a correct kernel's fp32 one may lie a hair above it and store a small positive value."""
    y = acc.clamp_min(0)
    return R.Expect(_sat(y, out), S, acc.abs())


def epi_geglu(acc, S, out):
    """Reference column order: the first half of the columns is wi_1 x (value), the second wi_0 x (gate)."""
    n = acc.shape[1] // 2
    a, g = acc[:, :n], acc[:, n:]
    gl = gelu_new(g)
    y = a * gl
    sens = gl.abs() * S[:, :n] + a.abs() * GELU_SLOPE_MAX * S[:, n:]
    return R.Expect(_sat(y, out), sens, y.abs() * (g.abs() + 4) + a.abs() + g.abs())
