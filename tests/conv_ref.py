"""float64 reference of one Oobleck VAE convolution step (csrc/oobleck.cu, csrc/conv_halo.cuh and EpiConv /
EpiStoreNCL of csrc/gemm.cuh) and a per-element error bound: the convolution counterpart of gemm_epilogue_ref.py,
whose accumulation bound, output roundings and report it reuses.

No GPU needed: every function runs on whatever device its tensors are on.  Activations are channels-last
[B, L, C] float64 holding the exact operands a kernel was given (16-bit values, hi + lo in fp16x3 mode); weights are
in the reference layout (Conv1d [cout, cin, k], ConvTranspose1d [cin, cout, k]).  Geometry and Snake follow
oracle/oobleck_oracle.py.

Bound.  For the pre-activation value v = conv + bias (+ skip), with S the same convolution of |A| and |W|:
    dv = e_acc(n) S + E_EPI (|acc| + |bias| + |skip|)      n = taps * K products (3 taps * K in fp16x3)
         + 2^-22 S                                        fp16x3: the dropped lo * lo product
Each output then adds its own terms:
    raw (un-activated) out       dv + E_OUT[raw] |v| + TAU
    Snake-activated 16-bit out   dv (1 + a ib) + ib 2 |sin(a v)| (2^-21 + |a v| 2^-23)   (the sin.approx error)
                                 + E_EPI (|v| + ib sin^2) + E_OUT |y| + TAU
    fused / two-launch unit      the inner snake2(conv7) value t is stored in 16 bits: its own bound dt (as above)
                                 enters the 1x1 conv as |W1| dt
    NCL fp32 out (final convs)   dv + 2^-22 |y| (tanhf, slope <= 1) + E_OUT["fp32"] |y|
    CUDA-core input conv         fp32 FMA chain of cin * k terms: (n + 1) 2^-24 (S + |bias|)
"""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from gemm_epilogue_ref import BLOCK_M, E_EPI, E_OUT, TAU, Report, e_acc
from oracle.oobleck_oracle import fold_weight_norm, snake_beta

OPERAND = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp16x3": torch.float16}
# half an ulp of what a 16-bit activation output holds: fp16x3 stores hi + fp16(y - hi), fp32-accurate up to the lo
# rounding (2^-11 of |lo| <= 2^-11 |y|) and the fp32 value it splits
E_OUT16 = {"fp16": E_OUT["fp16"], "bf16": E_OUT["bf16"], "fp16x3": 2.0 ** -22 + 2.0 ** -24}
TAU16 = {"fp16": TAU["fp16"], "bf16": TAU["bf16"], "fp16x3": TAU["fp16"]}
RAW = {"fp16": "fp16", "bf16": "fp32", "fp16x3": "fp32"}       # the raw skip stream's type per operand mode
RAW_DT = {"fp16": torch.float16, "fp32": torch.float32}
SIN_ABS, SIN_REL = 2.0 ** -21, 2.0 ** -23
LO_LO = 2.0 ** -22


# ---------------------------------------------------------------------------------------------------- operands
def split(x, dt):
    """x (any float) -> (hi, lo) as the kernels store it: hi = 16-bit(x), lo = fp16(x - hi) in fp16x3, else None."""
    x32 = x.float()
    hi = x32.to(OPERAND[dt])
    lo = (x32 - hi.float()).to(torch.float16) if dt == "fp16x3" else None
    return hi, lo


def value(hi, lo=None):
    """The exact float64 value of a 16-bit operand (hi + lo)."""
    return hi.double() + (lo.double() if lo is not None else 0)


def round16(x, dt):
    """x (float64) as a correct kernel may store it in a 16-bit activation output, back in float64."""
    return value(*split(x, dt))


def round_raw(x, raw):
    return x.to(RAW_DT[raw]).double()


# ---------------------------------------------------------------------------------------------------- weights
def fold(sd, pfx):
    """The weight-normed weight in float64 (oracle fold), reference layout."""
    return fold_weight_norm(sd[pfx + "weight_g"].double(), sd[pfx + "weight_v"].double())


def stored_to_ref(w, k, transposed, cin, cout, up=1, tap_flip=False):
    """The kernels' [tap][n][k] block -> reference layout.  Conv1d: row t * cout + co holds w[co, :, t].  ConvTranspose1d
    (2 taps over N = up * cout): row tap * up * cout + ph * cout + co holds w[:, co, ph + tap * up].  tap_flip restates
    a wrong read at ph + (1 - tap) * up (checker-sharpness test only)."""
    if not transposed:
        return w.view(k, cout, cin).permute(1, 2, 0)
    t = w.view(2, up, cout, cin)
    if tap_flip:
        t = t.flip(0)
    return t.permute(3, 2, 0, 1).reshape(cin, cout, 2 * up)


def ref_to_stored(w, k, transposed, cin, cout, up=1):
    """Inverse of stored_to_ref: the [tap * n, cin] block a correct load-time fold writes."""
    if not transposed:
        return w.permute(2, 0, 1).reshape(k * cout, cin)
    return w.view(cin, cout, 2, up).permute(2, 3, 1, 0).reshape(2 * up * cout, cin)


# ---------------------------------------------------------------------------------------------------- convolution
def _conv(x, w, kind, dil=1, s=1):
    """x [B, L, Cin] -> [B, L_out, Cout] with the oracle's geometry: "conv" (k taps, dilation, same padding),
    "up" (ConvTranspose1d k = 2s, stride s, padding ceil(s/2)), "down" (Conv1d k = 2s, stride s, padding ceil(s/2))."""
    xt = x.transpose(1, 2)
    k = w.shape[2]
    if kind == "conv":
        y = F.conv1d(xt, w, padding=dil * (k - 1) // 2, dilation=dil)
    elif kind == "up":
        y = F.conv_transpose1d(xt, w, stride=s, padding=math.ceil(s / 2))
    else:
        y = F.conv1d(xt, w, stride=s, padding=math.ceil(s / 2))
    return y.transpose(1, 2)


@dataclass
class Pre:
    v: torch.Tensor      # float64 pre-activation value
    dv: torch.Tensor     # its error bound


def conv(x, w, dt, kind="conv", bias=None, skip=None, dil=1, s=1):
    """v = conv(x, w) + bias (+ skip) on exact operands, and its bound for a tensor-core conv in operand mode dt."""
    acc = _conv(x, w, kind, dil, s)
    S = _conv(x.abs(), w.abs(), kind, dil, s)
    taps = w.shape[2] if kind != "up" else 2
    n = taps * x.shape[2] * (3 if dt == "fp16x3" else 1)
    b = bias.double() if bias is not None else torch.zeros(w.shape[1 if kind == "up" else 0], dtype=x.dtype, device=x.device)
    sk = skip.double() if skip is not None else torch.zeros_like(acc)
    v = acc + b + sk
    dv = e_acc(n) * S + E_EPI * (acc.abs() + b.abs() + sk.abs()) + (LO_LO * S if dt == "fp16x3" else 0)
    return Pre(v, dv)


def conv_in(audio, w32, bias):
    """The encoder's CUDA-core input conv (fp32 FMA): audio NCL [B, cin, T] fp32, w32 [cout, cin, k]."""
    a, w = audio.double(), w32.double()
    k = w.shape[2]
    acc = F.conv1d(a, w, padding=(k - 1) // 2).transpose(1, 2)
    S = F.conv1d(a.abs(), w.abs(), padding=(k - 1) // 2).transpose(1, 2)
    b = bias.double()
    return Pre(acc + b, (w.shape[1] * k + 1) * 2.0 ** -24 * (S + b.abs()))


def _ab(alpha, beta):
    return alpha.double().exp(), 1.0 / (beta.double().exp() + 1e-9)


def snake(p, alpha, beta, dt, exp_alpha=True):
    """y = snake(v) (oracle snake_beta, per channel) rounded to 16 bits: (y, bound).  exp_alpha=False restates a
    kernel that uses alpha itself as the frequency (checker-sharpness test only)."""
    if not exp_alpha:
        alpha = alpha.double().abs().log()        # sin^2 is even: a = |alpha| is a = alpha
    y = snake_beta(p.v.transpose(1, 2), alpha.double(), beta.double()).transpose(1, 2)
    a, ib = _ab(alpha, beta)
    av = p.v * a
    sn = torch.sin(av)
    dy = (p.dv * (1 + a * ib) + ib * 2 * sn.abs() * (SIN_ABS + av.abs() * SIN_REL)
          + E_EPI * (p.v.abs() + ib * sn * sn))
    return y, dy + E_OUT16[dt] * y.abs() + TAU16[dt]


def raw(p, dt):
    """The raw (un-activated) stream output: (v, bound)."""
    r = RAW[dt]
    return p.v, p.dv + E_OUT[r] * p.v.abs() + TAU[r]


def ncl_out(p, tanh=False):
    """The final convs' fp32 output (optional tanh): (y, bound)."""
    y = torch.tanh(p.v) if tanh else p.v
    return y, p.dv + (2.0 ** -22 * y.abs() if tanh else 0) + E_OUT["fp32"] * y.abs() + TAU["fp32"]


def residual_unit(x, skip, w7, b7, alpha2, beta2, w1, b1, dil, dt, inner_bias=True):
    """ResidualUnit (oracle residual_unit, from its snake1 output x on): v = skip + conv1(snake2(conv7_dil(x) + b7)) + b1.
    The kernel rounds the inner value t to 16 bits; its bound dt enters through |W1| dt.  inner_bias=False drops b7
    (checker-sharpness test only)."""
    p7 = conv(x, w7, dt, bias=b7 if inner_bias else None, dil=dil)
    t, dt_ = snake(p7, alpha2, beta2, dt)
    p = conv(t, w1, dt, bias=b1, skip=skip)
    return Pre(p.v, p.dv + _conv(dt_, w1.abs(), "conv"))


# ---------------------------------------------------------------------------------------------------- checker
@dataclass
class ConvReport(Report):
    item: int = 0
    pos: int = 0

    def __str__(self):
        return (f"worst err/bound {self.ratio:.3g} at item {self.item} pos {self.pos} ch {self.col} (m tile "
                f"{self.tile[0]}, n tile {self.tile[1]}): got {self.got!r} ref {self.ref!r} bound {self.bound:.3g}; "
                f"non-finite {self.nonfinite}")


def check(got, ref, bound, bn=64, up=1, pad=0):
    """Per-element check of a [B, L, C] output.  The worst element is reported as (item, position, channel) with the
    GEMM tile that wrote it: the 128-position m tile (over input positions l = (pos + pad) / up for a transposed conv,
    whose column is phase * C + channel) and the BN-wide n tile."""
    got = got.double()
    err = (got - ref).abs()
    finite = torch.isfinite(got)
    ratio = torch.where(finite, err / bound, torch.full_like(err, float("inf")))
    idx = int(torch.argmax(ratio))
    B, L, C = got.shape
    b, rem = divmod(idx, L * C)
    pos, ch = divmod(rem, C)
    l, ph = divmod(pos + pad, up) if up > 1 else (pos, 0)
    return ConvReport(float(ratio[b, pos, ch]), b * L + pos, ch, (l // BLOCK_M, (ph * C + ch) // bn),
                      float(got[b, pos, ch]), float(ref[b, pos, ch]), float(bound[b, pos, ch]),
                      int((~finite).sum()), b, pos)
