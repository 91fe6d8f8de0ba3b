"""float64 reference of the fused GEMM epilogues (csrc/gemm.cuh) and a per-element error bound.

No GPU needed: every function runs on whatever device its tensors are on (the GPU tests keep the bench-size
products on the device, the checker-sharpness test runs on the CPU).

Bound.  For one output element
    |got - ref| <= (1 + e_out) * (e_acc * sens + e_epi * mag) + e_out * |ref| + tau
  e_acc = (ceil(K / 16) + 1) * 2^-22   two fp32 ulps per 16-deep tensor-core step (the tensor core truncates when it
                                       aligns an addend), relative to S = |A| |W|^T;
  sens                                 the epilogue's first-order sensitivity to its accumulator inputs, times S
                                       (elementwise: e.g. SwiGLU |silu(g)| S_a + |a| max|silu'| S_g, rotary
                                       |cos| S_a + |sin| S_b);
  e_out                                half an ulp of the output type: 2^-11 fp16, 2^-8 bf16, 2^-24 fp32;
  e_epi * mag                          the fp32 arithmetic of the epilogue itself (mag: the size of its terms);
  tau                                  an absolute floor for fp16 subnormals.
The rotary step is the oracle's own (oracle/dit_oracle.py).  The two load-time weight layouts of
csrc/dit.cu are restated here from their comments (ff_perm, qkv_head_perm), so a test builds a weight in reference
order and hands the kernel the stored (permuted) one.
"""
import math
from dataclasses import dataclass

import torch

from oracle.dit_oracle import apply_rotary, rotary_freqs

BLOCK_M, BLOCK_K = 128, 64
SILU_SLOPE_MAX = 1.0998           # max |silu'(x)| (at x ~ 2.4)
E_EPI = 2.0 ** -21
E_OUT = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8, "fp32": 2.0 ** -24}
TAU = {"fp16": 2.0 ** -24, "bf16": 1e-37, "fp32": 1e-37}
TORCH_DT = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}


def gemm_stages(bn, k_cols, stage_bytes=0):
    """Depth of the shared-memory ring of gemm_wgmma_kernel (GemmCfg::kStages in csrc/gemm.cuh)."""
    k_stage = BLOCK_M * BLOCK_K * 2 + bn * BLOCK_K * 2
    acc_stage = 2 * 64 * (k_cols + 4) * 4
    fixed = 1024 + 256 + 2 * acc_stage + 8 * stage_bytes
    return min(8, (227 * 1024 - fixed) // k_stage)


def e_acc(K):
    return (math.ceil(K / 16) + 1) * 2.0 ** -22


def accumulate(a16, w16):
    """acc = A W^T in float64 on the same 16-bit operands, and S = |A| |W|^T (the scale of its rounding error)."""
    a, w = a16.double(), w16.double()
    return a @ w.T, a.abs() @ w.abs().T


def round_to(x, out):
    """x (float64) rounded to the output type, back in float64: what a correct kernel may store."""
    return x.to(TORCH_DT[out]).double()


@dataclass
class Expect:
    ref: torch.Tensor     # float64 result of the epilogue on the exact accumulator
    sens: torch.Tensor    # first-order sensitivity to the accumulator, times S
    mag: torch.Tensor     # size of the terms of the epilogue's fp32 arithmetic


# ---------------------------------------------------------------------------------------------------- layouts
def ff_perm(ffi):
    """Stored row n of ff.0.proj (2 ffi rows) holds reference row perm[n]: every 64-row group is 32 value rows followed
    by their 32 gate rows."""
    n = torch.arange(2 * ffi)
    g, w = n // 64, n % 64
    return torch.where(w < 32, g * 32 + w, ffi + g * 32 + (w - 32))


def qkv_head_perm(D, dh, nf):
    """Stored row n of to_qkv (3 D rows) holds reference row perm[n]: inside each q and k head, stored position
    32 ci + i (i < 16) holds dim 16 ci + i and 32 ci + 16 + i its rotary partner 16 ci + i + nf, for the first
    clamp(nf - 16 ci, 0, 16) pairs of 32-column chunk ci; the dims from 2 nf up fill the remaining positions in
    order.  v rows are untouched."""
    within, nxt = [], 2 * nf
    for s in range(dh):
        ci, w = divmod(s, 32)
        i = w % 16
        if i < min(max(nf - 16 * ci, 0), 16):
            within.append(16 * ci + i + (nf if w >= 16 else 0))
        else:
            within.append(nxt)
            nxt += 1
    within = torch.tensor(within)
    n = torch.arange(3 * D)
    return torch.where(n < 2 * D, (n // dh) * dh + within[n % dh], n)


def rope_nf(head_dim):
    """Rotary pairs per head: max(head_dim / 2, 32) / 2 (models/transformer.py:737)."""
    return max(head_dim // 2, 32) // 2


def inv_freq(nf):
    dim = 2 * nf
    return 1.0 / (10000 ** (torch.arange(0, dim, 2).float() / dim))


def rope_tables(seq_len, nf):
    """cos / sin tables [seq_len, nf] (fp32, correctly rounded) of the oracle's fp32 angles; the angles themselves
    [seq_len, 2 nf] as rotary_freqs returns them."""
    freqs = rotary_freqs(seq_len, inv_freq(nf))
    f = freqs[:, :nf].double()
    return f.cos().float(), f.sin().float(), freqs


def row_freqs(freqs, rows, seq_len):
    """Angles of each output row: position = row % seq_len (the prepend token is position 0 of every item)."""
    return freqs[torch.arange(rows) % seq_len]


# ---------------------------------------------------------------------------------------------------- epilogues
def _act(x, act):
    if act == 0:
        return x, torch.ones_like(x), x.abs()
    sg = torch.sigmoid(x)
    y = x * sg
    return y, (sg * (1 + x * (1 - sg))).abs(), y.abs() * (x.abs() + 4)


def epi_store(acc, S, bias=None, act=0):
    """EpiStore32 (act 0, fp32 out) / EpiStore16: act(acc + bias)."""
    x = acc + (bias.double() if bias is not None else 0)
    y, slope, mag = _act(x, act)
    return Expect(y, slope * S, mag + acc.abs() + (bias.double().abs() if bias is not None else 0))


def _rotate(x, S, freqs_rows, head_dim, nf, rope_cols):
    """Partial rotary of every head below rope_cols (reference column order), with the oracle's apply_rotary.  The
    sensitivity of a rotated pair element is |cos| S_a + |sin| S_b."""
    M, N = x.shape
    nr = rope_cols // head_dim
    if nr == 0:
        return x, S, x.abs()
    heads = lambda t: t[:, :rope_cols].reshape(M, nr, head_dim).transpose(0, 1)
    unheads = lambda t: t.transpose(0, 1).reshape(M, rope_cols)
    y = unheads(apply_rotary(heads(x), freqs_rows))
    cos = freqs_rows[:, :nf].double().cos().abs()
    sin = freqs_rows[:, :nf].double().sin().abs()
    ang = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)
    h = heads(S)
    rot = h[..., :2 * nf]
    swap = torch.cat([rot[..., nf:], rot[..., :nf]], -1)
    s_rot = torch.cat([rot * ang[0] + swap * ang[1], h[..., 2 * nf:]], -1)
    hx = heads(x.abs())[..., :2 * nf]
    m_rot = torch.cat([hx * ang[0] + torch.cat([hx[..., nf:], hx[..., :nf]], -1) * ang[1], heads(x.abs())[..., 2 * nf:]], -1)
    cat = lambda a, b: torch.cat([unheads(a), b[:, rope_cols:]], 1)
    return torch.cat([y, x[:, rope_cols:]], 1), cat(s_rot, S), cat(m_rot, x.abs())


def epi_qkv_rope(acc, S, freqs_rows, head_dim, nf, rope_cols):
    """EpiQkvRope in reference column order (callers permute with qkv_head_perm): q | k heads rotated, v as is."""
    y, s, m = _rotate(acc, S, freqs_rows, head_dim, nf, rope_cols)
    return Expect(y, s, m)


def epi_head_norm(acc, S, norm_cols, rope_cols, freqs_rows=None, norm_width=64):
    """EpiHeadNorm16: F.normalize (eps 1e-12) of every 64-wide head below norm_cols, then rotary (nf 16) below
    rope_cols.  norm_width < 64 restates a wrong kernel (checker-sharpness test only)."""
    M, N = acc.shape
    nh = norm_cols // norm_width
    x = acc.clone()
    s = S.clone()
    if nh:
        h = acc[:, :norm_cols].reshape(M, nh, norm_width)
        hs = S[:, :norm_cols].reshape(M, nh, norm_width)
        nrm = h.norm(dim=-1, keepdim=True)
        y = h / nrm.clamp_min(1e-12)
        # d(x / |x|) = (dx - y (y . dx)) / |x|
        sn = (hs + y.abs() * (y.abs() * hs).sum(-1, keepdim=True)) / nrm.clamp_min(1e-12)
        sn = torch.where(nrm > 0, sn, torch.zeros_like(sn))
        x[:, :norm_cols] = y.reshape(M, norm_cols)
        s[:, :norm_cols] = sn.reshape(M, norm_cols)
    if rope_cols and freqs_rows is not None:
        y, s, m = _rotate(x, s, freqs_rows, 64, 16, rope_cols)
        return Expect(y, s, m)
    return Expect(x, s, x.abs())


def epi_swiglu(acc, S, bias=None):
    """EpiSwiglu in reference order: u = acc + bias, value = first half, gate = second half, value * silu(gate)."""
    u = acc + (bias.double() if bias is not None else 0)
    n = u.shape[1] // 2
    a, g = u[:, :n], u[:, n:]
    sg = torch.sigmoid(g)
    y = a * g * sg
    sens = (g * sg).abs() * S[:, :n] + a.abs() * SILU_SLOPE_MAX * S[:, n:]
    return Expect(y, sens, y.abs() * (g.abs() + 4) + a.abs() + g.abs())


def gate_rows(gate, rows, rows_per_item, n_items):
    """The adaLN gate row of every output row: item = (row / rows_per_item) % n_items."""
    return gate[(torch.arange(rows, device=gate.device) // rows_per_item) % n_items]


def epi_residual(acc, S, h_old, bias=None, gate=None):
    """EpiResidual: h + (acc + bias) * gate.  gate: per-row gate values [M, N] (gate_rows) or None."""
    v = acc + (bias.double() if bias is not None else 0)
    g = gate.double() if gate is not None else torch.ones_like(v)
    y = h_old.double() + v * g
    return Expect(y, g.abs() * S, (acc.abs() + (bias.double().abs() if bias is not None else 0)) * g.abs()
                  + h_old.double().abs() + y.abs())


# ---------------------------------------------------------------------------------------------------- checker
@dataclass
class Report:
    ratio: float          # largest |got - ref| / bound
    row: int
    col: int
    tile: tuple           # (m tile, n tile) of the kernel's 128 x BN grid
    got: float
    ref: float
    bound: float
    nonfinite: int        # valid elements that are NaN / inf

    @property
    def ok(self):
        return self.nonfinite == 0 and self.ratio <= 1.0

    def __str__(self):
        return (f"worst err/bound {self.ratio:.3g} at row {self.row} col {self.col} tile {self.tile}: got {self.got!r} "
                f"ref {self.ref!r} bound {self.bound:.3g}; non-finite {self.nonfinite}")


def check(got, exp, K, out, bn=256, col_scale=1):
    """Per-element check of a kernel output against Expect.  col_scale: output columns per tile column (SwiGLU's
    output has half the GEMM's columns: 2)."""
    got = got.double()
    bound = (1 + E_OUT[out]) * (e_acc(K) * exp.sens + E_EPI * exp.mag) + E_OUT[out] * exp.ref.abs() + TAU[out]
    err = (got - exp.ref).abs()
    finite = torch.isfinite(got)
    ratio = torch.where(finite, err / bound, torch.full_like(err, float("inf")))
    idx = int(torch.argmax(ratio))
    r, c = divmod(idx, got.shape[1])
    return Report(float(ratio.view(-1)[idx]), r, c, (r // BLOCK_M, c * col_scale // bn), float(got[r, c]),
                  float(exp.ref[r, c]), float(bound[r, c]), int((~finite).sum()))
