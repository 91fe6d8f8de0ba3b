"""float64 reference of the attention core (csrc/attention_tc.cu) and a per-element error bound.

Every function but run() (the kernels in their guarded operand layouts) runs on whatever device its tensors are on:
the GPU tests keep the 6145 x 6145 references on the device, one head at a time; the checker-sharpness test runs on
the CPU.

Reference.  o = softmax(q k^T / sqrt(d)) v in float64 on the kernel's own 16-bit operands; head h reads kv head
h / (H / Hkv).  With s_j = q . k_j, S_j = |q| . |k_j|, z_j = c s_j (c = log2(e) / sqrt(d), scaled log2 units, the
kernels' own), p_j = 2^(z_j - max z) / l, l = sum_j 2^(z_j - max z) >= 1:

    |got - ref| <= e_out |ref| + tau_out
                   + (1 + e_out) F [ sum_j p_j eta_j (|v_jc| + |o_c|)                              weights
                                     + (e_P + e_pv + e_l + 2^-23) sum_j p_j |v_jc|                  P V and l
                                     + tau_P sum_j |v_jc| / l ]                                     P underflow

Weights.  Both kernels compute P_j = exp2(z~_j - m) in fp32 and use the same P_j (and the same alpha) in the row sum
l and in O, so every error of the exponent or of exp2f is a perturbation w_j = p_j (1 + eta_j) of one key's weight,
consistent between numerator and denominator.  Then |o(w) - o| = |sum_j p_j eta_j (v_j - o)| / (1 + sum_j p_j eta_j),
which is at most the first term over (1 - max eta) (folded into F).  eta_j = 2^|dz_j| - 1 + e_w with
    |dz_j| <= c e_acc(d) S_j + 2^-21 (|z_j| + max_j |z_j|)
  c e_acc(d) S_j        the tensor-core accumulation of s over d (gemm_epilogue_ref.e_acc: 2 fp32 ulps per k16 step
                        relative to S);
  2^-21 (...)           the fp32 scale c: 1 / sqrtf(d), the fp32 log2(e) and their product round once each (4 ulps,
                        2^-22 relative, a relative error of every z: (|z_j| + max |z|) 2^-22 after the shift by the
                        max cancels the common part); s * c (attn_kernel) or fmaf(s, c, -m) (attn_wgmma_kernel) and
                        the subtraction of the running max round once each (2^-24 (|z_j| + |m|)); alpha =
                        exp2f(m_old - m_new) rounds its argument once per tile, and those arguments telescope to at
                        most 2 max |z| (2^-23 max |z|).  Together below 2^-21 (|z_j| + max |z|).
  e_w = (n_tiles + 1) 2^-22    exp2f: no fast-math flag; the SASS is MUFU.EX2 with a halving / squaring
                        wrapper for results below 2^-126 (the CUDA math documentation gives 2 ulps, 2^-22 relative).
                        One exp2f for P_j, one for each alpha that rescales it later (at most one per key tile).
P V and l.
  e_P = e_out           P is rounded to the operand type before P V (2^-11 fp16, 2^-8 bf16); l sums the unrounded
                        P, so this error does not cancel in the normalisation.
  e_pv = e_acc(Nk) + n_tiles 2^-24   P V accumulates over Nk keys in k16 tensor-core steps, plus one fp32 rounding of
                        O per rescale (one per key tile).
  e_l = (ceil(Nk / 4) + n_tiles + 2) 2^-24   the fp32 row sum: each thread adds its quarter of the row's P values one
                        by one (attn_kernel), or per tile and then fmaf(l, alpha, sum) once per tile (attn_wgmma_kernel);
                        then the 4-lane shuffle reduction (2 additions).
  2^-23                 1 / l and o * (1 / l), one rounding each.
P underflow.
  tau_P = 2^-25 (fp16)  the absolute rounding error of a P value in fp16's subnormal range; P is computed relative to
                        a running max <= the final one and only scaled down (alpha <= 1) afterwards, and l >= 1.
  tau_P = 2^-126 (bf16) exp2f results below fp32's normal range (bf16 has fp32's exponent range).
Output.  e_out, tau_out = gemm_epilogue_ref.E_OUT / TAU: the rounding of the normalised fp32 output.
Second order.  F = (1 + e_P)(1 + max eta) / (1 - max eta) per row covers the products of the first-order terms (the
P V and l errors are relative to the perturbed, rounded weights) and the 1 / (1 - max eta) above.

Every term is a product over keys ((p o eta) |V|, p |V|, a column sum of |V|), so no [Nq, Nk, d] tensor is formed.
"""
import ctypes
import math
from dataclasses import dataclass

import torch

from gemm_epilogue_ref import E_OUT, TAU, TORCH_DT, Report, e_acc

LOG2E = 1.4426950408889634
E_EXP = 2.0 ** -22
E_SCORE = 2.0 ** -21
TAU_P = {"fp16": 2.0 ** -25, "bf16": 2.0 ** -126}
DISTS = ("random", "flat", "flat_offset", "dominant", "max_last", "max_first", "large")
V_OFFSET = 24.0                   # flat_offset: common offset of V
K_PAD = 16384.0                   # finite value of the K padding rows of run()
PADL, PADC, PADR = 8, 24, 3


def query_tile(d):
    """Query rows per CTA: attn_wgmma_kernel (head dim 64) 128, attn_kernel 64."""
    return 128 if d == 64 else 64


def key_tile(d):
    return 128 if d == 64 else 64


# ---------------------------------------------------------------------------------------------------- inputs
@dataclass(frozen=True)
class Case:
    """One GPU input: layout ("self" fused QKV, "cross" q + fused KV, "dense" satb_attention_hd), head dim, operand
    type, shape.  The seed follows from the rest, so the CPU checker and the GPU test build the same tensors."""
    layout: str
    d: int
    dt: str
    B: int
    H: int
    Hkv: int
    Nq: int
    Nk: int

    @property
    def seed(self):
        return (self.d * 7919 + self.Nq * 104729 + self.Nk * 31 + self.B * 13 + self.H * 3 + self.Hkv
                + {"self": 0, "cross": 1, "dense": 2}[self.layout] * 1000003 + (self.dt == "bf16") * 500009) % (2 ** 31)

    def __str__(self):
        return f"{self.layout} d{self.d} {self.dt} B{self.B} H{self.H}/{self.Hkv} Nq{self.Nq} Nk{self.Nk}"


def inputs(case):
    """q [B, Nq, H d], k / v [B, Nk, Hkv d] in the operand type (CPU).  kv head hk (and the q heads that read it)
    carries score distribution DISTS[hk % 7], each aimed at one part of the online softmax:
      random       q, k ~ 1.5 N(0, 1), v ~ N(0, 1) (|z| a few log2 units)
      flat         q = 0: o is the mean of v, so a dropped or extra key shows as a bias
      flat_offset  the same with V_OFFSET added to v: an extra zero key pulls o towards 0
      dominant     q_i along k_j(i), z = 30 on that key, the others near 30 +- 4 sqrt(64 / d) below: fp16 P
                   subnormals and zeros
      max_last     small random scores, key Nk - 1 (the last partial tile) 6 log2 units above: a rescale on the last
                   turn, with the earlier keys still carrying weight
      max_first    keys 0 .. 7 (the first tile) 200 log2 units above the rest: every later tile underflows
      large        q, k ~ 25 N(0, 1): |z| in the thousands"""
    c = case
    g = torch.Generator().manual_seed(c.seed)
    d, grp = c.d, c.H // c.Hkv
    cl = LOG2E / math.sqrt(d)
    q = torch.empty(c.B, c.Nq, c.H, d)
    k = torch.empty(c.B, c.Nk, c.Hkv, d)
    v = torch.empty(c.B, c.Nk, c.Hkv, d)
    rows = torch.arange(c.Nq)
    for hk in range(c.Hkv):
        dist = DISTS[hk % len(DISTS)]
        kk = torch.randn(c.B, c.Nk, d, generator=g)
        vv = torch.randn(c.B, c.Nk, d, generator=g)
        for h in range(hk * grp, (hk + 1) * grp):
            qq = torch.randn(c.B, c.Nq, d, generator=g)
            if dist == "random":
                qq, kq = qq * 1.5, kk * 1.5
            elif dist in ("flat", "flat_offset"):
                qq, kq = torch.zeros_like(qq), kk
            elif dist == "dominant":
                kq = kk
                j = (rows * 7919 + 13 * h) % c.Nk
                kj = kk[:, j]                                           # [B, Nq, d]
                qq = kj * (30.0 / (cl * (kj * kj).sum(-1, keepdim=True)))
            elif dist in ("max_last", "max_first"):
                qq, kq = qq * 0.5, kk * 0.5
                qq[..., 0] = 4.0
                kq[..., 0] = 0.0
                if dist == "max_last":
                    kq[:, c.Nk - 1, 0] = 6.0 / (4.0 * cl)
                else:
                    kq[:, :8, 0] = 200.0 / (4.0 * cl)
            else:
                qq, kq = qq * 25.0, kk * 25.0
            q[:, :, h] = qq
        k[:, :, hk] = kq
        v[:, :, hk] = vv + (V_OFFSET if dist == "flat_offset" else 0.0)
    dt = TORCH_DT[c.dt]
    return (q.reshape(c.B, c.Nq, c.H * d).to(dt), k.reshape(c.B, c.Nk, c.Hkv * d).to(dt),
            v.reshape(c.B, c.Nk, c.Hkv * d).to(dt))


# ---------------------------------------------------------------------------------------------------- reference
@dataclass
class Expect:
    ref: torch.Tensor       # [B, Nq, H d] float64
    bound: torch.Tensor     # [B, Nq, H d] float64
    max_key: torch.Tensor   # [B, Nq, H] key index of the row maximum (for the report)
    d: int


def _heads(t, n, d):
    B, N = t.shape[:2]
    return t.view(B, N, n, d).permute(0, 2, 1, 3)                       # [B, n, N, d]


def _one_head(qh, kh, vh, d, dt):
    """ref, bound and the argmax key of one head: qh [Nq, d], kh / vh [Nk, d] float64."""
    Nk = kh.shape[0]
    nt = math.ceil(Nk / key_tile(d))
    cl = LOG2E / math.sqrt(d)
    e_p = E_OUT[dt]
    z = (qh @ kh.T).mul_(cl)
    zmax = z.amax(-1, keepdim=True)
    max_key = z.argmax(-1)
    za = z.abs()
    dz = (qh.abs() @ kh.abs().T).mul_(cl * e_acc(d))
    dz.add_(za.add_(za.amax(-1, keepdim=True)), alpha=E_SCORE)
    del za
    p = z.sub_(zmax).exp2_()
    l = p.sum(-1, keepdim=True)
    p.div_(l)
    o = p @ vh
    va = vh.abs()
    eta = dz.mul_(math.log(2.0)).expm1_().add_((nt + 1) * E_EXP)
    eta_max = eta.amax(-1, keepdim=True)
    assert float(eta_max.max()) < 0.5, "score error too large for the first-order bound"
    pe = eta.mul_(p)
    weights = pe @ va + pe.sum(-1, keepdim=True) * o.abs()
    del pe
    coef = e_p + e_acc(Nk) + nt * 2.0 ** -24 + (math.ceil(Nk / 4) + nt + 2) * 2.0 ** -24 + 2.0 ** -23
    inner = weights + coef * (p @ va) + TAU_P[dt] * va.sum(0, keepdim=True) / l
    F = (1 + e_p) * (1 + eta_max) / (1 - eta_max)
    bound = E_OUT[dt] * o.abs() + TAU[dt] + (1 + E_OUT[dt]) * F * inner
    return o, bound, max_key


def expect(q, k, v, H, Hkv, dt):
    """Reference and bound of softmax(q k^T / sqrt(d)) v: q [B, Nq, H d], k / v [B, Nk, Hkv d] 16-bit, any device."""
    B, Nq = q.shape[:2]
    d = q.shape[2] // H
    grp = H // Hkv
    qh, kh, vh = _heads(q.double(), H, d), _heads(k.double(), Hkv, d), _heads(v.double(), Hkv, d)
    ref = torch.empty(B, H, Nq, d, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(ref)
    max_key = torch.empty(B, H, Nq, dtype=torch.int64, device=q.device)
    for b in range(B):
        for h in range(H):
            ref[b, h], bound[b, h], max_key[b, h] = _one_head(qh[b, h], kh[b, h // grp], vh[b, h // grp], d, dt)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B, Nq, H * d)
    return Expect(flat(ref), flat(bound), max_key.permute(0, 2, 1), d)


def round_to(x, dt):
    return x.to(TORCH_DT[dt]).double()


# ---------------------------------------------------------------------------------------------------- checker
@dataclass
class AttnReport(Report):
    """Report with the place of the worst element: tile = (the row's CTA, the key tile of the row's maximum)."""
    item: int = 0
    head: int = 0

    def __str__(self):
        return (f"worst err/bound {self.ratio:.3g} at item {self.item} head {self.head} row {self.row} col {self.col} "
                f"(CTA {self.tile[0]}, max in key tile {self.tile[1]}): got {self.got!r} ref {self.ref!r} "
                f"bound {self.bound:.3g}; non-finite {self.nonfinite}")


def check(got, exp):
    """Per-element check of a kernel output [B, Nq, H d] against Expect."""
    got = got.double().to(exp.ref.device)
    err = (got - exp.ref).abs()
    finite = torch.isfinite(got)
    ratio = torch.where(finite, err / exp.bound, torch.full_like(err, float("inf")))
    idx = int(torch.argmax(ratio))
    B, Nq, W = got.shape
    b, rest = divmod(idx, Nq * W)
    r, col = divmod(rest, W)
    h, c = divmod(col, exp.d)
    tile = (r // query_tile(exp.d), int(exp.max_key[b, r, h]) // key_tile(exp.d))
    return AttnReport(float(ratio.view(-1)[idx]), r, c, tile, float(got[b, r, col]), float(exp.ref[b, r, col]),
                      float(exp.bound[b, r, col]), int((~finite).sum()), b, h)


# ---------------------------------------------------------------------------------------------------- emulation
def emulate(q, k, v, H, Hkv, dt, skip_rescale_tile=None):
    """float32 restatement of the kernels' online softmax (checker-sharpness test): key tiles of key_tile(d), the
    running max (from -1e30), alpha = exp2(m_old - m_new) applied to O and l, P = exp2(s c - m) in fp32 (one fmaf for
    head dim 64, s c rounded first otherwise), l summed over the unrounded P, P rounded to the operand type before
    P V, O / l rounded to the output.  skip_rescale_tile: a wrong kernel that leaves O unscaled on that tile."""
    B, Nq = q.shape[:2]
    d = q.shape[2] // H
    kt = key_tile(d)
    Nk = k.shape[1]
    f32 = torch.float32
    scale = torch.tensor(1.0 / math.sqrt(d), dtype=f32) * torch.tensor(LOG2E, dtype=f32)
    qh = _heads(q.float(), H, d)
    kh = _heads(k.float(), Hkv, d).repeat_interleave(H // Hkv, dim=1)
    vh = _heads(v.float(), Hkv, d).repeat_interleave(H // Hkv, dim=1)
    m = torch.full((B, H, Nq, 1), -1e30, dtype=f32)
    l = torch.zeros(B, H, Nq, 1, dtype=f32)
    o = torch.zeros(B, H, Nq, d, dtype=f32)
    for t in range(math.ceil(Nk / kt)):
        s = qh @ kh[:, :, t * kt:(t + 1) * kt].transpose(-1, -2)
        if d == 64:
            mn = torch.maximum(m, s.amax(-1, keepdim=True) * scale)
            p = torch.exp2((s.double() * scale.double() - mn.double()).float())
        else:
            zs = s * scale
            mn = torch.maximum(m, zs.amax(-1, keepdim=True))
            p = torch.exp2(zs - mn)
        alpha = torch.exp2(m - mn)
        m = mn
        l = l * alpha + p.sum(-1, keepdim=True)
        if t != skip_rescale_tile:
            o = o * alpha
        o = o + p.to(TORCH_DT[dt]).float() @ vh[:, :, t * kt:(t + 1) * kt]
    out = (o * (1.0 / l)).to(TORCH_DT[dt])
    return out.permute(0, 2, 1, 3).reshape(B, Nq, H * d)


# ---------------------------------------------------------------------------------------------------- layouts (GPU)
class _Padded:
    """A [B, N, width] operand inside a NaN-filled buffer: PADR rows before the first item and after the last, and
    with pad=True PADR rows between items and PADL / PADC columns before / after every row."""

    def __init__(self, B, N, width, dt, pad=True):
        gap = PADR if pad else 0
        self.padl = PADL if pad else 0
        self.ld = self.padl + width + (PADC if pad else 0)
        self.bs = (N + gap) * self.ld
        self.buf = torch.full((B * (N + gap) + 2 * PADR - gap, self.ld), float("nan"), dtype=TORCH_DT[dt],
                              device="cuda")
        self.view = self.buf.view(-1).as_strided((B, N, width), (self.bs, self.ld, 1), PADR * self.ld + self.padl)
        self.pad_rows = torch.ones(self.buf.shape[0], dtype=torch.bool, device="cuda")
        for b in range(B):
            self.pad_rows[PADR + b * (N + gap):PADR + b * (N + gap) + N] = False


def _launch(case, xq, xk, xv, o, cols):
    from stable_audio_tools import _native as nat
    c = case
    if c.layout == "dense":
        nat.check(nat.lib().satb_attention_hd(xq.view.data_ptr(), xk.view.data_ptr(), xv.view.data_ptr(),
                                              o.view.data_ptr(), c.B, c.H, c.Hkv, c.Nq, c.Nk, c.d,
                                              int(c.dt == "bf16"), nat.stream_ptr()))
        return
    p = nat.SatbAttentionProbe(B=c.B, H=c.H, Hkv=c.Hkv, Nq=c.Nq, Nk=c.Nk, head_dim=c.d, bf16=int(c.dt == "bf16"),
                               q=xq.view.data_ptr(), k=xk.view.data_ptr(), v=xv.view.data_ptr(), o=o.view.data_ptr(),
                               ldq=xq.ld, ldk=xk.ld, ldv=xv.ld, ldo=o.ld, q_bs=xq.bs, k_bs=xk.bs, v_bs=xv.bs,
                               o_bs=o.bs, q_cols=xq.view.shape[2], k_cols=xk.view.shape[2],
                               v_cols=xv.view.shape[2], q_col=cols[0], k_col=cols[1], v_col=cols[2])
    nat.check(nat.lib().satb_attention_probe(ctypes.byref(p), nat.stream_ptr()))


def run(case, q, k, v):
    """The kernel's output [B, Nq, H d] for case.layout (a view into its guarded buffer).  Every operand and the
    output sit inside NaN-filled guards (_Padded): for "self" and "cross" 8 columns before and 24 after the used ones
    and 3 rows before every item and after the last (batch stride (N + 3) ld); for "dense" 3 rows before the first
    item and after the last.  The K columns of those rows hold K_PAD instead (a K score is selected, not multiplied: a
    read of such a row moves the row max), so a read outside the operands shows as a non-finite or wrong output.
    Asserts that no element of the output buffer outside the output changed its bits."""
    c = case
    Hd, Kd = c.H * c.d, c.Hkv * c.d
    q, k, v = q.cuda(), k.cuda(), v.cuda()
    o = _Padded(c.B, c.Nq, Hd, c.dt, pad=c.layout != "dense")
    if c.layout == "self":
        assert c.H == c.Hkv and c.Nq == c.Nk
        x = _Padded(c.B, c.Nq, 3 * Hd, c.dt)
        x.view[..., :Hd], x.view[..., Hd:2 * Hd], x.view[..., 2 * Hd:] = q, k, v
        x.buf[x.pad_rows, x.padl + Hd:x.padl + 2 * Hd] = K_PAD
        ops, cols = (x, x, x), (0, Hd, 2 * Hd)
    elif c.layout == "cross":
        xq = _Padded(c.B, c.Nq, Hd, c.dt)
        xq.view.copy_(q)
        kv = _Padded(c.B, c.Nk, 2 * Kd, c.dt)
        kv.view[..., :Kd], kv.view[..., Kd:] = k, v
        kv.buf[kv.pad_rows, kv.padl:kv.padl + Kd] = K_PAD
        ops, cols = (xq, kv, kv), (0, 0, Kd)
    else:
        ops, cols = tuple(_Padded(c.B, t.shape[1], t.shape[2], c.dt, pad=False) for t in (q, k, v)), (0, 0, 0)
        for x, t in zip(ops, (q, k, v)):
            x.view.copy_(t)
        ops[1].buf[ops[1].pad_rows] = K_PAD
    before = o.buf.view(torch.int16).clone()
    _launch(c, *ops, o, cols)
    torch.cuda.synchronize()
    inside = torch.zeros(o.buf.shape, dtype=torch.bool, device="cuda")
    inside.view(-1).as_strided(o.view.shape, o.view.stride(), o.view.storage_offset()).fill_(True)
    changed = (o.buf.view(torch.int16) != before) & ~inside
    assert not changed.any(), f"{case}: {int(changed.sum())} elements written outside the output"
    return o.view
