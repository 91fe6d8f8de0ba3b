"""float64 references of the DiT's small kernels (csrc/elementwise.cu, matmul_f64_kernel of csrc/conformer.cu) and a
per-element error bound for each, derived from the kernel's own arithmetic.

No GPU needed: every function is plain torch float64 and runs on whatever device its tensors are on (the GPU tests
keep the large cases on the device, tests/test_small_kernel_checker.py runs on the CPU).  Each function takes the
fp32 / 16-bit inputs the kernel takes and returns (ref, bound): the exact result in float64 and the largest error a
correct kernel can make, element by element.  `check` compares a kernel output with them; `check_bits` is for the
kernels that do one correctly rounded operation or none, whose output must be equal bit for bit.

Notation: u = 2^-24, the unit roundoff of fp32: one fp32 add / multiply / fma / divide / sqrtf has relative error
<= u.  expf, sinf, cosf and rsqrtf are within 2 ulp = 4 u (CUDA C Programming Guide, "Mathematical functions",
the accurate versions: what the library is built with, no -use_fast_math).  A sum of n fp32 terms added in a tree of
depth d has error <= d u sum |term| (first order).  E16 = 2^-11 (fp16) / 2^-8 (bf16): round-to-nearest of the 16-bit
output.  Second-order terms are dropped unless stated; the bounds are worst-case, so measured ratios sit well below 1.
"""
from dataclasses import dataclass

import torch

U = 2.0 ** -24
E16 = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}
TAU16 = {"fp16": 2.0 ** -24, "bf16": 2.0 ** -133}   # spacing of the 16-bit subnormals
DT16 = {"fp16": torch.float16, "bf16": torch.bfloat16}
SILU_SLOPE_MAX = 1.1
F32_TINY = 2.0 ** -126                               # below this an fp32 result may be a subnormal or 0
LN_EPS = 9.999999747378752e-06                       # 1e-5f, the kernel's constant


# ---------------------------------------------------------------------------------------------------- checker
@dataclass
class Report:
    ratio: float          # largest |got - ref| / bound (inf: a non-finite value where the reference is finite, a NaN
    index: tuple          # pattern that differs, or an error where the bound is 0)
    got: float
    ref: float
    bound: float
    nonfinite: int        # elements whose NaN / inf state differs from the reference's

    @property
    def ok(self):
        return self.nonfinite == 0 and self.ratio <= 1.0

    def __str__(self):
        return (f"worst err/bound {self.ratio:.3g} at {self.index}: got {self.got!r} ref {self.ref!r} "
                f"bound {self.bound:.3g}; non-finite mismatches {self.nonfinite}")


def check(got, ref, bound):
    """Per-element check.  Where the reference is NaN the output must be NaN, where it is +-inf the same inf; elsewhere
    it must be finite and within the bound (an exact match passes with any bound, 0 included)."""
    got, ref = got.double(), ref.double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    special = ~torch.isfinite(ref)
    same_special = (torch.isnan(ref) & torch.isnan(got)) | (got == ref)
    bad = torch.where(special, ~same_special, ~torch.isfinite(got))
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(special, torch.zeros_like(err), ratio)
    ratio = torch.where(bad | torch.isnan(ratio), torch.full_like(err, float("inf")), ratio)
    idx = int(torch.argmax(ratio))
    at = tuple(int(i) for i in torch.unravel_index(torch.tensor(idx), ref.shape)) if ref.dim() else ()
    pick = lambda t: float(t.reshape(-1)[idx])
    return Report(pick(ratio), at, pick(got), pick(ref), pick(bound), int(bad.sum()))


_INT_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def check_bits(got, ref):
    """Bit equality (so -0 != +0, and a NaN only equals the same NaN)."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (got.shape, ref.shape, got.dtype, ref.dtype)
    iv = _INT_VIEW[got.element_size()]
    diff = got.contiguous().view(iv) != ref.contiguous().view(iv)
    n = int(diff.sum())
    if n == 0:
        return Report(0.0, (), 0.0, 0.0, 0.0, 0)
    idx = int(torch.argmax(diff.reshape(-1).to(torch.uint8)))
    at = tuple(int(i) for i in torch.unravel_index(torch.tensor(idx), ref.shape))
    return Report(float("inf"), at, float(got.reshape(-1)[idx].float()), float(ref.reshape(-1)[idx].float()), 0.0, n)


def round16(x, out):
    """x (float64) rounded to the 16-bit output type: what a correct kernel may store."""
    return x.to(DT16[out])


# ---------------------------------------------------------------------------------------------------- LayerNorm
def item_of_row(rows, rows_per_item, n_items, device=None, shift=0):
    """The modulation vector of every row: item = (row / rows_per_item) % n_items (under CFG the unconditional rows
    wrap onto the conditional rows' vectors).  shift != 0 restates a kernel that takes a neighbour's vector."""
    return (torch.arange(rows, device=device) // rows_per_item + shift) % n_items


def layernorm_ref(x, gamma, beta=None, scale=None, shift=None, rows_per_item=1, n_items=1, out="fp16", item_shift=0):
    """layernorm_kernel: y = ((x - mean) rstd gamma (+ beta)) (* (1 + scale[item]) + shift[item]), rstd = (var + 1e-5f)^-1/2
    with the biased variance (models/transformer.py:188-206, adaLN :670-672 / :683-686), then the 16-bit rounding.
    x [rows, D] fp32, gamma / beta [D], scale / shift [n_items, D] (the vectors the kernel's pointer + item * mod_stride
    address).

    The kernel keeps a row in registers: D / 128 = nv float4 per lane.
      mean     each element passes 2 adds inside its float4, <= nv adds along the lane, 5 shuffle adds, one divide:
               |dmu| <= (nv + 8) u mean|x| =: delta.  This is the term that grows with the row mean.
      variance sum (x - mu^)^2 = sum (x - mu)^2 + D dmu^2 exactly; the subtraction, the square and the same tree add
               (nv + 12) u relative: |dv| <= delta^2 + (nv + 12) u (var + delta^2).
      rstd     relative error rho <= dv / (2 (var + eps)) + u (the + eps) + 4 u (rsqrtf).
      z        (x - mu^) rstd^ gamma + beta: |gamma| rstd delta + |z0| (rho + 3 u) + u |z|, z0 the value before beta.
               A variance-0 row has z0 = 0: it gives beta up to |gamma| rstd delta.
      adaLN    fl(1 + s), the product and the add: E_z |1 + s| + 2 u |z (1 + s)| + u |y|.
      output   (1 + E16) E_y + E16 |y| + the 16-bit subnormal spacing."""
    xd, g = x.double(), gamma.double()
    rows, D = xd.shape
    nv = D // 128
    mu = xd.mean(1, keepdim=True)
    xc = xd - mu
    var = (xc * xc).mean(1, keepdim=True)
    v = var + LN_EPS
    rstd = v.rsqrt()
    z0 = xc * rstd * g
    z = z0 + beta.double() if beta is not None else z0
    delta = (nv + 8) * U * xd.abs().mean(1, keepdim=True)
    dv = delta ** 2 + (nv + 12) * U * (var + delta ** 2)
    rho = 0.5 * dv / v + 5 * U
    err = g.abs() * rstd * delta + z0.abs() * (rho + 3 * U) + U * z.abs()
    y = z
    if scale is not None:
        item = item_of_row(rows, rows_per_item, n_items, xd.device, item_shift)
        s1, t = 1 + scale.double()[item], shift.double()[item]
        y = z * s1 + t
        err = err * s1.abs() + 2 * U * (z * s1).abs() + U * y.abs()
    return y, (1 + E16[out]) * err + E16[out] * y.abs() + TAU16[out]


# ---------------------------------------------------------------------------------------------------- timestep features
def fourier_ref(t, w):
    """fourier_kernel (models/blocks.py:95-97): out = [cos f | sin f], f = 2 pi t w.  The kernel forms f in fp32 as
    fl(fl(2pi_f32 t) w); its cosf / sinf are compared with float64 cos / sin of that same fp32 argument, so the bound
    holds only the functions' own error: 2 ulp of the result (<= 2 * 2^-23 |ref|) plus 2^-24 absolute for results
    near 0.  At |f| of tens of radians this tells the accurate functions from sin.approx / cos.approx (absolute error
    ~ 2^-21 |f|)."""
    two_pi = torch.tensor(6.283185307179586, dtype=torch.float32, device=t.device)
    f = ((two_pi * t.float())[:, None] * w.float()[None, :]).double()
    ref = torch.cat([f.cos(), f.sin()], 1)
    return ref, 2 * 2.0 ** -23 * ref.abs() + 2.0 ** -24


# ---------------------------------------------------------------------------------------------------- skinny linear
def skinny_linear_ref(x, W, bias=None, add=None, silu=False):
    """skinny_linear_kernel: out[r, n] = act(sum_k x[r, k] W[n, k] + bias[n] + add[r, n]), act = SiLU or identity
    (the timestep / global / prepend embedders, models/dit.py:41-81,149-161, and to_scale_shift_gate,
    models/transformer.py:648-651).  x [R, K], W [N, K] fp32.

    One warp per column: a lane chains K / 32 fma, the warp adds 32 partial sums in 5 steps, then the bias and the add:
    (K / 32 + 8) u sum_k |x w| covers the dot product (depth K / 32 + 5, and 3 to spare for the first-order model),
    u (|dot + bias| + |dot + bias + add|) the two adds.  SiLU x / (1 + expf(-x)): slope <= 1.1 on the input error, and
    4 u (expf) + u (add) + u (divide) <= 8 u |y| of its own; 1e-30 absolute where expf(-x) overflows and the kernel
    returns -0 for a value below 1e-36."""
    xd, wd = x.double(), W.double()
    K = xd.shape[1]
    acc, S = xd @ wd.T, xd.abs() @ wd.abs().T
    pre1 = acc + bias.double() if bias is not None else acc
    pre = pre1 + add.double() if add is not None else pre1
    err = (K / 32 + 8) * U * S + U * (pre1.abs() + pre.abs())
    if not silu:
        return pre, err + F32_TINY
    y = pre * torch.sigmoid(pre)
    return y, SILU_SLOPE_MAX * err + 8 * U * y.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------- prepend rows
def write_prepend_ref(tok, pre, pos, R, B, N_seq, D, Pp):
    """write_prepend_kernel: the Pp + 1 leading rows of every item of h [R, N_seq, D], as fp32 (bit-exact: at most one
    correctly rounded add).  Rows j < Pp: pre[r, j] for the conditional rows r < B, zeros for the unconditional CFG rows
    (models/dit.py:309-311) and without pre; row Pp: tok[r % B], the global-conditioning token, after the prepend
    tokens (models/dit.py:185-195); pos[j] added to row j (models/transformer.py:770-785)."""
    out = torch.zeros(R, Pp + 1, D, dtype=torch.float32, device=tok.device)
    if pre is not None and Pp > 0:
        out[:B, :Pp] = pre.view(B, Pp, D)
    out[:, Pp] = tok.view(B, D)[torch.arange(R, device=tok.device) % B]
    if pos is not None:
        out = out + pos.view(N_seq, D)[:Pp + 1]
    return out


# ---------------------------------------------------------------------------------------------------- adaLN gates
def gate_sigmoid_ref(ssg, depth, D, chunks=(2, 5)):
    """gate_sigmoid_kernel on ssg [rows, depth * 6 D]: chunks 2 and 5 of every 6 D-wide layer block become
    sigmoid(1 - g) (models/transformer.py:667,674,688); the other four chunks keep their bits.  Returns (ref, bound,
    changed): changed marks the transformed columns; elsewhere the bound is 0.

    a = fl(1 - g) has error u |a|, carried by sigmoid' = s (1 - s); 1 / (1 + expf(-a)) adds 4 u (expf) + u + u relative:
    u |a| s (1 - s) + 7 u s, and 2^-126 absolute where the result leaves the normal range (g >= 89 gives exactly 0)."""
    rows = ssg.shape[0]
    ref = ssg.double().clone().view(rows, depth, 6, D)
    bound = torch.zeros_like(ref)
    changed = torch.zeros_like(ref, dtype=torch.bool)
    for c in chunks:
        a = 1 - ref[:, :, c]
        s = torch.sigmoid(a)
        ref[:, :, c] = s
        bound[:, :, c] = U * a.abs() * s * (1 - s) + 7 * U * s + F32_TINY
        changed[:, :, c] = True
    flat = lambda t: t.view(rows, depth * 6 * D)
    return flat(ref), flat(bound), flat(changed)


# ---------------------------------------------------------------------------------------------------- DiT post
def dit_post_ref(y, B, C, L, N_seq, P, cfg, cfg_scale=1.0, scale_phi=0.0, unbiased=(True, True)):
    """dit_post_kernel: y [R * N_seq, ldy] fp32 token-major (R = 2 B with cfg, conditional rows first; ldy >= C, only the
    first C columns count) -> [B, C, L]: drop the P prepended rows (models/dit.py:219), cfg = u + (c - u) s, and with
    phi != 0 phi cfg std(c) / std(cfg) + (1 - phi) cfg, std unbiased over the channels (models/dit.py:338-347).  NaN
    where the reference formula gives NaN (0 / 0 standard deviations; one channel).  unbiased = (cond, cfg): False
    restates a kernel that divides that side's sum of squares by C.  (Dividing BOTH by C is the same function: the
    ratio of the two stds does not change, so no test can or should tell it apart.)

    No cfg: a copy, bound 0.  g = u + (c - u) s (an fma or two operations): E_g = 2 u |(c - u) s| + u |g|.
    Rescale, for each of the two stds: the mean (C sequential adds, a divide) is off by dm <= (C + 1) u mean|.| (+ mean
    E_g); sum (v - m^)^2 = V + C dm^2 for exact v, and for g^ = g + e at most V + 2 sqrt(V) eta + eta^2 with eta^2 =
    sum (E_g + dm)^2; the subtraction, square and C adds add (C + 3) u relative.  std = sqrtf(V / (C - 1)):
    |dstd| <= min(dV / ((C - 1) std), sqrt(dV / (C - 1))) + 2 u std.  ratio = std1 / std2: dstd1 / std2 + ratio dstd2 /
    (std2 - dstd2) + u ratio (infinite where dstd2 reaches std2: the kernel's result is then unconstrained, and the
    tests do not build such positions apart from the exact std-0 one).  out = phi (g ratio) + (1 - phi) g:
    E_g (phi ratio + |1 - phi|) + phi |g| dratio + 3 u (|phi g ratio| + |(1 - phi) g|) + u |out|."""
    f32 = lambda a: float(torch.tensor(a, dtype=torch.float32))
    s, phi = f32(cfg_scale), f32(scale_phi)
    R = 2 * B if cfg else B
    yd = y.double()[:, :C].reshape(R, N_seq, C)[:, P:P + L]          # [R, L, C]
    cv = yd[:B]
    if not cfg:
        return cv.transpose(1, 2).contiguous(), torch.zeros(B, C, L, dtype=torch.float64, device=y.device)
    uv = yd[B:]
    g = uv + (cv - uv) * s
    Eg = 2 * U * ((cv - uv) * s).abs() + U * g.abs()
    if phi == 0.0:
        return g.transpose(1, 2).contiguous(), (Eg + F32_TINY).transpose(1, 2).contiguous()

    def std_and_error(v, e, unbiased_side):
        div = C - 1 if unbiased_side else C
        m = v.mean(-1, keepdim=True)
        V = ((v - m) ** 2).sum(-1, keepdim=True)
        dm = (C + 1) * U * v.abs().mean(-1, keepdim=True) + e.mean(-1, keepdim=True)
        eta2 = ((e + dm) ** 2).sum(-1, keepdim=True)
        grow = 2 * V.sqrt() * eta2.sqrt() + eta2
        dV = grow + (C + 3) * U * (V + grow)
        std = (V / div).sqrt()                                        # 0 / 0 = NaN with one channel
        dstd = torch.minimum(dV / (div * std), (dV / div).sqrt()) + 2 * U * std
        return std, torch.where(std > 0, dstd, (dV / div).sqrt())

    s1, d1 = std_and_error(cv, torch.zeros_like(cv), unbiased[0])
    s2, d2 = std_and_error(g, Eg, unbiased[1])
    ratio = s1 / s2
    room = s2 - d2
    dratio = torch.where(room > 0, d1 / s2 + ratio * d2 / room + U * ratio, torch.full_like(ratio, float("inf")))
    out = phi * (g * ratio) + (1 - phi) * g
    err = (Eg * (phi * ratio + abs(1 - phi)) + phi * g.abs() * dratio
           + 3 * U * ((phi * g * ratio).abs() + ((1 - phi) * g).abs()) + U * out.abs() + F32_TINY)
    return out.transpose(1, 2).contiguous(), err.transpose(1, 2).contiguous()


# ---------------------------------------------------------------------------------------------------- weight prep
def cast_rows_ref(src, perm, cols, out):
    """cast_rows_kernel: dst[r, :cols] = 16-bit(src[perm[r], :cols]), round to nearest even, overflow to inf (fp16):
    torch's own cast.  Bit-exact."""
    rows = src if perm is None else src[perm.long()]
    return rows[:, :cols].to(DT16[out])


def quant_rows_fp8_ref(src, perm=None):
    """quant_rows_fp8_kernel: (e4m3 bytes [rows, cols] as uint8, row scales [rows] fp32) of src[perm] by the quantiser
    of tests/fp8_ref.py.  Bit-exact: the scale is a power of two picked by integer arithmetic on amax's bits, the
    scaling is exact, the e4m3 conversion is one round-to-nearest-even."""
    from fp8_ref import quantize_fp8_rows
    rows = src if perm is None else src[perm.long()]
    q, scale = quantize_fp8_rows(rows.float())
    return q.view(torch.uint8), scale[:, 0].contiguous()


def matmul_f64_ref(A, B):
    """matmul_f64_kernel: C = fp32(A B), fp64 fma chain over K.  The chain is off by <= K 2^-53 sum |a b|, the single
    rounding to fp32 by <= 2^-24 |C| (2^-149 in the subnormals): within one fp32 ulp of the rounded float64 product."""
    a, b = A.double(), B.double()
    ref = a @ b
    return ref, U * ref.abs() + A.shape[1] * 2.0 ** -53 * (a.abs() @ b.abs()) + 2.0 ** -149


# ---------------------------------------------------------------------------------------------------- sampler update
def sampler_update_ref(x, v, d1, d2, nz, c_skip, c_out, A, B, C, D, S, c_in_next):
    """sampler_update_kernel (inference/sampling.py:159,225-228 with k-diffusion's VDenoiser and DPM-Solver++ update):
    den = c_out v + c_skip x; x_next = A x + B den + C d1 + D d2 + S noise (null tensors skipped); x_in = x_next c_in.
    The scalars are the fp32 values the kernel receives.  Returns {name: (ref, bound)}.

    den = fma(c_out, v, fl(c_skip x)): u |c_skip x| + u |den|.  x_next starts as fma(A, x, fl(B den^)): |B| E_den +
    u |B den| + u |partial|, and every further fma adds u |partial|.  x_in: |c_in| E_next + u |x_in|."""
    f32 = lambda a: float(torch.tensor(a, dtype=torch.float32))
    c_skip, c_out, A, B, C, D, S, c_in_next = (f32(a) for a in (c_skip, c_out, A, B, C, D, S, c_in_next))
    xd, vd = x.double(), v.double()
    den = c_out * vd + c_skip * xd
    e_den = U * (c_skip * xd).abs() + U * den.abs()
    o = A * xd + B * den
    e = abs(B) * e_den + U * (B * den).abs() + U * o.abs()
    for coef, tns in ((C, d1), (D, d2), (S, nz)):
        if tns is not None:
            o = o + coef * tns.double()
            e = e + U * o.abs()
    x_in = o * c_in_next
    return {"den": (den, e_den + F32_TINY), "x_next": (o, e + F32_TINY),
            "x_in": (x_in, abs(c_in_next) * e + U * x_in.abs() + F32_TINY)}


# ---------------------------------------------------------------------------------------------------- SnakeBeta
def snake_beta_ref(x, alpha, beta, logscale=True):
    """snake_beta_kernel (models/blocks.py:318-319,350-358): y = x + sin^2(x a) / (b + 1e-9), a = e^alpha, b = e^beta
    per channel.  x [B, C, T].

    theta = x a with a = expf(alpha): 5 u |theta| (4 u expf, u the product), through d sin^2 = sin(2 theta) dtheta;
    sinf 4 u and the square u: 9 u s^2; 1 / (expf(beta) + 1e-9f): 6 u; the product with it u; the last add u |y|."""
    xd = x.double()
    a, b = alpha.double()[None, :, None], beta.double()[None, :, None]
    if logscale:
        a, b = a.exp(), b.exp()
    inv_b = 1.0 / (b + 1e-9)
    theta = xd * a
    s2 = theta.sin() ** 2
    y = xd + inv_b * s2
    err = inv_b * ((2 * theta).sin().abs() * 5 * U * theta.abs() + 9 * U * s2) + 7 * U * inv_b * s2 + U * y.abs()
    return y, err + F32_TINY
