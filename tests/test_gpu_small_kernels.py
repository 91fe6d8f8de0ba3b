"""GPU: the DiT's small kernels (csrc/elementwise.cu, matmul_f64_kernel) against the float64 references and derived
bounds of tests/small_kernel_ref.py, element by element, each through the launch function the forward calls
(include/satb200.h: satb_layernorm_mod, satb_*_probe, satb_sampler_update, satb_snake_beta).

Every output buffer has a guard band of NaN (0xAB bytes for e4m3) before and after it and is itself pre-filled the same
way: after the call the guards must be intact and every element the kernel owns finite unless the reference says
NaN.  Kernels that do one correctly rounded operation or none (write_prepend, cast_rows, quant_rows_fp8, the untouched
chunks of gate_sigmoid, dit_post without CFG) are compared bit for bit, buffer and guards at once.  The references run
in float64 on the device the inputs are on.  One `SMALLK {json}` line per case (pytest -s) with the worst err / bound."""
import json

import pytest
import torch

import small_kernel_ref as sk

pytestmark = pytest.mark.gpu

GUARD = 64          # elements on each side (a multiple of 16 bytes for every element size)
DEV = "cuda"


def report(kernel, rep=None, **kw):
    if rep is not None:
        kw.update(max_err_over_bound=rep.ratio, nonfinite=rep.nonfinite)
    print("SMALLK " + json.dumps(dict(kernel=kernel, **kw)), flush=True)


def nat():
    from stable_audio_tools import _native
    return _native


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, g, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


class Guarded:
    """A device buffer of `shape` between two guard bands, all of it pre-filled with NaN (0xAB for 1-byte types)."""

    def __init__(self, shape, dtype=torch.float32, fill=None):
        n = 1
        for s in shape:
            n *= s
        self.n, self.dtype = n, dtype
        if dtype == torch.uint8:
            self.buf = torch.full((n + 2 * GUARD,), 0xAB, dtype=dtype, device=DEV)
        else:
            self.buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device=DEV)
        self.view = self.buf[GUARD:GUARD + n].view(*shape)
        if fill is not None:
            self.view.copy_(fill)
        self.before = self.buf.clone()

    def ptr(self):
        return self.view.data_ptr()

    def guards_intact(self):
        iv = sk._INT_VIEW[self.buf.element_size()]
        a, b = self.buf.view(iv), self.before.view(iv)
        return bool(torch.equal(a[:GUARD], b[:GUARD]) and torch.equal(a[GUARD + self.n:], b[GUARD + self.n:]))


def call(fn, *args):
    n = nat()
    n.check(fn(*args, n.stream_ptr()))
    torch.cuda.synchronize()


def p(t):
    return t.data_ptr() if t is not None else None


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_rows(rows, D, g, offset):
    """Row r holds pattern (r + offset) % 8: N(0, 1); mean 4, 16, 1000 sigma; a constant; 1e-6-sized values (variance far
    below eps); one 1e4 outlier; N(0.5, 3)."""
    x = randn(rows, D, g=g)
    k = (torch.arange(rows, device=DEV) + offset) % 8
    x[k == 1] += 4.0
    x[k == 2] += 16.0
    x[k == 3] += 1000.0
    x[k == 4] = 2.5                       # every partial sum of equal 2.5s is exact: the kernel's mean is 2.5, z0 = 0
    x[k == 5] *= 1e-6
    r6 = torch.nonzero(k == 6).flatten()
    x[r6, r6 % D] = 1e4
    x[k == 7] = x[k == 7] * 3 + 0.5
    return x, k


def _ln_operands(D, g):
    return 1 + 0.3 * randn(D, g=g), 0.2 * randn(D, g=g)


@pytest.mark.parametrize("D", list(range(128, 2049, 128)))
def test_layernorm_every_width_vs_fp64(D):
    """All four register-array instances (NV 4 / 8 / 12 / 16) and every partial fill of each; a single row, the ragged
    last block (rows % 4 = 1, 3), one full block, and the forward's row counts; both output types, beta given and null."""
    g = gen(D)
    gamma, beta = _ln_operands(D, g)
    for i, rows in enumerate([1, 3, 4, 5, 1025, 8200]):
        x, k = _ln_rows(rows, D, g, offset=D // 128 + i)
        for bf16 in (0, 1):
            out = "bf16" if bf16 else "fp16"
            b = beta if (i + bf16) % 2 == 0 else None
            o = Guarded((rows, D), sk.DT16[out])
            call(nat().lib().satb_layernorm_mod, p(x), p(gamma), p(b), None, None, 0, 1, 1, o.ptr(), rows, D, bf16)
            y, bound = sk.layernorm_ref(x, gamma, b, out=out)
            rep = sk.check(o.view, y, bound)
            report("layernorm", rep, D=D, rows=rows, out=out, beta=b is not None)
            assert o.guards_intact() and rep.ok, str(rep)
            const = k == 4
            if const.any():             # variance 0: beta (0 without) up to the 16-bit rounding, nothing else
                want = (b if b is not None else torch.zeros_like(gamma)).to(sk.DT16[out]).expand(int(const.sum()), D)
                assert torch.equal(o.view[const], want)


MOD_CASES = [  # D, N_seq, B, bf16, beta
    (256, 1, 1, 0, 1), (256, 33, 3, 1, 0), (896, 1025, 4, 0, 1), (1152, 33, 1, 0, 1), (1536, 1025, 4, 0, 1),
    (1536, 33, 3, 1, 1), (1536, 1, 4, 0, 0), (2048, 1025, 3, 1, 1), (2048, 33, 4, 0, 0), (640, 1, 3, 1, 1)]


@pytest.mark.parametrize("D,N_seq,B,bf16,with_beta", MOD_CASES)
def test_layernorm_adaln_modulation_vs_fp64(D, N_seq, B, bf16, with_beta):
    """rows = 2 B N_seq as under CFG: the unconditional rows wrap onto the conditional rows' vectors.  The vectors sit
    where the forward keeps them: one [depth * 6 D] row per item, scale_ff / shift_ff of layer 1 at + 6 D + 3 D / + 4 D,
    NaN everywhere else in that buffer, the rows of B more items included."""
    g = gen(D + N_seq + B)
    depth, out = 3, "bf16" if bf16 else "fp16"
    rows, stride = 2 * B * N_seq, depth * 6 * D
    gamma, beta = _ln_operands(D, g)
    beta = beta if with_beta else None
    x, _ = _ln_rows(rows, D, g, offset=N_seq)
    ssg = torch.full((2 * B, stride), float("nan"), device=DEV)      # rows B ..: what a kernel that does not wrap reads
    ssg[:B, 9 * D:10 * D] = randn(B, D, g=g, scale=0.5)
    ssg[:B, 10 * D:11 * D] = randn(B, D, g=g)
    o = Guarded((rows, D), sk.DT16[out])
    call(nat().lib().satb_layernorm_mod, p(x), p(gamma), p(beta), ssg.data_ptr() + 9 * D * 4, ssg.data_ptr() + 10 * D * 4,
         stride, N_seq, B, o.ptr(), rows, D, bf16)
    scale, shift = ssg[:B, 9 * D:10 * D], ssg[:B, 10 * D:11 * D]
    y, bound = sk.layernorm_ref(x, gamma, beta, scale, shift, N_seq, B, out)
    rep = sk.check(o.view, y, bound)
    report("layernorm_mod", rep, D=D, N_seq=N_seq, B=B, out=out, beta=with_beta)
    assert o.guards_intact() and rep.ok, str(rep)
    if B > 1:   # the checker is sharp on the kernel's real output: a neighbour's vector is far outside
        shifted = sk.check(o.view, *sk.layernorm_ref(x, gamma, beta, scale, shift, N_seq, B, out, item_shift=1))
        report("layernorm_mod_shifted_reference", shifted, D=D, N_seq=N_seq, B=B)
        assert not shifted.ok and shifted.ratio > 100


# ------------------------------------------------------------------------------------------------ fourier
@pytest.mark.parametrize("B", [1, 8, 16])
@pytest.mark.parametrize("F", [3, 128])
@pytest.mark.parametrize("wscale", [1.0, 16.0])
def test_fourier_features_vs_fp64(B, F, wscale):
    """wscale 16: |2 pi t w| reaches ~100 rad and beyond, where an approximate sine would be off by 1e-5."""
    g = gen(B * 1000 + F)
    ts = torch.tensor([0.0, 1e-4, 0.5, 0.9365, 1.0], device=DEV)
    t = ts[(torch.arange(B, device=DEV) + 3) % 5].contiguous()
    w = randn(F, g=g, scale=wscale)
    o = Guarded((B, 2 * F))
    call(nat().lib().satb_fourier_probe, p(t), p(w), o.ptr(), B, F)
    ref, bound = sk.fourier_ref(t, w)
    rep = sk.check(o.view, ref, bound)
    report("fourier", rep, B=B, F=F, wscale=wscale, max_abs_arg=float((2 * torch.pi * t[:, None] * w[None]).abs().max()))
    assert o.guards_intact() and rep.ok, str(rep)
    assert torch.equal(o.view[t == 0][:, :F], torch.ones_like(o.view[t == 0][:, :F]))      # [cos | sin], t = 0: 1 | 0
    assert not sk.check(torch.cat([o.view[:, F:], o.view[:, :F]], 1), ref, bound).ok


# ------------------------------------------------------------------------------------------------ skinny linear
ALL8 = [(b, a, s) for b in (0, 1) for a in (0, 1) for s in (0, 1)]
SKINNY_SHAPES = [(1, 4, 1), (7, 128, 7), (8, 256, 8), (17, 768, 1536), (130, 1536, 9), (4096, 128, 9), (8, 1536, 9216),
                 (2, 2048, 1536), (3, 4096, 7), (5, 6400, 8), (16, 2052, 1536), (130, 6400, 1536)]
SKINNY_CASES = ([(9, 2052, 9) + c for c in ALL8] + [(9, 1536, 9) + c for c in ALL8]
                + [s + ALL8[(3 * i + 1) % 8] for i, s in enumerate(SKINNY_SHAPES)])


@pytest.mark.parametrize("R,K,N,bias,add,silu", SKINNY_CASES)
def test_skinny_linear_vs_fp64(R, K, N, bias, add, silu):
    """K <= 2048: the weights-in-registers pass; above: the fallback loop.  R > 8: several 8-row passes, the last one
    ragged.  N % 8 != 0: warps without a column."""
    g = gen(R + K + N)
    x, W = randn(R, K, g=g), randn(N, K, g=g, scale=K ** -0.5)
    b = randn(N, g=g) if bias else None
    a = randn(R, N, g=g) if add else None
    o = Guarded((R, N))
    call(nat().lib().satb_skinny_linear_probe, p(x), p(W), p(b), p(a), o.ptr(), R, K, N, silu)
    ref, bound = sk.skinny_linear_ref(x, W, b, a, bool(silu))
    rep = sk.check(o.view, ref, bound)
    report("skinny_linear", rep, R=R, K=K, N=N, bias=bias, add=add, silu=silu)
    assert o.guards_intact() and rep.ok, str(rep)
    if R > 1:
        assert not sk.check(torch.roll(o.view, 1, 0), ref, bound).ok


# ------------------------------------------------------------------------------------------------ prepend rows
@pytest.mark.parametrize("D", [256, 1536, 2048])
@pytest.mark.parametrize("B,Pp,with_pre,with_pos,cfg", [(1, 0, 0, 0, 1), (1, 1, 1, 1, 1), (3, 4, 1, 1, 1), (3, 4, 0, 1, 1),
                                                         (3, 1, 1, 0, 1), (1, 4, 1, 0, 0), (3, 0, 0, 1, 0)])
def test_write_prepend_bits(D, B, Pp, with_pre, with_pos, cfg):
    g = gen(D + B + Pp)
    R, N_seq = (2 * B if cfg else B), Pp + 1 + 5
    tok = randn(B, D, g=g)
    pre = randn(B, Pp, D, g=g) if with_pre and Pp else None
    pos = randn(N_seq, D, g=g) if with_pos else None
    h = Guarded((R, N_seq, D), fill=torch.full((R, N_seq, D), 7.25, device=DEV))
    call(nat().lib().satb_write_prepend_probe, p(tok), p(pre), p(pos), h.ptr(), R, B, N_seq, D, Pp)
    want = h.before.clone()
    want[GUARD:GUARD + h.n].view(R, N_seq, D)[:, :Pp + 1] = sk.write_prepend_ref(tok, pre, pos, R, B, N_seq, D, Pp)
    rep = sk.check_bits(h.buf, want)        # the rows past Pp keep their sentinel, the guards their NaN
    report("write_prepend", rep, D=D, B=B, R=R, Pp=Pp, pre=pre is not None, pos=with_pos)
    assert rep.ok, str(rep)
    if cfg and Pp:                          # the unconditional rows' prepend tokens are zeros (+ the position row)
        zero = pos[:Pp].expand(B, Pp, D) if pos is not None else torch.zeros(B, Pp, D, device=DEV)
        assert torch.equal(h.view[B:, :Pp], zero)


# ------------------------------------------------------------------------------------------------ gates
@pytest.mark.parametrize("depth", [1, 24])
@pytest.mark.parametrize("D", [128, 1536])
@pytest.mark.parametrize("rows", [1, 4])
def test_gate_sigmoid_vs_fp64_and_untouched_bits(depth, D, rows):
    g = gen(depth + D + rows)
    src = randn(rows, depth * 6 * D, g=g, scale=3.0)
    src.view(rows, depth, 6, D)[0, 0, 2, :4] = torch.tensor([100.0, -100.0, 1e4, -1e4], device=DEV)
    src.view(rows, depth, 6, D)[-1, -1, 5, -4:] = torch.tensor([-1e4, 1e4, -100.0, 100.0], device=DEV)
    o = Guarded(tuple(src.shape), fill=src)
    call(nat().lib().satb_gate_sigmoid_probe, o.ptr(), rows, depth, D)
    ref, bound, changed = sk.gate_sigmoid_ref(src, depth, D)
    rep = sk.check(o.view, ref, bound)
    kept = sk.check_bits(torch.where(changed, torch.zeros_like(src), o.view), torch.where(changed, torch.zeros_like(src), src))
    report("gate_sigmoid", rep, depth=depth, D=D, rows=rows, untouched_bits_equal=kept.ok)
    assert o.guards_intact() and rep.ok and kept.ok, f"{rep}; untouched: {kept}"
    assert o.view.view(rows, depth, 6, D)[0, 0, 2, :4].tolist() == [0.0, 1.0, 0.0, 1.0]
    assert not sk.check(o.view, *sk.gate_sigmoid_ref(src, depth, D, chunks=(1, 5))[:2]).ok


# ------------------------------------------------------------------------------------------------ DiT post
POST_CASES = [  # B, C, L, P, cfg, cfg_scale, phi
    (1, 1, 1, 0, 0, 1.0, 0.0), (1, 1, 127, 5, 1, 4.0, 0.0), (2, 1, 128, 1, 1, 4.0, 0.5), (3, 2, 129, 0, 1, 1.0, 1.0),
    (2, 3, 1024, 5, 1, 7.0, 0.5), (2, 16, 1, 1, 1, 4.0, 1.0), (1, 40, 127, 1, 1, 4.0, 0.5), (2, 40, 129, 5, 0, 1.0, 0.0),
    (2, 64, 1024, 1, 1, 4.0, 0.0), (3, 16, 128, 0, 1, 7.0, 1.0), (2, 64, 6144, 1, 1, 7.0, 0.5), (1, 64, 6144, 1, 0, 1.0, 0.0),
    (2, 3, 129, 1, 1, 1.0, 0.5), (1, 2, 1024, 0, 1, 7.0, 0.0)]


@pytest.mark.parametrize("B,C,L,P,cfg,cfg_scale,phi", POST_CASES)
def test_dit_post_vs_fp64(B, C, L, P, cfg, cfg_scale, phi):
    """y at the forward's pitch round_up(C, 32) with NaN in the pad columns and in the prepended rows: neither may be
    read.  Position 1 of item 0 has cond == uncond; position 2 has all channels equal in both (1.5: its sums are exact),
    so both stds are exactly 0 and the rescaled output is NaN there, as the reference formula's is."""
    g = gen(B * 100 + C + L + P)
    R, N_seq, ldy = (2 * B if cfg else B), L + P, (C + 31) // 32 * 32
    y = torch.full((R, N_seq, ldy), float("nan"), device=DEV)
    y[:, P:, :C] = randn(R, L, C, g=g)
    if cfg and L >= 3:
        y[B, P + 1, :C] = y[0, P + 1, :C]
        y[0, P + 2, :C] = 1.5
        y[B, P + 2, :C] = 1.5
    o = Guarded((B, C, L))
    call(nat().lib().satb_dit_post_probe, p(y), ldy, o.ptr(), B, C, L, N_seq, P, cfg, cfg_scale, phi)
    ref, bound = sk.dit_post_ref(y.view(R * N_seq, ldy), B, C, L, N_seq, P, cfg, cfg_scale, phi)
    rep = sk.check(o.view, ref, bound)
    nans = int(torch.isnan(ref).sum())
    report("dit_post", rep, B=B, C=C, L=L, P=P, cfg=cfg, cfg_scale=cfg_scale, phi=phi, reference_nans=nans)
    assert o.guards_intact() and rep.ok, str(rep)
    if not cfg:
        assert sk.check_bits(o.view, ref.float()).ok
    elif phi != 0.0:
        assert nans == (B * C * L if C == 1 else (C if L >= 3 else 0))
        if C > 1:   # one side's std over C instead of C - 1 is rejected on the kernel's output
            assert not sk.check(o.view, *sk.dit_post_ref(y.view(R * N_seq, ldy), B, C, L, N_seq, P, cfg, cfg_scale, phi,
                                                         unbiased=(True, False))).ok


# ------------------------------------------------------------------------------------------------ casts
@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("with_perm", [0, 1])
def test_cast_rows_70000_rows_bits(bf16, with_perm):
    """More rows than one launch's grid takes (65 535): the launcher's second chunk, with and without the row gather.
    Pitches differ from each other and from the column count; the source's pad columns hold NaN, the destination's
    must keep their fill.  Overflow to inf, fp16 subnormals, -0."""
    g = gen(70 + bf16 + 2 * with_perm)
    rows, cols, src_ld, dst_ld = 70000, 40, 56, 48
    out = "bf16" if bf16 else "fp16"
    src = torch.full((rows, src_ld), float("nan"), device=DEV)
    src[:, :cols] = randn(rows, cols, g=g)
    src[:, :6] = torch.tensor([70000.0, -1e9, 3e-6, -2e-8, -0.0, 65520.0], device=DEV)
    src[:, 6] = torch.arange(rows, device=DEV, dtype=torch.float32) / 64       # tells every row from every other
    perm = torch.randperm(rows, device=DEV, generator=g).int() if with_perm else None
    o = Guarded((rows, dst_ld), sk.DT16[out])
    call(nat().lib().satb_cast_rows_probe, p(src), o.ptr(), p(perm), rows, cols, src_ld, dst_ld, bf16)
    want = o.before.clone()
    want[GUARD:GUARD + o.n].view(rows, dst_ld)[:, :cols] = sk.cast_rows_ref(src, perm, cols, out)
    rep = sk.check_bits(o.buf, want)
    report("cast_rows", rep, rows=rows, cols=cols, out=out, perm=bool(with_perm), mismatches=rep.nonfinite)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("bf16,rows,cols,ld", [(0, 5, 1, 1), (1, 1, 17000, 17000), (0, 65535, 8, 8), (1, 65536, 8, 8)])
def test_cast_rows_edges_bits(bf16, rows, cols, ld):
    """One column; more columns than one pass of the 64-block column grid covers; exactly one chunk and one row more."""
    out = "bf16" if bf16 else "fp16"
    src = randn(rows, ld, g=gen(rows + cols))
    o = Guarded((rows, ld), sk.DT16[out])
    call(nat().lib().satb_cast_rows_probe, p(src), o.ptr(), None, rows, cols, ld, ld, bf16)
    want = o.before.clone()
    want[GUARD:GUARD + o.n].view(rows, ld)[:, :cols] = sk.cast_rows_ref(src, None, cols, out)
    rep = sk.check_bits(o.buf, want)
    report("cast_rows_edges", rep, rows=rows, cols=cols, out=out)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("cols", [4, 128, 1536, 6144])
@pytest.mark.parametrize("with_perm", [0, 1])
def test_quant_rows_fp8_bits(cols, with_perm):
    """Rows whose amax is exactly 448 * 2^e, one ulp above and one below (the scale steps between the first two), for
    several e; an all-zero row; a row of 1e-40-sized values (amax a subnormal: e clamps at -126)."""
    g = gen(cols + with_perm)
    rows = 37
    src = randn(rows, cols, g=g)
    nxt = lambda v, to: torch.nextafter(torch.tensor(v), torch.tensor(to)).item()
    for i, e in enumerate((-20, -8, -1, 0, 2, 9)):
        edge = 448.0 * 2.0 ** e
        for j, amax in enumerate((edge, nxt(edge, float("inf")), nxt(edge, 0.0))):
            r = 3 * i + j
            src[r] *= edge / 16
            src[r, (5 * r) % cols] = amax if r % 2 else -amax
    src[18] = 0.0
    src[19] = randn(cols, g=g) * 1e-40
    src[20] *= 1e-30
    perm = torch.randperm(rows, device=DEV, generator=g).int() if with_perm else None
    q, s = Guarded((rows, cols), torch.uint8), Guarded((rows,))
    call(nat().lib().satb_quant_rows_fp8_probe, p(src), q.ptr(), s.ptr(), p(perm), rows, cols)
    q_ref, s_ref = sk.quant_rows_fp8_ref(src.cpu(), perm.cpu() if with_perm else None)
    rq, rs = sk.check_bits(q.view.cpu(), q_ref), sk.check_bits(s.view.cpu(), s_ref)
    report("quant_rows_fp8", None, cols=cols, perm=bool(with_perm), byte_mismatches=rq.nonfinite, scale_mismatches=rs.nonfinite)
    assert q.guards_intact() and s.guards_intact() and rq.ok and rs.ok, f"bytes: {rq}; scales: {rs}"
    inv = torch.argsort(perm.long()) if with_perm else torch.arange(rows, device=DEV)
    got = s.view[inv]          # scales in source-row order: exact edge and one below share a scale, one above doubles it
    for i in range(6):
        assert float(got[3 * i]) == float(got[3 * i + 2]) and float(got[3 * i + 1]) == 2 * float(got[3 * i])
    assert float(got[18]) == 1.0 and float(got[19]) == 2.0 ** -126


# ------------------------------------------------------------------------------------------------ matmul_f64
@pytest.mark.parametrize("M,N,K", [(256, 128, 128), (512, 256, 256), (3072, 1536, 1536), (130, 70, 100), (1, 1, 1),
                                   (65, 129, 17), (64, 64, 16), (63, 65, 15)])
def test_matmul_f64_vs_fp64(M, N, K):
    """The conformer fold's shapes (2 D, D, D) and shapes that are no multiple of the 64 x 64 tile or the 16-deep step."""
    g = gen(M + N + K)
    A, B = randn(M, K, g=g), randn(K, N, g=g, scale=K ** -0.5)
    o = Guarded((M, N))
    call(nat().lib().satb_matmul_f64_probe, p(A), p(B), o.ptr(), M, N, K)
    ref, bound = sk.matmul_f64_ref(A, B)
    rep = sk.check(o.view, ref, bound)
    report("matmul_f64", rep, M=M, N=N, K=K)
    assert o.guards_intact() and rep.ok, str(rep)


# ------------------------------------------------------------------------------------------------ sampler update
COEF = dict(c_skip=0.8, c_out=-0.6, A=0.7, B=0.9, C=-0.35, D=0.05, S=0.3, c_in_next=0.83)
NULLS = [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)]


@pytest.mark.parametrize("n,combos", [(4, [NULLS[0], NULLS[15]]), (1028, NULLS), (8 * 64 * 6144, [NULLS[15], NULLS[6], NULLS[9]])])
def test_sampler_update_vs_fp64(n, combos):
    """n = 8 * 64 * 6144: more float4 than the capped grid has threads, so every thread loops.  (den_1, den_2, noise,
    x_in_next) given or null in every combination."""
    g = gen(n % 1000)
    x, v, d1, d2, nz = (randn(n, g=g) for _ in range(5))
    lib = nat().lib()
    for use in combos:
        t1, t2, tn = (t if u else None for t, u in zip((d1, d2, nz), use[:3]))
        den, nxt, xin = Guarded((n,)), Guarded((n,)), Guarded((n,))
        call(lib.satb_sampler_update, p(x), p(v), p(t1), p(t2), p(tn), den.ptr(), nxt.ptr(), xin.ptr() if use[3] else None,
             n, *COEF.values())
        r = sk.sampler_update_ref(x, v, t1, t2, tn, **COEF)
        reps = {"den": sk.check(den.view, *r["den"]), "x_next": sk.check(nxt.view, *r["x_next"])}
        if use[3]:
            reps["x_in"] = sk.check(xin.view, *r["x_in"])
        else:
            assert sk.check_bits(xin.buf, xin.before).ok            # a null x_in_next: nothing written anywhere near
        report("sampler_update", max(reps.values(), key=lambda q: q.ratio), n=n, given=use)
        assert den.guards_intact() and nxt.guards_intact() and xin.guards_intact()
        assert all(q.ok for q in reps.values()), {k: str(q) for k, q in reps.items()}


def test_sampler_update_refuses_a_ragged_count():
    x = torch.zeros(1030, device=DEV)
    lib = nat().lib()
    rc = lib.satb_sampler_update(p(x), p(x), None, None, None, p(x), p(x), None, 1030, *COEF.values(), nat().stream_ptr())
    assert rc != 0 and b"multiple of 4" in lib.satb_last_error()


# ------------------------------------------------------------------------------------------------ SnakeBeta
@pytest.mark.parametrize("offset", [1, 0])
def test_snake_beta_scalar_path_vs_fp64(offset):
    """T % 4 == 0 with x one float off 16-byte alignment: the kernel must take its scalar loop (offset 0: the float4 one)."""
    g = gen(5 + offset)
    B, C, T = 2, 3, 64
    xb = randn(B * C * T + 4, g=g, scale=4.0)
    x = xb[offset:offset + B * C * T].view(B, C, T)
    assert (x.data_ptr() % 16 != 0) == bool(offset)
    alpha, beta = randn(C, g=g, scale=0.4), randn(C, g=g, scale=0.4)
    o = Guarded((B, C, T))
    call(nat().lib().satb_snake_beta, p(x), p(alpha), p(beta), o.ptr(), B, C, T, 1)
    ref, bound = sk.snake_beta_ref(x, alpha, beta)
    rep = sk.check(o.view, ref, bound)
    report("snake_beta", rep, offset=offset)
    assert o.guards_intact() and rep.ok, str(rep)


# ------------------------------------------------------------------------------------------------ > 65535 token rows
def test_forward_with_more_than_65535_token_rows_equals_the_half_batch():
    """8 prompts with CFG at 6145 tokens: 98 320 token rows through every LayerNorm, GEMM and the final cast_rows, whose
    launcher splits at 65 535 rows.  The first 4 prompts' outputs equal, bit for bit, the same prompts run as a batch of
    4 (49 160 rows: below the split)."""
    free, _ = torch.cuda.mem_get_info()
    if free < 8 << 30:
        pytest.skip(f"needs about 8 GB of free device memory, {free >> 20} MB free")
    from helpers import build_native_dit
    from oracle import dit_oracle as do
    cfg = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
               project_cond_tokens=False, transformer_type="continuous_transformer")
    m = build_native_dit(cfg, do.make_dit_weights(cfg, seed=61))
    g = torch.Generator().manual_seed(62)
    B, L = 8, 6144
    x, t = torch.randn(B, 64, L, generator=g).cuda(), (torch.rand(B, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(B, 9, 128, generator=g).cuda(), torch.randn(B, 256, generator=g).cuda()
    sub = lambda n: dict(cross_attn_cond=c[:n].contiguous(), global_embed=ge[:n].contiguous(), cfg_scale=4.0, scale_phi=0.5)
    y8 = m(x, t, **sub(8)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(4)).clone()
    equal = bool(torch.equal(y8[:4], y4))
    report("forward_98320_rows", None, rows=2 * B * (L + 1), bit_equal=equal, finite=bool(torch.isfinite(y8).all()))
    assert torch.isfinite(y8).all() and float(y8[4:].abs().max()) > 0
    assert equal
