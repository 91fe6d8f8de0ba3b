"""CPU: the float64 references of tests/small_kernel_ref.py are the reference project's formulas, their checkers
reject the faults the kernels could have, and the probe entry points refuse bad arguments before any CUDA call.

1. Each reference equals an independent torch float64 evaluation of the reference project's code (F.layer_norm and the
   adaLN lines of models/transformer.py:188-206,670-688; the Fourier features of models/blocks.py:95-97; the prepend
   concat, prepend drop and CFG lines of models/dit.py:185-195,219,309-311,338-347).
2. A correct kernel's output (the reference rounded the way the kernel rounds) passes, and a planted fault of the kind
   the kernel could have is rejected: modulation taken from the neighbouring item, sin | cos swapped, the gate applied
   to chunk 1, a skinny-linear row shifted by one, the biased instead of the unbiased std, an e4m3 scale one exponent
   off at the 448 * 2^e boundary, a cast that drops the rows past a split, a pad column read.
3. The refusals: fake aligned addresses that are never dereferenced."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import small_kernel_ref as sk

FAKE = 1 << 20


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- LayerNorm
def _ln_case(seed=0, rows=24, D=256, B=2, rpi=4):
    g = _gen(seed)
    x = torch.randn(rows, D, generator=g) * 2 + 3
    gamma, beta = 1 + 0.2 * torch.randn(D, generator=g), 0.3 * torch.randn(D, generator=g)
    scale, shift = 0.5 * torch.randn(B, D, generator=g), torch.randn(B, D, generator=g)
    return x, gamma, beta, scale, shift, B, rpi


def test_layernorm_ref_is_the_reference_formula():
    x, gamma, beta, scale, shift, B, rpi = _ln_case()
    y, bound = sk.layernorm_ref(x, gamma, beta, scale, shift, rpi, B)
    # transformer.py:188-206 (F.layer_norm, eps 1e-5) and :670-672: x * (1 + scale) + shift with scale [b, 1, D]; the
    # 24 rows are [2 (cond | uncond), B, rpi]: the CFG half repeats the conditional vectors
    n = F.layer_norm(x.double(), (x.shape[1],), gamma.double(), beta.double(), 1e-5).view(-1, B, rpi, x.shape[1])
    want = n * (1 + scale.double()[None, :, None]) + shift.double()[None, :, None]
    assert float((y - want.reshape(y.shape)).abs().max()) < 1e-9
    assert float(bound.min()) > 0
    y0, _ = sk.layernorm_ref(x, gamma, None)
    assert float((y0 - F.layer_norm(x.double(), (x.shape[1],), gamma.double(), None, 1e-5)).abs().max()) < 1e-9


@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_layernorm_checker_accepts_the_rounded_reference_and_rejects_faults(out):
    x, gamma, beta, scale, shift, B, rpi = _ln_case(1)
    y, bound = sk.layernorm_ref(x, gamma, beta, scale, shift, rpi, B, out)
    assert sk.check(sk.round16(y, out), y, bound).ok
    # an fp32 evaluation (torch's own LayerNorm) is inside the bound as well
    y32 = F.layer_norm(x, (x.shape[1],), gamma, beta, 1e-5)
    item = sk.item_of_row(x.shape[0], rpi, B)
    assert sk.check((y32 * (1 + scale[item]) + shift[item]).to(sk.DT16[out]), y, bound).ok
    faults = {
        "neighbouring item": sk.layernorm_ref(x, gamma, beta, scale, shift, rpi, B, out, item_shift=1)[0],
        "rows_per_item + 1": sk.layernorm_ref(x, gamma, beta, scale, shift, rpi + 1, B, out)[0],
        "no wrap": sk.layernorm_ref(x, gamma, beta, torch.cat([scale, scale * 0]), torch.cat([shift, shift * 0]), rpi,
                                    2 * B, out)[0],
        "beta dropped": sk.layernorm_ref(x, gamma, None, scale, shift, rpi, B, out)[0],
        "unbiased variance": y * ((x.shape[1] - 1) / x.shape[1]) ** 0.5,
    }
    for name, bad in faults.items():
        r = sk.check(sk.round16(bad, out), y, bound)
        assert not r.ok, name
    one_row = y.clone()
    one_row[17] = y[16]
    assert sk.check(sk.round16(one_row, out), y, bound).index[0] == 17


def test_layernorm_bound_covers_the_mean_error_of_large_mean_and_constant_rows():
    """A row at 1000 sigma: an fp32 evaluation loses ~1e-4 of z to the mean's rounding, which the bound must allow and
    a plain 2^-11 |y| bound would not need to; a constant row gives beta (1 + s) + t."""
    g = _gen(2)
    D = 1024
    x = torch.randn(4, D, generator=g)
    x[1] += 1000.0
    x[2] = 2.5
    x[3] *= 1e-6
    gamma, beta = torch.ones(D), 0.1 * torch.randn(D, generator=g)
    y, bound = sk.layernorm_ref(x, gamma, beta, out="fp16")
    assert sk.check(F.layer_norm(x, (D,), gamma, beta, 1e-5).half(), y, bound).ok
    assert float((y[2] - beta.double()).abs().max()) == 0.0
    assert float((bound[1] / bound[0]).median()) > 1.05     # the mean term is visible at 1000 sigma
    assert float(bound[2].max()) < 2e-3


# ---------------------------------------------------------------------------------------------------- fourier
def test_fourier_ref_and_checker():
    g = _gen(3)
    t, w = torch.tensor([0.0, 1e-4, 0.5, 0.9365, 1.0]), torch.randn(128, generator=g) * 16
    ref, bound = sk.fourier_ref(t, w)
    # blocks.py:95-97: f = 2 pi t[:, None] w[None, :]; cat([f.cos(), f.sin()], -1)
    f = 2 * torch.pi * t.double()[:, None] * w.double()[None, :]
    want = torch.cat([f.cos(), f.sin()], -1)
    assert float((ref - want).abs().max()) < 1e-4           # the fp32 argument is off by up to 2^-23 |f|, |f| ~ 300
    assert sk.check(ref.float(), ref, bound).ok
    assert not sk.check(torch.cat([ref[:, 128:], ref[:, :128]], 1).float(), ref, bound).ok, "sin | cos"
    # the float64 argument instead of the kernel's fp32 one is already outside: the bound has no room for a sloppy sine
    assert not sk.check(want.float(), ref, bound).ok
    approx = ref + 2.0 ** -22 * torch.cat([f, f], 1).abs().clamp_min(1)
    assert not sk.check(approx.float(), ref, bound).ok, "sin.approx-sized error"


# ---------------------------------------------------------------------------------------------------- skinny linear
@pytest.mark.parametrize("bias,add,silu", [(b, a, s) for b in (0, 1) for a in (0, 1) for s in (0, 1)])
def test_skinny_linear_ref_and_checker(bias, add, silu):
    g = _gen(4)
    R, K, N = 9, 260, 17
    x, W = torch.randn(R, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) if bias else None
    a = torch.randn(R, N, generator=g) if add else None
    ref, bound = sk.skinny_linear_ref(x, W, b, a, silu)
    want = F.linear(x.double(), W.double(), b.double() if bias else None)
    want = want + a.double() if add else want
    want = F.silu(want) if silu else want
    assert float((ref - want).abs().max()) < 1e-12
    got = F.linear(x, W, b)
    got = got + a if add else got
    got = F.silu(got) if silu else got
    assert sk.check(got, ref, bound).ok
    assert not sk.check(torch.roll(got, 1, 0), ref, bound).ok, "row shifted by one"
    dropped = F.linear(x[:, :K - 4], W[:, :K - 4], b)
    dropped = dropped + a if add else dropped
    assert not sk.check(F.silu(dropped) if silu else dropped, ref, bound).ok, "last float4 of K dropped"
    if bias:
        assert not sk.check(got - b, ref, bound).ok, "bias dropped"


# ---------------------------------------------------------------------------------------------------- prepend rows
def test_write_prepend_ref_is_the_reference_concat():
    g = _gen(5)
    B, Pp, D, N_seq = 3, 4, 64, 9
    tok, pre = torch.randn(B, D, generator=g), torch.randn(B, Pp, D, generator=g)
    pos = torch.randn(N_seq, D, generator=g)
    ref = sk.write_prepend_ref(tok, pre, pos, 2 * B, B, N_seq, D, Pp)
    # dit.py:309-312: cat([prepend_cond, zeros]) over the batch; :185-195: cat([prepend_inputs, global_embed[:, None]], 1);
    # transformer.py:770-785: the positional embedding is added after the concat
    want = torch.cat([torch.cat([pre, torch.zeros_like(pre)], 0), torch.cat([tok, tok], 0)[:, None]], 1) + pos[:Pp + 1]
    assert sk.check_bits(ref, want).ok
    assert sk.check_bits(sk.write_prepend_ref(tok, None, None, 2 * B, B, N_seq, D, 0)[:, 0], torch.cat([tok, tok], 0)).ok
    bad = ref.clone()
    bad[B:, :Pp] = ref[:B, :Pp]                                   # unconditional rows given the conditional tokens
    assert not sk.check_bits(bad, want).ok
    assert not sk.check_bits(-torch.zeros(3), torch.zeros(3)).ok  # bit equality tells -0 from +0


# ---------------------------------------------------------------------------------------------------- gates
def test_gate_sigmoid_ref_and_checker():
    g = _gen(6)
    rows, depth, D = 3, 2, 128
    ssg = torch.randn(rows, depth * 6 * D, generator=g) * 3
    ssg[0, 2 * D:2 * D + 4] = torch.tensor([100.0, -100.0, 1e4, -1e4])
    ref, bound, changed = sk.gate_sigmoid_ref(ssg, depth, D)
    # transformer.py:667: chunk(6) = scale_self, shift_self, gate_self, scale_ff, shift_ff, gate_ff; :674 / :688:
    # x * sigmoid(1 - gate)
    want = ssg.double().clone().view(rows, depth, 6, D)
    for c in (2, 5):
        want[:, :, c] = torch.sigmoid(1 - want[:, :, c])
    assert torch.equal(ref, want.view(rows, -1))
    assert int(changed.sum()) == rows * depth * 2 * D and float(bound[~changed].max()) == 0.0
    assert torch.equal(ref[0, 2 * D:2 * D + 4], torch.tensor([torch.sigmoid(torch.tensor(-99.0, dtype=torch.float64)), 1, 0, 1]))

    def kernel_like(chunks):
        out = ssg.clone().view(rows, depth, 6, D)
        for c in chunks:
            out[:, :, c] = 1.0 / (1.0 + torch.exp(-(1.0 - out[:, :, c])))
        return out.view(rows, -1)

    assert sk.check(kernel_like((2, 5)), ref, bound).ok
    assert not sk.check(kernel_like((1, 5)), ref, bound).ok, "gate applied to chunk 1"
    assert not sk.check(kernel_like((2, 4)), ref, bound).ok
    touched = kernel_like((2, 5))
    touched[1, 7] = touched[1, 7] * (1 + 2.0 ** -23)              # one ulp on an element the kernel does not own
    assert not sk.check(touched, ref, bound).ok


# ---------------------------------------------------------------------------------------------------- DiT post
def _post_case(seed, B=2, C=16, L=37, P=2, ldy=32):
    g = _gen(seed)
    N_seq = L + P
    y = torch.full((2 * B * N_seq, ldy), float("nan"))
    y[:, :C] = torch.randn(2 * B * N_seq, C, generator=g)
    y.view(2 * B, N_seq, ldy)[:, :P] = float("nan")
    return y, B, C, L, N_seq, P


@pytest.mark.parametrize("cfg_scale,phi", [(1.0, 0.0), (4.0, 0.0), (7.0, 0.5), (4.0, 0.7), (3.0, 1.0)])
def test_dit_post_ref_is_the_reference_formula(cfg_scale, phi):
    y, B, C, L, N_seq, P = _post_case(7)
    ref, bound = sk.dit_post_ref(y, B, C, L, N_seq, P, 1, cfg_scale, phi)
    # dit.py:219: rearrange(output, "b t c -> b c t")[:, :, prepend_length:]; :338-347
    out = y[:, :C].double().view(2 * B, N_seq, C).transpose(1, 2)[:, :, P:]
    cond, uncond = torch.chunk(out, 2, dim=0)
    s, p = (float(torch.tensor(v, dtype=torch.float32)) for v in (cfg_scale, phi))
    cfg_out = uncond + (cond - uncond) * s
    want = cfg_out
    if phi != 0.0:
        want = p * (cfg_out * (cond.std(dim=1, keepdim=True) / cfg_out.std(dim=1, keepdim=True))) + (1 - p) * cfg_out
    assert ref.shape == (B, C, L) and float((ref - want).abs().max()) < 1e-12
    assert torch.isfinite(bound).all()
    nocfg, b0 = sk.dit_post_ref(y[:B * N_seq], B, C, L, N_seq, P, 0)
    assert torch.equal(nocfg, cond) and float(b0.max()) == 0.0


def test_dit_post_checker_rejects_faults_and_keeps_the_nan_pattern():
    y, B, C, L, N_seq, P = _post_case(8)
    y3 = y.view(2 * B, N_seq, -1)
    y3[0, P + 5, :C] = 1.5                                        # cond == uncond, all channels equal: std 0 / std 0
    y3[B, P + 5, :C] = 1.5
    ref, bound = sk.dit_post_ref(y, B, C, L, N_seq, P, 1, 4.0, 0.5)
    assert torch.isnan(ref[0, :, 5]).all() and int(torch.isnan(ref).sum()) == C
    assert sk.check(ref.float(), ref, bound).ok
    finite = torch.nan_to_num(ref.float(), nan=0.0)
    assert not sk.check(finite, ref, bound).ok, "a finite value where the formula gives NaN"
    # the std over C instead of C - 1 on one side moves the ratio by sqrt(C / (C - 1)); on both sides it cancels
    for sides in ((False, True), (True, False)):
        biased = sk.dit_post_ref(y, B, C, L, N_seq, P, 1, 4.0, 0.5, unbiased=sides)[0]
        assert not sk.check(biased.float(), ref, bound).ok, "biased std"
    both = sk.dit_post_ref(y, B, C, L, N_seq, P, 1, 4.0, 0.5, unbiased=(False, False))[0]
    assert sk.check(both.float(), ref, bound).ok
    assert not sk.check(sk.dit_post_ref(y, B, C, L, N_seq, P - 1, 1, 4.0, 0.5)[0][:, :, 1:].float(), ref[:, :, 1:], bound[:, :, 1:]).ok
    packed = y[:, :C].contiguous()                                # the row pitch taken as C: other rows' values
    wrong_pitch = torch.cat([packed.view(-1), torch.zeros(y.numel() - packed.numel())]).view_as(y)
    assert not sk.check(sk.dit_post_ref(wrong_pitch, B, C, L, N_seq, P, 1, 4.0, 0.5)[0].float(), ref, bound).ok
    one, b1 = sk.dit_post_ref(y, B, 1, L, N_seq, P, 1, 4.0, 0.5)  # one channel: the unbiased std is 0 / 0
    assert torch.isnan(one).all()


# ---------------------------------------------------------------------------------------------------- casts
@pytest.mark.parametrize("out", ["fp16", "bf16"])
def test_cast_rows_ref_and_checker(out):
    g = _gen(9)
    src = torch.randn(300, 12, generator=g)
    src[0, :6] = torch.tensor([70000.0, -1e9, 3e-6, -2e-8, -0.0, 65520.0])
    perm = torch.randperm(300, generator=g).int()
    ref = sk.cast_rows_ref(src, perm, 10, out)
    assert ref.shape == (300, 10) and sk.check_bits(ref, src[perm.long(), :10].to(sk.DT16[out])).ok
    dropped = ref.clone()
    dropped[256:] = 0                                             # rows past a launch split never written
    assert not sk.check_bits(dropped, ref).ok
    assert not sk.check_bits(sk.cast_rows_ref(src, None, 10, out), ref).ok


def test_quant_rows_fp8_ref_and_boundary_rows():
    from fp8_ref import fp8_row_exponent
    g = _gen(10)
    src = torch.randn(8, 128, generator=g)
    up = lambda v: float(torch.nextafter(torch.tensor(v), torch.tensor(float("inf"))))
    dn = lambda v: float(torch.nextafter(torch.tensor(v), torch.tensor(0.0)))
    src[0] *= 0.1
    src[0, 5] = 448.0 * 4                                         # amax exactly 448 * 2^2: e = 2
    src[1] *= 0.1
    src[1, 5] = -up(448.0 * 4)                                    # one ulp above: e = 3
    src[2] *= 0.1
    src[2, 5] = dn(448.0 * 4)                                     # one ulp below: e = 2
    src[3] = 0.0
    src[4] = torch.randn(128, generator=g) * 1e-40
    q, scale = sk.quant_rows_fp8_ref(src)
    assert scale[:4].tolist() == [4.0, 8.0, 4.0, 1.0] and float(scale[4]) == 2.0 ** -126
    assert int(q[3].max()) == 0 and q.dtype == torch.uint8
    assert float(q[0].view(torch.float8_e4m3fn).float()[5]) == 448.0
    # the rule, restated on the bits as the kernel does it
    amax = src.abs().amax(1)
    bits = amax.view(torch.int32)
    e_bits = torch.where((bits & 0x7FFFFF) <= 0x600000, (bits >> 23) - 127 - 8, (bits >> 23) - 127 - 7).clamp_min(-126)
    assert torch.equal(torch.where(amax > 0, e_bits, torch.zeros_like(e_bits)), fp8_row_exponent(amax).int())
    # a scale one exponent off at the boundary: row 1 quantised with e = 2 saturates, row 0 with e = 3 loses a bit
    q_bad = torch.ldexp(src[0], torch.tensor(-3)).to(torch.float8_e4m3fn).view(torch.uint8)
    assert not sk.check_bits(q_bad, q[0]).ok
    assert not sk.check_bits(torch.tensor([4.0, 4.0, 4.0, 1.0]), scale[:4]).ok
    perm = torch.tensor([3, 0, 7, 1], dtype=torch.int32)
    qp, sp = sk.quant_rows_fp8_ref(src, perm)
    assert torch.equal(qp, q[perm.long()]) and torch.equal(sp, scale[perm.long()])


def test_matmul_f64_ref_and_checker():
    g = _gen(11)
    A, B = torch.randn(70, 100, generator=g), torch.randn(100, 130, generator=g)
    ref, bound = sk.matmul_f64_ref(A, B)
    assert sk.check(ref.float(), ref, bound).ok
    got32 = A @ B                                                 # an fp32-accumulated product is NOT within the bound
    assert not sk.check(got32, ref, bound).ok
    assert not sk.check((A.double()[:, :96] @ B.double()[:96]).float(), ref, bound).ok, "ragged K tail dropped"


# ---------------------------------------------------------------------------------------------------- sampler, snake
def test_sampler_update_ref_and_checker():
    g = _gen(12)
    x, v, d1, d2, nz = (torch.randn(1028, generator=g) for _ in range(5))
    co = dict(c_skip=0.8, c_out=-0.6, A=0.7, B=0.9, C=-0.35, D=0.05, S=0.3, c_in_next=0.83)
    f = {k: torch.tensor(val, dtype=torch.float32).double() for k, val in co.items()}
    for use in [(1, 1, 1), (0, 0, 0), (1, 0, 1), (0, 1, 0)]:
        t1, t2, tn = (t if u else None for t, u in zip((d1, d2, nz), use))
        r = sk.sampler_update_ref(x, v, t1, t2, tn, **co)
        den = f["c_out"] * v.double() + f["c_skip"] * x.double()
        nxt = f["A"] * x.double() + f["B"] * den
        for c, t in (("C", t1), ("D", t2), ("S", tn)):
            nxt = nxt + f[c] * t.double() if t is not None else nxt
        assert float((r["den"][0] - den).abs().max()) < 1e-14 and float((r["x_next"][0] - nxt).abs().max()) < 1e-14
        assert float((r["x_in"][0] - nxt * f["c_in_next"]).abs().max()) < 1e-14
        for name in r:
            assert sk.check(r[name][0].float(), *r[name]).ok
    r = sk.sampler_update_ref(x, v, d1, d2, nz, **co)
    swapped = sk.sampler_update_ref(x, v, d2, d1, nz, **co)["x_next"][0]
    assert not sk.check(swapped.float(), *r["x_next"]).ok
    tail = r["x_next"][0].float().clone()
    tail[1024:] = 0                                               # the last float4 not reached by the loop
    assert not sk.check(tail, *r["x_next"]).ok


def test_snake_beta_ref_and_checker():
    g = _gen(13)
    x, alpha, beta = torch.randn(2, 5, 64, generator=g) * 4, torch.randn(5, generator=g) * 0.4, torch.randn(5, generator=g) * 0.4
    ref, bound = sk.snake_beta_ref(x, alpha, beta)
    a, b = alpha.exp()[None, :, None], beta.exp()[None, :, None]
    got = x + (1.0 / (b + 1e-9)) * torch.sin(x * a) ** 2          # blocks.py:350-358 in fp32
    assert sk.check(got, ref, bound).ok
    assert not sk.check(x + (1.0 / (a + 1e-9)) * torch.sin(x * b) ** 2, ref, bound).ok, "alpha / beta swapped"
    assert not sk.check(torch.roll(got, 1, 1), ref, bound).ok, "channel off by one"


# ---------------------------------------------------------------------------------------------------- refusals
def _refused(rc, lib, msg):
    err = lib.satb_last_error()
    assert rc != 0 and msg in err, (rc, err)


def test_small_kernel_probes_validate_before_any_cuda_call():
    """Fake addresses, never dereferenced: every call below must return before it touches CUDA (this machine may have no
    device at all)."""
    from stable_audio_tools import _native
    lib = _native.lib()
    f = FAKE
    ln = lambda **kw: lib.satb_layernorm_mod(*[kw.get(k, d) for k, d in (
        ("x", f), ("gamma", f), ("beta", f), ("scale", f), ("shift", f), ("stride", 1536), ("rpi", 5), ("items", 2),
        ("out", f), ("rows", 20), ("D", 256), ("bf16", 0))], None)
    _refused(ln(x=None), lib, b"null")
    _refused(ln(gamma=None), lib, b"null")
    _refused(ln(out=None), lib, b"null")
    _refused(ln(shift=None), lib, b"adaLN modulation")
    _refused(ln(rpi=0), lib, b"adaLN modulation")
    _refused(ln(items=0), lib, b"adaLN modulation")
    _refused(ln(stride=1538), lib, b"adaLN modulation")
    _refused(ln(x=f + 4), lib, b"aligned")
    _refused(ln(scale=f + 8), lib, b"aligned")
    _refused(ln(out=f + 4), lib, b"aligned")
    _refused(ln(D=200), lib, b"multiple of 128")
    _refused(ln(D=2176), lib, b"<= 2048")
    _refused(ln(rows=-1), lib, b"negative")
    assert ln(rows=0) == 0                                        # nothing to do: no launch

    _refused(lib.satb_fourier_probe(None, f, f, 2, 128, None), lib, b"null")
    _refused(lib.satb_fourier_probe(f, f, f, 0, 128, None), lib, b"B, F >= 1")
    _refused(lib.satb_fourier_probe(f, f, f, 2, 0, None), lib, b"B, F >= 1")

    sl = lambda **kw: lib.satb_skinny_linear_probe(*[kw.get(k, d) for k, d in (
        ("x", f), ("W", f), ("bias", None), ("add", None), ("out", f), ("R", 8), ("K", 256), ("N", 64), ("silu", 0))], None)
    _refused(sl(x=None), lib, b"null")
    _refused(sl(W=None), lib, b"null")
    _refused(sl(out=None), lib, b"null")
    _refused(sl(K=258), lib, b"multiple of 4")
    _refused(sl(K=0), lib, b"K >= 4")
    _refused(sl(R=0), lib, b"row count")
    _refused(sl(R=4097), lib, b"row count")
    _refused(sl(K=6404), lib, b"too large")
    _refused(sl(N=0), lib, b"N >= 1")
    _refused(sl(x=f + 4), lib, b"aligned")

    wp = lambda **kw: lib.satb_write_prepend_probe(*[kw.get(k, d) for k, d in (
        ("tok", f), ("pre", None), ("pos", None), ("h", f), ("R", 2), ("B", 1), ("N_seq", 10), ("D", 256), ("Pp", 1))], None)
    _refused(wp(tok=None), lib, b"null")
    _refused(wp(h=None), lib, b"null")
    _refused(wp(B=0), lib, b"write prepend")
    _refused(wp(R=65536), lib, b"write prepend")
    _refused(wp(Pp=10), lib, b"Pp < N_seq")
    _refused(wp(Pp=-1), lib, b"Pp < N_seq")

    _refused(lib.satb_gate_sigmoid_probe(None, 1, 1, 128, None), lib, b"null")
    _refused(lib.satb_gate_sigmoid_probe(f, 0, 1, 128, None), lib, b"gate sigmoid")
    _refused(lib.satb_gate_sigmoid_probe(f, 65536, 1, 128, None), lib, b"gate sigmoid")
    _refused(lib.satb_gate_sigmoid_probe(f, 1, 0, 128, None), lib, b"gate sigmoid")

    dp = lambda **kw: lib.satb_dit_post_probe(*[kw.get(k, d) for k, d in (
        ("y", f), ("ldy", 64), ("out", f), ("B", 1), ("C", 64), ("L", 10), ("N_seq", 11), ("P", 1), ("cfg", 1),
        ("s", 4.0), ("phi", 0.5))], None)
    _refused(dp(y=None), lib, b"null")
    _refused(dp(out=None), lib, b"null")
    _refused(dp(ldy=63), lib, b"row pitch")
    _refused(dp(C=65), lib, b"row pitch")
    _refused(dp(B=0), lib, b"dit post probe")
    _refused(dp(L=0), lib, b"dit post probe")
    _refused(dp(P=-1), lib, b"dit post probe")
    _refused(dp(N_seq=10), lib, b"N_seq >= P + L")

    cr = lambda **kw: lib.satb_cast_rows_probe(*[kw.get(k, d) for k, d in (
        ("src", f), ("dst", f), ("perm", None), ("rows", 100), ("cols", 40), ("src_ld", 40), ("dst_ld", 40), ("bf16", 0))], None)
    _refused(cr(src=None), lib, b"null")
    _refused(cr(dst=None), lib, b"null")
    _refused(cr(rows=0), lib, b"rows, cols >= 1")
    _refused(cr(cols=0), lib, b"rows, cols >= 1")
    _refused(cr(src_ld=39), lib, b"row pitches")
    _refused(cr(dst_ld=39), lib, b"row pitches")

    qr = lambda **kw: lib.satb_quant_rows_fp8_probe(*[kw.get(k, d) for k, d in (
        ("src", f), ("dst", f), ("scale", f), ("perm", None), ("rows", 8), ("cols", 128))], None)
    _refused(qr(src=None), lib, b"null")
    _refused(qr(dst=None), lib, b"null")
    _refused(qr(scale=None), lib, b"null")
    _refused(qr(cols=130), lib, b"multiple of 4")
    _refused(qr(cols=0), lib, b"cols >= 4")
    _refused(qr(rows=0), lib, b"rows >= 1")
    _refused(qr(src=f + 4), lib, b"16-byte aligned")
    _refused(qr(dst=f + 2), lib, b"4-byte aligned")

    _refused(lib.satb_matmul_f64_probe(None, f, f, 8, 8, 8, None), lib, b"null")
    _refused(lib.satb_matmul_f64_probe(f, f, None, 8, 8, 8, None), lib, b"null")
    _refused(lib.satb_matmul_f64_probe(f, f, f, 0, 8, 8, None), lib, b"matmul probe")
    _refused(lib.satb_matmul_f64_probe(f, f, f, 8, 8, 0, None), lib, b"matmul probe")

    _refused(lib.satb_sampler_update(f, f, None, None, None, f, f, None, 1030, *[0.5] * 8, None), lib, b"multiple of 4")
    _refused(lib.satb_sampler_update(f, f, None, None, None, None, f, None, 1028, *[0.5] * 8, None), lib, b"null")


def test_dit_create_refuses_widths_its_small_kernels_cannot_run():
    """embed_dim above the LayerNorm's 2048 and conditioning widths the embedding MLPs cannot stage (not a multiple of 4,
    above 6400) are refused when the model is created, not at the first prepare_cond / forward."""
    from stable_audio_tools import _native
    lib = _native.lib()
    base = dict(io_channels=64, embed_dim=2048, depth=1, num_heads=16, cond_token_dim=0, global_cond_dim=2048,
                project_cond_tokens=0, project_global_cond=1, global_cond_type=0, patch_size=1, operand_dtype=0)
    h = ctypes.c_void_p()
    assert lib.satb_dit_create(ctypes.byref(_native.SatbDitConfig(**base)), ctypes.byref(h)) == 0
    lib.satb_dit_destroy(h)
    for kw, msg in [(dict(embed_dim=2176, num_heads=17), b"embed_dim must be between 128 and 2048"),
                    (dict(embed_dim=0), b"embed_dim"),
                    (dict(global_cond_dim=130), b"global_cond_dim must be a multiple of 4"),
                    (dict(global_cond_dim=6404), b"at most 6400"),
                    (dict(global_cond_dim=-4), b"global_cond_dim"),
                    (dict(prepend_cond_dim=6404), b"prepend_cond_dim must be a multiple of 4, at most 6400"),
                    (dict(prepend_cond_dim=130), b"prepend_cond_dim must be a multiple of 4")]:
        rc = lib.satb_dit_create(ctypes.byref(_native.SatbDitConfig(**dict(base, **kw))), ctypes.byref(h))
        _refused(rc, lib, msg)
    wide = dict(base, global_cond_dim=6400, prepend_cond_dim=6400)
    assert lib.satb_dit_create(ctypes.byref(_native.SatbDitConfig(**wide)), ctypes.byref(h)) == 0
    lib.satb_dit_destroy(h)


def test_python_constructor_refuses_the_same_widths():
    from stable_audio_tools.models.dit import DiffusionTransformer
    base = dict(io_channels=64, embed_dim=256, depth=1, num_heads=4, transformer_type="continuous_transformer")
    for kw, msg in [(dict(embed_dim=2176, num_heads=17), "above 2048"), (dict(global_cond_dim=130), "global_cond_dim 130"),
                    (dict(global_cond_dim=6404), "global_cond_dim 6404"), (dict(prepend_cond_dim=6404), "prepend_cond_dim 6404")]:
        with pytest.raises(NotImplementedError, match=msg):
            DiffusionTransformer(**dict(base, **kw))
    DiffusionTransformer(**dict(base, embed_dim=2048, num_heads=16, global_cond_dim=2048, depth=0))
