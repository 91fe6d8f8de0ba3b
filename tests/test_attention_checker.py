"""CPU: the per-element checker of tests/attention_ref.py is sharp.  It accepts the float64 reference rounded to the
output type and a float32 emulation of the kernels' online softmax, and rejects the output of a subtly wrong kernel,
restated here as a mutation of the reference, on inputs that tests/test_gpu_attention_bound.py runs (same Case: same
layout, shape, distributions and seed).  This is the evidence, without a GPU, that the GPU tests fail on such
kernels."""
import pytest
import torch

import attention_ref as A

DTS = ["fp16", "bf16"]


def _self(d, dt, N):
    return A.Case("self", d, dt, 2, 7, 7, N, N)


def _cross(d, dt, Mctx):
    return A.Case("cross", d, dt, 2, 24, 12, 129, Mctx)


def _expect(case, q, k, v, H=None, Hkv=None):
    return A.expect(q, k, v, H or case.H, Hkv or case.Hkv, case.dt)


def _assert_rejects(case, exp, name, got):
    rep = A.check(got, exp)
    print(f"[ratio] {name} on {case}: {rep.ratio:.3g}")
    assert not rep.ok, f"accepts the mutation '{name}' on {case}: {rep}"


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [32, 64, 96, 128])
def test_accepts_the_rounded_reference_and_the_float32_emulation(d, dt):
    """Every score distribution at 1, 17, 129 and 257 keys.  The emulation rounds P before P V as the kernels do,
    which the rounded reference does not: its worst ratio is printed.  The bound reaches 1 only when every P rounding
    of a row pushes the output the same way; random signs stay well below, so 0.8 is asserted.  The emulation does
    not stand for every error source of the kernels: its float32 matmuls do not model the tensor cores' accumulation
    (alignment truncation, order), which the bound's e_acc terms cover, so the GPU tests may report higher ratios than
    this one (up to 0.76 on an H100 80GB HBM3 at a 400 W power limit) without a kernel being wrong."""
    worst = 0.0
    for N in (1, 17, 129, 257):
        c = _self(d, dt, N)
        q, k, v = A.inputs(c)
        exp = _expect(c, q, k, v)
        rep = A.check(A.round_to(exp.ref, dt), exp)
        assert rep.ok, f"rejects the rounded reference on {c}: {rep}"
        rep = A.check(A.emulate(q, k, v, c.H, c.Hkv, dt), exp)
        print(f"[ratio] float32 emulation on {c}: {rep}")
        assert rep.ok and rep.ratio <= 0.8, f"emulation on {c}: {rep}"
        worst = max(worst, rep.ratio)
    print(f"[ratio] float32 emulation, d {d} {dt}: worst {worst:.3g}")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [64, 128])
def test_rejects_key_mask_errors(d, dt):
    """17 keys (a last tile of 17 in both kernels): the last key dropped (mask at Nk - 1), one zero key admitted
    past Nk, and the last key of item 0 read from item 1 (a row past Nk of a dense batch)."""
    c = _self(d, dt, 17)
    q, k, v = A.inputs(c)
    exp = _expect(c, q, k, v)
    _assert_rejects(c, exp, "last key dropped", A.round_to(_expect(c, q, k[:, :-1], v[:, :-1]).ref, dt))
    z = torch.zeros_like(k[:, :1])
    _assert_rejects(c, exp, "zero key admitted", A.round_to(
        _expect(c, q, torch.cat([k, z], 1), torch.cat([v, z], 1)).ref, dt))
    k2, v2 = k.clone(), v.clone()
    k2[0, -1], v2[0, -1] = k[1, -1], v[1, -1]
    _assert_rejects(c, exp, "last key from the next item", A.round_to(_expect(c, q, k2, v2).ref, dt))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [64, 128])
def test_rejects_a_missing_rescale(d, dt):
    """129 keys: the max_last heads move the row max in the last (one-key) tile; O not rescaled there."""
    c = _self(d, dt, 129)
    q, k, v = A.inputs(c)
    exp = _expect(c, q, k, v)
    last = (c.Nk - 1) // A.key_tile(d)
    _assert_rejects(c, exp, "O not rescaled on the last tile", A.emulate(q, k, v, c.H, c.Hkv, dt, skip_rescale_tile=last))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [64, 128])
def test_rejects_the_wrong_kv_head(d, dt):
    """Cross-attention layout, 24 / 12 heads, 17 context tokens: kv head h % Hkv instead of h / group."""
    c = _cross(d, dt, 17)
    q, k, v = A.inputs(c)
    exp = _expect(c, q, k, v)
    idx = torch.tensor([h % c.Hkv for h in range(c.H)])
    per_head = lambda t: t.view(c.B, c.Nk, c.Hkv, d)[:, :, idx].reshape(c.B, c.Nk, c.H * d)
    _assert_rejects(c, exp, "kv head h % Hkv", A.round_to(_expect(c, q, per_head(k), per_head(v), c.H, c.H).ref, dt))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [96, 128])
def test_rejects_the_head_dim_64_scale(d, dt):
    """1 / 8 instead of 1 / sqrt(d): the scores of a head-dim-64 kernel applied to 96 / 128."""
    c = _self(d, dt, 17)
    q, k, v = A.inputs(c)
    exp = _expect(c, q, k, v)
    _assert_rejects(c, exp, "scale 1/8", A.round_to(_expect(c, q.double() * (d ** 0.5 / 8), k, v).ref, dt))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", [64, 128])
def test_rejects_misplaced_outputs(d, dt):
    """257 query rows: row 0 given the output of row 64 (the other consumer of a wgmma CTA, the next attn_kernel
    CTA) or of row 128 (the next CTA); head 0's output written into head 1's columns."""
    c = _self(d, dt, 257)
    q, k, v = A.inputs(c)
    exp = _expect(c, q, k, v)
    good = A.round_to(exp.ref, dt)
    for off in (64, 128):
        bad = good.clone()
        bad[:, 0] = good[:, off]
        _assert_rejects(c, exp, f"row 0 <- row {off}", bad)
    bad = good.clone()
    bad[..., d:2 * d] = good[..., :d]
    _assert_rejects(c, exp, "head 0 into head 1's columns", bad)
