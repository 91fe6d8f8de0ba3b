"""CPU: the per-element checker of tests/gemm_epilogue_ref.py is sharp.  For every fused GEMM epilogue at small shapes
(head dim 96, a 33-token sequence) it accepts the float64 reference rounded to the output type and rejects the
output of a subtly wrong kernel, restated here as a mutation of the reference.  This is the evidence, without a GPU,
that the GPU tests of tests/test_gpu_gemm_epilogues.py fail on such kernels."""
import pytest
import torch

import gemm_epilogue_ref as R

M, K = 300, 200        # three row tiles, the last one ragged; 13 k-blocks of 16 with a ragged last 64-block
OUTS = ["fp16", "bf16"]


def _operands(out, N, seed=0, k=K, m=M):
    g = torch.Generator().manual_seed(seed)
    dt = R.TORCH_DT[out]
    a = torch.randn(m, k, generator=g).to(dt)
    w = (torch.randn(N, k, generator=g) * k ** -0.5).to(dt)
    return a, w, g


def _assert_sharp(out, K_, exp, good, bad, bn=256, col_scale=1):
    rep = R.check(good, exp, K_, out, bn, col_scale)
    assert rep.ok, f"rejects the rounded reference: {rep}"
    for name, b in bad.items():
        rep = R.check(b, exp, K_, out, bn, col_scale)
        assert not rep.ok, f"accepts the mutation '{name}': {rep}"


@pytest.mark.parametrize("out", OUTS + ["fp32"])
def test_store_epilogue(out):
    """EpiStore16 (act 0 / 1) and EpiStore32: a dropped k-block, a row taken from the next tile, a bias chunk lost."""
    N = 256
    a, w, g = _operands("fp16" if out == "fp32" else out, N)
    acc, S = R.accumulate(a, w)
    bias = torch.randn(N, generator=g) * 0.5
    for act in ((0,) if out == "fp32" else (0, 1)):
        exp = R.epi_store(acc, S, bias, act)
        good = R.round_to(exp.ref, out)
        a_drop = a.clone()
        a_drop[:, 64:128] = 0
        acc_drop, _ = R.accumulate(a_drop, w)
        row = good.clone()
        row[5] = good[5 + 128]
        b_lost = bias.clone()
        b_lost[96:128] = 0
        bad = {"k-block dropped": R.round_to(R.epi_store(acc_drop, S, bias, act).ref, out),
               "row off by one tile": row,
               "bias missing on one chunk": R.round_to(R.epi_store(acc, S, b_lost, act).ref, out)}
        _assert_sharp(out, K, exp, good, bad)


@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("head_dim", [64, 96])
def test_qkv_rope_epilogue(out, head_dim):
    """EpiQkvRope over a 33-token sequence (every 128-row tile spans several items): the rotary position one off, the
    rotation by -theta, and (head dim 96, nf 24) the table read with a row stride of 16."""
    D = 2 * head_dim * (1 if head_dim == 96 else 2)
    nf = R.rope_nf(head_dim)
    seq = 33
    a, w, _ = _operands(out, 3 * D)
    acc, S = R.accumulate(a, w)
    cos, sin, freqs = R.rope_tables(seq, nf)
    fr = R.row_freqs(freqs, M, seq)
    exp = R.epi_qkv_rope(acc, S, fr, head_dim, nf, 2 * D)
    good = R.round_to(exp.ref, out)
    mut = lambda f: R.round_to(R.epi_qkv_rope(acc, S, f, head_dim, nf, 2 * D).ref, out)
    bad = {"position (row + 1) % seq_len": mut(freqs[(torch.arange(M) + 1) % seq]),
           "rotation by -theta": mut(-fr)}
    if nf != 16:
        flat = freqs[:, :nf].reshape(-1)
        idx = (torch.arange(M) % seq)[:, None] * 16 + torch.arange(nf)[None, :]
        f16 = flat[idx]
        bad["pair stride 16 where nf = 24"] = mut(torch.cat([f16, f16], -1))
    # the v columns pass through: a kernel that rotated them too is caught
    v_rot = exp.ref.clone()
    v_rot[:, 2 * D:] = R.epi_qkv_rope(acc[:, D:], S[:, D:], fr, head_dim, nf, 2 * D).ref[:, D:]
    bad["v columns rotated"] = R.round_to(v_rot, out)
    _assert_sharp(out, K, exp, good, bad)


def test_qkv_head_perm_matches_its_comment():
    """Head dim 96 (nf 24): chunk 0 = [0..15 | 24..39], chunk 1 = [16..23, 48..55 | 40..47, 56..63], 64..95; head dims
    32 and 64 give the identity; v rows are untouched."""
    p = R.qkv_head_perm(192, 96, 24)
    want = list(range(16)) + list(range(24, 40)) + list(range(16, 24)) + list(range(48, 56)) + \
        list(range(40, 48)) + list(range(56, 64)) + list(range(64, 96))
    assert p[:96].tolist() == want and p[96:192].tolist() == [96 + x for x in want]
    assert p[384:].tolist() == list(range(384, 576))
    assert R.qkv_head_perm(256, 64, 16).tolist() == list(range(768))
    assert R.qkv_head_perm(256, 32, 16).tolist() == list(range(768))
    assert R.ff_perm(128)[:70].tolist() == list(range(32)) + list(range(128, 160)) + list(range(32, 38))


@pytest.mark.parametrize("out", OUTS)
def test_head_norm_epilogue(out):
    """EpiHeadNorm16: the qk norm taken over one 32-column half instead of the whole 64-column head."""
    D = 128
    a, w, _ = _operands(out, 3 * D)
    w[64:128] = 0                                   # one all-zero head: the 1e-12 clamp
    acc, S = R.accumulate(a, w)
    cos, sin, freqs = R.rope_tables(33, 16)
    fr = R.row_freqs(freqs, M, 33)
    exp = R.epi_head_norm(acc, S, 2 * D, 2 * D, fr)
    good = R.round_to(exp.ref, out)
    assert torch.all(good[:, 64:128] == 0)
    bad = {"norm over 32 columns": R.round_to(R.epi_head_norm(acc, S, 2 * D, 2 * D, fr, norm_width=32).ref, out),
           "rotary position one off": R.round_to(R.epi_head_norm(acc, S, 2 * D, 2 * D, R.row_freqs(freqs, M + 1, 33)[1:]).ref, out)}
    _assert_sharp(out, K, exp, good, bad)


@pytest.mark.parametrize("out", OUTS)
def test_swiglu_epilogue(out):
    """EpiSwiglu with gate pre-activations out to +-20: value and gate swapped, a bias chunk lost."""
    ffi = 128
    a, w, g = _operands(out, 2 * ffi)
    w[ffi:] *= 6                                    # gate pre-activations into the __expf tails
    bias = torch.randn(2 * ffi, generator=g) * 0.5
    acc, S = R.accumulate(a, w)
    exp = R.epi_swiglu(acc, S, bias)
    good = R.round_to(exp.ref, out)
    sw = lambda t: torch.cat([t[..., ffi:], t[..., :ffi]], -1)
    b_lost = bias.clone()
    b_lost[32:64] = 0
    bad = {"value and gate swapped": R.round_to(R.epi_swiglu(sw(acc), sw(S), sw(bias)).ref, out),
           "bias missing on one chunk": R.round_to(R.epi_swiglu(acc, S, b_lost).ref, out)}
    _assert_sharp(out, K, exp, good, bad, col_scale=2)


def test_residual_epilogue():
    """EpiResidual with the adaLN gate over R = 4 CFG rows of 75 tokens, B = 2 items: the item index without % n_items."""
    N, rpi, B = 256, 75, 2
    a, w, g = _operands("fp16", N)
    acc, S = R.accumulate(a, w)
    h = torch.randn(M, N, generator=g, dtype=torch.float64).float()
    bias = torch.randn(N, generator=g) * 0.5
    gate = torch.rand(4, N, generator=g) + 0.2      # 4 rows: the unwrapped (wrong) index finds other values
    exp = R.epi_residual(acc, S, h, bias, R.gate_rows(gate, M, rpi, B))
    good = R.round_to(exp.ref, "fp32")
    unwrapped = gate[torch.arange(M) // rpi]
    bad = {"gate item without % n_items": R.round_to(R.epi_residual(acc, S, h, bias, unwrapped).ref, "fp32"),
           "gate missing": R.round_to(R.epi_residual(acc, S, h, bias, None).ref, "fp32")}
    _assert_sharp("fp32", K, exp, good, bad)

