"""GPU: the epilogues that run on the wgmma accumulator fragment (EpiSwiglu, EpiResidual: no staging through shared
memory, so their instances get a deeper ring than the staged epilogues), against the float64 reference of
tests/gemm_epilogue_ref.py, at K one k-block deeper than that ring, ragged M tails and partial row pairs (row0 valid,
row0 + 8 past M), with NaN / known-value guards; two identical calls must give the same bits, and b_static 0 and 1
too."""
import pytest
import torch

import gemm_epilogue_ref as R
from test_gpu_gemm_epilogues import DTS, GUARD_COLS, GUARD_ROWS, INT_VIEW, assert_guard, guarded, operands, probe, report, \
    swiglu_weight

pytestmark = pytest.mark.gpu


def fragment_stages(bn):
    """GemmCfg::kStages of an instance without accumulator staging (csrc/gemm.cuh)."""
    return min(8, (227 * 1024 - 1024 - 256) // (R.BLOCK_M * R.BLOCK_K * 2 + bn * R.BLOCK_K * 2))


def _bits(t):
    return t.view(INT_VIEW[t.dtype])


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("M", [1, 9, 1025, 8200])
def test_swiglu_deep_k(dt, M):
    from stable_audio_tools import _native as nat
    D = 256
    ffi, K = 4 * D, 64 * (fragment_stages(256) + 1)
    N = 2 * ffi
    tdt = R.TORCH_DT[dt]
    g = torch.Generator().manual_seed(M)
    w_ref = torch.randn(N, K, generator=g) * K ** -0.5
    w_ref[ffi:] *= 8.0
    perm = R.ff_perm(ffi)
    w_ref, w_st = w_ref.to(tdt).cuda(), w_ref[perm].to(tdt).cuda()
    a = torch.randn(M, K, generator=g).to(tdt).cuda()
    bias_ref = (torch.randn(N, generator=g) * 0.5).cuda()
    bias_st = bias_ref[perm.cuda()].contiguous()
    outs = []
    for b_static in (1, 1, 0):
        out = guarded(M, ffi, tdt)
        before = out.clone()
        probe(dt, nat.EPI_SWIGLU, 256, a, w_st, M, N, K, b_static=b_static, out=out, ld=out.shape[1], bias=bias_st)
        assert_guard(out, before, M, ffi, "swiglu")
        outs.append(out)
    acc, S = R.accumulate(a, w_ref)
    report(f"swiglu {dt} M{M} K{K}", R.check(outs[0][:M, :ffi], R.epi_swiglu(acc, S, bias_ref), K, dt, 256, 2))
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "two identical calls differ"
    assert torch.equal(_bits(outs[0]), _bits(outs[2])), "b_static 0 and 1 differ"


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("M", [1, 9, 1025])
def test_residual_deep_k(dt, bn, M):
    from stable_audio_tools import _native as nat
    N, K, rpi, B = 640, 64 * (fragment_stages(bn) + 1), 7, 2
    a, w, g = operands(dt, M, N, K, seed=M + bn)
    bias = torch.randn(N, device="cuda", generator=g) * 0.5
    gate = torch.rand(4, N, device="cuda", generator=g) + 0.2
    h0 = torch.randn(M + GUARD_ROWS, N + GUARD_COLS, device="cuda", generator=g)
    hs = []
    for b_static in (1, 1, 0):
        h = guarded(M, N, torch.float32, h0)
        probe(dt, nat.EPI_RESIDUAL, bn, a, w, M, N, K, b_static=b_static, h=h, ld=h.shape[1], bias=bias, gate=gate,
              rows_per_item=rpi, gate_ld=N, n_items=B)
        assert_guard(h, h0, M, N, "residual")
        hs.append(h)
    acc, S = R.accumulate(a, w)
    gr = R.gate_rows(gate, M, rpi, B)
    report(f"residual {dt} BN{bn} M{M} K{K}", R.check(hs[0][:M, :N], R.epi_residual(acc, S, h0[:M, :N], bias, gr), K,
                                                      "fp32", bn))
    assert torch.equal(hs[0], hs[1]), "two identical calls differ"
    assert torch.equal(hs[0], hs[2]), "b_static 0 and 1 differ"
