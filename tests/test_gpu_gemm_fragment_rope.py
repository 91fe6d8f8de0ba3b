"""GPU: EpiQkvRope on the wgmma accumulator fragment, element by element against the same accumulator.

The fp32 accumulator of a (BN, K) schedule does not depend on the epilogue, so each case runs the same A and W through
the EpiStore32 probe at BN 256 to get the accumulator bits, applies the rotary to them on the GPU and rounds to the
16-bit type.  The rotary is the kernel's: a' = fma(a, c, -fl32(b s)), b' = fma(a, s, fl32(b c)), with the fused
multiply-add emulated in float64 (the product of two floats is exact there).  Every rotated element must lie within one
16-bit ulp of that, and all but a double-rounding tie must match it bit for bit; every unrotated element (v columns,
pairs past n_rot, head dims past 2 nf) must be the accumulator rounded once.  Guard rows and columns stay NaN.

Head dims 32 / 64 / 96 (whose chunk 1 rotates 8 pairs) / 128 at widths with a partial last n-tile, M from one row to
the bench's 8200, items of 33 tokens (position 0 falls between the two fragment rows r and r + 8 of many threads) and
of 1025."""
import pytest
import torch

import gemm_epilogue_ref as R
from test_gpu_gemm_epilogues import INT_VIEW, assert_guard, guarded, probe

pytestmark = pytest.mark.gpu

DTS = ["fp16", "bf16"]
# head dim -> model width D: 3 D is not a multiple of 256 (the last n-tile is partial), D a multiple of the head dim
WIDTH = {32: 640, 64: 640, 96: 672, 128: 640}


def rope_reference(acc, D, head_dim, nf, seq, cos, sin):
    """acc [M, 3 D] fp32 (stored column order) -> (fp32 result of the kernel's rotary, mask of rotated elements)."""
    M, N = acc.shape
    dev = acc.device
    col = torch.arange(N, device=dev)
    s = col % head_dim
    ci, w = s // 32, s % 32
    i = w % 16
    rot = (col < 2 * D) & (i < (nf - 16 * ci).clamp(0, 16))
    first = w < 16                                       # column i of pair (i, i + 16), else column i + 16
    a_col = torch.where(first, col, col - 16)
    tcol = torch.where(rot, 16 * ci + i, torch.zeros_like(col))
    pos = torch.arange(M, device=dev) % seq
    c, sn = cos[pos][:, tcol], sin[pos][:, tcol]
    a, b = acc[:, a_col], acc[:, a_col + 16]
    f = first.unsqueeze(0)
    prod = torch.where(f, -(b * sn), b * c)              # fp32 products, rounded
    mul = torch.where(f, c, sn)
    val = (a.double() * mul.double() + prod.double()).float()
    return torch.where(rot.unsqueeze(0), val, acc), rot


def ordered(x):
    """16-bit values -> integers in the order of the values, one apart per ulp (+0 and -0 both 0)."""
    v = x.view(torch.int16).int()
    return torch.where(v < 0, -(v & 0x7FFF), v)


CASES = [(hd, M, 33) for hd in (32, 64, 96, 128) for M in (1, 8, 9, 129, 8200)]
CASES += [(64, 8200, 1025), (96, 1025, 1025)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("head_dim,M,seq", CASES)
def test_fragment_rope_against_accumulator(dt, head_dim, M, seq):
    from stable_audio_tools import _native as nat
    D = WIDTH[head_dim]
    nf = R.rope_nf(head_dim)
    N, K = 3 * D, D
    tdt = R.TORCH_DT[dt]
    g = torch.Generator(device="cuda").manual_seed(1000 * head_dim + M + seq)
    a = torch.randn(M, K, device="cuda", generator=g).to(tdt)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(tdt)
    cos, sin, _ = R.rope_tables(seq, nf)
    cos, sin = cos.cuda(), sin.cuda()

    acc = torch.empty(M, N, device="cuda")
    probe(dt, nat.EPI_STORE32, 256, a, w, M, N, K, out=acc, ld=N)
    out = guarded(M, N, tdt)
    before = out.clone()
    probe(dt, nat.EPI_QKV_ROPE, 256, a, w, M, N, K, out=out, ld=out.shape[1], rope_cols=2 * D, seq_len=seq,
          head_dim=head_dim, nf=nf, cos_tab=cos, sin_tab=sin)
    assert_guard(out, before, M, N, "qkv_rope")

    ref32, rot = rope_reference(acc, D, head_dim, nf, seq, cos, sin)
    ref = ref32.to(tdt)
    got = out[:M, :N]
    iv = INT_VIEW[tdt]
    keep = ~rot.unsqueeze(0).expand(M, N)
    assert torch.equal(got[keep].view(iv), ref[keep].view(iv)), "an unrotated element is not the rounded accumulator"
    rg, rr = got[~keep], ref[~keep]
    assert torch.isfinite(rg.float()).all(), "non-finite rotated element"
    dist = (ordered(rg) - ordered(rr)).abs()
    worst = int(dist.max()) if dist.numel() else 0
    n_diff = int((dist != 0).sum())
    print(f"[rope] {dt} hd{head_dim} M{M} seq{seq}: {rg.numel()} rotated, {n_diff} differ, worst {worst} ulp")
    assert worst <= 1, f"a rotated element is {worst} 16-bit ulps from the reference"
    assert n_diff <= 2, f"{n_diff} rotated elements differ from the kernel's fused multiply-add"
