"""GPU parity tests for the stand-alone primitives, through the C ABI (ctypes)."""
import ctypes

import pytest
import torch

from helpers import load_golden, max_abs, rel_l2

pytestmark = pytest.mark.gpu


def _native():
    from stable_audio_tools import _native
    return _native


def test_snake_beta_matches_reference_golden():
    """SnakeBeta vs the reference module's output (models/blocks.py:330-358); fp32, <= a few ulp of sinf."""
    from stable_audio_tools.models.blocks import SnakeBeta
    g = load_golden("snake_beta.npz")
    sn = SnakeBeta(24)
    with torch.no_grad():
        sn.alpha.copy_(torch.from_numpy(g["alpha"]))
        sn.beta.copy_(torch.from_numpy(g["beta"]))
    sn = sn.cuda()
    y = sn(torch.from_numpy(g["x"]).cuda()).cpu()
    ref = torch.from_numpy(g["y"])
    assert max_abs(y, ref) <= 2e-6 * float(ref.abs().max())


@pytest.mark.parametrize("T", [1, 7, 4096, 65537])
def test_snake_beta_ragged_lengths_vs_oracle(T):
    from oracle.oobleck_oracle import snake_beta
    nat = _native()
    torch.manual_seed(T)
    x = torch.randn(2, 5, T) * 4
    a, b = torch.randn(5) * 0.4, torch.randn(5) * 0.4
    xd, ad, bd = x.cuda(), a.cuda(), b.cuda()
    y = torch.empty_like(xd)
    nat.check(nat.lib().satb_snake_beta(nat.ptr(xd), nat.ptr(ad), nat.ptr(bd), nat.ptr(y), 2, 5,
                                        ctypes.c_longlong(T), 1, nat.stream_ptr()))
    ref = snake_beta(x, a, b)
    assert max_abs(y.cpu(), ref) <= 3e-6 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("rows,D", [(1, 128), (1025, 1536), (8200, 1536), (77, 256)])
def test_layernorm_vs_torch(rows, D):
    nat = _native()
    torch.manual_seed(0)
    x = (torch.randn(rows, D) * 3 + 0.5).cuda()
    g = (1 + 0.1 * torch.randn(D)).cuda()
    b = (0.1 * torch.randn(D)).cuda()
    out = torch.empty(rows, D, dtype=torch.float16, device="cuda")
    nat.check(nat.lib().satb_layernorm(nat.ptr(x), nat.ptr(g), nat.ptr(b), nat.ptr(out), rows, D, 0, nat.stream_ptr()))
    ref = torch.nn.functional.layer_norm(x, (D,), g, b, 1e-5)
    # fp16 output rounding: 2^-11 relative
    assert rel_l2(out.float(), ref) < 5e-4


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (1, 64, 64), (1025, 1536, 1536), (8200, 4608, 1536),
                                   (333, 128, 768), (2050, 64, 1536), (520, 768, 768), (300, 1536, 6144),
                                   (129, 384, 200)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_tcgen05_linear_vs_torch(M, N, K, bf16):
    """wgmma GEMM (TMA ring, fp32 register accumulators) vs torch matmul on the same 16-bit operands."""
    nat = _native()
    torch.manual_seed(M + N + K)
    dt = torch.bfloat16 if bf16 else torch.float16
    a = torch.randn(M, K, device="cuda").to(dt)
    w = (torch.randn(N, K, device="cuda") * 0.05).to(dt)
    c = torch.full((M, N), float("nan"), device="cuda")
    nat.check(nat.lib().satb_linear_f32out(nat.ptr(a), nat.ptr(w), nat.ptr(c), M, N, K, bf16, nat.stream_ptr()))
    ref = a.double() @ w.double().T
    err = rel_l2(c, ref)
    assert err < 1e-5, f"rel l2 {err}"


@pytest.mark.parametrize("B,H,Hkv,Nq,Nk", [(2, 4, 4, 1025, 1025), (1, 24, 12, 1025, 130), (2, 2, 1, 64, 1),
                                           (1, 3, 3, 65, 191), (1, 24, 24, 300, 300),
                                           # ragged query and key tiles (130 / 257); fewer query rows than one tile;
                                           # a key tile with only 2 keys; many CTAs per (item, head)
                                           (1, 2, 2, 130, 257), (1, 2, 1, 2, 130), (2, 4, 2, 128, 2), (3, 24, 24, 1024, 384),
                                           # small batch at the SA-Open length: the 1025th query row and the 1025th key
                                           # each in a tile of their own
                                           (2, 24, 24, 1025, 1025)])
def test_attention_vs_oracle(B, H, Hkv, Nq, Nk):
    """softmax(q k^T / 8) v vs the oracle's einsum path (models/transformer.py:510-536), fp16 operands."""
    from oracle.dit_oracle import attention_core
    nat = _native()
    torch.manual_seed(Nq * 7 + Nk)
    q = torch.randn(B, Nq, H * 64) * 1.5
    k = torch.randn(B, Nk, Hkv * 64) * 1.5
    v = torch.randn(B, Nk, Hkv * 64)
    qh, kh, vh = q.half(), k.half(), v.half()
    o = torch.empty(B, Nq, H * 64, dtype=torch.float16, device="cuda")
    qd, kd, vd = qh.cuda(), kh.cuda(), vh.cuda()
    nat.check(nat.lib().satb_attention(nat.ptr(qd), nat.ptr(kd), nat.ptr(vd), nat.ptr(o), B, H, Hkv, Nq, Nk, 0,
                                       nat.stream_ptr()))
    heads = lambda t, h: t.float().view(t.shape[0], t.shape[1], h, 64).permute(0, 2, 1, 3)
    ref = attention_core(heads(qh, H), heads(kh, Hkv), heads(vh, Hkv)).permute(0, 2, 1, 3).reshape(B, Nq, H * 64)
    assert rel_l2(o.float().cpu(), ref) < 2e-3


@pytest.mark.parametrize("Nk", [700, 641])
def test_attention_lazy_rescale_path_monotone_scores(Nk):
    """Scores that keep growing along the key axis force the running max to move in every 64-key tile: exercises
    the O rescale of the online softmax.  Nk = 641 = 10 x 64 + 1: the last, one-key tile (the other 63 rows
    zero-filled and masked) holds the row maximum of head 0 and rescales everything before it."""
    from oracle.dit_oracle import attention_core
    nat = _native()
    B, H, Nq = 1, 2, 200
    torch.manual_seed(0)
    q = torch.zeros(B, Nq, H * 64)
    k = torch.zeros(B, Nk, H * 64)
    q[..., 0::64] = 4.0                                   # q . k = 4 * k[..., 0]
    ramp = torch.arange(Nk, dtype=torch.float32) * 0.5    # logits / 8 grow by 0.25 per key (23 log2 units per tile)
    k[:, :, 0] = ramp
    k[:, :, 64] = ramp.flip(0)                            # second head: decreasing (max in the first tile)
    q = q + 0.05 * torch.randn_like(q)
    v = torch.randn(B, Nk, H * 64)
    qh, kh, vh = q.half(), k.half(), v.half()
    o = torch.empty(B, Nq, H * 64, dtype=torch.float16, device="cuda")
    qd, kd, vd = qh.cuda(), kh.cuda(), vh.cuda()
    nat.check(nat.lib().satb_attention(nat.ptr(qd), nat.ptr(kd), nat.ptr(vd), nat.ptr(o), B, H, H, Nq, Nk, 0, nat.stream_ptr()))
    heads = lambda t, h: t.float().view(t.shape[0], t.shape[1], h, 64).permute(0, 2, 1, 3)
    ref = attention_core(heads(qh, H), heads(kh, H), heads(vh, H)).permute(0, 2, 1, 3).reshape(B, Nq, H * 64)
    assert torch.isfinite(o).all()
    assert rel_l2(o.float().cpu(), ref) < 2e-3
