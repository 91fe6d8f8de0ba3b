"""GPU: the head-dim-64 attention kernel (wgmma, TMA-fed K / V ring, two ping-pong consumer warpgroups) through
satb_attention, on what the existing cases do not reach: bf16, every key-tail width of the last 128-key tile, query
tails around the two 64-row consumers of a 128-row CTA (a CTA whose second consumer has no rows: Nq = 1, 64, 129,
1025), GQA at the cross-attention shape, the rows around the output, and bit reproducibility (also across head dims
and the operand layouts of the DiT forward).  Tolerances are those of test_gpu_primitives.py / test_gpu_head_dims.py."""
import pytest
import torch

from helpers import rel_l2

pytestmark = pytest.mark.gpu

TOL = {0: 2e-3, 1: 1.5e-2}
DT = {0: torch.float16, 1: torch.bfloat16}
GUARD = 4096   # NaN-filled elements before and after the output


def _inputs(B, H, Hkv, Nq, Nk, bf16, seed, D=64):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, Nq, H * D, generator=g) * 1.5).to(DT[bf16]).cuda()
    k = (torch.randn(B, Nk, Hkv * D, generator=g) * 1.5).to(DT[bf16]).cuda()
    v = torch.randn(B, Nk, Hkv * D, generator=g).to(DT[bf16]).cuda()
    return q, k, v


def _attention(q, k, v, B, H, Hkv, Nq, Nk, bf16):
    """Runs satb_attention into the middle of a NaN-filled buffer; returns (o, the whole buffer)."""
    from stable_audio_tools import _native as nat
    n = B * Nq * H * 64
    buf = torch.full((GUARD + n + GUARD,), float("nan"), dtype=DT[bf16], device="cuda")
    o = buf[GUARD:GUARD + n].view(B, Nq, H * 64)
    nat.check(nat.lib().satb_attention(nat.ptr(q), nat.ptr(k), nat.ptr(v), nat.ptr(o), B, H, Hkv, Nq, Nk, bf16,
                                       nat.stream_ptr()))
    torch.cuda.synchronize()
    return o, buf


def _oracle(q, k, v, B, H, Hkv, Nq):
    from oracle.dit_oracle import attention_core
    heads = lambda t, h: t.float().cpu().view(t.shape[0], t.shape[1], h, 64).permute(0, 2, 1, 3)
    return attention_core(heads(q, H), heads(k, Hkv), heads(v, Hkv)).permute(0, 2, 1, 3).reshape(B, Nq, H * 64)


def _check(B, H, Hkv, Nq, Nk, bf16, seed):
    q, k, v = _inputs(B, H, Hkv, Nq, Nk, bf16, seed)
    o, buf = _attention(q, k, v, B, H, Hkv, Nq, Nk, bf16)
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all(), "write outside the output"
    assert torch.isfinite(o).all(), "output element not written"
    err = rel_l2(o.float().cpu(), _oracle(q, k, v, B, H, Hkv, Nq))
    assert err < TOL[bf16], f"rel l2 {err}"


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("Nk", [1, 2, 16, 17, 33, 64, 80, 96, 112, 127, 128, 129, 130, 224, 240, 1025])
def test_key_tails(Nk, bf16):
    """Last key tile of every width class: 1 .. 128 keys issued at 16 (1, 2, 16), 32 (17), 48 (33), 64, 80, 96, 112
    and 128 (127, 128) columns, and after a full tile at 16 (129, 130, 1025), 96 (224) and 112 (240); Nq = 129 adds a
    1-row CTA."""
    _check(2, 3, 3, 129, Nk, bf16, seed=Nk)


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("Nq", [1, 64, 65, 128, 129, 1025])
def test_query_tails(Nq, bf16):
    """Nq = 1, 64, 129, 1025: the last CTA's second consumer has no rows; 65, 128: both consumers have rows."""
    _check(2, 3, 3, Nq, 257, bf16, seed=1000 + Nq)


@pytest.mark.parametrize("bf16", [0, 1])
def test_gqa_group2_cross_attention_shape(bf16):
    """Cross-attention shape: GQA group 2, 130 keys (a full tile plus 2 keys)."""
    _check(2, 4, 2, 1025, 130, bf16, seed=7)


@pytest.mark.parametrize("bf16", [0, 1])
def test_two_calls_give_the_same_bits(bf16):
    B, H, Nq, Nk = 2, 4, 1025, 1025
    q, k, v = _inputs(B, H, H, Nq, Nk, bf16, seed=3)
    o1, _ = _attention(q, k, v, B, H, H, Nq, Nk, bf16)
    o2, _ = _attention(q, k, v, B, H, H, Nq, Nk, bf16)
    assert torch.equal(o1, o2)


# (bf16, head dim, layout of the batched run); the first two are satb_attention itself
_BITS = [pytest.param(bf16, 64, "dense", id=str(bf16)) for bf16 in (0, 1)] + [
    pytest.param(bf16, D, layout, id=f"{bf16}-hd{D}-{layout}") for layout in ("dense", "self", "cross")
    for D in (32, 64, 96, 128) for bf16 in (0, 1) if (D, layout) != (64, "dense")]


@pytest.mark.parametrize("bf16,D,layout", _BITS)
def test_one_head_alone_gives_the_bits_it_gets_in_a_batch(bf16, D, layout):
    """Item 1, head 2 of a 3 x 4-head batch (GQA group 2; group 1 in the fused QKV layout) against the same (item,
    head) run as a batch of one with one head through the contiguous layout: other CTA, other head offset and batch
    offset, and (attention_ref.run) the fused QKV or fused KV operand layout of the DiT forward, same bits."""
    import attention_ref as A
    B, H, Nq, Nk = 3, 4, 1025, 1025
    Hkv = H if layout == "self" else 2
    q, k, v = _inputs(B, H, Hkv, Nq, Nk, bf16, seed=11, D=D)
    dt = "bf16" if bf16 else "fp16"
    if D == 64 and layout == "dense":
        o, _ = _attention(q, k, v, B, H, Hkv, Nq, Nk, bf16)
    else:
        o = A.run(A.Case(layout, D, dt, B, H, Hkv, Nq, Nk), q, k, v)
    b, h = 1, 2
    hk = h // (H // Hkv)
    q1 = q[b:b + 1, :, h * D:(h + 1) * D].contiguous()
    k1 = k[b:b + 1, :, hk * D:(hk + 1) * D].contiguous()
    v1 = v[b:b + 1, :, hk * D:(hk + 1) * D].contiguous()
    if D == 64:
        o1, _ = _attention(q1, k1, v1, 1, 1, 1, Nq, Nk, bf16)
    else:
        o1 = A.run(A.Case("dense", D, dt, 1, 1, 1, Nq, Nk), q1, k1, v1)
    assert torch.equal(o1[0], o[b, :, h * D:(h + 1) * D])
