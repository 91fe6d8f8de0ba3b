"""GPU: both attention kernels (attn_wgmma_kernel, head dim 64; attn_kernel<D>, head dims 32 / 96 / 128) element by
element against the float64 reference and bound of tests/attention_ref.py, at the operand layouts the DiT forward
passes (csrc/dit.cu: self-attention reads q, k and v as column ranges 0 / Hd / 2Hd of one fused QKV buffer;
cross-attention reads q from its own buffer and k, v as columns 0 / Hkv d of one KV buffer, 24 / 12 heads) through
satb_attention_probe, and at the contiguous layout of satb_attention_hd.  Every operand and the output sit inside
NaN-filled guards (attention_ref.run), every valid element must be finite and within the bound, and every element of
the output buffer outside the output must keep its bits.  The reference runs on the device, one head at a time; every
case prints its worst err/bound."""
import pytest
import torch

import attention_ref as A

pytestmark = pytest.mark.gpu

DTS = ["fp16", "bf16"]
DIMS = [32, 64, 96, 128]


def _check(case):
    q, k, v = A.inputs(case)
    got = A.run(case, q, k, v)
    exp = A.expect(q.to(got.device), k.to(got.device), v.to(got.device), case.H, case.Hkv, case.dt)
    rep = A.check(got, exp)
    print(f"[ratio] {case}: {rep}")
    assert rep.ok, f"{case}: {rep}"


@pytest.mark.parametrize("N", [1, 2, 17, 33, 64, 65, 81, 97, 127, 128, 129, 224, 240, 257, 1025])
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", DIMS)
def test_self_attention_fused_qkv(d, dt, N):
    """Fused QKV layout, 2 items x 7 heads (one per score distribution), N_seq query and key rows: every query tail
    class of both kernels, and every width at which attn_wgmma_kernel issues its last key tile, alone (1, 2: 16;
    17: 32; 33: 48; 64: 64; 65: 80; 81: 96; 97: 112; 127, 128: 128) and after a full tile (224: 96; 240: 112;
    129, 257, 1025: 16)."""
    _check(A.Case("self", d, dt, 2, 7, 7, N, N))


@pytest.mark.parametrize("Mctx", [1, 16, 17, 128, 129, 130])
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", DIMS)
def test_cross_attention_fused_kv(d, dt, Mctx):
    """Cross-attention layout with GQA group 2 (24 / 12 heads), 129 query rows (a last CTA of one row)."""
    _check(A.Case("cross", d, dt, 2, 24, 12, 129, Mctx))


@pytest.mark.parametrize("Nq,Nk", [(65, 257), (1025, 130)])
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", DIMS)
def test_contiguous_layout(d, dt, Nq, Nk):
    """satb_attention_hd's contiguous [B, N, H d] operands (a row past Nk of item b is row 0 of item b + 1), GQA
    group 2."""
    _check(A.Case("dense", d, dt, 2, 14, 7, Nq, Nk))


@pytest.mark.parametrize("dt", DTS)
def test_bench_shape(dt):
    """The self-attention of the benchmark: 8 rows (4 items under CFG) x 24 heads x 1025 tokens, head dim 64."""
    _check(A.Case("self", 64, dt, 8, 24, 24, 1025, 1025))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("d", DIMS)
def test_sa20_length(d, dt):
    """6145 tokens (49 key tiles of 128: the 4-stage K / V ring wraps 12 times; 97 tiles of 64)."""
    _check(A.Case("self", d, dt, 2, 7, 7, 6145, 6145))
