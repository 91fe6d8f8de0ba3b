"""GPU: attention head dims 32, 96 and 128.  The attention core through satb_attention_hd against the oracle, the
drop-in DiffusionTransformer against golden outputs of the real reference (tests/golden/dit_hd*.npz) and against the
live oracle at SA-Open width, and the CUDA-graph replay.  Tolerances are those of test_gpu_dit.py /
test_gpu_primitives.py."""
import json
import math

import pytest
import torch

from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu

TOL = {"fp16": 2e-3, "bf16": 1.5e-2}


def tol(dtype, cfg_scale=1.0):
    return TOL[dtype] * max(1.0, cfg_scale / 1.5)


def _attention_hd(q, k, v, B, H, Hkv, Nq, Nk, D, bf16):
    from stable_audio_tools import _native as nat
    o = torch.full((B, Nq, H * D), float("nan"), dtype=q.dtype, device="cuda")
    nat.check(nat.lib().satb_attention_hd(nat.ptr(q), nat.ptr(k), nat.ptr(v), nat.ptr(o), B, H, Hkv, Nq, Nk, D, bf16,
                                          nat.stream_ptr()))
    return o


def _oracle_attention(q, k, v, B, H, Hkv, Nq, D):
    from oracle.dit_oracle import attention_core
    heads = lambda t, h: t.float().cpu().view(t.shape[0], t.shape[1], h, D).permute(0, 2, 1, 3)
    return attention_core(heads(q, H), heads(k, Hkv), heads(v, Hkv)).permute(0, 2, 1, 3).reshape(B, Nq, H * D)


@pytest.mark.parametrize("D", [32, 96, 128])
@pytest.mark.parametrize("B,H,Hkv,Nq,Nk", [(2, 4, 4, 1025, 1025), (1, 12, 6, 1025, 130), (2, 4, 2, 128, 2),
                                           (1, 2, 1, 2, 130), (1, 3, 3, 65, 191)])
def test_attention_hd_vs_oracle(D, B, H, Hkv, Nq, Nk):
    """softmax(q k^T / sqrt(D)) v: ragged query tiles (1025 rows), GQA with a ragged key tile (130 keys), a 2-key
    problem, fewer query rows than a tile; fp16 operands."""
    torch.manual_seed(Nq * 7 + Nk + D)
    q = (torch.randn(B, Nq, H * D) * 1.5).half().cuda()
    k = (torch.randn(B, Nk, Hkv * D) * 1.5).half().cuda()
    v = torch.randn(B, Nk, Hkv * D).half().cuda()
    o = _attention_hd(q, k, v, B, H, Hkv, Nq, Nk, D, 0)
    assert rel_l2(o.float().cpu(), _oracle_attention(q, k, v, B, H, Hkv, Nq, D)) < 2e-3


@pytest.mark.parametrize("D", [32, 96, 128])
def test_attention_hd_bf16_vs_oracle(D):
    B, H, Hkv, Nq, Nk = 2, 4, 2, 300, 257
    torch.manual_seed(D)
    q = (torch.randn(B, Nq, H * D) * 1.5).bfloat16().cuda()
    k = (torch.randn(B, Nk, Hkv * D) * 1.5).bfloat16().cuda()
    v = torch.randn(B, Nk, Hkv * D).bfloat16().cuda()
    o = _attention_hd(q, k, v, B, H, Hkv, Nq, Nk, D, 1)
    assert rel_l2(o.float().cpu(), _oracle_attention(q, k, v, B, H, Hkv, Nq, D)) < 1.5e-2


@pytest.mark.parametrize("D", [32, 96, 128])
@pytest.mark.parametrize("Nk", [700, 641])
def test_attention_hd_lazy_rescale_path_monotone_scores(D, Nk):
    """As test_gpu_primitives.py's monotone case: the running max moves in every 64-key tile (head 0), or sits in
    the first tile (head 1); logits / sqrt(D) grow by 0.25 per key at every D.  Nk = 641: a last tile of one key."""
    B, H, Nq = 1, 2, 200
    torch.manual_seed(0)
    q = torch.zeros(B, Nq, H * D)
    k = torch.zeros(B, Nk, H * D)
    q[..., 0::D] = 4.0
    ramp = torch.arange(Nk, dtype=torch.float32) * 0.5 * math.sqrt(D) / 8.0
    k[:, :, 0] = ramp
    k[:, :, D] = ramp.flip(0)
    q = q + 0.05 * torch.randn_like(q)
    v = torch.randn(B, Nk, H * D)
    q, k, v = q.half().cuda(), k.half().cuda(), v.half().cuda()
    o = _attention_hd(q, k, v, B, H, H, Nq, Nk, D, 0)
    assert torch.isfinite(o).all()
    assert rel_l2(o.float().cpu(), _oracle_attention(q, k, v, B, H, H, Nq, D)) < 2e-3


@pytest.mark.parametrize("bf16", [0, 1])
def test_attention_hd_64_gives_the_bits_of_satb_attention(bf16):
    from stable_audio_tools import _native as nat
    B, H, Hkv, Nq, Nk = 2, 24, 12, 1025, 1025
    dt = torch.bfloat16 if bf16 else torch.float16
    torch.manual_seed(1)
    q = (torch.randn(B, Nq, H * 64, device="cuda") * 1.5).to(dt)
    k = (torch.randn(B, Nk, Hkv * 64, device="cuda") * 1.5).to(dt)
    v = torch.randn(B, Nk, Hkv * 64, device="cuda").to(dt)
    o64 = torch.empty(B, Nq, H * 64, dtype=dt, device="cuda")
    nat.check(nat.lib().satb_attention(nat.ptr(q), nat.ptr(k), nat.ptr(v), nat.ptr(o64), B, H, Hkv, Nq, Nk, bf16,
                                       nat.stream_ptr()))
    assert torch.equal(_attention_hd(q, k, v, B, H, Hkv, Nq, Nk, 64, bf16), o64)


def test_attention_hd_rejects_other_head_dims():
    from stable_audio_tools import _native as nat
    q = torch.zeros(1, 64, 2 * 48, dtype=torch.float16, device="cuda")
    rc = nat.lib().satb_attention_hd(nat.ptr(q), nat.ptr(q), nat.ptr(q), nat.ptr(q), 1, 2, 2, 64, 64, 48, 0,
                                     nat.stream_ptr())
    assert rc != 0 and b"head dim" in nat.lib().satb_last_error()


def _golden_case(name):
    from oracle import dit_oracle as do
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = do.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), "synthetic weight RNG drifted from the golden run"
    return g, cfg, sd


@pytest.mark.parametrize("name", ["dit_hd128_small.npz", "dit_hd96_small.npz", "dit_hd32_small.npz",
                                  "dit_hd128_adaln_small.npz"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_dit_head_dims_vs_reference_golden(name, dtype):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    T = lambda k: torch.from_numpy(g[k]).cuda()
    x, t, c, ge, neg = T("x"), T("t"), T("cross"), T("glob"), T("neg")
    cases = {
        "y_nocfg": dict(cfg_scale=1.0),
        "y_cfg7": dict(cfg_scale=7.0),
        "y_cfg4_phi": dict(cfg_scale=4.0, scale_phi=0.7),
        "y_neg3": dict(cfg_scale=3.0, negative_cross_attn_cond=neg),
    }
    for key, kw in cases.items():
        y = m(x, t, cross_attn_cond=c, global_embed=ge, **kw).cpu()
        err = rel_l2(y, torch.from_numpy(g[key]))
        assert err < tol(dtype, kw["cfg_scale"]), f"{name} {key} {dtype}: rel l2 {err}"
    y, info = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=1.0, return_info=True)
    hid = info["hidden_states"][-1].cpu()
    err = rel_l2(hid, torch.from_numpy(g["hidden_last"]))
    assert err < TOL[dtype], f"{name} hidden {dtype}: rel l2 {err}"


@pytest.mark.parametrize("num_heads,cfg_scale", [(12, 7.0), (16, 1.0), (16, 7.0)])   # head dim 128, 96, 96
def test_dit_full_width_other_head_dims_vs_oracle(num_heads, cfg_scale):
    """SA-Open width (D=1536) with 12 heads of 128 or 16 heads of 96, a 130x768 context (6 or 8 kv heads), 1024
    latents + the prepend token, depth 2, B=2, against the CPU oracle computed live (fp32)."""
    from oracle import dit_oracle as do
    cfg = dict(SAO_DIT, depth=2, num_heads=num_heads)
    sd = do.make_dit_weights(cfg, seed=30 + num_heads)
    torch.manual_seed(2)
    B = 2
    x = torch.randn(B, 64, 1024)
    t = torch.rand(B) * 0.9 + 0.05
    c = torch.randn(B, 130, 768)
    c[:, 40:128] = 0.0   # padded T5 rows are exact zeros in the real pipeline (conditioners.py:343-344)
    ge = torch.randn(B, 1536)
    ref = do.dit_forward(sd, cfg, x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    m = build_native_dit(cfg, sd)
    y = m(x.cuda(), t.cuda(), cross_attn_cond=c.cuda(), global_embed=ge.cuda(), cfg_scale=cfg_scale).cpu()
    err = rel_l2(y, ref)
    assert err < tol("fp16", cfg_scale), f"rel l2 {err}"


def test_dit_head_dim_128_cuda_graph_call_equals_the_eager_call():
    g, cfg, sd = _golden_case("dit_hd128_small.npz")
    m = build_native_dit(cfg, sd)
    T = lambda k: torch.from_numpy(g[k]).cuda()
    x, t, c, ge = T("x"), T("t"), T("cross"), T("glob")
    eager = lambda xx: m(xx, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    y0 = eager(x)
    m.cuda_graph = True
    assert torch.equal(eager(x), y0)                      # capture + replay
    x2 = x * 0.5 + 0.1
    y2 = eager(x2)                                        # replay with new inputs
    m.cuda_graph = False
    assert torch.equal(y2, eager(x2))
