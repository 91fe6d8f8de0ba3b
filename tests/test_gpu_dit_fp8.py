"""GPU: the DiT's FP8 operand mode (operand_dtype "fp8": e4m3 operands with power-of-two row scales for the
self-attention QKV, cross-attention q and feed-forward input GEMMs).

1. The FP8 LayerNorm (satb_layernorm_fp8) against an fp64 LayerNorm: the row scales follow the rule of
   tests/fp8_ref.py, every dequantised element is within half an e4m3 ulp (plus the fp32 LayerNorm slack).
2. Every FP8 GEMM instance the forward launches (satb_gemm_probe_fp8) against the fp64 product of the dequantised
   operands, through the epilogue references of tests/gemm_epilogue_ref.py.
3. The forward in FP8 mode against the FP8 floor: rel-L2 to the fp32 oracle <= 1.25 x the rel-L2 of the oracle's own
   FP8 emulation (fp8_ref.fp8_operands) to the fp32 oracle.
4. Bit checks: the CUDA-graph call equals the eager call, a batch of 4 equals the same prompts inside a batch of 5.
Measured numbers are printed as `FP8 {...}` JSON lines (pytest -s)."""
import ctypes
import json
import math

import pytest
import torch

import gemm_epilogue_ref as ger
from fp8_ref import fp8_operands, fp8_row_exponent, quantize_fp8_rows
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu


def report(name, **kw):
    print("FP8 " + json.dumps(dict(test=name, **kw)), flush=True)


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


# ------------------------------------------------------------------------------------------------ 1. LayerNorm
def _e4m3_half_ulp(u):
    """Half an e4m3 ulp at |u| (u in scaled units, |u| <= 448): 2^(floor(log2 |u|) - 4) for normals (>= 2^-6),
    2^-10 in the subnormal range."""
    a = u.abs().clamp_min(2.0 ** -6)
    return torch.ldexp(torch.ones_like(a), torch.floor(torch.log2(a)).to(torch.int32) - 4)


@pytest.mark.parametrize("D", [256, 1536])
@pytest.mark.parametrize("adaln", [False, True])
def test_layernorm_fp8_vs_fp64(D, adaln):
    nat, lib = _lib()
    rows, items = 1025, 3
    g = torch.Generator(device="cuda").manual_seed(D + adaln)
    x = torch.randn(rows, D, device="cuda", generator=g) * 3 + 0.5
    x[7] = 0.0                                                            # constant row: y = beta
    x[11] *= 1e-4
    gamma = 1 + 0.3 * torch.randn(D, device="cuda", generator=g)
    beta = 0.1 * torch.randn(D, device="cuda", generator=g)
    gamma[:8] = 0.0
    ld = 6 * D
    mod = torch.randn(items, ld, device="cuda", generator=g) * 0.5 if adaln else None
    out8 = torch.empty(rows, D, dtype=torch.uint8, device="cuda")
    scale = torch.empty(rows, device="cuda")
    rpi = 400
    nat.check(lib.satb_layernorm_fp8(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                     mod.data_ptr() if adaln else None, mod[:, D:].data_ptr() if adaln else None,
                                     ld, rpi, items, out8.data_ptr(), scale.data_ptr(), rows, D, nat.stream_ptr()))
    torch.cuda.synchronize()
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    y = (xd - mu) / torch.sqrt(((xd - mu) ** 2).mean(-1, keepdim=True) + 1e-5) * gamma.double() + beta.double()
    slack_terms = y.abs() + 1
    if adaln:
        item = (torch.arange(rows, device="cuda") // rpi) % items
        sc, sh = mod[item, :D].double(), mod[item, D:2 * D].double()
        y = y * (1 + sc) + sh
        slack_terms = slack_terms * (1 + sc.abs()) + sh.abs()
    amax = y.abs().amax(-1)
    e_want = fp8_row_exponent(amax)
    s_got = scale.double()
    near = ((amax / (448.0 * torch.ldexp(torch.ones_like(amax), e_want)) - 1).abs() < 1e-6) | \
           ((amax / (224.0 * torch.ldexp(torch.ones_like(amax), e_want)) - 1).abs() < 1e-6)
    ok_scale = (s_got == torch.ldexp(torch.ones_like(amax), e_want)) | near
    assert bool(ok_scale.all()), f"row scales off the rule at rows {torch.nonzero(~ok_scale)[:8].flatten().tolist()}"
    dq = out8.view(torch.float8_e4m3fn).double() * s_got[:, None]
    bound = _e4m3_half_ulp(y / s_got[:, None]) * s_got[:, None] + 1e-5 * slack_terms
    err = (dq - y).abs()
    ratio = float((err / bound).max())
    report("layernorm_fp8", D=D, adaln=adaln, max_err_over_bound=ratio, rows_near_boundary=int(near.sum()))
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------ 2. GEMM probes
# FP8 wgmma accumulates in fp32, but with fewer addend bits than the 16-bit path (it is reported to align addends
# to about 13 mantissa bits).  Bound per output: |got - ref| <= e_acc8(K) * sum_k |a w| (through the epilogue's
# sensitivity) + the epilogue's own fp32 terms + half an fp16 ulp of the result.
def e_acc8(K):
    return (math.ceil(K / 32) + 1) * 2.0 ** -13


def _check8(got, exp, K):
    got = got.double()
    bound = (1 + ger.E_OUT["fp16"]) * (e_acc8(K) * exp.sens + ger.E_EPI * exp.mag) + ger.E_OUT["fp16"] * exp.ref.abs() \
        + ger.TAU["fp16"]
    err = (got - exp.ref).abs()
    assert torch.isfinite(got).all()
    # the accumulation error actually seen, relative to sum |a w| (output rounding removed)
    acc_err = ((err - ger.E_OUT["fp16"] * exp.ref.abs()).clamp_min(0) / exp.sens.clamp_min(1e-30))
    return float((err / bound).max()), float(acc_err.max())


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.exp(torch.randn(M, 1, device="cuda", generator=g))
    w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5 * torch.exp(0.5 * torch.randn(N, 1, device="cuda",
                                                                                               generator=g))
    qa, sa = quantize_fp8_rows(a)
    qw, sw = quantize_fp8_rows(w)
    ad, wd = qa.double() * sa.double(), qw.double() * sw.double()
    return (qa.view(torch.uint8).contiguous(), sa[:, 0].contiguous(), qw.view(torch.uint8).contiguous(),
            sw[:, 0].contiguous(), ad @ wd.T, ad.abs() @ wd.abs().T)


def _probe(M, N, K, a8, sa, w8, sw, bn, b_static, **f):
    nat, lib = _lib()
    p = nat.SatbGemmProbe()
    p.bn, p.bf16, p.b_static = bn, 0, b_static
    for k, v in f.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    nat.check(lib.satb_gemm_probe_fp8(a8.data_ptr(), w8.data_ptr(), sa.data_ptr(), sw.data_ptr(), M, N, K,
                                      ctypes.byref(p), nat.stream_ptr()))


CASES = [  # (name, epi, bn, M, N, K): N with a partial last tile where the instance allows one, ragged M
    ("qkv_rope", "qkv", 256, 1025, 960, 384), ("qkv_rope_bench", "qkv", 256, 8200, 4608, 1536),
    ("swiglu", "swiglu", 256, 1025, 1216, 384), ("swiglu_bench", "swiglu", 256, 8200, 12288, 1536),
    ("store16_bn128", "store16", 128, 1025, 480, 256), ("store16_bn256", "store16", 256, 1025, 480, 256),
    ("store16_cross_q", "store16", 128, 2050, 1536, 1536),
    ("head_norm16_bn128", "head_norm", 128, 1025, 960, 384),
]


@pytest.mark.parametrize("name,epi,bn,M,N,K", CASES, ids=[c[0] for c in CASES])
def test_gemm_probe_fp8_vs_fp64(name, epi, bn, M, N, K):
    nat, _ = _lib()
    a8, sa, w8, sw, acc, S = _operands(M, N, K, seed=M + N + K)
    g = torch.Generator(device="cuda").manual_seed(5)
    seq = 1025
    if epi == "qkv" or epi == "head_norm":
        D = N // 3
        cos, sin, freqs = ger.rope_tables(seq, 16)
        fr = ger.row_freqs(freqs, M, seq).cuda()
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        if epi == "qkv":
            f = dict(epi=nat.EPI_QKV_ROPE, out=out, ld=N, rope_cols=2 * D, seq_len=seq, head_dim=64, nf=16,
                     cos_tab=cos.cuda(), sin_tab=sin.cuda())
            exp = ger.epi_qkv_rope(acc, S, fr, 64, 16, 2 * D)
        else:
            f = dict(epi=nat.EPI_HEAD_NORM16, out=out, ld=N, norm_cols=2 * D, rope_cols=2 * D, seq_len=seq,
                     cos_tab=cos.cuda(), sin_tab=sin.cuda())
            exp = ger.epi_head_norm(acc, S, 2 * D, 2 * D, fr)
    elif epi == "swiglu":
        # weights / bias stored 32 / 32 value / gate interleaved (csrc/dit.cu ff_perm); the output is in reference order
        perm = ger.ff_perm(N // 2).cuda()
        bias = torch.randn(N, device="cuda", generator=g) * 0.1
        out = torch.empty(M, N // 2, dtype=torch.float16, device="cuda")
        f = dict(epi=nat.EPI_SWIGLU, out=out, ld=N // 2, bias=bias[perm].contiguous())
        w8, sw = w8[perm].contiguous(), sw[perm].contiguous()
        exp = ger.epi_swiglu(acc, S, bias)                     # acc in reference order (the rows before the perm)
    else:
        bias = torch.randn(N, device="cuda", generator=g) * 0.1
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        f = dict(epi=nat.EPI_STORE16, out=out, ld=N, bias=bias, act=1)
        exp = ger.epi_store(acc, S, bias, act=1)
    _probe(M, N, K, a8, sa, w8, sw, bn, 1, **f)
    first = out.clone()
    _probe(M, N, K, a8, sa, w8, sw, bn, 1, **f)
    again = out.clone()
    out.fill_(0)
    _probe(M, N, K, a8, sa, w8, sw, bn, 0, **f)
    torch.cuda.synchronize()
    assert torch.equal(first, again), "repeated calls differ"
    assert torch.equal(first, out), "b_static 0 and 1 differ"
    ratio, acc_rel = _check8(first, exp, K)
    report("gemm_probe_fp8", case=name, M=M, N=N, K=K, bn=bn, max_err_over_bound=ratio,
           max_acc_err_over_sum_abs_aw=acc_rel, e_acc8=e_acc8(K))
    assert ratio <= 1.0


def test_gemm_probe_fp8_refuses_other_instances():
    nat, lib = _lib()
    a8 = torch.zeros(128, 256, dtype=torch.uint8, device="cuda")
    s = torch.ones(256, device="cuda")
    out = torch.empty(128, 256, dtype=torch.float32, device="cuda")
    for epi, bn, bf16, K in [(nat.EPI_STORE32, 256, 0, 256), (nat.EPI_RESIDUAL, 128, 0, 256),
                             (nat.EPI_HEAD_NORM16, 256, 0, 256), (nat.EPI_QKV_ROPE, 128, 0, 256),
                             (nat.EPI_STORE16, 128, 1, 256), (nat.EPI_STORE16, 128, 0, 192)]:
        p = nat.SatbGemmProbe()
        p.epi, p.bn, p.bf16, p.out, p.ld, p.h, p.head_dim, p.nf = epi, bn, bf16, out.data_ptr(), 256, out.data_ptr(), 64, 16
        rc = lib.satb_gemm_probe_fp8(a8.data_ptr(), a8.data_ptr(), s.data_ptr(), s.data_ptr(), 128, 256, K,
                                     ctypes.byref(p), nat.stream_ptr())
        assert rc != 0, (epi, bn, bf16, K)


# ------------------------------------------------------------------------------------------------ 3. forward
GOLDEN_CONFIGS = ["dit_hd32_small.npz", "dit_prepend_small.npz", "dit_hd96_small.npz", "dit_hd128_small.npz",
                  "dit_adaln_small.npz", "dit_hd128_adaln_small.npz", "dit_qknorm_small.npz",
                  "dit_concat_prepend_small.npz"]


def _floor_and_native(cfg, sd, m, kw, device):
    from oracle import dit_oracle as do
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = do.dit_forward(sdd, cfg, **kwd)
    with fp8_operands(sdd):
        emu = do.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDEN_CONFIGS)
def test_forward_fp8_small_configs_vs_fp8_floor(name):
    from oracle import dit_oracle as do
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = do.make_dit_weights(cfg, seed=int(g["seed"]))
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    T = lambda k: torch.from_numpy(g[k])
    base = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "concat" in g:
        base.update(input_concat_cond=T("concat"), prepend_cond=T("prepend"))
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu")
        report("forward_fp8_small", config=name, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
        assert err <= 1.25 * floor, (name, cfg_scale, err, floor)


@pytest.mark.parametrize("cfg_scale", [1.0, 7.0])
def test_forward_fp8_sa_open_width_24_blocks_vs_fp8_floor(cfg_scale):
    """SA-Open width, all 24 blocks, 1024 latents + the prepend token = 1025 tokens; the oracle runs on the GPU in fp32
    (no TF32), its FP8 emulation likewise."""
    from oracle import dit_oracle as do
    assert not torch.backends.cuda.matmul.allow_tf32
    sd = do.make_dit_weights(SAO_DIT, seed=31)
    m = build_native_dit(SAO_DIT, sd, operand_dtype="fp8")
    g = torch.Generator().manual_seed(32)
    x, t = torch.randn(1, 64, 1024, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    c[:, 40:] = 0.0
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(SAO_DIT, sd, m, kw, "cuda")
    m16 = build_native_dit(SAO_DIT, sd)
    y16 = m16(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    y8 = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    report("forward_fp8_sa_open", cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor,
           rel_l2_fp8_vs_fp16=rel_l2(y8.cpu(), y16.cpu()))
    assert err <= 1.25 * floor, (cfg_scale, err, floor)


# ------------------------------------------------------------------------------------------------ 4. bit checks
def test_fp8_cuda_graph_call_equals_the_eager_call():
    from oracle import dit_oracle as do
    g = load_golden("dit_qknorm_small.npz")
    cfg = json.loads(str(g["cfg"]))
    sd = do.make_dit_weights(cfg, seed=int(g["seed"]))
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    T = lambda k: torch.from_numpy(g[k]).cuda()
    x, t, c, ge = T("x"), T("t"), T("cross"), T("glob")
    eager = lambda xx: m(xx, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    y0 = eager(x)
    m.cuda_graph = True
    y1 = eager(x)
    y2 = eager(x * 0.5)
    m.cuda_graph = False
    assert torch.equal(y0, y1)
    assert torch.equal(y2, eager(x * 0.5))


def test_fp8_batch_of_4_equals_the_same_prompts_in_a_batch_of_5():
    from oracle import dit_oracle as do
    sd = do.make_dit_weights(SAO_DIT, seed=33)
    m = build_native_dit(SAO_DIT, sd, operand_dtype="fp8")
    g = torch.Generator().manual_seed(34)
    x, t = torch.randn(5, 64, 1024, generator=g).cuda(), (torch.rand(5, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(5, 130, 768, generator=g).cuda(), torch.randn(5, 1536, generator=g).cuda()
    sub = lambda a, b: dict(cross_attn_cond=c[a:b].contiguous(), global_embed=ge[a:b].contiguous(), cfg_scale=7.0)
    y5 = m(x, t, **sub(0, 5)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(0, 4)).clone()
    report("fp8_batch_invariance", bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)
