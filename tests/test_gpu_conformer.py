"""GPU: DiTs built with conformer blocks (conformer=True, reference models/transformer.py:557-591).

1. conformer_dwconv_ln_silu through satb_conformer_dwconv against an fp64 reference, element by element.  Bound per
   output y = silu(z), z = mid_norm(conv(g)):
       |got - y| <= E16 |y| + 2^-24 + 1.1 (1e-5 (1 + |z|) + 64 u |gamma| rstd Smax)
   E16 = 2^-11 (fp16) / 2^-8 (bf16): rounding of the 16-bit output; u = 2^-24; Smax = the row's largest
   sum_k |w_k g_{r+k-8}| (the fp32 convolution's error, carried through the normalisation); 1e-5 (1 + |z|): the fp32
   mean / variance / rsqrt; 1.1 bounds silu'.
2. The DiT against the reference goldens (tests/golden/dit_conformer*.npz) at the gates of test_gpu_dit.py: rel-L2
   2e-3 (x max(1, cfg / 1.5) with CFG) in fp16, 1.5e-2 in bf16; the FP8 mode within 1.25 x its emulated floor
   (tests/fp8_ref.py: the conformer GEMMs fp16-rounded there, as they run).
3. SA-Open width (1536 wide, 24 heads, 1025 tokens, 2 blocks) against the oracle's fp16-operand floor.
4. Bit checks: the CUDA-graph call equals the eager call; a batch of 4 equals the same prompts inside a batch of 5.
Measured numbers are printed as `CONFORMER {...}` JSON lines (pytest -s)."""
import ctypes
import json

import pytest
import torch
import torch.nn.functional as F

from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu

GOLDENS = ["dit_conformer_small.npz", "dit_conformer_adaln_small.npz", "dit_conformer_hd128_small.npz"]
TOL = {"fp16": 2e-3, "bf16": 1.5e-2}
E16 = {0: 2.0 ** -11, 1: 2.0 ** -8}


def report(name, **kw):
    print("CONFORMER " + json.dumps(dict(test=name, **kw)), flush=True)


# ------------------------------------------------------------------------------------------------ 1. the kernel
def _run_kernel(g16, w, gamma, beta, items, n, D, bf16):
    from stable_audio_tools import _native as nat
    out = torch.full_like(g16, float("nan"))
    nat.check(nat.lib().satb_conformer_dwconv(g16.data_ptr(), w.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                              out.data_ptr(), items, n, D, bf16, nat.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _reference(g, w, gamma, beta, n, D):
    """fp64 per item: y, z and the bound terms."""
    x = g.double().view(-1, n, D).transpose(1, 2)
    wd = w.double()
    c = F.conv1d(x, wd, padding=8, groups=D).transpose(1, 2)
    S = F.conv1d(x.abs(), wd.abs(), padding=8, groups=D).transpose(1, 2)
    mu = c.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((c - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    z = (c - mu) * rstd * gamma.double() + beta.double()
    y = z * torch.sigmoid(z)
    slack = 1.1 * (1e-5 * (1 + z.abs()) + 64 * 2.0 ** -24 * gamma.double().abs() * rstd * S.amax(-1, keepdim=True))
    return y.reshape(-1, D), slack.reshape(-1, D)


def _operands(items, n, D, seed, dt):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    g = (torch.randn(items * n, D, device="cuda", generator=gen) * 0.6).to(dt)
    w = torch.randn(D, 1, 17, device="cuda", generator=gen) / 17 ** 0.5
    gamma = 1 + 0.3 * torch.randn(D, device="cuda", generator=gen)
    beta = 0.1 * torch.randn(D, device="cuda", generator=gen)
    return g, w, gamma, beta


def _check(got, y, slack, bf16, rows=None):
    got, y, slack = got.double(), y, slack
    if rows is not None:
        got, y, slack = got[rows], y[rows], slack[rows]
    bound = E16[bf16] * y.abs() + 2.0 ** -24 + slack
    err = (got - y).abs()
    assert torch.isfinite(got).all()
    return float((err / bound).max())


@pytest.mark.parametrize("D", [256, 384, 1536])
@pytest.mark.parametrize("n", [1, 5, 16, 17, 33, 1025])
def test_dwconv_kernel_vs_fp64(D, n):
    """3 items of n rows: every row of every item against its own item's zero-padded convolution, so a read across an
    item boundary shows as an error on the rows near it."""
    items = 3
    g, w, gamma, beta = _operands(items, n, D, seed=D * 7 + n, dt=torch.float16)
    if n == 1025:
        g[n + 300:n + 340] = 0   # item 1: the convolution is exactly 0 on rows 308..331: a constant row, variance 0
    got = _run_kernel(g, w, gamma, beta, items, n, D, 0)
    y, slack = _reference(g, w, gamma, beta, n, D)
    ratio = _check(got, y, slack, 0)
    report("dwconv_kernel", D=D, n=n, bf16=0, max_err_over_bound=ratio)
    assert ratio <= 1.0
    if n == 1025:   # the constant rows come out as silu(beta) exactly (up to the 16-bit rounding)
        r = slice(n + 308, n + 332)
        want = (beta.double() * torch.sigmoid(beta.double())).expand(24, D)
        assert float(((got[r].double() - want).abs() - E16[0] * want.abs()).max()) <= 2.0 ** -24


@pytest.mark.parametrize("D", [384, 1536])
@pytest.mark.parametrize("n", [17, 1025])
def test_dwconv_kernel_bf16_vs_fp64(D, n):
    g, w, gamma, beta = _operands(2, n, D, seed=D + n, dt=torch.bfloat16)
    got = _run_kernel(g, w, gamma, beta, 2, n, D, 1)
    y, slack = _reference(g, w, gamma, beta, n, D)
    ratio = _check(got, y, slack, 1)
    report("dwconv_kernel", D=D, n=n, bf16=1, max_err_over_bound=ratio)
    assert ratio <= 1.0


@pytest.mark.parametrize("D", [256, 1536])
@pytest.mark.parametrize("n", [5, 33, 1025])
def test_dwconv_kernel_never_reads_a_neighbouring_item(D, n):
    """Items 0 and 2 hold NaN (a sentinel any read would carry into a convolution sum): item 1 must still equal its
    zero-padded reference, and be finite."""
    items = 3
    g, w, gamma, beta = _operands(items, n, D, seed=D + 3 * n, dt=torch.float16)
    g[:n] = float("nan")
    g[2 * n:] = float("nan")
    got = _run_kernel(g, w, gamma, beta, items, n, D, 0)
    y, slack = _reference(g[n:2 * n], w, gamma, beta, n, D)
    ratio = _check(got[n:2 * n], y, slack, 0)
    report("dwconv_sentinel", D=D, n=n, max_err_over_bound=ratio)
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------ 2. the DiT
def _golden_case(name):
    from oracle import conformer_oracle as co
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = co.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), "synthetic weight RNG drifted from the golden run"
    return g, cfg, sd


@pytest.mark.parametrize("name", GOLDENS)
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_dit_conformer_vs_reference_golden(name, dtype):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    T = lambda k: torch.from_numpy(g[k]).cuda()
    x, t, c, ge, neg = T("x"), T("t"), T("cross"), T("glob"), T("neg")
    cases = {"y_nocfg": dict(cfg_scale=1.0), "y_cfg7": dict(cfg_scale=7.0),
             "y_cfg4_phi": dict(cfg_scale=4.0, scale_phi=0.7),
             "y_neg3": dict(cfg_scale=3.0, negative_cross_attn_cond=neg)}
    for key, kw in cases.items():
        y = m(x, t, cross_attn_cond=c, global_embed=ge, **kw).cpu()
        err = rel_l2(y, torch.from_numpy(g[key]))
        report("dit_golden", config=name, dtype=dtype, case=key, rel_l2=err)
        assert err < TOL[dtype] * max(1.0, kw["cfg_scale"] / 1.5), f"{name} {key} {dtype}: rel l2 {err}"
    y, info = m(x, t, cross_attn_cond=c, global_embed=ge, cfg_scale=1.0, return_info=True)
    err = rel_l2(info["hidden_states"][-1].cpu(), torch.from_numpy(g["hidden_last"]))
    assert err < TOL[dtype], f"{name} hidden {dtype}: rel l2 {err}"


def _floor_and_native(cfg, sd, m, kw, device, floor_ctx):
    from oracle import conformer_oracle as co
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = co.dit_forward(sdd, cfg, **kwd)
    with floor_ctx(sdd):
        emu = co.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDENS)
def test_dit_conformer_fp8_vs_fp8_floor(name):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    T = lambda k: torch.from_numpy(g[k])
    base = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", fp8_operands)
        report("dit_fp8", config=name, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
        assert err <= 1.25 * floor, (name, cfg_scale, err, floor)


@pytest.mark.parametrize("cfg_scale", [1.0, 7.0])
def test_dit_conformer_sa_open_width_vs_fp16_floor(cfg_scale):
    """1536 wide, 24 heads, 1024 latents + the prepend token = 1025 tokens, 2 blocks; the oracle runs on the GPU in fp32
    (no TF32), its fp16-operand emulation likewise."""
    from oracle import conformer_oracle as co
    from oracle import dit_oracle as do
    assert not torch.backends.cuda.matmul.allow_tf32
    cfg = dict(SAO_DIT, depth=2, conformer=True)
    sd = co.make_dit_weights(cfg, seed=50)
    m = build_native_dit(cfg, sd)
    g = torch.Generator().manual_seed(51)
    x, t = torch.randn(1, 64, 1024, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    c[:, 40:] = 0.0
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(cfg, sd, m, kw, "cuda", lambda sdd: do.operand_rounding(torch.float16))
    report("dit_sa_open", cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
    assert err <= 1.25 * floor, (cfg_scale, err, floor)


def test_finalize_with_a_conformer_tensor_missing_fails_with_a_message():
    from stable_audio_tools import _native as nat
    from stable_audio_tools.models.dit import DiffusionTransformer
    g, cfg, sd = _golden_case("dit_conformer_small.npz")
    lib = nat.lib()
    h = ctypes.c_void_p()
    nat.check(lib.satb_dit_create(ctypes.byref(DiffusionTransformer(**cfg).native_config()), ctypes.byref(h)))
    try:
        nat.check(lib.satb_dit_set_conformer(h, 1))
        st = nat.stream_ptr()
        for k, v in sd.items():
            if k == "transformer.layers.1.conformer.glu.proj.weight":
                continue
            src = v.cuda().contiguous()
            nat.check(lib.satb_dit_load_weight(h, k.encode(), src.data_ptr(), src.numel(), st))
            torch.cuda.synchronize()
        rc = lib.satb_dit_finalize(h, st)
        msg = lib.satb_last_error()
        assert rc != 0 and b"conformer weights missing in layer 1" in msg
        assert lib.satb_dit_set_conformer(h, 0) != 0 and b"before the first weight" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


# ------------------------------------------------------------------------------------------------ 4. bit checks
def test_conformer_cuda_graph_call_equals_the_eager_call():
    g, cfg, sd = _golden_case("dit_conformer_small.npz")
    m = build_native_dit(cfg, sd)
    T = lambda k: torch.from_numpy(g[k]).cuda()
    x, t, c, ge = T("x"), T("t"), T("cross"), T("glob")
    eager = lambda xx: m(xx, t, cross_attn_cond=c, global_embed=ge, cfg_scale=7.0).clone()
    y0 = eager(x)
    m.cuda_graph = True
    y1 = eager(x)
    y2 = eager(x * 0.5 + 0.1)
    m.cuda_graph = False
    assert torch.equal(y0, y1)
    assert torch.equal(y2, eager(x * 0.5 + 0.1))


def test_conformer_batch_of_4_equals_the_same_prompts_in_a_batch_of_5():
    from oracle import conformer_oracle as co
    cfg = dict(SAO_DIT, depth=2, conformer=True)
    sd = co.make_dit_weights(cfg, seed=52)
    m = build_native_dit(cfg, sd)
    g = torch.Generator().manual_seed(53)
    x, t = torch.randn(5, 64, 1024, generator=g).cuda(), (torch.rand(5, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(5, 130, 768, generator=g).cuda(), torch.randn(5, 1536, generator=g).cuda()
    sub = lambda a, b: dict(cross_attn_cond=c[a:b].contiguous(), global_embed=ge[a:b].contiguous(), cfg_scale=7.0)
    y5 = m(x, t, **sub(0, 5)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(0, 4)).clone()
    report("batch_invariance", bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)
