"""GPU: DiTs built with the reference's other feed-forward options (ff_kwargs; reference models/transformer.py:211-287).

1. The token convolution through satb_token_conv_probe (the forward's GEMM launch, both epilogues, fp16 and bf16)
   against float64, element by element, with the bound of tests/gemm_epilogue_ref.py over the k K-deep reduction; NaN
   rows between the items must never be read, and a reference whose taps are shifted by one is rejected on the
   kernel's own output.
2. The DiT against the reference goldens (tests/golden/dit_ff_*.npz) at the gates of test_gpu_dit.py: rel-L2 2e-3
   (x max(1, cfg / 1.5) with CFG) in fp16, 1.5e-2 in bf16; the FP8 mode within 1.25 x its emulated floor
   (tests/fp8_ref.py, with a plain Linear FF-in on e4m3 operands like the SwiGLU one, and a convolutional FF-in in
   fp16, as they run).
3. SA-Open width (1536 wide, 24 heads, 1025 tokens, 2 blocks) for mult 8/3, SwiGLU + Conv1d k 3 and plain Conv1d k 3
   against the oracle's fp16-operand floor.
4. Bit checks: the CUDA-graph call equals the eager call; a batch of 4 equals the same prompts inside a batch of 5.
Measured numbers are printed as `FFVAR {...}` JSON lines (pytest -s)."""
import ctypes
import json

import pytest
import torch
import torch.nn.functional as F

import gemm_epilogue_ref as ger
from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu

GOLDENS = ["dit_ff_mult83_small.npz", "dit_ff_glu_conv3_nobias_small.npz", "dit_ff_conv5_adaln_hd128_small.npz",
           "dit_ff_plain_nobias_hd32_small.npz", "dit_ff_conformer_conv3_small.npz"]
TOL = {"fp16": 2e-3, "bf16": 1.5e-2}
SA_OPEN_FF = {"mult83": dict(mult=8 / 3), "swiglu_conv3": dict(use_conv=True, conv_kernel_size=3),
              "plain_conv3": dict(glu=False, use_conv=True, conv_kernel_size=3)}


def report(name, **kw):
    print("FFVAR " + json.dumps(dict(test=name, **kw)), flush=True)


# ------------------------------------------------------------------------------------------------ 1. the probe
def _unfold(a, k, shift=0):
    """a [R, n, K] (float64) -> [R n, k K]: row (r, l) holds a[r, l + t - k // 2 + shift] for t = 0..k-1 (zeros
    outside the item)."""
    R, n, K = a.shape
    p = k // 2 + 1
    ap = F.pad(a, (0, 0, p, p))
    return torch.cat([ap[:, 1 + t + shift:1 + t + shift + n] for t in range(k)], dim=-1).reshape(R * n, k * K)


def _conv_case(k, n_seq, R, K, N, bf16, seed):
    dt = torch.bfloat16 if bf16 else torch.float16
    gen = torch.Generator(device="cuda").manual_seed(seed)
    stride = n_seq + 3                                       # three NaN rows after every item
    a_buf = torch.full((R, stride, K), float("nan"), dtype=dt, device="cuda")
    a_buf[:, :n_seq] = (torch.randn(R, n_seq, K, device="cuda", generator=gen) * 0.5).to(dt)
    w = (torch.randn(k * N, K, device="cuda", generator=gen) / (k * K) ** 0.5).to(dt)   # tap-major [k N, K]
    bias = torch.randn(N, device="cuda", generator=gen) * 0.1
    gate = torch.rand(max(1, R // 2), N, device="cuda", generator=gen)
    return a_buf, w, bias, gate, gen


def _reference_acc(a_buf, w, k, n_seq, N, shift=0):
    xu = _unfold(a_buf[:, :n_seq].double(), k, shift)
    wu = w.double().view(k, N, -1).permute(1, 0, 2).reshape(N, -1)
    return xu @ wu.T, xu.abs() @ wu.abs().T


def _run_probe(a_buf, w, R, n_seq, K, N, k, **fields):
    from stable_audio_tools import _native as nat
    p = nat.SatbGemmProbe(**fields)
    nat.check(nat.lib().satb_token_conv_probe(a_buf.data_ptr(), a_buf.shape[1], w.data_ptr(), R, n_seq, K, N, k,
                                              ctypes.byref(p), nat.stream_ptr()))
    torch.cuda.synchronize()


def _store16(a_buf, w, bias, R, n_seq, K, N, k, bf16, act, bn=0):
    from stable_audio_tools import _native as nat
    out = torch.full((R * n_seq, N), float("nan"), dtype=torch.bfloat16 if bf16 else torch.float16, device="cuda")
    _run_probe(a_buf, w, R, n_seq, K, N, k, epi=nat.EPI_STORE16, bn=bn, bf16=bf16, out=out.data_ptr(), ld=N,
               bias=bias.data_ptr() if bias is not None else None, act=act)
    return out


def _residual(a_buf, w, bias, gate, R, n_seq, K, N, k, bf16, gen, bn=0):
    from stable_audio_tools import _native as nat
    h0 = torch.randn(R * n_seq, N, device="cuda", generator=gen)
    h = h0.clone()
    n_items = gate.shape[0] if gate is not None else 1
    _run_probe(a_buf, w, R, n_seq, K, N, k, epi=nat.EPI_RESIDUAL, bn=bn, bf16=bf16, h=h.data_ptr(), ld=N,
               bias=bias.data_ptr() if bias is not None else None, gate=gate.data_ptr() if gate is not None else None,
               rows_per_item=n_seq, gate_ld=N, n_items=n_items)
    return h0, h


def _check_all(k, n_seq, R, bf16, K=192, seed=0):
    """Both epilogues, with and without bias / SiLU / gate, on one case; returns the worst report."""
    out_t = "bf16" if bf16 else "fp16"
    worst = None
    Ns, Nr = 320, 256                                          # 320: a partial last N tile at BN 256
    for N, kind in ((Ns, "store16"), (Nr, "residual")):
        a_buf, w, bias, gate, gen = _conv_case(k, n_seq, R, K, N, bf16, seed + N)
        acc, S = _reference_acc(a_buf, w, k, n_seq, N)
        for with_bias in (True, False):
            b = bias if with_bias else None
            if kind == "store16":
                act = 1 if with_bias else 0
                got = _store16(a_buf, w, b, R, n_seq, K, N, k, bf16, act)
                rep = ger.check(got, ger.epi_store(acc, S, b, act), k * K, out_t)
            else:
                g = gate if with_bias else None
                h0, got = _residual(a_buf, w, b, g, R, n_seq, K, N, k, bf16, gen)
                gr = ger.gate_rows(g, R * n_seq, n_seq, g.shape[0]) if g is not None else None
                rep = ger.check(got, ger.epi_residual(acc, S, h0, b, gr), k * K, "fp32")
            assert rep.ok, f"{kind} bias={with_bias} k={k} n_seq={n_seq} R={R}: {rep}"
            if worst is None or rep.ratio > worst.ratio:
                worst = rep
    return worst


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("n_seq", [1, 2, 3, 33, 129, 1025])
def test_token_conv_probe_vs_fp64(k, n_seq):
    for R in (1, 3, 8):
        rep = _check_all(k, n_seq, R, bf16=0, seed=100 * k + n_seq + R)
        report("probe", k=k, n_seq=n_seq, R=R, dtype="fp16", max_err_over_bound=rep.ratio)


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("n_seq", [33, 1025])
def test_token_conv_probe_bf16_vs_fp64(k, n_seq):
    rep = _check_all(k, n_seq, 3, bf16=1, seed=7 * k + n_seq)
    report("probe", k=k, n_seq=n_seq, R=3, dtype="bf16", max_err_over_bound=rep.ratio)


@pytest.mark.parametrize("bn", [128, 256])
def test_token_conv_probe_both_n_tiles(bn):
    k, n_seq, R, K, N = 3, 129, 3, 192, 256
    a_buf, w, bias, gate, gen = _conv_case(k, n_seq, R, K, N, 0, 5 + bn)
    acc, S = _reference_acc(a_buf, w, k, n_seq, N)
    got = _store16(a_buf, w, bias, R, n_seq, K, N, k, 0, 1, bn=bn)
    rep = ger.check(got, ger.epi_store(acc, S, bias, 1), k * K, "fp16", bn=bn)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("shift", [-1, 1])
def test_shifted_tap_reference_is_rejected(shift):
    """The checker is sharp enough to see a one-token shift of the taps on the kernel's real output."""
    k, n_seq, R, K, N = 3, 129, 3, 192, 256
    a_buf, w, bias, gate, gen = _conv_case(k, n_seq, R, K, N, 0, 17)
    got = _store16(a_buf, w, bias, R, n_seq, K, N, k, 0, 1)
    acc, S = _reference_acc(a_buf, w, k, n_seq, N)
    assert ger.check(got, ger.epi_store(acc, S, bias, 1), k * K, "fp16").ok
    acc_s, S_s = _reference_acc(a_buf, w, k, n_seq, N, shift=shift)
    rep = ger.check(got, ger.epi_store(acc_s, S_s, bias, 1), k * K, "fp16")
    report("shifted_reference", shift=shift, max_err_over_bound=rep.ratio)
    assert not rep.ok and rep.ratio > 10


# ------------------------------------------------------------------------------------------------ 2. the DiT
def _golden_case(name):
    from oracle import feedforward_oracle as fo
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = fo.make_dit_weights(cfg, seed=int(g["seed"]))
    wsum = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(wsum - float(g["wsum"])) <= 1e-6 * abs(wsum), "synthetic weight RNG drifted from the golden run"
    return g, cfg, sd


def _golden_kw(g, dev):
    T = lambda k: torch.from_numpy(g[k]).to(dev)
    kw = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "prepend" in g:
        kw["prepend_cond"] = T("prepend")
    return kw


@pytest.mark.parametrize("name", GOLDENS)
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_dit_feedforward_vs_reference_golden(name, dtype):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype=dtype)
    kw = _golden_kw(g, "cuda")
    neg = torch.from_numpy(g["neg"]).cuda()
    cases = {"y_nocfg": dict(cfg_scale=1.0), "y_cfg7": dict(cfg_scale=7.0),
             "y_cfg4_phi": dict(cfg_scale=4.0, scale_phi=0.7),
             "y_neg3": dict(cfg_scale=3.0, negative_cross_attn_cond=neg)}
    for key, ck in cases.items():
        y = m(**kw, **ck).cpu()
        err = rel_l2(y, torch.from_numpy(g[key]))
        report("dit_golden", config=name, dtype=dtype, case=key, rel_l2=err)
        assert err < TOL[dtype] * max(1.0, ck["cfg_scale"] / 1.5), f"{name} {key} {dtype}: rel l2 {err}"
    y, info = m(**kw, cfg_scale=1.0, return_info=True)
    err = rel_l2(info["hidden_states"][-1].cpu(), torch.from_numpy(g["hidden_last"]))
    assert err < TOL[dtype], f"{name} hidden {dtype}: rel l2 {err}"


def fp8_floor(sdd):
    """fp8_ref's emulation with a plain Linear FF-in (ff.ff.0.1, 2-D) on e4m3 operands as well, as the FP8 mode runs
    it; a convolutional FF-in (3-D weight) stays fp16-rounded."""
    ctx = fp8_operands(sdd)
    ctx.ids |= {id(v) for k, v in sdd.items() if k.endswith("ff.ff.0.1.weight") and v.dim() == 2}
    return ctx


def _floor_and_native(cfg, sd, m, kw, device, floor_ctx):
    from oracle import feedforward_oracle as fo
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = fo.dit_forward(sdd, cfg, **kwd)
    with floor_ctx(sdd):
        emu = fo.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDENS)
def test_dit_feedforward_fp8_vs_fp8_floor(name):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    base = _golden_kw(g, "cpu")
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", fp8_floor)
        report("dit_fp8", config=name, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
        assert err <= 1.25 * floor, (name, cfg_scale, err, floor)


def _sa_open_inputs(seed, B=1):
    g = torch.Generator().manual_seed(seed)
    x, t = torch.randn(B, 64, 1024, generator=g), torch.rand(B, generator=g) * 0.9 + 0.05
    c, ge = torch.randn(B, 130, 768, generator=g), torch.randn(B, 1536, generator=g)
    c[:, 40:] = 0.0
    return x, t, c, ge


@pytest.mark.parametrize("variant", sorted(SA_OPEN_FF))
@pytest.mark.parametrize("cfg_scale", [1.0, 7.0])
def test_dit_feedforward_sa_open_width_vs_fp16_floor(variant, cfg_scale):
    """1536 wide, 24 heads, 1024 latents + the prepend token = 1025 tokens, 2 blocks; the oracle runs on the GPU in fp32
    (no TF32), its fp16-operand emulation likewise."""
    from oracle import dit_oracle as do
    from oracle import feedforward_oracle as fo
    assert not torch.backends.cuda.matmul.allow_tf32
    cfg = dict(SAO_DIT, depth=2, ff_kwargs=SA_OPEN_FF[variant])
    sd = fo.make_dit_weights(cfg, seed=70)
    m = build_native_dit(cfg, sd)
    x, t, c, ge = _sa_open_inputs(71)
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(cfg, sd, m, kw, "cuda", lambda sdd: do.operand_rounding(torch.float16))
    report("dit_sa_open", variant=variant, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
    assert err <= 1.25 * floor, (variant, cfg_scale, err, floor)


def test_set_feedforward_after_a_weight_and_finalize_with_a_key_missing_fail_with_messages():
    from stable_audio_tools import _native as nat
    from stable_audio_tools.models.dit import DiffusionTransformer
    g, cfg, sd = _golden_case("dit_ff_conv5_adaln_hd128_small.npz")
    lib = nat.lib()
    h = ctypes.c_void_p()
    nat.check(lib.satb_dit_create(ctypes.byref(DiffusionTransformer(**cfg).native_config()), ctypes.byref(h)))
    try:
        nat.check(lib.satb_dit_set_feedforward(h, 1024, 0, 5, 1))
        st = nat.stream_ptr()
        for k, v in sd.items():
            if k == "transformer.layers.1.ff.ff.0.1.bias":
                continue
            src = v.cuda().contiguous()
            nat.check(lib.satb_dit_load_weight(h, k.encode(), src.data_ptr(), src.numel(), st))
            torch.cuda.synchronize()
        rc = lib.satb_dit_finalize(h, st)
        msg = lib.satb_last_error()
        assert rc != 0 and b"feed-forward weights missing in layer 1: transformer.layers.1.ff.ff.0.1.bias" in msg
        assert lib.satb_dit_set_feedforward(h, 1024, 0, 3, 1) != 0 and b"before the first weight" in lib.satb_last_error()
    finally:
        lib.satb_dit_destroy(h)


# ------------------------------------------------------------------------------------------------ 4. bit checks
@pytest.mark.parametrize("name", ["dit_ff_glu_conv3_nobias_small.npz", "dit_ff_conv5_adaln_hd128_small.npz"])
def test_feedforward_cuda_graph_call_equals_the_eager_call(name):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd)
    kw = _golden_kw(g, "cuda")
    x = kw.pop("x")
    eager = lambda xx: m(xx, cfg_scale=7.0, **kw).clone()
    y0 = eager(x)
    m.cuda_graph = True
    y1 = eager(x)
    y2 = eager(x * 0.5 + 0.1)
    m.cuda_graph = False
    assert torch.equal(y0, y1)
    assert torch.equal(y2, eager(x * 0.5 + 0.1))


@pytest.mark.parametrize("variant", ["plain_conv3", "mult83"])
def test_feedforward_batch_of_4_equals_the_same_prompts_in_a_batch_of_5(variant):
    from oracle import feedforward_oracle as fo
    cfg = dict(SAO_DIT, depth=2, ff_kwargs=SA_OPEN_FF[variant])
    m = build_native_dit(cfg, fo.make_dit_weights(cfg, seed=72))
    x, t, c, ge = (v.cuda() for v in _sa_open_inputs(73, B=5))
    sub = lambda a, b: dict(cross_attn_cond=c[a:b].contiguous(), global_embed=ge[a:b].contiguous(), cfg_scale=7.0)
    y5 = m(x, t, **sub(0, 5)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(0, 4)).clone()
    report("batch_invariance", variant=variant, bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)
