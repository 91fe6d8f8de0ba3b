"""GPU: DiTs built with the reference's positional options (rotary_pos_emb=False, use_sinusoidal_emb, use_abs_pos_emb;
reference models/transformer.py:50-96, 705-809).

1. The project_in GEMM with the position table (satb_gemm_probe kind SATB_EPI_STORE32_POS, the forward's instance,
   fp16 and bf16) against float64, element by element, with the bound of tests/gemm_epilogue_ref.py: items of 1025
   and 6145 rows (partial last m-tiles, sinusoidal positions beyond 6000, no prepended row: P = 0).
2. The table and the prepended rows through a depth-0 model (its last hidden state is project_in + prepend + table):
   P = 1 and 4, 6144 latents; the difference to the same model with scale 0 is the float64 sinusoid of the fp32
   products, to fp32 rounding.
3. The DiT against the reference goldens (tests/golden/dit_pos_*.npz) at the gates of test_gpu_dit.py: rel-L2 2e-3
   (x max(1, cfg / 1.5) with CFG) in fp16, 1.5e-2 in bf16; FP8 within 1.25 x its emulated floor.
4. SA-Open width (1536 wide, 24 heads, 2 blocks) at 1025 and 6145 tokens against the oracle's fp16-operand floor.
5. Bit checks: the CUDA-graph call equals the eager call; a batch of 4 equals the same prompts inside a batch of 5;
   changing pos_emb.scale and reloading changes the output, eagerly and through the graph.
Measured numbers are printed as `POSVAR {...}` JSON lines (pytest -s)."""
import ctypes
import json

import pytest
import torch

import gemm_epilogue_ref as ger
from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu

GOLDENS = ["dit_pos_sin_small.npz", "dit_pos_abs_prepcond_small.npz", "dit_pos_norope_abs_adaln_hd128_small.npz",
           "dit_pos_norope_qknorm_small.npz", "dit_pos_sin_conformer_patch2_conv3_small.npz"]
TOL = {"fp16": 2e-3, "bf16": 1.5e-2}
SA_OPEN_POS = {"sin": dict(use_sinusoidal_emb=True), "abs": dict(use_abs_pos_emb=True),
               "norope_sin": dict(rotary_pos_emb=False, use_sinusoidal_emb=True)}


def report(name, **kw):
    print("POSVAR " + json.dumps(dict(test=name, **kw)), flush=True)


def _sinusoid64(n, dim, scale):
    """The table in float64 from the fp32 products p * inv_freq (the reference's own rounding of the argument)."""
    from oracle import positions_oracle as po
    f = (torch.arange(n).float()[:, None] * po.sinusoid_inv_freq(dim)[None, :]).double()
    return torch.cat((f.sin(), f.cos()), dim=-1) * float(scale)


# ------------------------------------------------------------------------------------------------ 1. the probe
@pytest.mark.parametrize("n_seq,R", [(1025, 3), (6145, 2), (77, 5)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_project_in_position_epilogue_vs_fp64(n_seq, R, bf16):
    from stable_audio_tools import _native as nat
    dt = torch.bfloat16 if bf16 else torch.float16
    K, N = 64, 1536
    M = R * n_seq
    gen = torch.Generator(device="cuda").manual_seed(n_seq + R + bf16)
    a = torch.randn(M, K, device="cuda", generator=gen).to(dt)
    w = (torch.randn(N, K, device="cuda", generator=gen) / K ** 0.5).to(dt)
    pos = _sinusoid64(n_seq, N, 0.75).float().cuda().contiguous()
    for with_bias in (False, True):
        bias = torch.randn(N, device="cuda", generator=gen) * 0.1 if with_bias else None
        out = torch.full((M, N), float("nan"), device="cuda")
        p = nat.SatbGemmProbe(epi=nat.EPI_STORE32_POS, bn=256, bf16=bf16, b_static=1, out=out.data_ptr(), ld=N,
                              bias=bias.data_ptr() if bias is not None else None, seq_len=n_seq, pos_tab=pos.data_ptr())
        nat.check(nat.lib().satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, N, K, ctypes.byref(p), nat.stream_ptr()))
        torch.cuda.synchronize()
        acc, S = ger.accumulate(a.cpu(), w.cpu())
        e = ger.epi_store(acc, S, bias.cpu() if bias is not None else None)
        rows = pos.cpu().double().repeat(R, 1)
        rep = ger.check(out.cpu(), ger.Expect(e.ref + rows, e.sens, e.mag + rows.abs()), K, "fp32")
        report("probe", n_seq=n_seq, R=R, bf16=bf16, bias=with_bias, max_err_over_bound=rep.ratio)
        assert rep.ok, str(rep)
        # the table row is that of the position inside the item: a table shifted by one row is rejected
        shifted = torch.roll(pos.cpu().double(), 1, dims=0).repeat(R, 1)
        assert not ger.check(out.cpu(), ger.Expect(e.ref + shifted, e.sens, e.mag + shifted.abs()), K, "fp32").ok


# ------------------------------------------------------------------------------------------------ 2. prepended rows
@pytest.mark.parametrize("n_prepend", [0, 3])
def test_table_and_prepended_rows_through_a_depth0_model(n_prepend):
    from oracle import positions_oracle as po
    cfg = dict(SAO_DIT, depth=0, use_sinusoidal_emb=True, prepend_cond_dim=64 if n_prepend else 0)
    sd = po.make_dit_weights(cfg, seed=80)
    m = build_native_dit(cfg, sd)
    g = torch.Generator().manual_seed(81)
    L = 6144
    kw = dict(cross_attn_cond=torch.randn(1, 20, 768, generator=g).cuda(),
              global_embed=torch.randn(1, 1536, generator=g).cuda(), cfg_scale=1.0, return_info=True)
    if n_prepend:
        kw["prepend_cond"] = torch.randn(1, n_prepend, 64, generator=g).cuda()
    x, t = torch.randn(1, 64, L, generator=g).cuda(), torch.rand(1, generator=g).cuda()
    h_pos = m(x, t, **kw)[1]["hidden_states"][-1][0].cpu().double()
    scale = float(m.transformer.pos_emb.scale)
    with torch.no_grad():
        m.transformer.pos_emb.scale.zero_()
    m.refresh_native_weights()
    h_0 = m(x, t, **kw)[1]["hidden_states"][-1][0].cpu().double()
    n = L + 1 + n_prepend
    assert h_pos.shape == (n, 1536)
    want = _sinusoid64(n, 1536, scale)
    bound = 2.0 ** -23 * (h_pos.abs() + 2 * want.abs()) + 1e-30
    ratio = float(((h_pos - h_0 - want).abs() / bound).max())
    report("depth0_rows", n_prepend=n_prepend, n_seq=n, max_err_over_bound=ratio)
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------ 3. the goldens
def _golden_case(name):
    from oracle import positions_oracle as po
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    sd = po.make_dit_weights(cfg, seed=int(g["seed"]))
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
def test_dit_positions_vs_reference_golden(name, dtype):
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
    """fp8_ref's emulation; a convolutional FF-in would stay fp16, as in the feed-forward tests (none here)."""
    return fp8_operands(sdd)


def _floor_and_native(cfg, sd, m, kw, device, floor_ctx):
    from oracle import positions_oracle as po
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = po.dit_forward(sdd, cfg, **kwd)
    with floor_ctx(sdd):
        emu = po.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDENS)
def test_dit_positions_fp8_vs_fp8_floor(name):
    g, cfg, sd = _golden_case(name)
    m = build_native_dit(cfg, sd, operand_dtype="fp8")
    base = _golden_kw(g, "cpu")
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", fp8_floor)
        report("dit_fp8", config=name, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
        assert err <= 1.25 * floor, (name, cfg_scale, err, floor)


# ------------------------------------------------------------------------------------------------ 4. SA-Open width
def _sa_open_inputs(seed, B=1, L=1024):
    g = torch.Generator().manual_seed(seed)
    x, t = torch.randn(B, 64, L, generator=g), torch.rand(B, generator=g) * 0.9 + 0.05
    c, ge = torch.randn(B, 130, 768, generator=g), torch.randn(B, 1536, generator=g)
    c[:, 40:] = 0.0
    return x, t, c, ge


@pytest.mark.parametrize("variant", sorted(SA_OPEN_POS))
@pytest.mark.parametrize("L,cfg_scale", [(1024, 7.0), (6144, 1.0)])
def test_dit_positions_sa_open_width_vs_fp16_floor(variant, L, cfg_scale):
    """1536 wide, 24 heads, L latents + the prepend token (1025 and 6145 tokens), 2 blocks; the oracle runs on the GPU
    in fp32 (no TF32), its fp16-operand emulation likewise."""
    from oracle import dit_oracle as do
    from oracle import positions_oracle as po
    assert not torch.backends.cuda.matmul.allow_tf32
    cfg = dict(SAO_DIT, depth=2, **SA_OPEN_POS[variant])
    sd = po.make_dit_weights(cfg, seed=82)
    m = build_native_dit(cfg, sd)
    x, t, c, ge = _sa_open_inputs(83, L=L)
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(cfg, sd, m, kw, "cuda", lambda sdd: do.operand_rounding(torch.float16))
    report("dit_sa_open", variant=variant, tokens=L + 1, cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor)
    assert err <= 1.25 * floor, (variant, L, err, floor)


def test_forward_refuses_a_sequence_longer_than_the_absolute_embedding():
    from oracle import positions_oracle as po
    cfg = dict(SAO_DIT, depth=1, use_abs_pos_emb=True, abs_pos_emb_max_length=40)
    m = build_native_dit(cfg, po.make_dit_weights(cfg, seed=84))
    x, t, c, ge = (v.cuda() for v in _sa_open_inputs(85, L=39))
    y = m(x, t, cross_attn_cond=c, global_embed=ge)
    assert torch.isfinite(y).all()
    with pytest.raises(AssertionError, match="max sequence length of 40"):
        m(torch.cat([x, x[:, :, :1]], dim=2), t, cross_attn_cond=c, global_embed=ge)


# ------------------------------------------------------------------------------------------------ 5. bit checks
@pytest.mark.parametrize("name", ["dit_pos_sin_small.npz", "dit_pos_abs_prepcond_small.npz",
                                  "dit_pos_norope_abs_adaln_hd128_small.npz"])
def test_positions_cuda_graph_call_equals_the_eager_call(name):
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


@pytest.mark.parametrize("variant", ["sin", "abs"])
def test_positions_batch_of_4_equals_the_same_prompts_in_a_batch_of_5(variant):
    from oracle import positions_oracle as po
    cfg = dict(SAO_DIT, depth=2, **SA_OPEN_POS[variant])
    m = build_native_dit(cfg, po.make_dit_weights(cfg, seed=86))
    x, t, c, ge = (v.cuda() for v in _sa_open_inputs(87, B=5))
    sub = lambda a, b: dict(cross_attn_cond=c[a:b].contiguous(), global_embed=ge[a:b].contiguous(), cfg_scale=7.0)
    y5 = m(x, t, **sub(0, 5)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(0, 4)).clone()
    report("batch_invariance", variant=variant, bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)


@pytest.mark.parametrize("graph", [False, True])
def test_reloading_the_scale_changes_the_output(graph):
    """finalize invalidates the table, so a reloaded pos_emb.scale takes effect (same shapes, so no regrowth forces it)."""
    g, cfg, sd = _golden_case("dit_pos_sin_small.npz")
    m = build_native_dit(cfg, sd)
    m.cuda_graph = graph
    kw = _golden_kw(g, "cuda")
    y0 = m(**kw, cfg_scale=7.0).clone()
    sd2 = dict(sd, **{"transformer.pos_emb.scale": sd["transformer.pos_emb.scale"] * 0.25})
    m.load_state_dict(sd2, strict=True)
    y1 = m(**kw, cfg_scale=7.0).clone()
    m.load_state_dict(sd, strict=True)
    y2 = m(**kw, cfg_scale=7.0).clone()
    report("reload", graph=graph, moved=rel_l2(y1.cpu(), y0.cpu()))
    assert rel_l2(y1.cpu(), y0.cpu()) > 0.05
    assert torch.equal(y0, y2)
