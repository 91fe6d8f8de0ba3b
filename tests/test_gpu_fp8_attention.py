"""GPU: the DiT's FP8 self-attention (attention_dtype "fp8", head dim 64).

1. The operand quantisers.  The e4m3 QKV epilogues (satb_gemm_probe_qk8: EpiQkvRopeE4m3, EpiHeadNormE4m3, with 16-bit
   and e4m3 GEMM operands): q8 / k8 bits and scales equal torch's float8_e4m3fn rounding, under the rule of
   tests/fp8_attn_ref.py, of the very 16-bit values the 16-bit epilogue of the same schedule stores (which
   test_gpu_gemm_fragment_rope.py / test_gpu_gemm_epilogues.py pin to the EpiStore32 accumulator through the rotary
   and qk_norm emulation), and the v columns equal its v columns bit for bit; M from 1 to 8200, items of 33 and 1025
   tokens, a partial last n-tile.  The V transpose-quantiser (satb_attention_fp8_vt): V^T bits and channel scales
   equal torch's rounding of v * 2^-e in the stored key order, zero past N.
2. The core (satb_attention_fp8_core) against float64 softmax attention on the dequantised q, k, v, element by element
   within the bound of P's e4m3 rounding: sum_j max(2^-4 p_j, 2^-10) |v_j| / l (relative half-ulp of a normal e4m3,
   half the subnormal step), plus the 16-bit output rounding and a small fp32 slack.
3. The forward against its floor: rel-L2 to the fp32 oracle <= 1.25 x the rel-L2 of the oracle's FP8-attention
   emulation (stacked on the operand mode's emulation) to the fp32 oracle.
4. Bit checks: the CUDA-graph call equals the eager call; a batch of 4 equals the same prompts inside a batch of 5.
Measured numbers are printed as `FP8ATTN {...}` JSON lines (pytest -s)."""
import ctypes
import json

import pytest
import torch

from fp8_attn_ref import dequant, fp8_attention, quantize_heads, quantize_v, stored_key_order
from fp8_ref import fp8_operands
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu


def report(name, **kw):
    print("FP8ATTN " + json.dumps(dict(test=name, **kw)), flush=True)


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


def _pad(n):
    return (n + 127) // 128 * 128


def _vt_native(v, bf16):
    nat, lib = _lib()
    B, N, D = v.shape
    H = D // 64
    vt = torch.full((B * H, 64, _pad(N)), 0x7F, dtype=torch.uint8, device="cuda")   # NaN bytes: all must be written
    sv = torch.full((B * H, 64), float("nan"), device="cuda")
    nat.check(lib.satb_attention_fp8_vt(v.data_ptr(), vt.data_ptr(), sv.data_ptr(), B, H, N, int(bf16), nat.stream_ptr()))
    torch.cuda.synchronize()
    return vt, sv


def _heads(x, H):   # [B, N, H*64] -> [B, H, N, 64]
    B, N, _ = x.shape
    return x.view(B, N, H, 64).permute(0, 2, 1, 3)


def _qk_operand(x):
    """q or k [B, N, H*64] -> (e4m3 bytes [B, N, H*64], scales [B*H, pad(N)]) by the fp32 CPU-rule of fp8_attn_ref."""
    B, N, D = x.shape
    H = D // 64
    x8, s = quantize_heads(_heads(x.float(), H))
    sp = torch.zeros(B * H, _pad(N), device=x.device)
    sp[:, :N] = s.reshape(B * H, N)
    return x8.permute(0, 2, 1, 3).reshape(B, N, D).view(torch.uint8), sp


def _v_operand(v):
    """v [B, N, H*64] -> (V^T e4m3 bytes [B*H, 64, pad(N)] in the stored key order, scales [B*H, 64])."""
    B, N, D = v.shape
    H, Np = D // 64, _pad(N)
    v8, s = quantize_v(_heads(v.float(), H))                   # [B, H, N, 64], [B, H, 1, 64]
    vt = torch.zeros(B * H, 64, Np, dtype=torch.uint8, device=v.device)
    vt[:, :, :N] = v8.reshape(B * H, N, 64).transpose(1, 2).view(torch.uint8)
    return vt[:, :, stored_key_order(Np).to(v.device)].contiguous(), s.reshape(B * H, 64)


# ------------------------------------------------------------------------------------------------ 1. quantisers
QK_WIDTH = 640                                   # 10 heads: N = 1920 is not a multiple of 256 (partial last n-tile)
QK_CASES = [(M, 33) for M in (1, 9, 129, 8200)] + [(8200, 1025)]


def _probe16(mode, epi, bn, a, w, sa, sw, M, N, K, **f):
    nat, lib = _lib()
    p = nat.SatbGemmProbe()
    p.epi, p.bn, p.bf16, p.b_static = epi, bn, int(mode == "bf16"), 1
    for k, v in f.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    if mode == "fp8":
        nat.check(lib.satb_gemm_probe_fp8(a.data_ptr(), w.data_ptr(), sa.data_ptr(), sw.data_ptr(), M, N, K,
                                          ctypes.byref(p), nat.stream_ptr()))
    else:
        nat.check(lib.satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, N, K, ctypes.byref(p), nat.stream_ptr()))
    return p


@pytest.mark.parametrize("mode", ["fp16", "bf16", "fp8"])
@pytest.mark.parametrize("kind", ["rope", "norm"])
@pytest.mark.parametrize("M,seq", QK_CASES)
def test_qkv_e4m3_epilogue_quantises_the_16bit_epilogue_values(mode, kind, M, seq):
    import gemm_epilogue_ref as R
    from fp8_ref import quantize_fp8_rows
    nat, lib = _lib()
    D, H = QK_WIDTH, QK_WIDTH // 64
    N, K = 3 * D, D
    dt = torch.bfloat16 if mode == "bf16" else torch.float16
    g = torch.Generator(device="cuda").manual_seed(M + seq + len(kind) + len(mode))
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
    w[5 * 64: 6 * 64] *= 1e-3                     # one head (q head 5) with small values
    sa = sw = None
    if mode == "fp8":
        qa, sa = quantize_fp8_rows(a)
        qw, sw = quantize_fp8_rows(w)
        a, w = qa.view(torch.uint8).contiguous(), qw.view(torch.uint8).contiguous()
        sa, sw = sa[:, 0].contiguous(), sw[:, 0].contiguous()
    else:
        a, w = a.to(dt), w.to(dt)
    cos, sin, _ = R.rope_tables(seq, 16)
    cos, sin = cos.cuda(), sin.cuda()
    f = dict(rope_cols=2 * D, seq_len=seq, cos_tab=cos, sin_tab=sin)
    if kind == "rope":
        epi16, epi8, bn16 = nat.EPI_QKV_ROPE, nat.EPI_QKV_ROPE_E4M3, 256
        f.update(head_dim=64, nf=16)
    else:
        epi16, epi8 = nat.EPI_HEAD_NORM16, nat.EPI_HEAD_NORM_E4M3
        bn16 = 128 if mode == "fp8" else 256
        f.update(norm_cols=2 * D)
    ref16 = torch.full((M, N), float("nan"), dtype=dt, device="cuda")
    _probe16(mode, epi16, bn16, a, w, sa, sw, M, N, K, out=ref16, ld=N, **f)

    R_items, Np = (M + seq - 1) // seq, _pad(seq)
    out = torch.full((M + 3, N), float("nan"), dtype=dt, device="cuda")
    q8 = torch.full((M + 3, D), 0x7F, dtype=torch.uint8, device="cuda")
    k8 = torch.full_like(q8, 0x7F)
    sq = torch.full((R_items * H, Np), -1.0, device="cuda")
    sk = torch.full_like(sq, -1.0)
    o = nat.SatbQkE4m3(q8=q8.data_ptr(), k8=k8.data_ptr(), sq=sq.data_ptr(), sk=sk.data_ptr(), heads=H, scale_ld=Np)
    p = nat.SatbGemmProbe()
    p.epi, p.bn, p.bf16, p.b_static = epi8, bn16, int(mode == "bf16"), 1
    p.out, p.ld, p.rope_cols, p.seq_len = out.data_ptr(), N, 2 * D, seq
    p.cos_tab, p.sin_tab = cos.data_ptr(), sin.data_ptr()
    nat.check(lib.satb_gemm_probe_qk8(a.data_ptr(), w.data_ptr(), sa.data_ptr() if sa is not None else None,
                                      sw.data_ptr() if sw is not None else None, M, N, K, ctypes.byref(p),
                                      ctypes.byref(o), nat.stream_ptr()))
    torch.cuda.synchronize()

    iv = torch.int16
    assert torch.equal(out[:M, 2 * D:].view(iv), ref16[:, 2 * D:].view(iv)), "v columns differ from the 16-bit epilogue"
    assert bool(torch.isnan(out[:, :2 * D].float()).all()) and bool(torch.isnan(out[M:].float()).all()), \
        "the e4m3 epilogue wrote a q / k column or a row past M of the 16-bit output"
    tok = torch.arange(M, device="cuda")
    for name, x8, sx, c0 in (("q", q8, sq, 0), ("k", k8, sk, D)):
        want8, want_s = quantize_fp8_rows(ref16[:, c0:c0 + D].float().view(M, H, 64))
        assert torch.equal(x8[:M], want8.view(torch.uint8).view(M, D)), f"{name}8 bits differ"
        assert bool((x8[M:] == 0x7F).all()), f"{name}8: a row past M was written"
        idx = (tok // seq)[:, None] * H + torch.arange(H, device="cuda")[None, :]
        got_s = sx[idx, (tok % seq)[:, None]]
        assert torch.equal(got_s, want_s[..., 0]), f"{name} scales differ"
        written = torch.zeros_like(sx, dtype=torch.bool)
        written[idx, (tok % seq)[:, None].expand(M, H)] = True
        assert bool((sx[~written] == -1.0).all()), f"{name} scale written outside its (row, head) slots"
    report("qkv_e4m3_epilogue", mode=mode, kind=kind, M=M, seq=seq, bit_equal=True)


def test_qkv_e4m3_epilogues_are_refused_by_the_other_probes_and_epi_6_stays_retired():
    nat, lib = _lib()
    a = torch.zeros(128, 256, dtype=torch.float16, device="cuda")
    out = torch.empty(128, 256, dtype=torch.float16, device="cuda")
    s = torch.ones(256, device="cuda")
    for epi in (nat.EPI_QKV_ROPE_E4M3, nat.EPI_HEAD_NORM_E4M3, nat.EPI_RESIDUAL_LN):
        p = nat.SatbGemmProbe()
        p.epi, p.bn, p.out, p.ld, p.h, p.seq_len, p.head_dim, p.nf = epi, 256, out.data_ptr(), 256, out.data_ptr(), 1, 64, 16
        assert lib.satb_gemm_probe(a.data_ptr(), a.data_ptr(), 128, 256, 256, ctypes.byref(p), nat.stream_ptr()) != 0
        assert lib.satb_gemm_probe_fp8(a.data_ptr(), a.data_ptr(), s.data_ptr(), s.data_ptr(), 128, 256, 256,
                                       ctypes.byref(p), nat.stream_ptr()) != 0
    o = nat.SatbQkE4m3(q8=a.data_ptr(), k8=a.data_ptr(), sq=s.data_ptr(), sk=s.data_ptr(), heads=1, scale_ld=128)
    for epi, bn in ((nat.EPI_RESIDUAL_LN, 256), (nat.EPI_QKV_ROPE, 256), (nat.EPI_HEAD_NORM16, 256),
                    (nat.EPI_QKV_ROPE_E4M3, 128)):
        p = nat.SatbGemmProbe()
        p.epi, p.bn, p.out, p.ld, p.seq_len = epi, bn, out.data_ptr(), 256, 1
        rc = lib.satb_gemm_probe_qk8(a.data_ptr(), a.data_ptr(), None, None, 128, 256, 256, ctypes.byref(p),
                                     ctypes.byref(o), nat.stream_ptr())
        assert rc != 0, (epi, bn)
    torch.cuda.synchronize()


@pytest.mark.parametrize("N", [1025, 130, 2, 33])
@pytest.mark.parametrize("bf16", [False, True])
def test_v_transpose_quantiser_bits_equal_torch_e4m3_rounding(N, bf16):
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator(device="cuda").manual_seed(N + bf16)
    B, H = 2, 3
    v = torch.randn(B, N, H * 64, device="cuda", generator=g) * 4
    v[1, :, 7] = 0.0                                           # an all-zero channel
    v[0, :, 70] *= 2.0 ** -10                                  # a small channel
    v[0, :, 71] = 0.003                                        # values in the e4m3 subnormals after scaling
    v[0, N // 2, 71] = 400.0
    v[1, 0, 130] = 448.0                                       # amax exactly 448 * 2^0
    v = v.to(dt)
    vt, sv = _vt_native(v, bf16)
    want_vt, want_sv = _v_operand(v)
    if not torch.equal(vt, want_vt):
        pytest.fail(f"vt8 differs at {torch.nonzero(vt != want_vt)[:4].tolist()} (N={N}, bf16={bf16})")
    assert torch.equal(sv, want_sv), "channel scales differ"
    report("v_quantiser", N=N, bf16=bf16, bit_equal=True)


# ------------------------------------------------------------------------------------------------ 2. core
def _core_native(q8, k8, sq, sk, vt, sv, B, H, Nq, Nk, bf16):
    nat, lib = _lib()
    o = torch.full((B, Nq, H * 64), float("nan"), dtype=torch.bfloat16 if bf16 else torch.float16, device="cuda")
    nat.check(lib.satb_attention_fp8_core(q8.data_ptr(), k8.data_ptr(), sq.data_ptr(), sk.data_ptr(), vt.data_ptr(),
                                          sv.data_ptr(), o.data_ptr(), B, H, Nq, Nk, int(bf16), nat.stream_ptr()))
    torch.cuda.synchronize()
    return o


def _check_core(q, k, v, bf16, name):
    """q [B, Nq, D], k / v [B, Nk, D] fp32 on the GPU: quantise in torch, run the native core, compare with fp64."""
    B, Nq, D = q.shape
    Nk, H = k.shape[1], D // 64
    q8, sq = _qk_operand(q)
    k8, sk = _qk_operand(k)
    vt, sv = _v_operand(v)
    o = _core_native(q8, k8, sq, sk, vt, sv, B, H, Nq, Nk, bf16)
    qd = dequant(*quantize_heads(_heads(q, H))).double()
    kd = dequant(*quantize_heads(_heads(k, H))).double()
    vd = dequant(*quantize_v(_heads(v, H))).double()
    s = qd @ kd.transpose(-1, -2) / 8
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    ref = (p @ vd) / l
    p_err = torch.maximum(p * 2.0 ** -4, torch.full_like(p, 2.0 ** -10))
    bound = (p_err @ vd.abs()) / l
    half_ulp = 2.0 ** -8 if bf16 else 2.0 ** -11
    bound = bound + ref.abs() * (half_ulp + 1e-5) + 1e-6 * vd.abs().amax(-2, keepdim=True)
    got = _heads(o.double(), H)
    err = (got - ref).abs()
    ratio = float((err / bound).max())
    worst = torch.nonzero((err / bound) == (err / bound).max())[0].tolist()
    report("core", case=name, bf16=bf16, max_err_over_bound=ratio, worst=worst,
           rel_l2=rel_l2(got.cpu(), ref.cpu()))
    assert bool(torch.isfinite(got).all())
    assert ratio <= 1.0, (name, ratio, worst)


CORE_SHAPES = [(2, 24, 1025, 1025), (1, 2, 2, 130), (1, 3, 65, 191), (1, 2, 300, 641)]


@pytest.mark.parametrize("B,H,Nq,Nk", CORE_SHAPES)
@pytest.mark.parametrize("bf16", [False, True])
def test_core_vs_fp64_on_the_dequantised_operands(B, H, Nq, Nk, bf16):
    g = torch.Generator(device="cuda").manual_seed(Nq * 7 + Nk + bf16)
    q = torch.randn(B, Nq, H * 64, device="cuda", generator=g) * 1.5
    k = torch.randn(B, Nk, H * 64, device="cuda", generator=g) * 1.5
    v = torch.randn(B, Nk, H * 64, device="cuda", generator=g)
    _check_core(q, k, v, bf16, f"{B}x{H}x{Nq}x{Nk}")


@pytest.mark.parametrize("bf16", [False, True])
def test_core_monotone_scores_move_the_running_max_every_tile(bf16):
    """Scores grow with the key index, so every key tile raises the row maximum and rescales O and l."""
    B, H, Nq, Nk = 1, 2, 130, 1025
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.zeros(B, Nq, H * 64, device="cuda")
    q[..., 0::64] = 4.0
    k = torch.randn(B, Nk, H * 64, device="cuda", generator=g) * 0.05
    k[..., 0::64] = torch.linspace(0, 6, Nk, device="cuda").view(1, Nk, 1)
    v = torch.randn(B, Nk, H * 64, device="cuda", generator=g)
    _check_core(q, k, v, bf16, "monotone")


# ------------------------------------------------------------------------------------------------ 3. forward
def _oracle(name):
    from oracle import conformer_oracle as co
    from oracle import dit_oracle as do
    from oracle import feedforward_oracle as fo
    if "conformer" in name:
        return co
    if "_ff_" in name:
        return fo
    return do


GOLDEN_HD64 = ["dit_prepend_small.npz", "dit_adaln_small.npz", "dit_qknorm_small.npz", "dit_concat_prepend_small.npz",
               "dit_conformer_small.npz", "dit_ff_mult83_small.npz"]


def _floor_ctx(sdd, operand_dtype):
    from oracle import dit_oracle as do
    return fp8_operands(sdd) if operand_dtype == "fp8" else do.operand_rounding(torch.float16)


def _floor_and_native(orc, cfg, sd, m, kw, device, operand_dtype):
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = orc.dit_forward(sdd, cfg, **kwd)
    with _floor_ctx(sdd, operand_dtype), fp8_attention():
        emu = orc.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


@pytest.mark.parametrize("name", GOLDEN_HD64)
@pytest.mark.parametrize("operand_dtype", ["fp16", "fp8"])
def test_forward_small_configs_vs_fp8_attention_floor(name, operand_dtype):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    orc = _oracle(name)
    sd = orc.make_dit_weights(cfg, seed=int(g["seed"]))
    m = build_native_dit(dict(cfg, attention_dtype="fp8"), sd, operand_dtype=operand_dtype)
    T = lambda k: torch.from_numpy(g[k])
    base = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "concat" in g:
        base.update(input_concat_cond=T("concat"), prepend_cond=T("prepend"))
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(orc, cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", operand_dtype)
        report("forward_small", config=name, operand_dtype=operand_dtype, cfg_scale=cfg_scale, rel_l2=err, floor=floor,
               ratio=err / floor)
        assert err <= 1.25 * floor, (name, operand_dtype, cfg_scale, err, floor)


@pytest.mark.parametrize("cfg_scale", [1.0, 7.0])
@pytest.mark.parametrize("operand_dtype", ["fp16", "fp8"])
def test_forward_sa_open_width_24_blocks_vs_fp8_attention_floor(cfg_scale, operand_dtype):
    from oracle import dit_oracle as do
    assert not torch.backends.cuda.matmul.allow_tf32
    sd = do.make_dit_weights(SAO_DIT, seed=41)
    m = build_native_dit(dict(SAO_DIT, attention_dtype="fp8"), sd, operand_dtype=operand_dtype)
    g = torch.Generator().manual_seed(42)
    x, t = torch.randn(1, 64, 1024, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    c[:, 40:] = 0.0
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(do, SAO_DIT, sd, m, kw, "cuda", operand_dtype)
    report("forward_sa_open", operand_dtype=operand_dtype, cfg_scale=cfg_scale, rel_l2=err, floor=floor,
           ratio=err / floor)
    assert err <= 1.25 * floor, (operand_dtype, cfg_scale, err, floor)


# ------------------------------------------------------------------------------------------------ 4. bit checks
def test_fp8_attention_cuda_graph_call_equals_the_eager_call():
    from oracle import dit_oracle as do
    g = load_golden("dit_qknorm_small.npz")
    cfg = json.loads(str(g["cfg"]))
    sd = do.make_dit_weights(cfg, seed=int(g["seed"]))
    m = build_native_dit(dict(cfg, attention_dtype="fp8"), sd)
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


def test_fp8_attention_batch_of_4_equals_the_same_prompts_in_a_batch_of_5():
    from oracle import dit_oracle as do
    sd = do.make_dit_weights(SAO_DIT, seed=43)
    m = build_native_dit(dict(SAO_DIT, attention_dtype="fp8"), sd)
    g = torch.Generator().manual_seed(44)
    x, t = torch.randn(5, 64, 1024, generator=g).cuda(), (torch.rand(5, generator=g) * 0.9 + 0.05).cuda()
    c, ge = torch.randn(5, 130, 768, generator=g).cuda(), torch.randn(5, 1536, generator=g).cuda()
    sub = lambda a, b: dict(cross_attn_cond=c[a:b].contiguous(), global_embed=ge[a:b].contiguous(), cfg_scale=7.0)
    y5 = m(x, t, **sub(0, 5)).clone()
    y4 = m(x[:4].contiguous(), t[:4].contiguous(), **sub(0, 4)).clone()
    report("batch_invariance", bit_equal=bool(torch.equal(y5[:4], y4)))
    assert torch.isfinite(y5).all()
    assert torch.equal(y5[:4], y4)


def test_setter_refuses_a_call_after_finalize():
    from oracle import dit_oracle as do
    g = load_golden("dit_prepend_small.npz")
    cfg = json.loads(str(g["cfg"]))
    m = build_native_dit(cfg, do.make_dit_weights(cfg, seed=int(g["seed"])))
    T = lambda k: torch.from_numpy(g[k]).cuda()
    m(T("x"), T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))   # loads the weights and finalizes
    nat, lib = _lib()
    h = m.__dict__["_h"]
    assert lib.satb_dit_set_attention_fp8(h, 1) != 0
    assert b"before satb_dit_finalize" in lib.satb_last_error()
