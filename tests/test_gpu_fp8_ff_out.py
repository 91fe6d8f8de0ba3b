"""GPU: the FP8 FF-out option (ff_out_dtype "fp8" with operand_dtype "fp8"; satb_dit_set_ff_out_fp8).

1. FF-in's e4m3 block epilogues (satb_gemm_probe_ff8: EpiSwigluE4m3, EpiSiluE4m3) against the fp64 SwiGLU / SiLU of
   the dequantised FP8 operands: every (row, 128-column) scale follows the rule of tests/fp8_ref.py applied to the fp64
   block amax (except an amax within the GEMM's accumulation error of a power-of-two boundary), and every dequantised
   element is within half an e4m3 ulp at its block scale plus the accumulation bound.
2. The block-scaled FF-out GEMM (BlockScaledA<EpiResidual>, BN 128) element by element against the fp64 product of the
   dequantised operands, within the (ceil(K / 32) + 1) 2^-13 sum |a w| bound of the FP8 GEMM tests.
3. The forward against the option's floor: rel-L2 to the fp32 oracle within 0.95-1.05 x the rel-L2 of the oracle's
   emulation (fp8_ref.fp8_operands + fp8_ff_out_ref.fp8_ff_out_operands, + fp8_attn_ref.fp8_attention with FP8
   self-attention) to the fp32 oracle.
4. Token sharding and the CFG split give the unsharded forward bit for bit, eagerly and from the group's graph.
Measured numbers are printed as `FF8 {...}` JSON lines (pytest -s)."""
import ctypes
import json
import math

import pytest
import torch

import gemm_epilogue_ref as ger
from fp8_attn_ref import fp8_attention
from fp8_ff_out_ref import fp8_ff_out_operands, quantize_fp8_blocks
from fp8_ref import fp8_operands, fp8_row_exponent, quantize_fp8_rows
from helpers import SAO_DIT, build_native_dit, load_golden, rel_l2

pytestmark = pytest.mark.gpu


def report(name, **kw):
    print("FF8 " + json.dumps(dict(test=name, **kw)), flush=True)


def _lib():
    from stable_audio_tools import _native
    return _native, _native.lib()


def e_acc8(K):
    return (math.ceil(K / 32) + 1) * 2.0 ** -13


def _half_ulp(u):
    """Half an e4m3 ulp at |u| (scaled units): 2^(floor(log2 |u|) - 4) for normals (>= 2^-6), 2^-10 below."""
    a = u.abs().clamp_min(2.0 ** -6)
    return torch.ldexp(torch.ones_like(a), torch.floor(torch.log2(a)).to(torch.int32) - 4)


def _pow2(e):
    return torch.ldexp(torch.ones_like(e, dtype=torch.float64), e)


def _probe(M, N, K, a8, sa, w8, sw, p_fields, ff8=None, ffs=None):
    nat, lib = _lib()
    p = nat.SatbGemmProbe()
    p.bf16, p.b_static = 0, 1
    for k, v in p_fields.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    nat.check(lib.satb_gemm_probe_ff8(a8.data_ptr(), w8.data_ptr(), sa.data_ptr(), sw.data_ptr(), M, N, K,
                                      ctypes.byref(p), ff8.data_ptr() if ff8 is not None else None,
                                      ffs.data_ptr() if ffs is not None else None, nat.stream_ptr()))


# ------------------------------------------------------------------------------------------------ 1. FF-in epilogues
def _row_operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.exp(torch.randn(M, 1, device="cuda", generator=g))
    w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5 * torch.exp(0.5 * torch.randn(N, 1, device="cuda",
                                                                                               generator=g))
    a[3] = 0.0                                                   # an all-zero row
    qa, sa = quantize_fp8_rows(a)
    qw, sw = quantize_fp8_rows(w)
    ad, wd = qa.double() * sa.double(), qw.double() * sw.double()
    return (qa.view(torch.uint8).contiguous(), sa[:, 0].contiguous(), qw.view(torch.uint8).contiguous(),
            sw[:, 0].contiguous(), ad @ wd.T, ad.abs() @ wd.abs().T)


EPI_CASES = [  # (name, kind, bn, M, N, K): ragged M; the SiLU BN 256 case has a half last tile (N = 384)
    ("swiglu", "swiglu", 256, 1025, 768, 256), ("swiglu_bench", "swiglu", 256, 8200, 12288, 1536),
    ("silu_bn128", "silu", 128, 1025, 384, 256), ("silu_bn256", "silu", 256, 1025, 384, 384),
    ("silu_nobias_bn256", "silu_nobias", 256, 300, 512, 128),
]


@pytest.mark.parametrize("name,kind,bn,M,N,K", EPI_CASES, ids=[c[0] for c in EPI_CASES])
def test_ff_in_e4m3_epilogue_vs_fp64(name, kind, bn, M, N, K):
    nat, _ = _lib()
    a8, sa, w8, sw, acc, S = _row_operands(M, N, K, seed=M + N + K)
    g = torch.Generator(device="cuda").manual_seed(7)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    if kind == "swiglu":
        perm = ger.ff_perm(N // 2).cuda()
        w8, sw = w8[perm].contiguous(), sw[perm].contiguous()
        exp = ger.epi_swiglu(acc, S, bias)
        f = dict(epi=nat.EPI_SWIGLU_E4M3, bn=bn, bias=bias[perm].contiguous())
    else:
        b = bias if kind == "silu" else None
        exp = ger.epi_store(acc, S, b, act=1)
        f = dict(epi=nat.EPI_SILU_E4M3, bn=bn, bias=b if b is not None else 0)
    cols = exp.ref.shape[1]
    f["ld"] = cols
    ff8 = torch.full((M + 1, cols), 0xAB, dtype=torch.uint8, device="cuda")        # row M: a canary
    ffs = torch.full((M + 1, cols // 128), -1.0, device="cuda")
    _probe(M, N, K, a8, sa, w8, sw, f, ff8, ffs)
    first8, firsts = ff8.clone(), ffs.clone()
    _probe(M, N, K, a8, sa, w8, sw, f, ff8, ffs)
    torch.cuda.synchronize()
    assert torch.equal(first8, ff8) and torch.equal(firsts, ffs), "repeated calls differ"
    assert bool((ff8[M] == 0xAB).all()) and bool((ffs[M] == -1.0).all()), "a row past M was written"
    ref = exp.ref
    bnd = e_acc8(K) * exp.sens + ger.E_EPI * exp.mag                # what the fp32 value may differ from ref by
    blocks = lambda t: t.reshape(M, cols // 128, 128)
    amax = blocks(ref).abs().amax(-1)
    e_want = fp8_row_exponent(amax)
    s_got = ffs[:M].double()
    b_blk = blocks(bnd).amax(-1)
    top = 448.0 * _pow2(e_want)
    near = ((amax - top).abs() <= b_blk) | ((amax - top / 2).abs() <= b_blk)
    ok = (s_got == _pow2(e_want)) | near
    assert bool(ok.all()), f"block scales off the rule at {torch.nonzero(~ok)[:8].tolist()}"
    s_el = s_got.repeat_interleave(128, dim=1)
    dq = ff8[:M].view(torch.float8_e4m3fn).double() * s_el
    bound = _half_ulp((ref.abs() + bnd) / s_el) * s_el + bnd
    err = (dq - ref).abs()
    ratio = float((err / bound).max())
    report("ff_in_e4m3", case=name, M=M, N=N, K=K, bn=bn, max_err_over_bound=ratio, blocks_near_boundary=int(near.sum()))
    assert ratio <= 1.0
    if kind == "silu_nobias":                                      # a zero row without bias: all-zero blocks, scale 1
        assert bool((s_got[3] == 1.0).all()) and bool((ff8[3] == 0).all())


# ------------------------------------------------------------------------------------------------ 2. block-scaled GEMM
def _block_operands(M, N, K, seed, alt_scale):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.exp(torch.randn(M, 1, device="cuda", generator=g))
    if alt_scale:                         # every odd k-block = the even one before it times 2^-20: so are its scales
        ab = a.view(M, K // 256, 2, 128)
        ab[:, :, 1] = ab[:, :, 0] * 2.0 ** -20
    else:
        a = a * torch.exp(torch.randn(M, K // 128, device="cuda", generator=g)).repeat_interleave(128, dim=1)
    w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5 * torch.exp(0.5 * torch.randn(N, 1, device="cuda",
                                                                                               generator=g))
    qa, sa = quantize_fp8_blocks(a)
    qw, sw = quantize_fp8_rows(w)
    ad = qa.double() * sa.double().repeat_interleave(128, dim=1)
    wd = qw.double() * sw.double()
    return (qa.view(torch.uint8).contiguous(), sa.contiguous(), qw.view(torch.uint8).contiguous(),
            sw[:, 0].contiguous(), ad @ wd.T, ad.abs() @ wd.abs().T, sa)


GEMM_CASES = [  # (name, M, N, K, alt_scale, gate): N = 992 has a partial last BN 128 tile, M = 1025 a partial m tile
    ("k128_one_block", 1025, 992, 128, False, False), ("k6144", 1025, 1536, 6144, False, True),
    ("alt_scales_2pow20", 1025, 992, 1024, True, False), ("bench", 8200, 1536, 6144, False, True),
]


@pytest.mark.parametrize("name,M,N,K,alt,gate", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_block_scaled_ff_out_gemm_vs_fp64(name, M, N, K, alt, gate):
    nat, _ = _lib()
    a8, sa, w8, sw, acc, S, sblk = _block_operands(M, N, K, M + N + K, alt)
    if alt:
        assert bool((sblk[:, 1::2] == sblk[:, 0::2] * 2.0 ** -20).all())
    g = torch.Generator(device="cuda").manual_seed(9)
    h0 = torch.randn(M, N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    f = dict(epi=nat.EPI_RESIDUAL_A8, bn=128, ld=N, bias=bias)
    gate_rows = None
    if gate:
        items, rpi = 3, 400
        gt = torch.rand(items, N, device="cuda", generator=g)
        f.update(gate=gt, rows_per_item=rpi, gate_ld=N, n_items=items)
        gate_rows = ger.gate_rows(gt, M, rpi, items)
    h = h0.clone()
    f["h"] = h
    _probe(M, N, K, a8, sa, w8, sw, f)
    torch.cuda.synchronize()
    exp = ger.epi_residual(acc, S, h0, bias, gate_rows)
    bound = (1 + 2.0 ** -24) * (e_acc8(K) * exp.sens + ger.E_EPI * exp.mag) + 2.0 ** -24 * exp.ref.abs() + 1e-37
    err = (h.double() - exp.ref).abs()
    assert torch.isfinite(h).all()
    ratio = float((err / bound).max())
    acc_rel = float(((err - 2.0 ** -24 * exp.ref.abs()).clamp_min(0) / exp.sens.clamp_min(1e-30)).max())
    report("block_scaled_gemm", case=name, M=M, N=N, K=K, max_err_over_bound=ratio, max_acc_err_over_sum_abs_aw=acc_rel,
           e_acc8=e_acc8(K))
    assert ratio <= 1.0


def test_probe_ff8_refuses_other_instances():
    nat, lib = _lib()
    a8 = torch.zeros(128, 512, dtype=torch.uint8, device="cuda")
    s = torch.ones(512, device="cuda")
    ff8 = torch.zeros(128, 512, dtype=torch.uint8, device="cuda")
    out = torch.zeros(128, 512, device="cuda")
    for epi, bn, bf16, N, K in [(nat.EPI_SWIGLU_E4M3, 128, 0, 512, 256), (nat.EPI_RESIDUAL_A8, 256, 0, 512, 256),
                                (nat.EPI_SILU_E4M3, 64, 0, 512, 256), (nat.EPI_RESIDUAL, 128, 0, 512, 256),
                                (nat.EPI_STORE16, 128, 0, 512, 256), (nat.EPI_SILU_E4M3, 128, 1, 512, 256),
                                (nat.EPI_SILU_E4M3, 128, 0, 512, 192)]:
        p = nat.SatbGemmProbe()
        p.epi, p.bn, p.bf16, p.ld, p.h, p.out = epi, bn, bf16, 512, out.data_ptr(), out.data_ptr()
        rc = lib.satb_gemm_probe_ff8(a8.data_ptr(), a8.data_ptr(), s.data_ptr(), s.data_ptr(), 128, N, K,
                                     ctypes.byref(p), ff8.data_ptr(), s.data_ptr(), nat.stream_ptr())
        assert rc != 0, (epi, bn, bf16, K)


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


class _floor:
    """The option's emulation: FP8 operands (a plain Linear FF-in on e4m3 operands too, as the FP8 mode runs it), the
    FF-out block quantiser and, with FP8 self-attention, its emulation."""

    def __init__(self, sdd, attn):
        self.ctx = [fp8_operands(sdd), fp8_ff_out_operands(sdd)] + ([fp8_attention()] if attn else [])
        self.ctx[0].ids |= {id(v) for k, v in sdd.items() if k.endswith("ff.ff.0.1.weight") and v.dim() == 2}

    def __enter__(self):
        for c in self.ctx:
            c.__enter__()

    def __exit__(self, *exc):
        for c in reversed(self.ctx):
            c.__exit__(*exc)


def _floor_and_native(orc, cfg, sd, m, kw, device, attn):
    sdd = {k: v.to(device) for k, v in sd.items()}
    kwd = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
    ref = orc.dit_forward(sdd, cfg, **kwd)
    with _floor(sdd, attn):
        emu = orc.dit_forward(sdd, cfg, **kwd)
    y = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    return rel_l2(emu.cpu(), ref.cpu()), rel_l2(y.cpu(), ref.cpu())


GOLDENS = ["dit_prepend_small.npz", "dit_adaln_small.npz", "dit_concat_prepend_small.npz", "dit_hd32_small.npz",
           "dit_hd128_small.npz", "dit_hd128_adaln_small.npz", "dit_ff_plain_nobias_hd32_small.npz",
           "dit_conformer_small.npz", "dit_conformer_adaln_small.npz"]
HD64 = {"dit_prepend_small.npz", "dit_adaln_small.npz", "dit_concat_prepend_small.npz", "dit_conformer_small.npz",
        "dit_conformer_adaln_small.npz"}
FORWARD_CASES = [(n, False) for n in GOLDENS] + [(n, True) for n in GOLDENS if n in HD64]


@pytest.mark.parametrize("name,attn", FORWARD_CASES, ids=[f"{n[:-4]}{'-attn8' if a else ''}" for n, a in FORWARD_CASES])
def test_forward_small_configs_vs_floor(name, attn):
    g = load_golden(name)
    cfg = json.loads(str(g["cfg"]))
    orc = _oracle(name)
    sd = orc.make_dit_weights(cfg, seed=int(g["seed"]))
    extra = dict(ff_out_dtype="fp8", attention_dtype="fp8" if attn else None)
    m = build_native_dit(dict(cfg, **extra), sd, operand_dtype="fp8")
    T = lambda k: torch.from_numpy(g[k])
    base = dict(x=T("x"), t=T("t"), cross_attn_cond=T("cross"), global_embed=T("glob"))
    if "concat" in g:
        base.update(input_concat_cond=T("concat"), prepend_cond=T("prepend"))
    for cfg_scale in (1.0, 7.0):
        floor, err = _floor_and_native(orc, cfg, sd, m, dict(base, cfg_scale=cfg_scale), "cpu", attn)
        report("forward_small", config=name, attn_fp8=attn, cfg_scale=cfg_scale, rel_l2=err, floor=floor,
               ratio=err / floor)
        assert 0.95 * floor <= err <= 1.05 * floor, (name, attn, cfg_scale, err, floor)


@pytest.mark.parametrize("cfg_scale", [1.0, 7.0])
def test_forward_sa_open_width_24_blocks_vs_floor(cfg_scale):
    """SA-Open width, all 24 blocks, 1024 latents + the prepend token = 1025 tokens; the oracle and its emulation run
    on the GPU in fp32 (no TF32)."""
    from oracle import dit_oracle as do
    assert not torch.backends.cuda.matmul.allow_tf32
    sd = do.make_dit_weights(SAO_DIT, seed=31)
    m = build_native_dit(dict(SAO_DIT, ff_out_dtype="fp8"), sd, operand_dtype="fp8")
    g = torch.Generator().manual_seed(32)
    x, t = torch.randn(1, 64, 1024, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 130, 768, generator=g), torch.randn(1, 1536, generator=g)
    c[:, 40:] = 0.0
    kw = dict(x=x, t=t, cross_attn_cond=c, global_embed=ge, cfg_scale=cfg_scale)
    floor, err = _floor_and_native(do, SAO_DIT, sd, m, kw, "cuda", False)
    m8 = build_native_dit(SAO_DIT, sd, operand_dtype="fp8")
    y8 = m8(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    y88 = m(**{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    report("forward_sa_open", cfg_scale=cfg_scale, rel_l2=err, floor=floor, ratio=err / floor,
           rel_l2_vs_fp8_mode=rel_l2(y88.cpu(), y8.cpu()))
    assert 0.95 * floor <= err <= 1.05 * floor, (cfg_scale, err, floor)


# ------------------------------------------------------------------------------------------------ 4. sharding
SMALL = dict(io_channels=64, embed_dim=256, depth=2, num_heads=4, cond_token_dim=128, global_cond_dim=256,
             project_cond_tokens=False, transformer_type="continuous_transformer")


def _shard_inputs(L):
    g = torch.Generator().manual_seed(92 + L)
    x, t = torch.randn(1, 64, L, generator=g), torch.tensor([0.4])
    c, ge = torch.randn(1, 19, 128, generator=g), torch.randn(1, 256, generator=g)
    c[:, 12:] = 0.0
    return {k: v.cuda() for k, v in dict(x=x, t=t, cross_attn_cond=c, global_embed=ge).items()}


@pytest.mark.parametrize("gtype", ["prepend", "adaLN"])
@pytest.mark.parametrize("L", [300, 1100])
def test_sharded_and_cfg_split_equal_the_unsharded_forward(L, gtype):
    from oracle import dit_oracle as do
    cfg = dict(SMALL, global_cond_type=gtype)
    sd = do.make_dit_weights(cfg, seed=91)
    m = build_native_dit(dict(cfg, ff_out_dtype="fp8"), sd, operand_dtype="fp8")
    kw = _shard_inputs(L)
    y1 = {s: m(**kw, cfg_scale=s).clone() for s in (1.0, 7.0)}
    layouts = [["cuda:0"] * w for w in (2, 3, 4, 8)] + [[["cuda:0"], ["cuda:0"]], [["cuda:0"] * 2, ["cuda:0"] * 2]]
    for layout in layouts:
        m.shard_tokens(layout)
        for graph in (False, True):
            m.cuda_graph = graph
            for s in (1.0, 7.0):
                y = m(**kw, cfg_scale=s).clone()
                report("sharded", L=L, gtype=gtype, layout=str(layout), graph=graph, cfg_scale=s,
                       bit_identical=bool(torch.equal(y, y1[s])))
                assert torch.equal(y, y1[s]), (layout, graph, s)
        m.cuda_graph = False
    m.shard_tokens(None)
    assert torch.equal(m(**kw, cfg_scale=7.0), y1[7.0])


def test_group_refuses_handles_that_differ_in_the_option():
    from oracle import dit_oracle as do
    nat, lib = _lib()
    sd = do.make_dit_weights(SMALL, seed=5)
    m_on = build_native_dit(dict(SMALL, ff_out_dtype="fp8"), sd, operand_dtype="fp8")
    m_off = build_native_dit(SMALL, sd, operand_dtype="fp8")
    dev = torch.device("cuda", torch.cuda.current_device())
    hs = [m._handle(dev) for m in (m_on, m_off)]
    g = ctypes.c_void_p()
    handles = (ctypes.c_void_p * 2)(*[h.value for h in hs])
    ids = (ctypes.c_int * 2)(dev.index, dev.index)
    assert lib.satb_dit_group_create(handles, ids, 2, ctypes.byref(g)) != 0
    # and the setter refuses a call after the first weight is loaded
    assert lib.satb_dit_set_ff_out_fp8(hs[1], 1) != 0 and b"before the first weight" in lib.satb_last_error()
