"""GPU: every fused epilogue of the DiT's wgmma GEMM (csrc/gemm.cuh), at every tile width the forward instantiates,
against the float64 reference of tests/gemm_epilogue_ref.py, element by element, through satb_gemm_probe (the very
kernel instances the forward launches).

Every output carries guard rows and columns: 16-bit and fp32 outputs are filled with NaN bits, the fp32 residual
stream h with known random values; every valid element must be finite and within the bound, every guard element
bit-unchanged.  Shapes cover the ragged M tail (1, 127, 129), the SA-Open item (1025 rows) and the bench (8200
rows), a persistent grid of exactly `sms` and `sms + 1` tiles, N not a multiple of BN (3 x 640), K from 64 to 6144
and K one k-block deeper than the shared-memory ring.  The last tests pin bit properties of the schedule.
Each test prints its largest err/bound ratio ("[ratio] ...")."""
import ctypes

import pytest
import torch

import gemm_epilogue_ref as R

pytestmark = pytest.mark.gpu

DTS = ["fp16", "bf16"]
GUARD_ROWS, GUARD_COLS = 3, 16
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000}
INT_VIEW = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}


def _nat():
    from stable_audio_tools import _native
    return _native


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------- plumbing
def probe(dt, epi, bn, a, w, M, N, K, b_static=1, **f):
    nat = _nat()
    p = nat.SatbGemmProbe()
    p.epi, p.bn, p.bf16, p.b_static = epi, bn, int(dt == "bf16"), b_static
    for k, v in f.items():
        setattr(p, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    nat.check(nat.lib().satb_gemm_probe(a.data_ptr(), w.data_ptr(), M, N, K, ctypes.byref(p), nat.stream_ptr()))
    torch.cuda.synchronize()


def guarded(rows, cols, dtype, fill=None):
    """[rows + GUARD_ROWS, cols + GUARD_COLS]: NaN bits, or the given values (then the guard gets random values too)."""
    buf = torch.empty(rows + GUARD_ROWS, cols + GUARD_COLS, dtype=dtype, device="cuda")
    if fill is None:
        buf.view(INT_VIEW[dtype]).fill_(NAN_BITS[dtype])
    else:
        buf.copy_(fill)
    return buf


def assert_guard(after, before, rows, cols, what):
    iv = INT_VIEW[after.dtype]
    a, b = after.view(iv), before.view(iv)
    assert torch.equal(a[rows:], b[rows:]), f"{what}: a guard row was written"
    assert torch.equal(a[:rows, cols:], b[:rows, cols:]), f"{what}: a guard column was written"


def operands(dt, M, N, K, seed, w_scale=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    tdt = R.TORCH_DT[dt]
    a = torch.randn(M, K, device="cuda", generator=g).to(tdt)
    w = (torch.randn(N, K, device="cuda", generator=g) * (w_scale or K ** -0.5)).to(tdt)
    return a, w, g


def report(tag, rep):
    print(f"[ratio] {tag}: {rep.ratio:.3f}  ({rep})")
    assert rep.ok, f"{tag}: {rep}"


def shapes_sweep(bn, k_cols):
    """(M, N, K) of the shape sweep for one tile width; M "sms" / "sms+1": exactly `sms` tiles, then one more
    (resolved on the device by rows())."""
    ring = 64 * (R.gemm_stages(bn, k_cols) + 1)
    out = [(m, 1536, 1536) for m in (1, 127, 128, 129, 1025, 8200)]
    out += [(1025, 1536, k) for k in (64, 72, 200, 6144)]
    out += [(1025, 1920, 640), (1025, 1536, ring)]
    out += [("sms", bn, 256), ("sms+1", bn, 256)]
    return out


def rows(M):
    return {"sms": 128 * _sms(), "sms+1": 128 * _sms() + 1}.get(M, M)


# ------------------------------------------------------------------------------------------------- EpiStore32
STORE32 = [(64, m, 64, 1536) for m in (1, 127, 129, 1025, 8200)] + [(64, 1025, 64, 64 * (R.gemm_stages(64, 32) + 1))]
STORE32 += [(256, m, 1536, k) for m in (1, 129, 8200) for k in (64, 72)] + [(256, 1025, 1536, 256), (256, 1025, 1920, 200)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bn,M,N,K", STORE32)
def test_store32(dt, bn, M, N, K):
    """project_out (BN 64, N = 64) and project_in (BN 256, K = io 64 + concat 8)."""
    nat = _nat()
    a, w, g = operands(dt, M, N, K, seed=M + N + K)
    bias = torch.randn(N, device="cuda", generator=g) * 0.5 if M % 2 else None
    out = guarded(M, N, torch.float32)
    before = out.clone()
    probe(dt, nat.EPI_STORE32, bn, a, w, M, N, K, out=out, ld=out.shape[1], bias=bias)
    assert_guard(out, before, M, N, "store32")
    acc, S = R.accumulate(a, w)
    report(f"store32 {dt} BN{bn} M{M} N{N} K{K}", R.check(out[:M, :N], R.epi_store(acc, S, bias), K, "fp32", bn))


# ------------------------------------------------------------------------------------------------- EpiStore16
def _store16_cases():
    cases = []
    for bn in (128, 256):
        for i, (M, N, K) in enumerate(shapes_sweep(bn, 32)):
            cases.append((bn, M, N, K, i % 2, (i // 2) % 2))
    cases.append((256, "sms+1", 1920, 200, 1, 1))
    return cases


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bn,M,N,K,act,has_bias", _store16_cases())
def test_store16(dt, bn, M, N, K, act, has_bias):
    nat = _nat()
    M = rows(M)
    a, w, g = operands(dt, M, N, K, seed=7 * M + N + K)
    bias = torch.randn(N, device="cuda", generator=g) * 0.5 if has_bias else None
    tdt = R.TORCH_DT[dt]
    out = guarded(M, N, tdt)
    before = out.clone()
    probe(dt, nat.EPI_STORE16, bn, a, w, M, N, K, out=out, ld=out.shape[1], bias=bias, act=act)
    assert_guard(out, before, M, N, "store16")
    acc, S = R.accumulate(a, w)
    report(f"store16 {dt} BN{bn} M{M} N{N} K{K} act{act} bias{has_bias}",
           R.check(out[:M, :N], R.epi_store(acc, S, bias, act), K, dt, bn))


# ------------------------------------------------------------------------------------------------- EpiHeadNorm16
HEAD_NORM = [(bn, M, mode, seq) for bn in (128, 256) for (M, mode, seq) in
             ((129, "kv", 1), (1025, "qkv", 1025), (2050, "qkv", 33), (8200, "qkv", 1025), (1025, "q", 1))]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bn,M,mode,seq", HEAD_NORM)
def test_head_norm16(dt, bn, M, mode, seq):
    """qk_norm heads: k | v (norm_cols < N, no rotary), q | k | v (norm and rotary below 2 D), q alone; one head
    whose accumulator is all zeros (the 1e-12 clamp)."""
    nat = _nat()
    D, K = 768, 768
    N = {"kv": 2 * D, "qkv": 3 * D, "q": D}[mode]
    norm_cols = D if mode != "qkv" else 2 * D
    rope_cols = 2 * D if mode == "qkv" else 0
    a, w, _ = operands(dt, M, N, K, seed=M + N)
    w[128:192] = 0                                                  # head 2: all-zero accumulator
    out = guarded(M, N, R.TORCH_DT[dt])
    before = out.clone()
    cos, sin, freqs = R.rope_tables(seq, 16)
    tabs = dict(cos_tab=cos.cuda(), sin_tab=sin.cuda(), seq_len=seq) if rope_cols else {}
    probe(dt, nat.EPI_HEAD_NORM16, bn, a, w, M, N, K, out=out, ld=out.shape[1], norm_cols=norm_cols,
          rope_cols=rope_cols, **tabs)
    assert_guard(out, before, M, N, "head_norm16")
    assert torch.all(out[:M, 128:192].float() == 0)
    acc, S = R.accumulate(a, w)
    fr = R.row_freqs(freqs, M, seq).cuda() if rope_cols else None
    report(f"head_norm16 {dt} BN{bn} M{M} {mode} seq{seq}",
           R.check(out[:M, :N], R.epi_head_norm(acc, S, norm_cols, rope_cols, fr), K, dt, bn))


# ------------------------------------------------------------------------------------------------- EpiQkvRope
QKV = [(1536, 64, 8200, 1025), (1536, 96, 1025, 1025), (1536, 128, 2050, 33), (768, 64, 1025, 33),
       (768, 96, 330, 33), (768, 128, 1025, 1025), (256, 32, 1025, 33), (256, 32, 129, 1025), (640, 64, 1025, 1025),
       (640, 128, 127, 33)]


def qkv_weight(D, head_dim, seed):
    """to_qkv in reference row order and as stored (qkv_head_perm)."""
    nf = R.rope_nf(head_dim)
    g = torch.Generator().manual_seed(seed)
    w_ref = torch.randn(3 * D, D, generator=g) * D ** -0.5
    perm = R.qkv_head_perm(D, head_dim, nf)
    return w_ref, w_ref[perm], perm


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("D,head_dim,M,seq", QKV)
def test_qkv_rope(dt, D, head_dim, M, seq):
    """Rotary of every q | k head at head dims 32 / 64 / 96 / 128 over items of 1025 or 33 rows (a 128-row tile spans
    several items, position 0 falls mid-tile); v columns unrotated.  The weight is built in reference order and
    stored permuted; the reference is the oracle's rotary on the reference columns, permuted like the weight."""
    nat = _nat()
    nf = R.rope_nf(head_dim)
    N, K = 3 * D, D
    tdt = R.TORCH_DT[dt]
    w_ref, w_st, perm = qkv_weight(D, head_dim, seed=D + head_dim)
    w_ref, w_st = w_ref.to(tdt).cuda(), w_st.to(tdt).cuda()
    a = torch.randn(M, K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(M)).to(tdt)
    cos, sin, freqs = R.rope_tables(seq, nf)
    out = guarded(M, N, tdt)
    before = out.clone()
    probe(dt, nat.EPI_QKV_ROPE, 256, a, w_st, M, N, K, out=out, ld=out.shape[1], rope_cols=2 * D, seq_len=seq,
          head_dim=head_dim, nf=nf, cos_tab=cos.cuda(), sin_tab=sin.cuda())
    assert_guard(out, before, M, N, "qkv_rope")
    acc, S = R.accumulate(a, w_ref)
    e = R.epi_qkv_rope(acc, S, R.row_freqs(freqs, M, seq).cuda(), head_dim, nf, 2 * D)
    pc = perm.cuda()
    e = R.Expect(e.ref[:, pc], e.sens[:, pc], e.mag[:, pc])
    report(f"qkv_rope {dt} D{D} hd{head_dim} M{M} seq{seq}", R.check(out[:M, :N], e, K, dt, 256))


# ------------------------------------------------------------------------------------------------- EpiSwiglu
def swiglu_weight(D, ffi, seed, gate_std=8.0):
    """ff.0.proj in reference order (value rows, then gate rows scaled so the gate pre-activations reach +-20 for
    unit inputs) and as stored (ff_perm)."""
    g = torch.Generator().manual_seed(seed)
    w_ref = torch.randn(2 * ffi, D, generator=g) * D ** -0.5
    w_ref[ffi:] *= gate_std
    perm = R.ff_perm(ffi)
    return w_ref, w_ref[perm], perm


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("M,D,has_bias", [(8200, 1536, True), (129, 1536, False), (1025, 640, True), (1, 768, True)])
def test_swiglu(dt, M, D, has_bias):
    nat = _nat()
    ffi = 4 * D
    N, K = 2 * ffi, D
    tdt = R.TORCH_DT[dt]
    w_ref, w_st, perm = swiglu_weight(D, ffi, seed=D)
    w_ref, w_st = w_ref.to(tdt).cuda(), w_st.to(tdt).cuda()
    a = torch.randn(M, K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(M)).to(tdt)
    bias_ref = (torch.randn(N) * 0.5).cuda() if has_bias else None
    out = guarded(M, ffi, tdt)
    before = out.clone()
    probe(dt, nat.EPI_SWIGLU, 256, a, w_st, M, N, K, out=out, ld=out.shape[1],
          bias=bias_ref[perm.cuda()].contiguous() if has_bias else None)
    assert_guard(out, before, M, ffi, "swiglu")
    acc, S = R.accumulate(a, w_ref)
    gmax = float((acc[:, ffi:] + (bias_ref[ffi:].double() if has_bias else 0)).abs().max())
    assert M == 1 or gmax > 15, gmax                                 # the gate reaches the __expf tails
    report(f"swiglu {dt} M{M} D{D} bias{has_bias}", R.check(out[:M, :ffi], R.epi_swiglu(acc, S, bias_ref), K, dt, 256, 2))


# ------------------------------------------------------------------------------------------------- EpiResidual
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("K,has_bias,has_gate", [(1536, True, True), (6144, True, False), (1536, False, True),
                                                 (200, False, False)])
def test_residual(dt, bn, K, has_bias, has_gate):
    """h += (acc + bias) * gate with the adaLN gate of B = 2 items on R = 4 CFG rows of 1025 tokens: rows of the
    unconditional half use the gate rows of their item (the % n_items wrap); the buffer holds 4 gate rows so that
    an unwrapped index would read other values.  At BN 256 the result must be h_old + v in a single fp32 add, v
    formed from EpiStore32's accumulator bits."""
    nat = _nat()
    M, N, rpi, B = 4100, 1536, 1025, 2
    a, w, g = operands(dt, M, N, K, seed=K + bn)
    bias = torch.randn(N, device="cuda", generator=g) * 0.5 if has_bias else None
    gate = (torch.rand(4, N, device="cuda", generator=g) + 0.2) if has_gate else None
    h0 = torch.randn(M + GUARD_ROWS, N + GUARD_COLS, device="cuda", generator=g)
    h = guarded(M, N, torch.float32, h0)
    probe(dt, nat.EPI_RESIDUAL, bn, a, w, M, N, K, h=h, ld=h.shape[1], bias=bias, gate=gate, rows_per_item=rpi,
          gate_ld=N, n_items=B)
    assert_guard(h, h0, M, N, "residual")
    acc, S = R.accumulate(a, w)
    gr = R.gate_rows(gate, M, rpi, B) if has_gate else None
    report(f"residual {dt} BN{bn} K{K} bias{has_bias} gate{has_gate}",
           R.check(h[:M, :N], R.epi_residual(acc, S, h0[:M, :N], bias, gr), K, "fp32", bn))
    if bn == 256:
        s32 = torch.empty(M, N, device="cuda")
        probe(dt, nat.EPI_STORE32, 256, a, w, M, N, K, out=s32, ld=N, bias=bias)
        v = s32 * gr if has_gate else s32
        assert torch.equal(h[:M, :N], h0[:M, :N] + v), "h is not h_old + v in one fp32 add"


# ------------------------------------------------------------------------------------------------- schedule / bits
def _schedule(M, N, bn, num_kb, stages, row_off=0):
    """(n tile, m tile of the rows starting at row_off) -> (CTA, ring position at the tile's start), as the persistent
    kernel walks its tiles: tile = n_tile * m_tiles + m_tile, CTA = tile % grid, start = (tile // grid) * num_kb k-blocks
    into a ring of `stages` slots with a phase bit."""
    m_tiles, n_tiles = -(-M // 128), -(-N // bn)
    total = m_tiles * n_tiles
    grid = min(_sms(), total)
    out = {}
    for nt in range(n_tiles):
        for mt in range(row_off // 128, m_tiles):
            t = nt * m_tiles + mt
            out[(nt, mt - row_off // 128)] = (t % grid, ((t // grid) * num_kb) % (2 * stages))
    return out


def _prop_n(kind, bn):
    return {"store32": 64 if bn == 64 else 1024, "swiglu": 1024, "qkv_rope": 3 * 256}.get(kind, 768)


def _prop_case(kind, dt, M, bn, K, seed):
    """A launchable case of each epilogue on M rows whose row-dependent parameters repeat every 128 rows (seq_len
    128, rows_per_item 64 of 2 items), so its rows can be computed at any 128-aligned offset."""
    nat = _nat()
    tdt = R.TORCH_DT[dt]
    g = torch.Generator(device="cuda").manual_seed(seed)
    kc = 64 if kind in ("head_norm16", "swiglu") else 32
    N = _prop_n(kind, bn)
    a = torch.randn(M, K, device="cuda", generator=g).to(tdt)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(tdt)
    f, outs = {}, {}
    if kind == "residual":
        h = torch.randn(M, N, device="cuda", generator=g)
        f.update(h=h, ld=N, bias=torch.randn(N, device="cuda", generator=g))
        outs["h"] = h
        # as many gate rows as items of 64 rows: an index without the % n_items wrap stays inside the buffer
        f.update(gate=torch.rand(-(-M // 64), N, device="cuda", generator=g) + 0.2, rows_per_item=64, gate_ld=N,
                 n_items=2)
    else:
        ld = N // 2 if kind == "swiglu" else N
        out = torch.zeros(M, ld, dtype=torch.float32 if kind == "store32" else tdt, device="cuda")
        f.update(out=out, ld=ld)
        outs["out"] = out
        if kind in ("store16", "store32", "swiglu"):
            f["bias"] = torch.randn(N, device="cuda", generator=g)
        if kind == "store16":
            f["act"] = 1
        if kind in ("qkv_rope", "head_norm16"):
            nf = 16
            cos, sin, _ = R.rope_tables(128, nf)
            f.update(rope_cols=2 * N // 3, seq_len=128, cos_tab=cos.cuda(), sin_tab=sin.cuda())
            if kind == "qkv_rope":
                f.update(head_dim=64, nf=nf)
            else:
                f.update(norm_cols=2 * N // 3)
    epi = {"store32": nat.EPI_STORE32, "store16": nat.EPI_STORE16, "head_norm16": nat.EPI_HEAD_NORM16,
           "qkv_rope": nat.EPI_QKV_ROPE, "swiglu": nat.EPI_SWIGLU, "residual": nat.EPI_RESIDUAL}[kind]
    return dict(epi=epi, a=a, w=w, N=N, f=f, outs=outs, kc=kc)


def _run_prop(c, dt, M, bn, K, b_static=1):
    f = dict(c["f"])
    if "h" in f:
        f["h"] = f["h"].clone()
        c["outs"]["h"] = f["h"]
    probe(dt, c["epi"], bn, c["a"], c["w"], M, c["N"], K, b_static=b_static, **f)
    return {k: v.clone() for k, v in c["outs"].items()}


PROP_KINDS = [("store32", 256), ("store32", 64), ("store16", 128), ("store16", 256), ("head_norm16", 128),
              ("head_norm16", 256), ("qkv_rope", 256), ("swiglu", 256), ("residual", 128), ("residual", 256)]


def _bits(d):
    return {k: v.view(INT_VIEW[v.dtype]) for k, v in d.items()}


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("kind,bn", PROP_KINDS)
def test_schedule_bit_properties(dt, kind, bn):
    """Bit-exact, every epilogue: (1) two identical calls; (2) b_static 1 (weight prefetch before the dependency wait)
    and 0; (3) rows [0, M1) against the same rows computed at row offset P = 128 (sms + 1) inside a larger M2 = P +
    M1 + 77: another tile count, another CTA for every tile, another ring position at every tile's start (K = one
    k-block more than the ring depth)."""
    M1 = 1025
    kc = 64 if kind in ("head_norm16", "swiglu") else 32
    stages = R.gemm_stages(bn, kc)
    P = 128 * (_sms() + 1)
    M2 = P + M1 + 77
    N = _prop_n(kind, bn)
    K = None
    for nkb in range(stages + 1, 6 * stages):       # the first k-block count that moves every tile's ring position
        small, big = _schedule(M1, N, bn, nkb, stages), _schedule(M2, N, bn, nkb, stages, P)
        if all(small[t][0] != big[t][0] and small[t][1] != big[t][1] for t in small):
            K = 64 * nkb
            break
    assert K is not None, "no K gives every tile another CTA and ring position"
    c = _prop_case(kind, dt, M1, bn, K, seed=11)
    r1 = _run_prop(c, dt, M1, bn, K)
    r2 = _run_prop(c, dt, M1, bn, K)
    r0 = _run_prop(c, dt, M1, bn, K, b_static=0)
    for k in r1:
        assert torch.equal(_bits(r1)[k], _bits(r2)[k]), f"{kind}: two identical calls differ ({k})"
        assert torch.equal(_bits(r1)[k], _bits(r0)[k]), f"{kind}: b_static 0 and 1 differ ({k})"
    # the same rows inside a larger problem
    cb = _prop_case(kind, dt, M2, bn, K, seed=12)
    cb["a"][P:P + M1] = c["a"]
    for key in ("h",):
        if key in cb["f"]:
            cb["f"][key][P:P + M1] = c["f"][key]
    if "gate" in cb["f"]:
        cb["f"]["gate"][:c["f"]["gate"].shape[0]] = c["f"]["gate"]
    if "bias" in cb["f"]:
        cb["f"]["bias"] = c["f"]["bias"]
    cb["w"] = c["w"]
    rb = _run_prop(cb, dt, M2, bn, K)
    for k in r1:
        assert torch.equal(_bits(r1)[k], _bits(rb)[k][P:P + M1]), f"{kind}: rows differ inside a larger M ({k})"


@pytest.mark.parametrize("dt", DTS)
def test_report_bn128_vs_bn256_bits(dt):
    """Not gated: whether the 128- and 256-wide tiles give the same bits (linear_auto picks either)."""
    for kind in ("store16", "head_norm16", "residual"):
        c = _prop_case(kind, dt, 1025, 128, 1536, seed=13)
        r128 = _run_prop(c, dt, 1025, 128, 1536)
        r256 = _run_prop(c, dt, 1025, 256, 1536)
        same = all(torch.equal(_bits(r128)[k], _bits(r256)[k]) for k in r128)
        print(f"[bn] {kind} {dt}: BN 128 and BN 256 bit-identical: {same}")


def test_probe_refuses_instances_the_forward_does_not_have():
    nat = _nat()
    a = torch.zeros(128, 64, dtype=torch.float16, device="cuda")
    w = torch.zeros(256, 64, dtype=torch.float16, device="cuda")
    out = torch.zeros(128, 256, dtype=torch.float16, device="cuda")
    for epi, bn in ((nat.EPI_QKV_ROPE, 128), (nat.EPI_STORE16, 64), (nat.EPI_RESIDUAL_LN, 128), (nat.EPI_SWIGLU, 128)):
        with pytest.raises(nat.NativeError, match="instances"):
            probe("fp16", epi, bn, a, w, 128, 256, 64, out=out, ld=256, head_dim=64, nf=16, h=out)
    with pytest.raises(nat.NativeError, match="multiple of 64"):
        probe("fp16", nat.EPI_SWIGLU, 256, a, w, 128, 96, 64, out=out, ld=256)
    with pytest.raises(nat.NativeError, match="K % 8"):
        probe("fp16", nat.EPI_STORE16, 256, a, w, 128, 256, 60, out=out, ld=256)

