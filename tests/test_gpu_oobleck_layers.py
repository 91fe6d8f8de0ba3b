"""GPU: every step of the Oobleck decoder and encoder, one layer at a time, against the float64 reference of
tests/conv_ref.py, element by element, through satb_oobleck_probe (the host functions, and so the kernel instances,
routes, next Snakes and raw streams, of the product decode / encode).

Each step reads random operands (exactly representable in the operand type; hi + lo in fp16x3) and the weights the
handle stored (satb_oobleck_weights), so the check measures the kernels, not the load-time rounding; the stored
weights are checked against the weight-norm fold on their own.  Every input and output buffer, and every lo half,
sits between NaN guard regions: no kernel may read them into a valid output (a NaN would show) or write them.
Shapes: L = 1, 2, 40 (dilation 9 halo longer than the item), 127, 128, 129, 257 at B = 1 and 3; channel widths 32,
64, 96, 128, 256, 512 and a 2048-channel layer; transposed-conv strides 2, 4, 8 with N = s * cout on BN 64, 128 and
256; strided-conv strides 2, 3, 4, 5, 8; a length whose tiles outnumber the SMs.  Snake parameters reach the largest
slope e^alpha / e^beta of SA-Open's synthetic weights.  Each step prints "[ratio] ..." and the module prints the worst
err/bound per route and dtype at the end."""
import ctypes
import functools
import math

import pytest
import torch

import conv_ref as C

pytestmark = pytest.mark.gpu

DTS = ["fp16", "bf16", "fp16x3"]
G = 8192     # guard elements around every buffer and lo half: more than a transposed conv reaches past either end
NAN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000}
INT_VIEW = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}
DILS = (1, 3, 9)
LATENT = 16
WORST = {}                                           # (route, dtype, output) -> worst err/bound


def _nat():
    from stable_audio_tools import _native
    return _native


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def worst_table():
    yield
    print("\n[table] worst err/bound per route and dtype")
    for (route, dt, out), r in sorted(WORST.items()):
        print(f"[table] {route:28s} {dt:7s} {out:10s} {r:.3f}")


@functools.lru_cache(maxsize=None)
def sao_slope():
    """The largest Snake slope term e^alpha / e^beta of SA-Open's synthetic decoder weights."""
    from oracle import oobleck_oracle as oo
    cfg = dict(out_channels=2, channels=128, c_mults=[1, 2, 4, 8, 16], strides=[2, 4, 4, 8, 8], latent_dim=64)
    sd = oo.make_oobleck_weights(oo.decoder_param_shapes(cfg), seed=0, transposed=oo.decoder_transposed_prefixes(cfg))
    return max(float((sd[k] - sd[k[:-5] + "beta"]).exp().max()) for k in sd if k.endswith("alpha"))


# ------------------------------------------------------------------------------------------------- models
class Model:
    """A finalized native handle: a one-stage decoder (chans [c, m c], stride s) or a two-stage encoder (chans
    [c, m c, m c], strides [s, 2]), with synthetic weights whose Snakes are spread to SA-Open's largest slope."""

    def __init__(self, dec, dt, c, m, s):
        from oracle import oobleck_oracle as oo
        nat = _nat()
        self.dec, self.dt, self.s = dec, dt, s
        mults, strides = ([m], [s]) if dec else ([m, m], [s, 2])
        self.chans = [c] + [k * c for k in mults]
        if dec:
            shapes = oo.decoder_param_shapes(dict(channels=c, c_mults=mults, strides=strides, latent_dim=LATENT,
                                                  out_channels=2))
            sd = oo.make_oobleck_weights(shapes, seed=c + s, transposed={"layers.1.layers.1."})
        else:
            shapes = oo.encoder_param_shapes(dict(channels=c, c_mults=mults, strides=strides, latent_dim=LATENT,
                                                  in_channels=2))
            sd = oo.make_oobleck_weights(shapes, seed=c + s)
        g = torch.Generator().manual_seed(c * 7 + s)
        half = math.log(sao_slope()) / 2 + 0.05
        for k in sd:
            if k.endswith("alpha"):
                n = sd[k].numel()
                sd[k] = torch.rand(n, generator=g) * (half + 1) - 1                # [-1, half]
                sd[k[:-5] + "beta"] = torch.rand(n, generator=g) * (half + 1) - half   # [-half, 1]
                sd[k][n // 3], sd[k[:-5] + "beta"][n // 3] = half, -half        # e^alpha / e^beta past SA-Open's max
            elif k.endswith("bias"):
                sd[k] = torch.randn(sd[k].shape, generator=g) * 0.3
        self.sd = {k: v.cuda().contiguous() for k, v in sd.items()}
        cfg = nat.SatbOobleckConfig()
        cfg.in_channels, cfg.channels, cfg.latent_dim, cfg.n_stages = 2, c, LATENT, len(mults)
        for i, (mm, ss) in enumerate(zip(mults, strides)):
            cfg.c_mults[i], cfg.strides[i] = mm, ss
        cfg.final_tanh, cfg.is_decoder, cfg.operand_dtype = 1, int(dec), DTS.index(dt)
        self.h = ctypes.c_void_p()
        lib = nat.lib()
        nat.check(lib.satb_oobleck_create(ctypes.byref(cfg), ctypes.byref(self.h)))
        for k, v in self.sd.items():
            nat.check(lib.satb_oobleck_load_weight(self.h, k.encode(), v.data_ptr(), v.numel(), nat.stream_ptr()))
        nat.check(lib.satb_oobleck_finalize(self.h, nat.stream_ptr()))

    def stored(self, pfx):
        """The handle's stored weights of conv pfx: raw bytes as a uint8 tensor."""
        nat = _nat()
        n = ctypes.c_longlong()
        nat.check(nat.lib().satb_oobleck_weights(self.h, pfx.encode(), None, ctypes.byref(n), nat.stream_ptr()))
        out = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        nat.check(nat.lib().satb_oobleck_weights(self.h, pfx.encode(), out.data_ptr(), ctypes.byref(n), nat.stream_ptr()))
        torch.cuda.synchronize()
        return out

    def weight(self, pfx, k, transposed, cin, cout, up=1):
        """The stored 16-bit weights (hi + lo) in the reference layout, float64."""
        b = self.stored(pfx)
        w = b.view(C.OPERAND[self.dt])
        total = cin * cout * k
        val = C.value(w[:total], w[total:2 * total] if self.dt == "fp16x3" else None)
        return C.stored_to_ref(val.view(-1, cin), k, transposed, cin, cout, up)

    def bias(self, pfx):
        return self.sd.get(pfx + "bias")

    def snake(self, pfx):
        return self.sd[pfx + "alpha"], self.sd[pfx + "beta"]


@functools.lru_cache(maxsize=None)
def model(dec, dt, c, m, s):
    return Model(dec, dt, c, m, s)


# ------------------------------------------------------------------------------------------------- buffers
def _pad8(n):
    return (n + 7) // 8 * 8


class Buf:
    """n elements between NaN guards; in fp16x3 mode a lo half of n elements starts lo_span elements after hi."""

    def __init__(self, n, dtype, lo_span=0):
        self.n, self.lo_span, self.dtype = n, lo_span, dtype
        self.t = torch.empty(G + lo_span + _pad8(n) + G, dtype=dtype, device="cuda")
        self.t.view(INT_VIEW[dtype]).fill_(NAN_BITS[dtype])

    @property
    def ptr(self):
        return self.t[G:].data_ptr()

    def hi(self):
        return self.t[G:G + self.n]

    def lo(self):
        return self.t[G + self.lo_span:G + self.lo_span + self.n] if self.lo_span else None

    def set(self, hi, lo=None):
        self.hi().copy_(hi.reshape(-1))
        if lo is not None:
            self.lo().copy_(lo.reshape(-1))
        return self

    def value(self, shape):
        return C.value(self.hi(), self.lo()).view(shape)

    def guards_ok(self):
        keep = torch.ones(self.t.numel(), dtype=torch.bool, device="cuda")
        keep[G:G + self.n] = False
        if self.lo_span:
            keep[G + self.lo_span:G + self.lo_span + self.n] = False
        return bool((self.t.view(INT_VIEW[self.dtype])[keep] == NAN_BITS[self.dtype]).all())


def act16(shape, dt, g):
    """A random 16-bit activation input: (hi, lo), the exact operand value being hi + lo."""
    return C.split(torch.randn(*shape, device="cuda", generator=g), dt)


# ------------------------------------------------------------------------------------------------- one step
class Step:
    """Buffers and result of one probe call.  inputs: name -> tensors (16-bit (hi, lo) pairs, or one fp32 tensor)."""

    def __init__(self, md, step, B, L, block=1, unit=0, **shapes):
        self.md, self.step, self.B, self.L, self.block, self.unit = md, step, B, L, block, unit
        self.shapes = shapes
        dt = md.dt
        n16 = [math.prod(v) for k, v in shapes.items() if k in ("in16", "out16", "scratch")]
        self.lo_span = _pad8(max(n16)) + G if dt == "fp16x3" and n16 else 0
        self.op = C.OPERAND[dt]
        self.raw_dt = C.RAW_DT[C.RAW[dt]]

    def run(self, inputs):
        nat = _nat()
        sh = self.shapes
        bufs = {}
        for name, shape in sh.items():
            if name in ("in16", "out16", "scratch"):
                bufs[name] = Buf(math.prod(shape), self.op, self.lo_span)
            elif name in ("raw_in", "raw_out"):
                bufs[name] = Buf(math.prod(shape), self.raw_dt)
            else:                                   # in32, out32
                bufs[name] = Buf(math.prod(shape), torch.float32)
        for name, val in inputs.items():
            bufs[name].set(*val) if isinstance(val, tuple) else bufs[name].set(val)
        p = nat.SatbOobleckProbe()
        p.step, p.block, p.unit, p.B, p.L = self.step, self.block, self.unit, self.B, self.L
        p.in_ = (bufs.get("in16") or bufs.get("in32")).ptr
        for f in ("raw_in", "raw_out", "out16", "scratch", "out32"):
            if f in bufs:
                setattr(p, f, bufs[f].ptr)
        p.lo_off = self.lo_span * 2
        nat.check(nat.lib().satb_oobleck_probe(self.md.h, ctypes.byref(p), nat.stream_ptr()))
        torch.cuda.synchronize()
        self.p, self.bufs = p, bufs
        for name, b in bufs.items():
            assert b.guards_ok(), f"{self.label()}: a guard region of {name} changed"
        return self

    def route(self):
        return "+".join(v for k, v in sorted(_nat().OOB_ROUTES.items()) if self.p.routes & k)

    def label(self):
        names = ["dec_in", "dec_up", "dec_res", "dec_out", "enc_in", "enc_res", "enc_down", "enc_out"]
        return f"{names[self.step]} b{self.block} j{self.unit} {self.md.dt} C{self.md.chans} s{self.md.s} B{self.B} L{self.L}"

    def result16(self):
        """The 16-bit result buffer: out16, or the ResidualUnit's in16 / scratch, whichever the probe reports."""
        if "out16" in self.bufs:
            return self.bufs["out16"]
        return self.bufs["scratch"] if self.p.result_in_scratch else self.bufs["in16"]

    def bits(self):
        """Every output's bits, for bit-identity comparisons."""
        out = {}
        for name in ("out16", "raw_out", "out32"):
            if name in self.bufs:
                out[name] = self.bufs[name].t.clone()
        if self.step in (_nat().OOB_DEC_RES, _nat().OOB_ENC_RES):
            out["res"] = self.result16().t.clone()
        return out


def report(st, out, got, ref, bound, **kw):
    rep = C.check(got, ref, bound, **kw)
    key = (st.route(), st.md.dt, out)
    WORST[key] = max(WORST.get(key, 0.0), rep.ratio)
    print(f"[ratio] {st.label()} {out} [{st.route()}]: {rep.ratio:.3f}  ({rep})")
    return rep


# ------------------------------------------------------------------------------------------------- step cases
def dec_steps(md, B, L, g):
    """(Step, inputs, check) for every step of a one-stage decoder at L latents."""
    nat = _nat()
    dt = md.dt
    c0, c1 = md.chans
    s = md.s
    L2 = L * s
    cases = []

    z = torch.randn(B, LATENT, L, device="cuda", generator=g)
    st = Step(md, nat.OOB_DEC_IN, B, L, in32=(B, LATENT, L), scratch=(B, L, LATENT), out16=(B, L, c1))

    def chk_in(st, z=z):
        hi, lo = C.split(z.transpose(1, 2), dt)
        copy = st.bufs["scratch"]
        assert torch.equal(copy.hi().view(hi.shape), hi) and (lo is None or torch.equal(copy.lo().view(lo.shape), lo)), \
            f"{st.label()}: the 16-bit copy of the latents is not their rounding"
        x = C.value(hi, lo)
        y, bd = C.snake(C.conv(x, md.weight("layers.0.", 7, False, LATENT, c1), dt, bias=md.bias("layers.0.")),
                        *md.snake("layers.1.layers.0."), dt)
        return [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, bn=min(256, max(64, c1)))]
    cases.append((st, {"in32": z}, chk_in))

    x = act16((B, L, c1), dt, g)
    st = Step(md, nat.OOB_DEC_UP, B, L, in16=(B, L, c1), raw_out=(B, L2, c0), out16=(B, L2, c0))

    def chk_up(st, x=x):
        p = C.conv(C.value(*x), md.weight("layers.1.layers.1.", 2 * s, True, c1, c0, s), dt, "up",
                   bias=md.bias("layers.1.layers.1."), s=s)
        y, bd = C.snake(p, *md.snake("layers.1.layers.2.layers.0."), dt)
        v, bv = C.raw(p, dt)
        bn = 256 if s * c0 >= 256 else (128 if s * c0 > 64 else 64)
        kw = dict(bn=bn, up=s, pad=math.ceil(s / 2))
        return [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, **kw),
                report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, **kw)]
    cases.append((st, {"in16": x}, chk_up))

    for j in range(3):
        nxt = f"layers.1.layers.{3 + j}.layers.0." if j < 2 else "layers.2."
        cases.append(res_case(md, nat.OOB_DEC_RES, 1, j, f"layers.1.layers.{2 + j}.", nxt, c0, B, L2, g))

    x = act16((B, L2, c0), dt, g)
    st = Step(md, nat.OOB_DEC_OUT, B, L2, in16=(B, L2, c0), out32=(B, 2, L2))

    def chk_out(st, x=x):
        y, bd = C.ncl_out(C.conv(C.value(*x), md.weight("layers.3.", 7, False, c0, 2), dt), tanh=True)
        return [report(st, "out32", st.bufs["out32"].value((B, 2, L2)).transpose(1, 2), y, bd)]
    cases.append((st, {"in16": x}, chk_out))
    return cases


def res_case(md, step, b, j, pfx, nxt, c, B, L, g):
    dt = md.dt
    x = act16((B, L, c), dt, g)
    skip = torch.randn(B, L, c, device="cuda", generator=g).to(C.RAW_DT[C.RAW[dt]])
    st = Step(md, step, B, L, block=b, unit=j, in16=(B, L, c), raw_in=(B, L, c), raw_out=(B, L, c), scratch=(B, L, c))

    def chk(st):
        p = C.residual_unit(C.value(*x), skip.double(), md.weight(pfx + "layers.1.", 7, False, c, c),
                            md.bias(pfx + "layers.1."), *md.snake(pfx + "layers.2."),
                            md.weight(pfx + "layers.3.", 1, False, c, c), md.bias(pfx + "layers.3."), DILS[j], dt)
        y, bd = C.snake(p, *md.snake(nxt), dt)
        reps = [report(st, "out16", st.result16().value(y.shape), y, bd, bn=min(256, c))]
        v, bv = C.raw(p, dt)
        if st.p.wrote_raw:
            reps.append(report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, bn=min(256, c)))
        else:
            assert torch.equal(st.bufs["raw_out"].hi(), skip.reshape(-1)), f"{st.label()}: raw stream changed"
        assert st.p.wrote_raw == (j < 2), f"{st.label()}: the raw output of unit {j} is written iff a later skip reads it"
        return reps
    return st, {"in16": x, "raw_in": skip}, chk


def enc_steps(md, B, L, g):
    """(Step, inputs, check) for every step of block 1 of a two-stage encoder at T = L * s samples, block 2's strided
    conv and the final conv."""
    nat = _nat()
    dt = md.dt
    c0, c1, c2 = md.chans
    s = md.s
    T = L * s
    cases = []

    a = torch.randn(B, 2, T, device="cuda", generator=g)
    st = Step(md, nat.OOB_ENC_IN, B, T, in32=(B, 2, T), raw_out=(B, T, c0), out16=(B, T, c0))

    def chk_in(st, a=a):
        w32 = md.stored("layers.0.").view(torch.float32).view(c0, 2, 7)
        p = C.conv_in(a, w32, md.bias("layers.0."))
        y, bd = C.snake(p, *md.snake("layers.1.layers.0.layers.0."), dt)
        v, bv = C.raw(p, dt)
        return [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd),
                report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv)]
    cases.append((st, {"in32": a}, chk_in))

    for j in range(3):
        nxt = f"layers.1.layers.{j + 1}.layers.0." if j < 2 else "layers.1.layers.3."
        cases.append(res_case(md, nat.OOB_ENC_RES, 1, j, f"layers.1.layers.{j}.", nxt, c0, B, T, g))

    for b, (cin, cout, ss, Lin, nxt) in enumerate([(c0, c1, s, T, "layers.2.layers.0.layers.0."),
                                                   (c1, c2, 2, 2 * L, "layers.3.")], start=1):
        x = act16((B, Lin, cin), dt, g)
        Lo = Lin // ss
        st = Step(md, nat.OOB_ENC_DOWN, B, Lin, block=b, in16=(B, Lin, cin), raw_out=(B, Lo, cout), out16=(B, Lo, cout))

        def chk_down(st, x=x, b=b, cin=cin, cout=cout, ss=ss, nxt=nxt):
            pfx = f"layers.{b}.layers.4."
            p = C.conv(C.value(*x), md.weight(pfx, 2 * ss, False, cin, cout), dt, "down", bias=md.bias(pfx), s=ss)
            y, bd = C.snake(p, *md.snake(nxt), dt)
            bn = 256 if cout >= 256 else (128 if cout > 64 else 64)
            reps = [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, bn=bn)]
            assert st.p.wrote_raw == (b < 2), f"{st.label()}: raw written iff a next block reads it"
            if st.p.wrote_raw:
                v, bv = C.raw(p, dt)
                reps.append(report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, bn=bn))
            return reps
        cases.append((st, {"in16": x}, chk_down))

    x = act16((B, L, c2), dt, g)
    st = Step(md, nat.OOB_ENC_OUT, B, L, in16=(B, L, c2), out32=(B, LATENT, L))

    def chk_out(st, x=x):
        y, bd = C.ncl_out(C.conv(C.value(*x), md.weight("layers.4.", 3, False, c2, LATENT), dt, bias=md.bias("layers.4.")))
        return [report(st, "out32", st.bufs["out32"].value((B, LATENT, L)).transpose(1, 2), y, bd)]
    cases.append((st, {"in16": x}, chk_out))
    return cases


def _item(val, i, step):
    """Item i of a batched input (keeping the batch dim)."""
    if isinstance(val, tuple):
        return tuple(v[i:i + 1] if v is not None else None for v in val)
    return val[i:i + 1]


def run_all(dec, dt, c, m, s, B, L, bits=False):
    md = model(dec, dt, c, m, s)
    g = torch.Generator(device="cuda").manual_seed(1000 * c + 10 * s + B + L)
    failed = []
    for st, inputs, chk in (dec_steps if dec else enc_steps)(md, B, L, g):
        st.run(inputs)
        for rep in chk(st):
            if not rep.ok:
                failed.append(f"{st.label()} [{st.route()}]: {rep}")
        if bits and B == 3:
            first = st.bits()
            again = Step(md, st.step, B, st.L, st.block, st.unit, **st.shapes).run(inputs).bits()
            for k in first:
                assert torch.equal(first[k].view(INT_VIEW[first[k].dtype]), again[k].view(INT_VIEW[again[k].dtype])), \
                    f"{st.label()}: {k} differs between two identical calls"
            one_shapes = {k: (1,) + v[1:] for k, v in st.shapes.items()}
            one = Step(md, st.step, 1, st.L, st.block, st.unit, **one_shapes).run(
                {k: _item(v, 1, st.step) for k, v in inputs.items()})
            for name in ("out16", "raw_out", "out32"):
                if name in st.bufs and (name != "raw_out" or st.p.wrote_raw):
                    n1 = one.bufs[name].n
                    for half in ("hi", "lo"):
                        a, b1 = getattr(st.bufs[name], half)(), getattr(one.bufs[name], half)()
                        if a is not None:
                            assert torch.equal(a[n1:2 * n1].view(INT_VIEW[a.dtype]), b1.view(INT_VIEW[b1.dtype])), \
                                f"{st.label()}: item 1 of 3 differs from the same item alone ({name} {half})"
            if st.step in (_nat().OOB_DEC_RES, _nat().OOB_ENC_RES):
                r3, r1 = st.result16(), one.result16()
                assert torch.equal(r3.hi()[r1.n:2 * r1.n].view(torch.int16), r1.hi().view(torch.int16)), \
                    f"{st.label()}: item 1 of 3 differs from the same item alone"
    assert not failed, "\n".join(failed)


# ------------------------------------------------------------------------------------------------- tests
DEC_CFGS = [(32, 2, 2), (64, 1, 2), (32, 4, 4), (96, 1, 4), (128, 2, 2), (256, 1, 8), (512, 1, 2)]
ENC_CFGS = [(32, 2, 2), (96, 1, 3), (128, 2, 4), (256, 1, 5), (64, 1, 8), (512, 1, 2)]
BL = [(1, 1), (3, 2), (1, 40), (1, 127), (3, 128), (1, 129), (3, 257)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c,m,s", DEC_CFGS)
@pytest.mark.parametrize("B,L", BL)
def test_decoder_steps(dt, c, m, s, B, L):
    run_all(True, dt, c, m, s, B, L, bits=True)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c,m,s", ENC_CFGS)
@pytest.mark.parametrize("B,L", BL)
def test_encoder_steps(dt, c, m, s, B, L):
    run_all(False, dt, c, m, s, B, L, bits=True)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("B,L", [(1, 1), (3, 2)])
def test_2048_channel_layers(dt, B, L):
    """SA-Open's widest layers at small L: the decoder's input conv to 2048 channels and its 2048 -> 1024 stride-8
    transposed conv (N = 8192), the encoder's 1024 -> 2048 strided conv and 2048-channel final conv."""
    run_all(True, dt, 1024, 2, 8, B, L)
    run_all(False, dt, 1024, 2, 8, B, L)


@pytest.mark.parametrize("dt", DTS)
def test_persistent_loop_wraps(dt):
    """More 128-position tiles than SMs: the decoder's input conv and transposed conv (lean GEMM in fp16, general in
    bf16) and the fused 128-channel ResidualUnit (fp16, bf16) each loop over the grid more than once."""
    run_all(True, dt, 128, 2, 2, 1, 128 * _sms() + 1)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("dec,c,m,s", [(True, cfg[0], cfg[1], cfg[2]) for cfg in DEC_CFGS]
                         + [(False, cfg[0], cfg[1], cfg[2]) for cfg in ENC_CFGS] + [(True, 1024, 2, 8), (False, 1024, 2, 8)])
def test_stored_weights_are_the_fold(dt, dec, c, m, s):
    """Every stored weight is the weight-norm fold g v / ||v|| rounded to the operand type (exactly, or one 16-bit ulp
    off where the fp32 fold sits on a rounding boundary) in the [tap][n][k] layout; the lo block holds the rounded
    remainder; the CUDA-core input conv keeps the fp32 fold."""
    md = model(dec, dt, c, m, s)
    for k in md.sd:
        if not k.endswith("weight_v"):
            continue
        pfx = k[:-len("weight_v")]
        w64 = C.fold(md.sd, pfx)
        transposed = dec and pfx == "layers.1.layers.1."
        d0, d1, kk = w64.shape
        cin, cout = (d0, d1) if transposed else (d1, d0)
        raw = md.stored(pfx)
        if not dec and pfx == "layers.0.":
            w32 = raw.view(torch.float32).view(cout, cin, kk).double()
            assert float(((w32 - w64).abs() / w64.abs().clamp_min(1e-30)).max()) <= 2.0 ** -17, pfx
            continue
        total = cin * cout * kk
        w = raw.view(C.OPERAND[dt])
        want = C.ref_to_stored(w64, kk, transposed, cin, cout, md.s).to(C.OPERAND[dt]).reshape(-1)
        got = w[:total]
        ib = got.view(torch.int16).int() - want.view(torch.int16).int()
        exact = ib == 0
        w64s = C.ref_to_stored(w64, kk, transposed, cin, cout, md.s).reshape(-1)
        mid = (got.double() + want.double()) / 2
        near_mid = (w64s - mid).abs() <= 2.0 ** -16 * w64s.abs()
        bad = ~exact & ~((ib.abs() == 1) & near_mid)
        assert not bool(bad.any()), f"{pfx}: {int(bad.sum())} of {total} stored weights are not the rounded fold"
        assert int((~exact).sum()) <= max(4, total // 500), f"{pfx}: too many one-ulp roundings ({int((~exact).sum())})"
        if dt == "fp16x3":
            lo = w[total:2 * total]
            err = (got.double() + lo.double() - w64s).abs()
            assert bool((err <= 2.0 ** -17 * w64s.abs() + 2.0 ** -24).all()), f"{pfx}: lo block is not the remainder"
