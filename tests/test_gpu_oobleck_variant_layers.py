"""GPU: every step of ELU Oobleck decoders and encoders, and the nearest-upsample conv of Snake and ELU decoders, one
layer at a time through satb_oobleck_probe, element by element against the float64 reference of tests/conv_ref.py and
tests/oobleck_variant_ref.py, with the NaN guards of tests/test_gpu_oobleck_layers.py around every buffer and lo half.

Routes: the lean and general EpiConv epilogues (fp16 / bf16, fp16x3), the fused ResidualUnit (128 / 256 channels) and
the two-launch one (512 channels, fp16x3), the CUDA-core encoder input conv, and the 3-tap nearest-upsample GEMM at
strides 2, 3, 4, 5, 8 with N = s * cout on BN 64, 128 and 256, L = 1 .. 257, B = 1 and 3.  Batch item 1 of 3 is
bit-identical to the same item run alone."""
import ctypes
import functools
import math

import pytest
import torch

import conv_ref as C
import oobleck_variant_ref as V
from test_gpu_oobleck_layers import DILS, INT_VIEW, LATENT, Step, _item, act16, report, sao_slope

pytestmark = pytest.mark.gpu

DTS = ["fp16", "bf16", "fp16x3"]


def _nat():
    from stable_audio_tools import _native
    return _native


class VariantModel:
    """A finalized native handle like test_gpu_oobleck_layers.Model (one-stage decoder, two-stage encoder), built with
    satb_oobleck_create_variant: ELU or Snake activations, nearest or transposed upsampling."""

    def __init__(self, dec, dt, c, m, s, snake, nearest):
        from oracle import oobleck_oracle as oo
        from oracle import oobleck_variants_oracle as ov
        nat = _nat()
        self.dec, self.dt, self.s, self.snake_act, self.nearest = dec, dt, s, snake, nearest
        mults, strides = ([m], [s]) if dec else ([m, m], [s, 2])
        self.chans = [c] + [k * c for k in mults]
        opts = dict(use_snake=snake, use_nearest_upsample=nearest)
        if dec:
            cfg = dict(channels=c, c_mults=mults, strides=strides, latent_dim=LATENT, out_channels=2, **opts)
            sd = ov.make_decoder_weights(cfg, seed=c + s)
        else:
            cfg = dict(channels=c, c_mults=mults, strides=strides, latent_dim=LATENT, in_channels=2, use_snake=snake)
            sd = ov.make_encoder_weights(cfg, seed=c + s)
        g = torch.Generator().manual_seed(c * 7 + s)
        half = math.log(sao_slope()) / 2 + 0.05
        for k in sd:
            if k.endswith("alpha"):
                n = sd[k].numel()
                sd[k] = torch.rand(n, generator=g) * (half + 1) - 1
                sd[k[:-5] + "beta"] = torch.rand(n, generator=g) * (half + 1) - half
                sd[k][n // 3], sd[k[:-5] + "beta"][n // 3] = half, -half
            elif k.endswith("bias"):
                sd[k] = torch.randn(sd[k].shape, generator=g) * 0.3
        self.sd = {k: v.cuda().contiguous() for k, v in sd.items()}
        ncfg = nat.SatbOobleckConfig()
        ncfg.in_channels, ncfg.channels, ncfg.latent_dim, ncfg.n_stages = 2, c, LATENT, len(mults)
        for i, (mm, ss) in enumerate(zip(mults, strides)):
            ncfg.c_mults[i], ncfg.strides[i] = mm, ss
        ncfg.final_tanh, ncfg.is_decoder, ncfg.operand_dtype = 1, int(dec), DTS.index(dt)
        self.h = ctypes.c_void_p()
        lib = nat.lib()
        act = nat.OOB_ACT_SNAKE if snake else nat.OOB_ACT_ELU
        nat.check(lib.satb_oobleck_create_variant(ctypes.byref(ncfg), act, int(nearest), ctypes.byref(self.h)))
        for k, v in self.sd.items():
            nat.check(lib.satb_oobleck_load_weight(self.h, k.encode(), v.data_ptr(), v.numel(), nat.stream_ptr()))
        nat.check(lib.satb_oobleck_finalize(self.h, nat.stream_ptr()))

    def stored(self, pfx):
        nat = _nat()
        n = ctypes.c_longlong()
        nat.check(nat.lib().satb_oobleck_weights(self.h, pfx.encode(), None, ctypes.byref(n), nat.stream_ptr()))
        out = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        nat.check(nat.lib().satb_oobleck_weights(self.h, pfx.encode(), out.data_ptr(), ctypes.byref(n), nat.stream_ptr()))
        torch.cuda.synchronize()
        return out

    def _val(self, pfx, total):
        w = self.stored(pfx).view(C.OPERAND[self.dt])
        assert w.numel() == total * (2 if self.dt == "fp16x3" else 1)
        return C.value(w[:total], w[total:2 * total] if self.dt == "fp16x3" else None)

    def weight(self, pfx, k, transposed, cin, cout, up=1):
        return C.stored_to_ref(self._val(pfx, cin * cout * k).view(-1, cin), k, transposed, cin, cout, up)

    def nearest_weight(self, pfx, cin, cout, s, tap_shift=0):
        return V.nearest_stored_to_ref(self._val(pfx, 3 * s * cout * cin), s, cout, cin, tap_shift)

    def bias(self, pfx):
        return self.sd.get(pfx + "bias")

    def act(self, p, pfx):
        """The activation at pfx applied to Pre p, rounded to 16 bits: (y, bound)."""
        if self.snake_act:
            return C.snake(p, self.sd[pfx + "alpha"], self.sd[pfx + "beta"], self.dt)
        assert pfx + "alpha" not in self.sd
        return V.elu(p, self.dt)


@functools.lru_cache(maxsize=None)
def model(dec, dt, c, m, s, snake=False, nearest=False):
    return VariantModel(dec, dt, c, m, s, snake, nearest)


def _bn(n):
    return 256 if n >= 256 else (128 if n > 64 else 64)


def res_case(md, step, b, j, pfx, nxt, c, B, L, g):
    dt = md.dt
    x = act16((B, L, c), dt, g)
    skip = torch.randn(B, L, c, device="cuda", generator=g).to(C.RAW_DT[C.RAW[dt]])
    st = Step(md, step, B, L, block=b, unit=j, in16=(B, L, c), raw_in=(B, L, c), raw_out=(B, L, c), scratch=(B, L, c))

    def chk(st):
        # the inner activation (snake2 / ELU) of the unit, then the 1x1 conv: conv_ref.residual_unit with the act's bound
        p7 = C.conv(C.value(*x), md.weight(pfx + "layers.1.", 7, False, c, c), dt, bias=md.bias(pfx + "layers.1."),
                    dil=DILS[j])
        t, dt_ = md.act(p7, pfx + "layers.2.")
        w1 = md.weight(pfx + "layers.3.", 1, False, c, c)
        p1 = C.conv(t, w1, dt, bias=md.bias(pfx + "layers.3."), skip=skip.double())
        p = C.Pre(p1.v, p1.dv + C._conv(dt_, w1.abs(), "conv"))
        y, bd = md.act(p, nxt)
        reps = [report(st, "out16", st.result16().value(y.shape), y, bd, bn=min(256, c))]
        if st.p.wrote_raw:
            v, bv = C.raw(p, dt)
            reps.append(report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, bn=min(256, c)))
        else:
            assert torch.equal(st.bufs["raw_out"].hi(), skip.reshape(-1)), f"{st.label()}: raw stream changed"
        assert st.p.wrote_raw == (j < 2)
        return reps
    return st, {"in16": x, "raw_in": skip}, chk


def up_case(md, B, L, g, tap_shift=0):
    """The decoder block's upsampling step (DEC_UP): transposed conv, or the nearest 3-tap GEMM."""
    nat = _nat()
    dt = md.dt
    c0, c1 = md.chans
    s = md.s
    x = act16((B, L, c1), dt, g)
    st = Step(md, nat.OOB_DEC_UP, B, L, in16=(B, L, c1), raw_out=(B, L * s, c0), out16=(B, L * s, c0))

    def chk(st):
        if md.nearest:
            p = V.conv_nearest(C.value(*x), md.nearest_weight("layers.1.layers.1.1.", c1, c0, s, tap_shift), dt)
            kw = dict(bn=_bn(s * c0), up=s, pad=0)
        else:
            p = C.conv(C.value(*x), md.weight("layers.1.layers.1.", 2 * s, True, c1, c0, s), dt, "up",
                       bias=md.bias("layers.1.layers.1."), s=s)
            kw = dict(bn=_bn(s * c0), up=s, pad=math.ceil(s / 2))
        y, bd = md.act(p, "layers.1.layers.2.layers.0.")
        v, bv = C.raw(p, dt)
        return [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, **kw),
                report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, **kw)]
    return st, {"in16": x}, chk


def dec_steps(md, B, L, g):
    nat = _nat()
    dt = md.dt
    c0, c1 = md.chans
    L2 = L * md.s
    cases = []
    z = torch.randn(B, LATENT, L, device="cuda", generator=g)
    st = Step(md, nat.OOB_DEC_IN, B, L, in32=(B, LATENT, L), scratch=(B, L, LATENT), out16=(B, L, c1))

    def chk_in(st, z=z):
        x = C.value(*C.split(z.transpose(1, 2), dt))
        y, bd = md.act(C.conv(x, md.weight("layers.0.", 7, False, LATENT, c1), dt, bias=md.bias("layers.0.")),
                       "layers.1.layers.0.")
        return [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, bn=min(256, max(64, c1)))]
    cases.append((st, {"in32": z}, chk_in))
    cases.append(up_case(md, B, L, g))
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


def enc_steps(md, B, L, g):
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
        y, bd = md.act(p, "layers.1.layers.0.layers.0.")
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
        st = Step(md, nat.OOB_ENC_DOWN, B, Lin, block=b, in16=(B, Lin, cin), raw_out=(B, Lin // ss, cout),
                  out16=(B, Lin // ss, cout))

        def chk_down(st, x=x, b=b, cin=cin, cout=cout, ss=ss, nxt=nxt):
            pfx = f"layers.{b}.layers.4."
            p = C.conv(C.value(*x), md.weight(pfx, 2 * ss, False, cin, cout), dt, "down", bias=md.bias(pfx), s=ss)
            y, bd = md.act(p, nxt)
            reps = [report(st, "out16", st.bufs["out16"].value(y.shape), y, bd, bn=_bn(cout))]
            if st.p.wrote_raw:
                v, bv = C.raw(p, dt)
                reps.append(report(st, "raw", st.bufs["raw_out"].value(v.shape), v, bv, bn=_bn(cout)))
            return reps
        cases.append((st, {"in16": x}, chk_down))
    x = act16((B, L, c2), dt, g)
    st = Step(md, nat.OOB_ENC_OUT, B, L, in16=(B, L, c2), out32=(B, LATENT, L))

    def chk_out(st, x=x):
        y, bd = C.ncl_out(C.conv(C.value(*x), md.weight("layers.4.", 3, False, c2, LATENT), dt, bias=md.bias("layers.4.")))
        return [report(st, "out32", st.bufs["out32"].value((B, LATENT, L)).transpose(1, 2), y, bd)]
    cases.append((st, {"in16": x}, chk_out))
    return cases


def run_cases(md, cases, B):
    failed, routes = [], set()
    for st, inputs, chk in cases:
        st.run(inputs)
        routes.add(st.route())
        for rep in chk(st):
            if not rep.ok:
                failed.append(f"{st.label()} [{st.route()}]: {rep}")
        if B == 3:
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
    assert not failed, "\n".join(failed)
    return routes


BL = [(1, 1), (3, 2), (1, 40), (3, 129), (1, 257)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c,m,s", [(32, 2, 2), (128, 2, 4), (256, 1, 2), (512, 1, 2)])
@pytest.mark.parametrize("B,L", BL)
def test_elu_decoder_steps(dt, c, m, s, B, L):
    md = model(True, dt, c, m, s)
    g = torch.Generator(device="cuda").manual_seed(1000 * c + 10 * s + B + L)
    routes = run_cases(md, dec_steps(md, B, L, g), B)
    if dt == "fp16" and c in (128, 256):
        assert any("fused_lean" in r for r in routes), routes
    if c == 512 or dt == "fp16x3":
        assert not any("fused" in r for r in routes), routes


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c,m,s", [(32, 2, 2), (128, 2, 3), (256, 1, 5), (512, 1, 2)])
@pytest.mark.parametrize("B,L", BL)
def test_elu_encoder_steps(dt, c, m, s, B, L):
    md = model(False, dt, c, m, s)
    g = torch.Generator(device="cuda").manual_seed(2000 * c + 10 * s + B + L)
    routes = run_cases(md, enc_steps(md, B, L, g), B)
    assert any("cuda_core" in r for r in routes), routes


# (c0, m, s): N = s * c0 on BN 64 (s * c0 <= 64), 128 (<= 128) and 256
NEAREST = [(32, 2, 2), (32, 1, 3), (32, 2, 4), (32, 2, 5), (32, 1, 8), (64, 2, 2), (64, 1, 3), (64, 2, 5), (128, 1, 8)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("snake", [True, False])
@pytest.mark.parametrize("c,m,s", NEAREST)
def test_nearest_upsample_conv(dt, snake, c, m, s):
    md = model(True, dt, c, m, s, snake=snake, nearest=True)
    for B, L in [(1, 1), (3, 2), (1, 7), (3, 64), (1, 127), (3, 128), (1, 129), (3, 257)]:
        g = torch.Generator(device="cuda").manual_seed(3000 * c + 10 * s + B + L)
        run_cases(md, [up_case(md, B, L, g)], B)


@pytest.mark.parametrize("dt", ["fp16", "fp16x3"])
def test_nearest_decoder_all_steps(dt):
    """Every step of a nearest-upsampling decoder (ELU, stride 3): the same kernels as the transposed decoder after the
    upsampling step, fed by its output layout."""
    md = model(True, dt, 64, 2, 3, snake=False, nearest=True)
    g = torch.Generator(device="cuda").manual_seed(7)
    run_cases(md, dec_steps(md, 3, 43, g), 3)


def test_checker_catches_a_wrong_phase_tap():
    """The reference with every phase's taps read one block over (o shifted by one) is rejected on the kernel's real
    output: the check can see a kernel that misplaces the 3-tap offsets."""
    md = model(True, "fp16", 32, 2, 3, snake=True, nearest=True)
    for shift in (1, -1):
        g = torch.Generator(device="cuda").manual_seed(11)
        st, inputs, chk = up_case(md, 3, 40, g, tap_shift=shift)
        st.run(inputs)
        reps = chk(st)
        assert not reps[0].ok and reps[0].ratio > 10, reps[0]
