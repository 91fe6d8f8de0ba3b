"""CPU: the Oobleck convolution checker of tests/conv_ref.py is sharp.  It accepts the float64 reference rounded to
the output type, and rejects each of the wrong kernels a per-layer test is there to catch (the mutated reference,
rounded the same way), at the fp16, bf16 and fp16x3 bounds."""
import math

import pytest
import torch

import conv_ref as C

DTS = ["fp16", "bf16", "fp16x3"]
B, L, CH = 2, 40, 64


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def act(shape, dt, g):
    """Exact operand values of a 16-bit activation input (hi + lo in fp16x3)."""
    return C.round16(torch.randn(*shape, generator=g, dtype=torch.float64), dt)


def weight(shape, fan_in, dt, g):
    return C.round16(torch.randn(*shape, generator=g, dtype=torch.float64) * 0.7 / math.sqrt(fan_in), dt)


def snake_params(c, g):
    """alpha, beta spread wide enough that e^alpha / e^beta reaches ~6 (the largest Snake slope of SA-Open's synthetic
    weights)."""
    return torch.rand(c, generator=g) * 1.8 - 0.9, torch.rand(c, generator=g) * 1.8 - 0.9


def assert_sharp(dt, got_ok, got_bad, ref, bound, what, **kw):
    ok = C.check(got_ok, ref, bound, **kw)
    assert ok.ok, f"{dt} {what}: the correct result is rejected: {ok}"
    bad = C.check(got_bad, ref, bound, **kw)
    assert not bad.ok, f"{dt} {what}: the mutation passes: {bad}"


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("s", [2, 4])
@pytest.mark.parametrize("mutation", ["phase", "shift"])
def test_transposed_conv_geometry(dt, s, mutation):
    g = _gen(1 + s)
    cin, cout = CH, 32
    x = act((B, L, cin), dt, g)
    w = weight((cin, cout, 2 * s), 2 * cin, dt, g)
    bias = torch.randn(cout, generator=g) * 0.3
    al, be = snake_params(cout, g)
    p = C.conv(x, w, dt, "up", bias=bias, s=s)
    y, bound = C.snake(p, al, be, dt)
    if mutation == "shift":                 # output position l*s + ph - pad + 1
        bad = torch.cat([y[:, 1:], y[:, -1:]], 1)
    else:                                   # phase (pos + pad) % s taken from the next phase
        pos = torch.arange(L * s)
        src = (pos // s) * s + (pos % s + 1) % s
        bad = y[:, src]
    pad = math.ceil(s / 2)
    assert_sharp(dt, C.round16(y, dt), C.round16(bad, dt), y, bound, f"up s{s} {mutation}", bn=128, up=s, pad=pad)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("s", [3, 5])
def test_strided_conv_padding(dt, s):
    """pad floor(s/2) instead of ceil(s/2): only odd strides tell them apart."""
    g = _gen(10 + s)
    x = act((B, L * s, CH), dt, g)
    w = weight((CH, CH, 2 * s), 2 * s * CH, dt, g)
    bias = torch.randn(CH, generator=g) * 0.3
    al, be = snake_params(CH, g)
    y, bound = C.snake(C.conv(x, w, dt, "down", bias=bias, s=s), al, be, dt)
    # output l reads x[l s - floor(s/2) + t] = x[l s - ceil(s/2) + t + 1]: the input moved one position left
    x_left = torch.cat([x[:, 1:], torch.zeros_like(x[:, :1])], 1)
    bad, _ = C.snake(C.conv(x_left, w, dt, "down", bias=bias, s=s), al, be, dt)
    assert_sharp(dt, C.round16(y, dt), C.round16(bad, dt), y, bound, f"down s{s} floor pad")


def _unit(dt, g, c=CH):
    x = act((B, L, c), dt, g)
    skip = C.round_raw(torch.randn(B, L, c, generator=g, dtype=torch.float64), C.RAW[dt])
    w7 = weight((c, c, 7), 7 * c, dt, g)
    w1 = weight((c, c, 1), c, dt, g)
    b7, b1 = torch.randn(c, generator=g) * 0.3, torch.randn(c, generator=g) * 0.3
    a2, be2 = snake_params(c, g)
    an, ben = snake_params(c, g)
    return x, skip, w7, b7, a2, be2, w1, b1, an, ben


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("mutation", ["dilation", "halo_first", "halo_last", "skip_chunk", "snake_channel",
                                      "snake_not_exp", "inner_bias"])
def test_residual_unit_mutations(dt, mutation):
    g = _gen(20)
    x, skip, w7, b7, a2, be2, w1, b1, an, ben = _unit(dt, g)
    dil = 3 if mutation != "dilation" else 9
    p = C.residual_unit(x, skip, w7, b7, a2, be2, w1, b1, dil, dt)
    y, bound = C.snake(p, an, ben, dt)
    if mutation == "dilation":              # dilation 9 run where 3 was asked (and vice versa)
        bad, _ = C.snake(C.residual_unit(x, skip, w7, b7, a2, be2, w1, b1, 3, dt), an, ben, dt)
    elif mutation.startswith("halo"):       # the item's edge position computed over the neighbouring item's rows
        flat = C.residual_unit(x.reshape(1, B * L, CH), skip.reshape(1, B * L, CH), w7, b7, a2, be2, w1, b1, dil, dt)
        fy, _ = C.snake(flat, an, ben, dt)
        fy = fy.reshape(B, L, CH)
        bad = y.clone()
        if mutation == "halo_first":
            bad[1, 0] = fy[1, 0]
        else:
            bad[0, L - 1] = fy[0, L - 1]
    elif mutation == "skip_chunk":          # skip dropped on channels 32 .. 63
        sk = skip.clone()
        sk[..., 32:64] = 0
        bad, _ = C.snake(C.residual_unit(x, sk, w7, b7, a2, be2, w1, b1, dil, dt), an, ben, dt)
    elif mutation == "snake_channel":       # next Snake with channel co + 1's parameters
        bad, _ = C.snake(p, an.roll(-1), ben.roll(-1), dt)
    elif mutation == "snake_not_exp":
        bad, _ = C.snake(p, an, ben, dt, exp_alpha=False)
    else:                                   # conv7 bias missing inside the fused unit
        bad, _ = C.snake(C.residual_unit(x, skip, w7, b7, a2, be2, w1, b1, dil, dt, inner_bias=False), an, ben, dt)
    assert_sharp(dt, C.round16(y, dt), C.round16(bad, dt), y, bound, mutation, bn=CH)


@pytest.mark.parametrize("dt", DTS)
def test_raw_stream_is_checked(dt):
    """The raw output at its own type's bound: a raw stream that lost the skip on one chunk fails."""
    g = _gen(30)
    x, skip, w7, b7, a2, be2, w1, b1, _, _ = _unit(dt, g)
    p = C.residual_unit(x, skip, w7, b7, a2, be2, w1, b1, 1, dt)
    v, bound = C.raw(p, dt)
    sk = skip.clone()
    sk[..., :32] = 0
    bad = C.residual_unit(x, sk, w7, b7, a2, be2, w1, b1, 1, dt).v
    assert_sharp(dt, C.round_raw(v, C.RAW[dt]), C.round_raw(bad, C.RAW[dt]), v, bound, "raw skip chunk")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("s", [2, 4, 8])
def test_transposed_weight_layout(dt, s):
    """A kernel that reads the mode-1 layout at ph + (1 - tap) * up computes a different convolution; the layout
    functions round-trip."""
    g = _gen(40 + s)
    cin, cout = CH, 32
    w = weight((cin, cout, 2 * s), 2 * cin, dt, g)
    stored = C.ref_to_stored(w, 2 * s, True, cin, cout, s)
    assert torch.equal(C.stored_to_ref(stored, 2 * s, True, cin, cout, s), w)
    flipped = C.stored_to_ref(stored, 2 * s, True, cin, cout, s, tap_flip=True)
    x = act((B, L, cin), dt, g)
    bias = torch.randn(cout, generator=g) * 0.3
    al, be = snake_params(cout, g)
    y, bound = C.snake(C.conv(x, w, dt, "up", bias=bias, s=s), al, be, dt)
    bad, _ = C.snake(C.conv(x, flipped, dt, "up", bias=bias, s=s), al, be, dt)
    assert_sharp(dt, C.round16(y, dt), C.round16(bad, dt), y, bound, "tap flip", bn=128, up=s, pad=math.ceil(s / 2))


def test_conv_weight_layout_round_trips():
    w = torch.randn(48, 32, 7, dtype=torch.float64)
    stored = C.ref_to_stored(w, 7, False, 32, 48)
    assert stored.shape == (7 * 48, 32) and torch.equal(stored[2 * 48 + 5], w[5, :, 2])
    assert torch.equal(C.stored_to_ref(stored, 7, False, 32, 48), w)
    wt = torch.randn(32, 16, 8, dtype=torch.float64)           # ConvTranspose1d, stride 4
    st = C.ref_to_stored(wt, 8, True, 32, 16, 4)
    # row tap * up * cout + ph * cout + co holds w[:, co, ph + tap * up]
    assert torch.equal(st[1 * 4 * 16 + 2 * 16 + 3], wt[:, 3, 2 + 1 * 4])


@pytest.mark.parametrize("dt", DTS)
def test_final_conv_and_input_conv(dt):
    g = _gen(50)
    x = act((B, L, CH), dt, g)
    w = weight((2, CH, 7), 7 * CH, dt, g)
    y, bound = C.ncl_out(C.conv(x, w, dt), tanh=True)
    bad = torch.cat([y[:, 1:], y[:, -1:]], 1)
    assert_sharp(dt, y.float().double(), bad.float().double(), y, bound, "final conv shift")
    audio = torch.randn(B, 2, L, generator=g)
    w32 = torch.randn(CH, 2, 7, generator=g) * 0.3
    bias = torch.randn(CH, generator=g) * 0.1
    p = C.conv_in(audio, w32, bias)
    al, be = snake_params(CH, g)
    y, bound = C.snake(p, al, be, dt)
    bad = C.conv_in(audio.roll(1, 2), w32, bias)
    assert_sharp(dt, C.round16(y, dt), C.round16(C.snake(bad, al, be, dt)[0], dt), y, bound, "input conv shift")
