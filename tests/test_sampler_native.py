"""CPU: the native step path of inference/sampling.py (one satb_sampler_step launch per model call).

- the ctypes parameter block and the entry point's refusals (checked before any CUDA call);
- the host scalars of every fused step: with the kernel replaced by its torch restatement (sampler_step_ref.py) and
  the gate forced open, each sampler run in float64 must give the torch path's result, callback arguments and random
  draws, so every coefficient, index and draw order is the torch path's;
- the gate: which (sampler, callback, device) combinations take the native path, and how many launches they make."""
import ctypes
import os
import re
import types

import pytest
import torch

from sampler_step_ref import sampler_step_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sampling():
    from stable_audio_tools.inference import sampling
    return sampling


def model_fn(x, t, gain=1.0, **kw):            # a smooth stand-in for the v-prediction network
    return torch.tanh(x * gain) * (0.5 + t.view(-1, 1, 1)) - 0.1 * x


class Recorder:
    def __init__(self):
        self.seen = []

    def __call__(self, args):
        self.seen.append((args["i"], float(args.get("sigma", args.get("t"))), args["denoised"].clone(), args["x"].clone()))


def test_parameter_block_matches_the_header():
    from stable_audio_tools import _native
    text = open(os.path.join(ROOT, "include", "satb200.h")).read()
    body = re.search(r"typedef struct SatbSamplerStep \{(.*?)\} SatbSamplerStep;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            for part in decl.split(","):
                names.append(re.search(r"(\w+)\s*(\[\w+\])?\s*$", part.strip()).group(1))
    assert [f[0] for f in _native.SatbSamplerStep._fields_] == names
    assert ctypes.sizeof(_native.SatbSamplerStep) == 14 * 8 + 8 + 4 + 15 * 4      # no padding anywhere
    assert _native.SIGNATURES["satb_sampler_step"] == (ctypes.c_int, [ctypes.POINTER(_native.SatbSamplerStep),
                                                                      ctypes.c_void_p])


def test_entry_point_refuses_bad_arguments():
    """Fake 16-byte-aligned addresses: every refusal comes before a CUDA call, so nothing is dereferenced."""
    from stable_audio_tools import _native
    lib = _native.lib()
    fake = 1 << 20

    def call(**kw):
        p = _native.SatbSamplerStep(x=fake, y=fake, x_next=fake + 4096, n=1024, L=64)
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.satb_sampler_step(ctypes.byref(p), None), lib.satb_last_error()

    assert lib.satb_sampler_step(None, None) != 0 and b"null" in lib.satb_last_error()
    for kw, msg in [(dict(n=1030), b"multiple of 4"), (dict(n=0), b"multiple of 4"), (dict(y=None), b"null x or y"),
                    (dict(x_next=None), b"no output"), (dict(mask=fake), b"inpainting blend"),
                    (dict(mask=fake, init=fake, renoise=fake, L=100), b"inpainting blend"),
                    (dict(x_in_next=fake + 8), b"16-byte aligned")]:
        rc, err = call(**kw)
        assert rc != 0 and msg in err, (kw, err)
    p = _native.SatbSamplerStep(x=fake, y=fake, x_next=fake, n=1024, L=64)
    p.buf[2] = fake + 4
    assert lib.satb_sampler_step(ctypes.byref(p), None) != 0 and b"16-byte aligned" in lib.satb_last_error()


def _run(name, x, sigmas, callback=None, **kw):
    s = _sampling()
    fn = s.SAMPLERS[name]
    return fn(s.VDenoiser(model_fn), x, sigmas, callback=callback, extra_args={"gain": 0.7}, **kw)


def _case(seed=0, shape=(2, 4, 16)):
    torch.manual_seed(seed)
    x = torch.randn(*shape, dtype=torch.float64) * 20
    sigmas = _sampling().get_sigmas_polyexponential(7, 0.3, 20.0).to(torch.float64)
    return x, sigmas


FIXED = ["k-heun", "k-dpm-2", "k-lms", "k-dpmpp-2s-ancestral"]
CALLBACKS = ["none", "user", "inpaint", "inpaint+user"]


def _callback(kind, x, steps):
    s = _sampling()
    rec = Recorder()
    if kind == "none":
        return None, rec
    if kind == "user":
        return rec, rec
    g = torch.Generator().manual_seed(3)
    mask = torch.rand(x.shape[-1], generator=g)
    inp = s.InpaintingCallback(torch.randn(x.shape, generator=g, dtype=x.dtype), mask, steps)
    if kind == "inpaint":
        return inp, rec
    return (lambda args: (inp(args), rec(args))), rec


# the multistep SDE samplers without a callback run satb_sampler_update, unchanged, on the GPU only
@pytest.mark.parametrize("name,kind", [(n, k) for n in FIXED for k in CALLBACKS]
                         + [(n, k) for n in ("dpmpp-2m-sde", "dpmpp-3m-sde") for k in CALLBACKS[1:]])
def test_native_steps_reproduce_the_torch_path(name, kind, monkeypatch):
    """float64 on the CPU: the native path with the kernel's restatement equals the torch samplers to rounding, with
    the same callback arguments and the same random draws (the state after the run is compared, so a changed draw
    order would show)."""
    x0, sigmas = _case()
    steps = len(sigmas) - 1
    results = []
    for native in (False, True):
        with monkeypatch.context() as m:
            log = []
            if native:
                s = _sampling()
                m.setattr(s, "_fusable", lambda x: True)
                m.setattr(s, "_launch_step", lambda p: (log.append(p), sampler_step_ref(p)))
            cb, rec = _callback(kind, x0, steps)
            torch.manual_seed(11)
            out = _run(name, x0.clone(), sigmas, callback=cb)
            results.append((out, rec.seen, torch.randn(3), log))
    (ref, ref_seen, ref_next, _), (got, seen, nxt, log) = results
    assert len(log) > 0
    scale = float(ref.abs().max())
    assert float((got - ref).abs().max()) <= 1e-10 * scale, name
    assert torch.equal(nxt, ref_next), "the native path drew a different number of random values"
    assert [(i, sg) for i, sg, _, _ in seen] == [(i, sg) for i, sg, _, _ in ref_seen]
    for (_, _, d, xx), (_, _, rd, rx) in zip(seen, ref_seen):
        assert float((d - rd).abs().max()) <= 1e-10 * scale
        assert float((xx - rx).abs().max()) <= 1e-10 * scale


@pytest.mark.parametrize("with_callback", [False, True])
def test_native_rectified_flow_reproduces_the_torch_path(with_callback, monkeypatch):
    s = _sampling()
    torch.manual_seed(0)
    x0 = torch.randn(2, 4, 16, dtype=torch.float64)
    results = []
    for native in (False, True):
        with monkeypatch.context() as m:
            log = []
            if native:
                m.setattr(s, "_fusable", lambda x: True)
                m.setattr(s, "_launch_step", lambda p: (log.append(p), sampler_step_ref(p)))
            rec = Recorder()
            out = s.sample_discrete_euler(model_fn, x0.clone(), 9, sigma_max=0.9,
                                          callback=rec if with_callback else None, gain=0.7)
            results.append((out, rec.seen, log))
    (ref, ref_seen, _), (got, seen, log) = results
    assert len(log) == 9 * (2 if with_callback else 1)
    assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    assert [(i, t) for i, t, _, _ in seen] == [(i, t) for i, t, _, _ in ref_seen]
    for (_, _, d, _), (_, _, rd, _) in zip(seen, ref_seen):
        assert float((d - rd).abs().max()) <= 1e-12 * float(rd.abs().max())


def test_fused_blend_equals_the_torch_callback_bit_for_bit(monkeypatch):
    """The kernel's blend (restated) selects init + renoise * sigma exactly where the torch callback does, in fp32."""
    s = _sampling()
    monkeypatch.setattr(s, "_launch_step", sampler_step_ref)
    torch.manual_seed(1)
    x = torch.randn(2, 3, 40)
    inp = s.InpaintingCallback(torch.randn(2, 3, 40), torch.rand(40), 10)
    for i in range(10):
        sigma = torch.tensor(3.7 - 0.3 * i)
        torch.manual_seed(i)
        eager = x.clone()
        inp({"i": i, "x": eager, "sigma": sigma})
        torch.manual_seed(i)
        fused = x.clone()
        s._step(fused, torch.zeros_like(x), blend=(inp, i, torch.randn_like(inp.init_data), float(sigma)))
        assert torch.equal(fused, eager), i


def _launches(name, x, sigmas, callback, monkeypatch, fusable=None):
    s = _sampling()
    log, calls = [], []

    def counted(xx, t, **kw):
        calls.append(1)
        return model_fn(xx, t, **kw)
    with monkeypatch.context() as m:
        if fusable is not None:
            m.setattr(s, "_fusable", fusable)
        m.setattr(s, "_launch_step", lambda p: (log.append(p), sampler_step_ref(p)))
        fn = s.SAMPLERS[name]
        if name in ("k-dpm-fast", "k-dpm-adaptive"):
            fn(s.VDenoiser(counted), x, 0.3, 20.0, **({"n": 6} if name == "k-dpm-fast" else {}), callback=callback)
        else:
            fn(s.VDenoiser(counted), x, sigmas, callback=callback)
    return len(log), len(calls)


def test_gate():
    s = _sampling()
    fake = lambda **kw: types.SimpleNamespace(**dict(dict(is_cuda=True, dtype=torch.float32, numel=lambda: 64), **kw))
    assert s._fusable(fake())
    assert not s._fusable(fake(is_cuda=False))
    assert not s._fusable(fake(dtype=torch.float16))
    assert not s._fusable(fake(numel=lambda: 66))
    assert not s._fusable(torch.zeros(4, 4))


@pytest.mark.parametrize("name", FIXED + ["k-dpm-fast", "k-dpm-adaptive"])
@pytest.mark.parametrize("kind", CALLBACKS)
def test_which_combinations_fuse(name, kind, monkeypatch):
    """CPU tensors never launch; with the gate open, every fixed-step sampler makes one launch per model call, plus
    one denoised-only launch per step for a callback other than the bare inpainting one; the DPM-Solver samplers
    keep their torch arithmetic."""
    x, sigmas = _case()
    steps = len(sigmas) - 1
    x = x.float()
    cb, _ = _callback(kind, x, steps)
    assert _launches(name, x.clone(), sigmas.float(), cb, monkeypatch)[0] == 0
    cb, _ = _callback(kind, x, steps)
    launches, calls = _launches(name, x.clone(), sigmas.float(), cb, monkeypatch, fusable=lambda t: True)
    if name in ("k-dpm-fast", "k-dpm-adaptive"):
        assert launches == 0
    else:
        extra = steps if kind in ("user", "inpaint+user") else 0
        assert launches == calls + extra, (launches, calls)


def test_other_wrappers_keep_the_torch_path(monkeypatch):
    """A denoiser that is not the standard VDenoiser is not fused, even with the gate open."""
    s = _sampling()
    x, sigmas = _case()
    log = []
    monkeypatch.setattr(s, "_fusable", lambda t: True)
    monkeypatch.setattr(s, "_launch_step", lambda p: log.append(p))
    den = lambda xx, sigma, **kw: xx * 0.5
    for name in FIXED:
        s.SAMPLERS[name](den, x.clone(), sigmas)
    assert log == []


def test_inpainting_fold_needs_a_matching_mask_and_init():
    s = _sampling()
    x = torch.zeros(2, 3, 8)
    good = s.InpaintingCallback(torch.zeros(2, 3, 8), torch.zeros(8), 4)
    assert good.foldable(x)
    assert not s.InpaintingCallback(torch.zeros(2, 3, 8), torch.zeros(1, 8), 4).foldable(x)
    assert not s.InpaintingCallback(torch.zeros(2, 3, 8), torch.zeros(8, dtype=torch.float64), 4).foldable(x)
    assert not s.InpaintingCallback(torch.zeros(1, 3, 8), torch.zeros(8), 4).foldable(x)
    assert not s.InpaintingCallback(torch.zeros(2, 8, 3).transpose(1, 2), torch.zeros(8), 4).foldable(x)
