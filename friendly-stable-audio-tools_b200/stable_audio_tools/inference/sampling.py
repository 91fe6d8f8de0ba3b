"""Samplers for the v-objective denoiser.

``sample`` is the reference's v-diffusion DDIM sampler (``inference/sampling.py:64-118``), the decode loop of
diffusion autoencoders.  ``sample_k`` keeps the reference signature and behaviour (``inference/sampling.py:144-228``):
polyexponential sigma schedule, initial noise scaled by sigma_0, variation / inpainting
initialisation and the inpainting callback, sampler dispatch by name.  The k-diffusion 0.1.1
pieces it relies on (``VDenoiser``, ``get_sigmas_polyexponential``, DPM-Solver++(2M/3M) SDE, and
the ``k-*`` samplers: Heun, linear multistep, DPM-2, DPM-Solver++(2S) ancestral, DPM-Solver
fast / adaptive) are an un-vendored third-party dependency of the reference (``setup.py:21``) that
is absent offline, so they are restated here from the published algorithms (Karras et al. 2022,
Alg. 1/2; Lu et al. 2022, DPM-Solver and DPM-Solver++) - parity for those is unpinned by the
reference (see DESIGN.md); ``tests/test_host_logic.py`` checks every one of them against the
closed-form probability-flow solution of a Gaussian toy problem.
k-diffusion's Brownian-tree noise (torchsde) is replaced by one ``randn_like`` draw per
step, which has the same distribution over the disjoint sigma intervals; pass
``noise_sampler=`` to inject an explicit sequence.
"""
import contextlib
import ctypes
import math

import torch


def exists(x):
    return x is not None


def append_dims(x, target_dims):
    extra = target_dims - x.ndim
    if extra < 0:
        raise ValueError("input has more dims than the target")
    return x[(...,) + (None,) * extra]


def get_sigmas_polyexponential(n, sigma_min, sigma_max, rho=1.0, device="cpu"):
    ramp = torch.linspace(1, 0, n, device=device) ** rho
    lo, hi = math.log(sigma_min), math.log(sigma_max)
    sigmas = torch.exp(ramp * (hi - lo) + lo)
    return torch.cat([sigmas, sigmas.new_zeros([1])])


class VDenoiser(torch.nn.Module):
    """D(x, sigma) = F(x c_in, atan(sigma) 2/pi) c_out + x c_skip with sigma_data = 1."""

    def __init__(self, inner_model):
        super().__init__()
        self.inner_model = inner_model
        self.sigma_data = 1.0

    def get_scalings(self, sigma):
        denom = sigma ** 2 + self.sigma_data ** 2
        return self.sigma_data ** 2 / denom, -sigma * self.sigma_data / denom ** 0.5, 1 / denom ** 0.5

    def sigma_to_t(self, sigma):
        return sigma.atan() / math.pi * 2

    def forward(self, input, sigma, **kwargs):
        c_skip, c_out, c_in = (append_dims(c, input.ndim) for c in self.get_scalings(sigma))
        return self.inner_model(input * c_in, self.sigma_to_t(sigma), **kwargs) * c_out + input * c_skip


def _noise_fn(x, noise_sampler):
    if noise_sampler is not None:
        return noise_sampler
    return lambda sigma, sigma_next: torch.randn_like(x)


# ---- the native step path: one satb_sampler_step launch per model call (include/satb200.h gives the algebra)
def _fusable(x):
    """The native step path's condition on the sampler state: CUDA fp32 in whole 16-byte vectors."""
    return x.is_cuda and x.dtype == torch.float32 and x.numel() % 4 == 0


def _graph_dit(model):
    """The native DiT behind a model callable (a DiffusionTransformer, or a DiTWrapper holding one as ``.model``),
    which can run each call as one CUDA-graph replay; None for any other callable."""
    dit = None
    for cand in (model, getattr(model, "model", None)):
        if cand is not None and hasattr(cand, "cuda_graph") and hasattr(cand, "_graph_forward"):
            dit = cand
    return dit


@contextlib.contextmanager
def _graph_replay(dit):
    """Switch the DiT's ``cuda_graph`` on for a sampling loop and restore it after.  A graph call returns a static buffer
    that the next call overwrites, so inside the loop no raw model output may be kept across two calls."""
    if dit is None:
        yield
        return
    prev, dit.cuda_graph = dit.cuda_graph, True
    try:
        yield
    finally:
        dit.cuda_graph = prev


def _launch_step(p):
    """satb_sampler_step on the parameter dict built by ``_step`` (the CPU tests substitute a torch restatement)."""
    from .. import _native
    s = _native.SatbSamplerStep()
    for k in ("x", "y", "noise", "mask", "init", "renoise", "den", "d", "x_next", "x_in_next"):
        setattr(s, k, _native.ptr(p[k]))
    for j, (c, t) in enumerate(zip(p["c"], p["buf"])):
        s.buf[j], s.c[j] = _native.ptr(t), c
    for k in ("n", "L", "c_skip", "c_out", "inv_sigma", "a", "b", "g", "s", "c_in_next", "blend_sigma", "blend_thr"):
        setattr(s, k, p[k])
    _native.check(_native.lib().satb_sampler_step(ctypes.byref(s), _native.stream_ptr(p["x"].device)))


def _step(x, y, c_skip=0.0, c_out=1.0, inv_sigma=0.0, a=0.0, b=0.0, g=0.0, bufs=(), noise=None, s=0.0, blend=None,
          den=False, d=False, x_next=True, c_in_next=None):
    """One launch: den = c_out y + c_skip x, the optional inpainting blend of x (in place), d = (x - den) inv_sigma,
    x_next = a x + b den + g d + sum c buf + s noise and x_in_next = x_next c_in_next.  ``bufs`` holds (c, tensor)
    pairs, ``blend`` is (inpainting callback, step index, re-noise, sigma).  The default c_out = 1, c_skip = 0 takes y
    as den.  Returns fresh (den, d, x_next, x_in_next) tensors, None for those not asked for."""
    if len(bufs) > 4:
        raise ValueError("satb_sampler_step reads at most 4 stored tensors")
    new = lambda want: torch.empty_like(x) if want else None
    p = dict(x=x, y=y, buf=[t for _, t in bufs] + [None] * (4 - len(bufs)),
             c=[float(c) for c, _ in bufs] + [0.0] * (4 - len(bufs)),
             noise=None if noise is None else noise.to(x.dtype).contiguous(), mask=None, init=None, renoise=None,
             den=new(den), d=new(d), x_next=new(x_next), x_in_next=new(c_in_next is not None), n=x.numel(),
             L=x.shape[-1], c_skip=c_skip, c_out=c_out, inv_sigma=inv_sigma, a=a, b=b, g=g, s=s,
             c_in_next=c_in_next or 0.0, blend_sigma=0.0, blend_thr=0.0)
    if blend is not None:
        inpaint, i, renoise, sigma = blend
        p.update(mask=inpaint.mask, init=inpaint.init_data, renoise=renoise, blend_sigma=sigma,
                 blend_thr=(i + 1) / inpaint.steps)
    _launch_step(p)
    return p["den"], p["d"], p["x_next"], p["x_in_next"]


class _NativeSteps:
    """The fixed-step k-samplers over a ``VDenoiser`` on the native step path: the inner model is called on
    x * c_in(sigma) produced by the previous launch, and each call is followed by ONE ``satb_sampler_step`` launch
    that makes the VDenoiser combine, the update and the next model input.  A step's first call keeps the callback
    semantics of the torch samplers: the inpainting callback of ``sample_k`` alone is folded into that launch (its
    re-noise drawn with the same ``torch.randn_like`` call); any other callback gets fresh x / denoised tensors from a
    denoised-only launch first and may change x in place before the update launch reads it.  Every kept tensor (the
    state before a two-stage step, derivatives, denoised estimates) is a fresh launch output, never the model's own
    output buffer, so a graph-replayed DiT may overwrite that at its next call."""

    def __init__(self, model, x, sigmas, extra_args, callback):
        self.model, self.sigmas, self.extra = model, sigmas, extra_args or {}
        self.sig = [float(v) for v in sigmas]          # host copies: no device sync inside the loop
        self.ones = x.new_ones([x.shape[0]])
        self.inpaint = callback if isinstance(callback, InpaintingCallback) and callback.foldable(x) else None
        self.callback = None if self.inpaint is not None else callback
        self.dit = _graph_dit(model.inner_model)

    def scalings(self, sigma):
        """(c_skip, c_out, c_in) of the VDenoiser at sigma, in float64."""
        return tuple(float(c) for c in self.model.get_scalings(torch.tensor(float(sigma), dtype=torch.float64)))

    def c_in_after(self, i, sigma):
        """c_in of the model call that follows step i's last launch (None after the last step)."""
        return self.scalings(sigma)[2] if i + 2 < len(self.sig) else None

    def call(self, x_in, sigma):
        """The inner model on an already scaled input; sigma is a schedule entry or a float, as the torch samplers
        pass it to the VDenoiser (so t is the same fp32 value)."""
        t = self.model.sigma_to_t(sigma * self.ones)
        return self.model.inner_model(x_in, t, **self.extra).to(x_in.dtype).contiguous()

    def after_call(self, x, v, i, noise=None, **upd):
        """The launch(es) after the model call at the start of step i, whose output is v; ``noise`` is a callable drawn
        after the callback's own draws, as the torch samplers draw it."""
        c_skip, c_out, _ = self.scalings(self.sig[i])
        if self.callback is not None:
            den = _step(x, v, c_skip, c_out, den=True, x_next=False)[0]
            self.callback({"x": x, "i": i, "sigma": self.sigmas[i], "sigma_hat": self.sigmas[i], "denoised": den})
            out = _step(x, den, noise=noise() if noise else None, **dict(upd, den=False))
            return (den,) + out[1:]
        blend = None
        if self.inpaint is not None:
            blend = (self.inpaint, i, torch.randn_like(self.inpaint.init_data), self.sig[i])
        return _step(x, v, c_skip, c_out, noise=noise() if noise else None, blend=blend, **upd)

    def first(self, x, i, x_in, noise=None, **upd):
        return self.after_call(x, self.call(x_in, self.sigmas[i]), i, noise, **upd)

    def second(self, x, sigma, x_in, noise=None, **upd):
        """The launch after a step's second model call at sigma (no callback there)."""
        v = self.call(x_in, sigma)
        c_skip, c_out, _ = self.scalings(sigma)
        return _step(x, v, c_skip, c_out, noise=noise() if noise else None, **upd)

    def run(self, sampler, x, *args):
        with _graph_replay(self.dit):
            x = x.contiguous()
            return sampler(x, x * self.scalings(self.sig[0])[2], *args)

    def heun(self, x, x_in):
        sig = self.sig
        for i in range(len(sig) - 1):
            dt = sig[i + 1] - sig[i]
            if sig[i + 1] == 0:
                x = self.first(x, i, x_in, inv_sigma=1.0 / sig[i], a=1.0, g=dt)[2]
            else:
                _, d, x_2, x_in_2 = self.first(x, i, x_in, inv_sigma=1.0 / sig[i], a=1.0, g=dt, d=True,
                                               c_in_next=self.scalings(sig[i + 1])[2])
                _, _, x, x_in = self.second(x_2, self.sigmas[i + 1], x_in_2, inv_sigma=1.0 / sig[i + 1], g=0.5 * dt,
                                            bufs=((1.0, x), (0.5 * dt, d)), c_in_next=self.c_in_after(i, sig[i + 1]))
        return x

    def dpm_2(self, x, x_in):
        sig = self.sig
        for i in range(len(sig) - 1):
            if sig[i + 1] == 0:
                x = self.first(x, i, x_in, inv_sigma=1.0 / sig[i], a=1.0, g=sig[i + 1] - sig[i])[2]
            else:
                sigma_mid = math.exp(0.5 * (math.log(sig[i]) + math.log(sig[i + 1])))
                _, _, x_2, x_in_2 = self.first(x, i, x_in, inv_sigma=1.0 / sig[i], a=1.0, g=sigma_mid - sig[i],
                                               c_in_next=self.scalings(sigma_mid)[2])
                _, _, x, x_in = self.second(x_2, sigma_mid, x_in_2, inv_sigma=1.0 / sigma_mid, g=sig[i + 1] - sig[i],
                                            bufs=((1.0, x),), c_in_next=self.c_in_after(i, sig[i + 1]))
        return x

    def lms(self, x, x_in, order):
        sig, ds = self.sig, []                         # ds: the derivatives of the previous steps, oldest first
        for i in range(len(sig) - 1):
            cur = min(i + 1, order)
            coef = [_lms_coeff(cur, sig, i, j) for j in range(cur)]
            _, d, x, x_in = self.first(x, i, x_in, inv_sigma=1.0 / sig[i], a=1.0, g=coef[0],
                                       bufs=tuple((coef[j], ds[-j]) for j in range(1, cur)), d=i + 2 < len(sig),
                                       c_in_next=self.c_in_after(i, sig[i + 1]))
            ds = (ds + [d])[-(order - 1):] if order > 1 else []
        return x

    def dpmpp_2s_ancestral(self, x, x_in, eta, s_noise, noise):
        sig = self.sig
        for i in range(len(sig) - 1):
            sigma_down, sigma_up = get_ancestral_step(sig[i], sig[i + 1], eta)
            nz, s = None, 0.0
            if sig[i + 1] > 0 and sigma_up > 0:
                nz, s = (lambda i=i: noise(self.sigmas[i], self.sigmas[i + 1])), s_noise * sigma_up
            if sigma_down == 0:
                x, x_in = self.first(x, i, x_in, nz, s=s, inv_sigma=1.0 / sig[i], a=1.0, g=sigma_down - sig[i],
                                     c_in_next=self.c_in_after(i, sig[i + 1]))[2:]
            else:
                t, t_next = -math.log(sig[i]), -math.log(sigma_down)
                h = t_next - t
                s_mid = t + 0.5 * h
                sigma_mid = math.exp(-s_mid)
                _, _, x_2, x_in_2 = self.first(x, i, x_in, a=sigma_mid / math.exp(-t), b=-math.expm1(-0.5 * h),
                                               c_in_next=self.scalings(sigma_mid)[2])
                x, x_in = self.second(x_2, sigma_mid, x_in_2, nz, s=s, b=-math.expm1(-h),
                                      bufs=((math.exp(-t_next) / math.exp(-t), x),),
                                      c_in_next=self.c_in_after(i, sig[i + 1]))[2:]
        return x


def _native_steps(model, x, sigmas, extra_args, callback):
    """A ``_NativeSteps`` when the native step path applies to (model, x), else None (CPU tensors, other dtypes and
    wrappers other than ``VDenoiser`` keep the torch samplers)."""
    if isinstance(model, VDenoiser) and _fusable(x):
        return _NativeSteps(model, x, sigmas, extra_args, callback)
    return None


class MultistepSdeStepper:
    """DPM-Solver++(2M) SDE / DPM-Solver++(3M) SDE as a state machine with one model call per ``step()``.

    Every update of both samplers is linear in the tensors involved,
        x_next = A x + B den + C den_1 + D den_2 + S noise,
    with scalars that depend only on the sigma schedule (``coeffs``).  On CUDA, with the standard ``VDenoiser``
    wrapper, the denoiser scalings, this update and the scaling of the next model input run as ONE kernel instead
    of ~20 elementwise launches: ``satb_sampler_update`` without a callback, ``satb_sampler_step`` with the inpainting
    blend folded in for ``sample_k``'s inpainting callback, and a denoised-only launch, the callback, then the update
    launch for any other callback (``_NativeSteps.after_call``).  Otherwise the same algebra is evaluated with torch
    ops (CPU tensors, other dtypes and wrappers).
    """

    def __init__(self, model, x, sigmas, order=3, extra_args=None, callback=None, eta=1.0, s_noise=1.0,
                 noise_sampler=None, solver_type="midpoint"):
        self.model, self.x, self.sigmas, self.order = model, x, sigmas, order
        self.extra_args, self.callback = extra_args or {}, callback
        self.eta, self.s_noise, self.solver_type = eta, s_noise, solver_type
        self.noise = _noise_fn(x, noise_sampler)
        self.sig = [float(v) for v in sigmas]          # host copies: no device sync inside the loop
        self.ones = x.new_ones([x.shape[0]])
        self.i = 0
        self.den_1 = self.den_2 = None
        self.h_1 = self.h_2 = None
        self.fused = isinstance(model, VDenoiser) and _fusable(x)
        # the native DiT (directly, or as DiTWrapper.model) can run a call as one CUDA-graph launch; its output is then a
        # static buffer, which is safe here because the fused update consumes v before the next model call
        self.graph_dit = _graph_dit(model.inner_model) if self.fused else None
        self.native = None
        if self.fused and callback is not None:
            self.x = x.contiguous()
            self.native = _NativeSteps(model, x, sigmas, self.extra_args, callback)
        self.x_in = None                               # x * c_in(sigma_i), produced by the previous fused update

    def coeffs(self, i):
        """(A, B, C, D, S, h) of step i; C / D are 0 while the history is shorter than the order."""
        sig, eta = self.sig, self.eta
        if sig[i + 1] == 0:
            return 0.0, 1.0, 0.0, 0.0, 0.0, None
        h = math.log(sig[i]) - math.log(sig[i + 1])
        C = D = 0.0
        if self.order == 2:
            eta_h = eta * h
            A = sig[i + 1] / sig[i] * math.exp(-eta_h)
            E = -math.expm1(-h - eta_h)
            B = E
            if self.den_1 is not None:
                r = self.h_1 / h
                K = (E / (-h - eta_h) + 1) / r if self.solver_type == "heun" else 0.5 * E / r
                B, C = B + K, -K
            S = sig[i + 1] * math.sqrt(-math.expm1(-2 * eta_h)) * self.s_noise if eta else 0.0
        else:
            h_eta = h * (eta + 1)
            A = math.exp(-h_eta)
            B = -math.expm1(-h_eta)
            phi_2 = math.expm1(-h_eta) / h_eta + 1
            if self.h_2 is not None:
                r0, r1 = self.h_1 / h, self.h_2 / h
                w, q = r0 / (r0 + r1), 1.0 / (r0 + r1)
                phi_3 = phi_2 / h_eta - 0.5
                P, Q = phi_2 * (1 + w) - phi_3 * q, -phi_2 * w + phi_3 * q
                B, C, D = B + P / r0, -P / r0 + Q / r1, -Q / r1
            elif self.h_1 is not None:
                r = self.h_1 / h
                B, C = B + phi_2 / r, -phi_2 / r
            S = sig[i + 1] * math.sqrt(-math.expm1(-2 * h * eta)) * self.s_noise if eta else 0.0
        return A, B, C, D, S, h

    def step(self, i=None):
        """One model evaluation + update at schedule index i (default: the next one); returns the new x."""
        i = self.i if i is None else i
        x, sig = self.x, self.sig
        A, B, C, D, S, h = self.coeffs(i)
        nz = self.noise(self.sigmas[i], self.sigmas[i + 1]) if S != 0.0 else None
        if self.fused:
            from .. import _native
            c_skip, c_out, c_in = (float(c) for c in self.model.get_scalings(torch.tensor(sig[i], dtype=torch.float64)))
            if self.x_in is None:
                self.x_in = x * c_in
            t = self.model.sigma_to_t(self.sigmas[i]) * self.ones
            v = self.model.inner_model(self.x_in, t, **self.extra_args)
            v = v.to(x.dtype).contiguous()
            c_in_next = 1.0 / math.sqrt(sig[i + 1] ** 2 + self.model.sigma_data ** 2)
            if self.native is not None:
                bufs = tuple((c, t) for c, t in ((C, self.den_1), (D, self.den_2)) if c != 0.0)
                den, _, x_next, x_in_next = self.native.after_call(x, v, i, a=A, b=B, bufs=bufs, s=S,
                                                                   noise=(lambda: nz) if nz is not None else None,
                                                                   den=True, c_in_next=c_in_next)
            else:
                den, x_next, x_in_next = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
                xc = x.contiguous()
                _native.check(_native.lib().satb_sampler_update(
                    _native.ptr(xc), _native.ptr(v), _native.ptr(self.den_1 if C != 0.0 else None),
                    _native.ptr(self.den_2 if D != 0.0 else None),
                    _native.ptr(nz.contiguous() if nz is not None else None), _native.ptr(den), _native.ptr(x_next),
                    _native.ptr(x_in_next), x.numel(), c_skip, c_out, A, B, C, D, S, c_in_next,
                    _native.stream_ptr(x.device)))
            self.x_in = x_in_next
        else:
            den = self.model(x, self.sigmas[i] * self.ones, **self.extra_args)
            if self.callback is not None:
                self.callback({"x": x, "i": i, "sigma": self.sigmas[i], "sigma_hat": self.sigmas[i], "denoised": den})
            x_next = den if (A == 0.0 and B == 1.0) else A * x + B * den
            if C != 0.0:
                x_next = x_next + C * self.den_1
            if D != 0.0:
                x_next = x_next + D * self.den_2
            if nz is not None:
                x_next = x_next + S * nz
        self.den_1, self.den_2 = den, self.den_1
        self.h_1, self.h_2 = h, self.h_1
        self.x = x_next
        self.i = i + 1
        return x_next

    def run(self):
        with _graph_replay(self.graph_dit):
            for _ in range(len(self.sig) - 1):
                self.step()
        return self.x


@torch.no_grad()
def sample_dpmpp_2m_sde(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                        noise_sampler=None, solver_type="midpoint"):
    """DPM-Solver++(2M) SDE (Lu et al. 2022; k-diffusion's sample_dpmpp_2m_sde, eta = 1, 'midpoint')."""
    return MultistepSdeStepper(model, x, sigmas, 2, extra_args, callback, eta, s_noise, noise_sampler, solver_type).run()


@torch.no_grad()
def sample_dpmpp_3m_sde(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                        noise_sampler=None):
    """DPM-Solver++(3M) SDE (k-diffusion's sample_dpmpp_3m_sde, eta = 1)."""
    return MultistepSdeStepper(model, x, sigmas, 3, extra_args, callback, eta, s_noise, noise_sampler).run()


def _to_d(x, sigma, denoised):
    """Karras ODE derivative dx/dsigma = (x - D(x, sigma)) / sigma."""
    return (x - denoised) / sigma


@torch.no_grad()
def sample_heun(model, x, sigmas, extra_args=None, callback=None, disable=None, **_):
    """Karras et al. 2022, Algorithm 1 without churn: Euler step + trapezoidal correction."""
    native = _native_steps(model, x, sigmas, extra_args, callback)
    if native is not None:
        return native.run(native.heun, x)
    extra_args = extra_args or {}
    ones = x.new_ones([x.shape[0]])
    sig = [float(v) for v in sigmas]
    for i in range(len(sig) - 1):
        den = model(x, sigmas[i] * ones, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": den})
        d = _to_d(x, sig[i], den)
        dt = sig[i + 1] - sig[i]
        if sig[i + 1] == 0:
            x = x + d * dt
        else:
            x_2 = x + d * dt
            den_2 = model(x_2, sigmas[i + 1] * ones, **extra_args)
            x = x + (d + _to_d(x_2, sig[i + 1], den_2)) * (0.5 * dt)
    return x


@torch.no_grad()
def sample_dpm_2(model, x, sigmas, extra_args=None, callback=None, disable=None, **_):
    """Second-order sampler with the midpoint taken in log-sigma (Karras et al. 2022, Algorithm 2 without churn)."""
    native = _native_steps(model, x, sigmas, extra_args, callback)
    if native is not None:
        return native.run(native.dpm_2, x)
    extra_args = extra_args or {}
    ones = x.new_ones([x.shape[0]])
    sig = [float(v) for v in sigmas]
    for i in range(len(sig) - 1):
        den = model(x, sigmas[i] * ones, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": den})
        d = _to_d(x, sig[i], den)
        if sig[i + 1] == 0:
            x = x + d * (sig[i + 1] - sig[i])
        else:
            sigma_mid = math.exp(0.5 * (math.log(sig[i]) + math.log(sig[i + 1])))
            x_2 = x + d * (sigma_mid - sig[i])
            den_2 = model(x_2, sigma_mid * ones, **extra_args)
            x = x + _to_d(x_2, sigma_mid, den_2) * (sig[i + 1] - sig[i])
    return x


def _lms_coeff(order, t, i, j):
    """Integral over [t_i, t_{i+1}] of the j-th Lagrange basis polynomial through t_i, t_{i-1}, ..., t_{i-order+1}
    (exact polynomial integration)."""
    import numpy as np
    poly = np.poly1d([1.0])
    for k in range(order):
        if k != j:
            poly = poly * np.poly1d([1.0, -t[i - k]]) / (t[i - j] - t[i - k])
    integ = poly.integ()
    return float(integ(t[i + 1]) - integ(t[i]))


@torch.no_grad()
def sample_lms(model, x, sigmas, extra_args=None, callback=None, disable=None, order=4, **_):
    """Linear multistep (Adams-Bashforth in sigma) of order <= 4 over the derivative history."""
    native = _native_steps(model, x, sigmas, extra_args, callback)
    if native is not None and 1 <= order <= 4:
        return native.run(native.lms, x, order)
    extra_args = extra_args or {}
    ones = x.new_ones([x.shape[0]])
    sig = [float(v) for v in sigmas]
    ds = []
    for i in range(len(sig) - 1):
        den = model(x, sigmas[i] * ones, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": den})
        ds.append(_to_d(x, sig[i], den))
        if len(ds) > order:
            ds.pop(0)
        cur = min(i + 1, order)
        for j, d in zip(range(cur), reversed(ds)):
            x = x + d * _lms_coeff(cur, sig, i, j)
    return x


def get_ancestral_step(sigma_from, sigma_to, eta=1.0):
    """Split a step into a deterministic part down to sigma_down and fresh noise of scale sigma_up."""
    if not eta:
        return sigma_to, 0.0
    sigma_up = min(sigma_to, eta * math.sqrt(sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2))
    return math.sqrt(sigma_to ** 2 - sigma_up ** 2), sigma_up


@torch.no_grad()
def sample_dpmpp_2s_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                              noise_sampler=None):
    """DPM-Solver++(2S) with ancestral noise (Lu et al. 2022, data-prediction, single-step second order)."""
    noise = _noise_fn(x, noise_sampler)
    native = _native_steps(model, x, sigmas, extra_args, callback)
    if native is not None:
        return native.run(native.dpmpp_2s_ancestral, x, eta, s_noise, noise)
    extra_args = extra_args or {}
    ones = x.new_ones([x.shape[0]])
    sig = [float(v) for v in sigmas]
    for i in range(len(sig) - 1):
        den = model(x, sigmas[i] * ones, **extra_args)
        sigma_down, sigma_up = get_ancestral_step(sig[i], sig[i + 1], eta)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": den})
        if sigma_down == 0:
            x = x + _to_d(x, sig[i], den) * (sigma_down - sig[i])
        else:
            t, t_next = -math.log(sig[i]), -math.log(sigma_down)
            h = t_next - t
            s_mid = t + 0.5 * h
            x_2 = (math.exp(-s_mid) / math.exp(-t)) * x - math.expm1(-0.5 * h) * den
            den_2 = model(x_2, math.exp(-s_mid) * ones, **extra_args)
            x = (math.exp(-t_next) / math.exp(-t)) * x - math.expm1(-h) * den_2
        if sig[i + 1] > 0 and sigma_up > 0:
            x = x + noise(sigmas[i], sigmas[i + 1]) * (s_noise * sigma_up)
    return x


class _DPMSolver:
    """DPM-Solver (Lu et al. 2022) in t = -log(sigma) with noise prediction eps = (x - D(x, sigma)) / sigma:
    singlestep orders 1-3, the fixed-budget schedule ("fast") and the adaptive order-2/3 pair with a
    PID step-size controller ("adaptive")."""

    def __init__(self, model, extra_args=None, callback=None):
        self.model, self.extra_args, self.callback = model, extra_args or {}, callback
        self.nfe = 0

    @staticmethod
    def sigma(t):
        return math.exp(-t)

    def eps(self, cache, key, x, t):
        if key in cache:
            return cache[key], cache
        sig = self.sigma(t)
        eps = (x - self.model(x, x.new_ones([x.shape[0]]) * sig, **self.extra_args)) / sig
        self.nfe += 1
        return eps, {key: eps, **cache}

    def step1(self, x, t, t_next, cache=None):
        cache = cache or {}
        h = t_next - t
        eps, cache = self.eps(cache, "eps", x, t)
        return x - self.sigma(t_next) * math.expm1(h) * eps, cache

    def step2(self, x, t, t_next, r1=0.5, cache=None):
        cache = cache or {}
        h = t_next - t
        eps, cache = self.eps(cache, "eps", x, t)
        s1 = t + r1 * h
        u1 = x - self.sigma(s1) * math.expm1(r1 * h) * eps
        eps_r1, cache = self.eps(cache, "eps_r1", u1, s1)
        x_2 = x - self.sigma(t_next) * math.expm1(h) * eps - self.sigma(t_next) / (2 * r1) * math.expm1(h) * (eps_r1 - eps)
        return x_2, cache

    def step3(self, x, t, t_next, r1=1 / 3, r2=2 / 3, cache=None):
        cache = cache or {}
        h = t_next - t
        eps, cache = self.eps(cache, "eps", x, t)
        s1, s2 = t + r1 * h, t + r2 * h
        u1 = x - self.sigma(s1) * math.expm1(r1 * h) * eps
        eps_r1, cache = self.eps(cache, "eps_r1", u1, s1)
        u2 = (x - self.sigma(s2) * math.expm1(r2 * h) * eps
              - self.sigma(s2) * (r2 / r1) * (math.expm1(r2 * h) / (r2 * h) - 1) * (eps_r1 - eps))
        eps_r2, cache = self.eps(cache, "eps_r2", u2, s2)
        x_3 = (x - self.sigma(t_next) * math.expm1(h) * eps
               - self.sigma(t_next) / r2 * (math.expm1(h) / h - 1) * (eps_r2 - eps))
        return x_3, cache

    def _report(self, x, i, t, cache):
        if self.callback is not None and "eps" in cache:
            sig = self.sigma(t)
            self.callback({"x": x, "i": i, "t": t, "sigma": x.new_tensor(sig), "sigma_hat": x.new_tensor(sig),
                           "denoised": x - sig * cache["eps"]})

    def fast(self, x, t_start, t_end, nfe):
        if nfe < 1:
            raise ValueError("nfe must be at least 1")
        m = nfe // 3 + 1
        ts = [t_start + (t_end - t_start) * k / m for k in range(m + 1)]
        orders = [3] * (m - 2) + [2, 1] if nfe % 3 == 0 else [3] * (m - 1) + [nfe % 3]
        for i, order in enumerate(orders):
            t, t_next = ts[i], ts[i + 1]
            eps, cache = self.eps({}, "eps", x, t)
            self._report(x, i, t, cache)
            if order == 1:
                x, _ = self.step1(x, t, t_next, cache=cache)
            elif order == 2:
                x, _ = self.step2(x, t, t_next, cache=cache)
            else:
                x, _ = self.step3(x, t, t_next, cache=cache)
        return x

    def adaptive(self, x, t_start, t_end, order=3, rtol=0.05, atol=0.0078, h_init=0.05, pcoeff=0.0, icoeff=1.0,
                 dcoeff=0.0, accept_safety=0.81):
        if order not in (2, 3):
            raise ValueError("order should be 2 or 3")
        forward = t_end > t_start
        h = abs(h_init) * (1 if forward else -1)
        b1, b2, b3 = (pcoeff + icoeff + dcoeff) / order, -(pcoeff + 2 * dcoeff) / order, dcoeff / order
        errs = None
        s, x_prev, n_steps = t_start, x, 0
        while (s < t_end - 1e-5) if forward else (s > t_end + 1e-5):
            t = min(t_end, s + h) if forward else max(t_end, s + h)
            eps, cache = self.eps({}, "eps", x, s)
            denoised = x - self.sigma(s) * eps          # reported below: the estimate at the OLD (x, s)
            if order == 2:
                x_low, cache = self.step1(x, s, t, cache=cache)
                x_high, cache = self.step2(x, s, t, cache=cache)
            else:
                x_low, cache = self.step2(x, s, t, r1=1 / 3, cache=cache)
                x_high, cache = self.step3(x, s, t, cache=cache)
            delta = torch.maximum(torch.full_like(x_low, atol), rtol * torch.maximum(x_low.abs(), x_prev.abs()))
            error = float(torch.linalg.norm((x_low - x_high) / delta) / x.numel() ** 0.5)
            inv = 1.0 / (error + 1e-8)
            if errs is None:
                errs = [inv, inv, inv]
            errs[0] = inv
            factor = errs[0] ** b1 * errs[1] ** b2 * errs[2] ** b3
            factor = 1 + math.atan(factor - 1)
            accept = factor >= accept_safety
            if accept:
                errs[2], errs[1] = errs[1], errs[0]
                x_prev, x, s = x_low, x_high, t
            h *= factor
            n_steps += 1
            # k-diffusion's contract (the inpainting callback relies on it): the callback fires on EVERY iteration,
            # accepted or rejected, with i = the iteration count, x = the state after this iteration and sigma at
            # the proposed t
            if self.callback is not None:
                sig = x.new_tensor(self.sigma(t))
                self.callback({"x": x, "i": n_steps - 1, "t": t, "sigma": sig, "sigma_hat": sig, "denoised": denoised})
        return x


@torch.no_grad()
def sample_dpm_fast(model, x, sigma_min, sigma_max, n, extra_args=None, callback=None, disable=None, **_):
    """DPM-Solver with a fixed budget of n model evaluations between sigma_max and sigma_min."""
    if sigma_min <= 0 or sigma_max <= 0:
        raise ValueError("sigma_min and sigma_max must not be 0")
    with _graph_replay(_dpm_solver_dit(model, x)):
        return _DPMSolver(model, extra_args, callback).fast(x, -math.log(sigma_max), -math.log(sigma_min), n)


def _dpm_solver_dit(model, x):
    """The DPM-Solver samplers keep their torch arithmetic (the adaptive one needs the error norm on the host every
    step) and only replay the DiT from its graph, under the native step path's condition.  Safe: every eps they keep
    is computed from the VDenoiser's output, a fresh tensor, never the graph's output buffer itself."""
    return _graph_dit(model.inner_model) if isinstance(model, VDenoiser) and _fusable(x) else None


@torch.no_grad()
def sample_dpm_adaptive(model, x, sigma_min, sigma_max, extra_args=None, callback=None, disable=None, order=3,
                        rtol=0.05, atol=0.0078, h_init=0.05, pcoeff=0.0, icoeff=1.0, dcoeff=0.0, accept_safety=0.81, **_):
    """DPM-Solver-12/23 with adaptive step size (PID controller on the embedded error estimate)."""
    if sigma_min <= 0 or sigma_max <= 0:
        raise ValueError("sigma_min and sigma_max must not be 0")
    with _graph_replay(_dpm_solver_dit(model, x)):
        return _DPMSolver(model, extra_args, callback).adaptive(x, -math.log(sigma_max), -math.log(sigma_min), order,
                                                                rtol, atol, h_init, pcoeff, icoeff, dcoeff, accept_safety)


# sampler_type -> (function, takes a sigma schedule?)  (reference inference/sampling.py:211-228)
SAMPLERS = {
    "k-heun": sample_heun, "k-lms": sample_lms, "k-dpmpp-2s-ancestral": sample_dpmpp_2s_ancestral, "k-dpm-2": sample_dpm_2,
    "k-dpm-fast": sample_dpm_fast, "k-dpm-adaptive": sample_dpm_adaptive,
    "dpmpp-2m-sde": sample_dpmpp_2m_sde, "dpmpp-3m-sde": sample_dpmpp_3m_sde,
}


def get_bmask(i, steps, mask):
    """Shrinking hard mask for soft-mask inpainting (reference generation.py:277-281)."""
    return torch.where(mask <= (i + 1) / steps, 1, 0)


class InpaintingCallback:
    """The k-diffusion callback of soft-mask inpainting (reference inference/sampling.py:187-198): after each step's first
    model call it re-noises init_data to that step's sigma and pastes it into x, in place, where the shrinking hard
    mask keeps the input.  A class rather than a closure so that the native step path recognises it and folds the
    blend into its update launch (``foldable``)."""

    def __init__(self, init_data, mask, steps):
        self.init_data, self.mask, self.steps = init_data, mask, steps

    def __call__(self, args):
        i, xx, sigma = args["i"], args["x"], args["sigma"]
        noised = self.init_data + torch.randn_like(self.init_data) * sigma
        bm = get_bmask(i, self.steps, self.mask)
        xx[:, :, :] = (noised * bm + xx * (1 - bm))[:, :, :]

    def foldable(self, x):
        """Whether satb_sampler_step can apply the blend to the state x: a [L] fp32 mask over its last dim and an
        init_data of its own shape and dtype, contiguous and on its device."""
        m, d = self.mask, self.init_data
        return (m.dim() == 1 and m.shape[0] == x.shape[-1] and m.dtype == torch.float32 and m.device == x.device
                and m.is_contiguous() and d.shape == x.shape and d.dtype == x.dtype and d.device == x.device
                and d.is_contiguous())


def sample_k(model_fn, noise, init_data=None, mask=None, steps=100, sampler_type="dpmpp-2m-sde", sigma_min=0.5,
             sigma_max=50, rho=1.0, device="cuda", callback=None, cond_fn=None, disable_tqdm: bool = False,
             noise_sampler=None, **extra_args):
    if cond_fn is not None:
        raise NotImplementedError("guidance through cond_fn needs autograd through the denoiser (inference-only here)")
    if sampler_type not in SAMPLERS:
        raise NotImplementedError(f"sampler '{sampler_type}' is not restated; available: {sorted(SAMPLERS)}")
    denoiser = VDenoiser(model_fn)
    sigmas = get_sigmas_polyexponential(steps, sigma_min, sigma_max, rho, device=device)
    noise = noise * sigmas[0]
    wrapped_callback = callback
    if mask is None and exists(init_data):
        x = init_data + noise                                   # variation
    elif exists(mask) and exists(init_data):
        bmask = get_bmask(0, steps, mask)                       # inpainting
        x = (init_data + noise) * bmask + noise * (1 - bmask)
        inpainting_callback = InpaintingCallback(init_data, mask, steps)
        if callback is None:
            wrapped_callback = inpainting_callback
        else:
            def wrapped_callback(args):
                return inpainting_callback(args), callback(args)
    else:
        x = noise
    if sampler_type == "k-dpm-fast":
        return sample_dpm_fast(denoiser, x, sigma_min, sigma_max, steps, disable=disable_tqdm, callback=wrapped_callback,
                               extra_args=extra_args)
    if sampler_type == "k-dpm-adaptive":
        return sample_dpm_adaptive(denoiser, x, sigma_min, sigma_max, rtol=0.01, atol=0.01, disable=disable_tqdm,
                                   callback=wrapped_callback, extra_args=extra_args)
    return SAMPLERS[sampler_type](denoiser, x, sigmas, disable=disable_tqdm, callback=wrapped_callback,
                                  extra_args=extra_args, noise_sampler=noise_sampler)


def get_alphas_sigmas(t):
    """The scales of the clean signal (alpha) and of the noise (sigma) at timestep t (reference sampling.py:10-13)."""
    return torch.cos(t * math.pi / 2), torch.sin(t * math.pi / 2)


def vdiffusion_schedule(steps, eta):
    """Per-step scalars of ``sample`` as Python floats: (t, alpha, sigma, alpha_next, adjusted_sigma, ddim_sigma) for
    every step, the last step's three next-step values None.  Computed once per call with the reference's fp32 CPU
    tensor expressions (sampling.py:69-70,94-96), so the floats are the very values its fp32 loop multiplies by."""
    t = torch.linspace(1, 0, steps + 1)[:-1]
    alphas, sigmas = get_alphas_sigmas(t)
    out = []
    for i in range(steps):
        nxt = (None, None, None)
        if i < steps - 1:
            ddim_sigma = eta * (sigmas[i + 1] ** 2 / sigmas[i] ** 2).sqrt() * (1 - alphas[i] ** 2 / alphas[i + 1] ** 2).sqrt()
            adjusted_sigma = (sigmas[i + 1] ** 2 - ddim_sigma ** 2).sqrt()
            nxt = (float(alphas[i + 1]), float(adjusted_sigma), float(ddim_sigma))
        out.append((float(t[i]), float(alphas[i]), float(sigmas[i])) + nxt)
    return out


@torch.no_grad()
def sample(model, x, steps, eta, verbose: bool = True, noise_sampler=None, **extra_args):
    """v-diffusion DDIM sampling from the start noise x (reference sampling.py:64-118): with alpha, sigma = cos, sin of
    t pi / 2 over t = linspace(1, 0, steps + 1)[:-1] and v = model(x, t_i, **extra_args),
        pred = x alpha_i - v sigma_i,  eps = x sigma_i + v alpha_i,
        x = pred alpha_{i+1} + eps adjusted_sigma + ddim_sigma noise   (every step but the last),
    and returns the last step's pred.  ``noise_sampler(i)`` returns step i's noise (default ``torch.randn_like(x)``;
    drawn only when eta != 0).  ``verbose`` is accepted for the reference's signature; no progress is printed (the
    reference times every tenth step with a device synchronise).

    CUDA fp32 state: each step's update is one launch of ``satb_vdiffusion_update``, which equals the fp32 torch
    expressions below bit for bit, and a native DiT (a DiTWrapper or a DiffusionTransformer) runs each forward as one
    CUDA-graph replay.  Other inputs (CPU tensors, other dtypes) take the torch expressions themselves."""
    if steps < 1:
        raise ValueError(f"sample needs steps >= 1, got {steps}")
    sched = vdiffusion_schedule(steps, eta)
    noise = noise_sampler if noise_sampler is not None else (lambda i: torch.randn_like(x))
    ones = x.new_ones([x.shape[0]])
    fused = x.is_cuda and x.dtype == torch.float32
    with _graph_replay(_graph_dit(model) if fused else None):
        pred = None
        for i, (t_i, a, s, a_next, adj, ddim) in enumerate(sched):
            v = model(x, ones * t_i, **extra_args).float()
            last = a_next is None
            nz = noise(i) if (not last and eta) else None
            if fused:
                from .. import _native
                xc, vc = x.contiguous(), v.contiguous()
                pred = torch.empty_like(xc) if last else None
                x_next = None if last else torch.empty_like(xc)
                _native.check(_native.lib().satb_vdiffusion_update(
                    _native.ptr(xc), _native.ptr(vc), _native.ptr(nz.float().contiguous() if nz is not None else None),
                    _native.ptr(x_next), _native.ptr(pred), xc.numel(), a, s, a_next or 0.0, adj or 0.0, ddim or 0.0,
                    _native.stream_ptr(x.device)))
                if not last:
                    x = x_next
            else:
                pred = x * a - v * s
                if not last:
                    eps = x * s + v * a
                    x = pred * a_next + eps * adj
                    if nz is not None:
                        x += nz * ddim
    return pred


@torch.no_grad()
def sample_discrete_euler(model, x, steps, sigma_max=1, callback=None, **extra_args):
    """Rectified-flow sampling (reference inference/sampling.py:29-60): the network predicts the velocity and
    the state is integrated from t = sigma_max down to 0 on a uniform grid, x += (t_next - t) * v(x, t).

    CUDA fp32 state (``_fusable``): the update is one ``satb_sampler_step`` launch per call, and a native DiT (a
    DiTWrapper or a DiffusionTransformer) runs each call as one CUDA-graph replay; a callback gets x and a fresh
    denoised = x - t v from a launch of its own, before the update launch reads x."""
    ts = torch.linspace(sigma_max, 0, steps + 1)
    ones = x.new_ones([x.shape[0]])
    if _fusable(x):
        with _graph_replay(_graph_dit(model)):
            x = x.contiguous()
            for i in range(steps):
                t_curr, t_next = float(ts[i]), float(ts[i + 1])
                v = model(x, t_curr * ones, **extra_args).to(x.dtype).contiguous()
                if callback is not None:
                    den = _step(x, v, c_skip=1.0, c_out=-t_curr, den=True, x_next=False)[0]
                    callback({"x": x, "i": i, "t": t_curr, "denoised": den})
                x = _step(x, v, a=1.0, b=t_next - t_curr)[2]
        return x
    for i in range(steps):
        t_curr, t_next = float(ts[i]), float(ts[i + 1])
        v = model(x, t_curr * ones, **extra_args)
        if callback is not None:
            callback({"x": x, "i": i, "t": t_curr, "denoised": x - t_curr * v})
        x = x + (t_next - t_curr) * v
    return x


def sample_rf(model_fn, noise, init_data=None, steps=100, sigma_max=1, device="cuda", callback=None, cond_fn=None,
              disable_tqdm: bool = False, **extra_args):
    """Reference inference/sampling.py:236-270: plain noise, or a variation that starts from the
    (1 - sigma_max, sigma_max) interpolation of init_data and noise."""
    if cond_fn is not None:
        raise NotImplementedError("guidance through cond_fn needs autograd through the model (inference-only here)")
    sigma_max = min(sigma_max, 1)
    x = noise if init_data is None else init_data * (1 - sigma_max) + noise * sigma_max
    return sample_discrete_euler(model_fn, x, steps, sigma_max, callback=callback, **extra_args)
