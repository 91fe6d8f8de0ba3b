"""Pretransform adapters (interface parity with reference ``models/pretransforms.py:6-133``): the autoencoder
pretransform and the PQMF filterbank (``models/pqmf.py``), whose analysis and synthesis run in ``libsatb200.so``
(``satb_pqmf_*``)."""
import ctypes
import math

import numpy as np
import torch
from torch import nn

from .. import _native


class Pretransform(nn.Module):
    def __init__(self, enable_grad: bool, io_channels: int, is_discrete: bool):
        super().__init__()
        self.is_discrete = is_discrete
        self.io_channels = io_channels
        self.encoded_channels = None
        self.downsampling_ratio = None
        self.enable_grad = enable_grad

    def encode(self, x):
        raise NotImplementedError

    def decode(self, z):
        raise NotImplementedError


class AutoencoderPretransform(Pretransform):
    """``encode = encode_audio(x) / scale``, ``decode = decode_audio(z * scale)``.

    ``model_half`` is accepted for config compatibility; the native convolutions always use
    16-bit operands with fp32 accumulation and return fp32, so it changes nothing."""

    def __init__(self, model, scale=1.0, model_half=False, iterate_batch=False, chunked=False):
        is_discrete = model.bottleneck is not None and model.bottleneck.is_discrete
        super().__init__(enable_grad=False, io_channels=model.io_channels, is_discrete=is_discrete)
        self.model = model
        self.model.requires_grad_(False).eval()
        self.scale = scale
        self.downsampling_ratio = model.downsampling_ratio
        self.io_channels = model.io_channels
        self.sample_rate = model.sample_rate
        self.model_half = model_half
        self.iterate_batch = iterate_batch
        self.encoded_channels = model.latent_dim
        self.chunked = chunked
        self.num_quantizers = None
        self.codebook_size = None

    def encode(self, x, **kwargs):
        z = self.model.encode_audio(x.float(), chunked=self.chunked, iterate_batch=self.iterate_batch, **kwargs)
        return z.float() / self.scale

    def decode(self, z, **kwargs):
        z = z.float() * self.scale
        return self.model.decode_audio(z, chunked=self.chunked, iterate_batch=self.iterate_batch, **kwargs).float()

    def load_state_dict(self, state_dict, strict=True):
        self.model.load_state_dict(state_dict, strict=strict)

    def shard_time(self, devices):
        """The autoencoder's ``shard_time``: time-shard its unchunked encode / decode over ``devices`` (None: one
        device)."""
        self.model.shard_time(devices)
        return self


# ---------------------------------------------------------------------------------------------------- PQMF
def check_pqmf_bands(num_bands):
    """The band counts the native filterbank runs: a power of 2 (as the reference asserts), at least 2."""
    if not (isinstance(num_bands, int) and 2 <= num_bands <= 256 and num_bands & (num_bands - 1) == 0):
        raise ValueError(f"PQMF: num_bands must be a power of 2 between 2 and 256, got {num_bands!r}")


def _kaiser_lowpass(cutoff, attenuation):
    """Odd-length Kaiser-window lowpass at angular cutoff `cutoff` (rad / sample) whose length and shape kaiserord
    picks for `attenuation` dB, unscaled."""
    from scipy.signal import firwin, kaiserord
    numtaps, beta = kaiserord(attenuation, cutoff / math.pi)
    numtaps = 2 * (numtaps // 2) + 1
    return firwin(numtaps, cutoff, window=("kaiser", beta), scale=False, fs=2 * math.pi)


def _reconstruction_error(cutoff, attenuation, num_bands):
    """Largest off-centre tap, at multiples of 2 * num_bands, of the prototype's autocorrelation: zero for a perfect
    power-complementary prototype (Lin & Vaidyanathan's near-PR criterion, IEEE SPL 1998)."""
    h = _kaiser_lowpass(float(np.asarray(cutoff).reshape(-1)[0]), attenuation)
    r = np.convolve(h, h[::-1])
    return np.max(np.abs(r[r.shape[-1] // 2::2 * num_bands][1:]))


def design_pqmf_prototype(attenuation, num_bands):
    """Prototype lowpass: the cutoff that minimises the reconstruction error, searched by Nelder-Mead from 1 / n."""
    from scipy.optimize import fmin
    cutoff = fmin(lambda wc: _reconstruction_error(wc, attenuation, num_bands), 1 / num_bands, disp=0)[0]
    return torch.tensor(_kaiser_lowpass(cutoff, attenuation), dtype=torch.float32)


def design_pqmf_bank(prototype, num_bands):
    """Cosine-modulated bank [n, 2^ceil(log2 L)]: band k is 2 p[i] cos((2k + 1) pi / (2n) (i - (L-1)/2) + (-1)^k pi/4),
    zero-padded on both sides (the extra zero on the right) to a power-of-two length."""
    L = prototype.shape[-1]
    k = np.arange(num_bands)[:, None]
    t = np.arange(L)[None, :] - (L - 1) // 2
    phase = (2 * k + 1) * np.pi / (2 * num_bands) * t + np.where(k % 2 == 0, 1.0, -1.0) * np.pi / 4
    bank = 2 * prototype.double().numpy()[None, :] * np.cos(phase)
    P = 1 << math.ceil(math.log2(L))
    left = (P - L) // 2
    bank = np.pad(bank, ((0, 0), (left, P - L - left)))
    return torch.from_numpy(bank).to(torch.float32)


class PQMF(nn.Module):
    """reference models/pqmf.py:10-50: buffers "filter_bank" [n, taps] and "prototype" [L], designed on the host at
    construction time.  forward / inverse run on the device: the bank loaded into a native handle (reloaded after
    a state-dict load or a device move)."""

    def __init__(self, attenuation, num_bands):
        super().__init__()
        check_pqmf_bands(num_bands)
        prototype = design_pqmf_prototype(attenuation, num_bands)
        self.register_buffer("filter_bank", design_pqmf_bank(prototype, num_bands))
        self.register_buffer("prototype", prototype)
        self.num_bands = num_bands
        self.__dict__["_h"] = None
        self.__dict__["_dirty"] = True
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.refresh_native_weights())

    def _apply(self, fn, *a, **k):
        self.__dict__["_dirty"] = True
        return super()._apply(fn, *a, **k)

    def refresh_native_weights(self):
        self.__dict__["_dirty"] = True

    def __del__(self):
        h = self.__dict__.get("_h")
        if h is not None:
            try:
                _native.lib().satb_pqmf_destroy(h)
            except Exception:
                pass

    def _handle(self, device):
        lib = _native.lib()
        fb = self.filter_bank
        if not fb.is_cuda:
            raise _native.NativeError(f"pqmf.filter_bank is on {fb.device}: move the model to a CUDA device "
                                      "(this package has no CPU path)")
        if self.__dict__["_h"] is None:
            h = ctypes.c_void_p()
            _native.check(lib.satb_pqmf_create(self.num_bands, fb.shape[-1], ctypes.byref(h)))
            self.__dict__["_h"] = h
        if self.__dict__["_dirty"]:
            # kept alive until the prep kernel has read it: the handle's load is stream-ordered
            self.__dict__["_fb32"] = fb.detach().to(torch.float32).contiguous()
            _native.check(lib.satb_pqmf_load_filter(self.__dict__["_h"], _native.ptr(self.__dict__["_fb32"]),
                                                    _native.stream_ptr(device)))
            self.__dict__["_dirty"] = False
        return self.__dict__["_h"]

    @staticmethod
    def _check_input(x, what):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise _native.NativeError(f"PQMF.{what} needs a CUDA tensor (no CPU fallback)")
        if x.dim() != 3:
            raise ValueError(f"PQMF.{what}: expected [batch, channels, time], got shape {tuple(x.shape)}")

    @torch.no_grad()
    def forward(self, signal):
        """[B, C, T] -> [B, C, n, ceil(T / n)] (reference PQMF.forward)."""
        self._check_input(signal, "forward")
        return self.analysis(signal).unflatten(1, (signal.shape[1], self.num_bands))

    @torch.no_grad()
    def inverse(self, bands):
        """[B, C, n, t] -> [B, C, t * n] (reference PQMF.inverse)."""
        if bands.dim() != 4:
            raise ValueError(f"PQMF.inverse: expected [batch, channels, bands, time], got shape {tuple(bands.shape)}")
        return self.synthesis(bands.flatten(1, 2))

    @torch.no_grad()
    def analysis(self, x):
        """[B, C, T] -> [B, C * n, ceil(T / n)]."""
        self._check_input(x, "analysis")
        with torch.cuda.device(x.device):
            h = self._handle(x.device)
            xin = x.detach().to(torch.float32).contiguous()
            B, C, T = xin.shape
            out = torch.empty(B, C * self.num_bands, -(-T // self.num_bands), device=x.device, dtype=torch.float32)
            _native.check(_native.lib().satb_pqmf_analysis(h, _native.ptr(xin), _native.ptr(out), B, C,
                                                           ctypes.c_longlong(T), _native.stream_ptr(x.device)))
        return out.to(x.dtype)

    @torch.no_grad()
    def synthesis(self, z):
        """[B, C * n, t] -> [B, C, t * n]."""
        self._check_input(z, "synthesis")
        B, CN, t = z.shape
        if CN % self.num_bands:
            raise ValueError(f"PQMF.synthesis: {CN} channels is not a multiple of num_bands={self.num_bands}")
        with torch.cuda.device(z.device):
            h = self._handle(z.device)
            zin = z.detach().to(torch.float32).contiguous()
            out = torch.empty(B, CN // self.num_bands, t * self.num_bands, device=z.device, dtype=torch.float32)
            _native.check(_native.lib().satb_pqmf_synthesis(h, _native.ptr(zin), _native.ptr(out), B,
                                                            CN // self.num_bands, t, _native.stream_ptr(z.device)))
        return out.to(z.dtype)


class PQMFPretransform(Pretransform):
    """reference models/pretransforms.py:114-133: encode = PQMF analysis with channels and bands flattened
    ([B, C, T] -> [B, C * n, T / n]), decode = its synthesis.  ``downsampling_ratio`` stays None, as in the
    reference."""

    def __init__(self, attenuation=100, num_bands=16):
        super().__init__(enable_grad=False, io_channels=1, is_discrete=False)
        self.pqmf = PQMF(attenuation, num_bands)

    def encode(self, x):
        return self.pqmf.analysis(x)

    def decode(self, x):
        return self.pqmf.synthesis(x)
