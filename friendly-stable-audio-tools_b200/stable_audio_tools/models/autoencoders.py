"""Oobleck VAE: the reference's module interface over the native conv kernels.

Interface parity with reference ``models/autoencoders.py`` for the Oobleck path:
``ResidualUnit`` / ``EncoderBlock`` / ``DecoderBlock`` / ``OobleckEncoder`` /
``OobleckDecoder`` (:45-194, same constructor kwargs and state-dict keys incl. the
weight-norm ``weight_g`` / ``weight_v`` pairs), ``AudioAutoencoder`` (:234-645: encode /
decode with ``iterate_batch`` micro-batching, chunked ``encode_audio`` / ``decode_audio`` /
``reconstruct_audio`` with Bartlett cross-fades), ``DiffusionAutoencoder`` (:648-690, a DiT decoder sampled with
``inference.sampling.sample``) and the config factories (:693-847).

The encoder / decoder ``forward`` run in ``libsatb200.so`` (``satb_oobleck_*``): wgmma
implicit-GEMM convolutions with the activation (SnakeBeta for ``use_snake=True``, ELU otherwise)
fused into the producing epilogue.  Decoders upsample by transposed convolution or, with
``use_nearest_upsample=True``, by nearest-neighbour repetition + a 'same' convolution.  The
inner blocks are parameter containers.  ``antialias_activation=True`` is refused: it needs
``alias_free_torch``, which this package does not ship.  The chunking / cross-fade orchestration is host-side tensor
slicing on the device, exactly as in the reference.  A nested ``pqmf`` pretransform (``PQMFPretransform``) runs around
the encoder and decoder where the reference runs it; the encoder then reads, and the decoder writes, io_channels x
num_bands sub-bands.  Other nested pretransform kinds are refused.  ``AudioAutoencoder.shard_time(devices)`` runs the
unchunked encode / decode time-sharded over several ranks (``satb_oobleck_group_*``), bit-identical to one device.
"""
import contextlib
import ctypes
import math
import typing as tp

import torch
from torch import nn
from torch.nn import functional as F
from torch.nn.utils import weight_norm

from .. import _native
from .blocks import SnakeBeta
from .bottleneck import Bottleneck
from .factory import create_bottleneck_from_config, create_pretransform_from_config
from .pretransforms import AutoencoderPretransform, PQMFPretransform
from .transformer import _FusedModule


def WNConv1d(*args, **kwargs):
    """dac.nn.layers.WNConv1d: a weight-normed Conv1d (parameters weight_g, weight_v, bias)."""
    return weight_norm(nn.Conv1d(*args, **kwargs))


def WNConvTranspose1d(*args, **kwargs):
    return weight_norm(nn.ConvTranspose1d(*args, **kwargs))


_ANTIALIAS_REFUSAL = ("antialias_activation=True is not supported: the anti-aliased activation (alias_free_torch's "
                      "Activation1d) needs the alias_free_torch package, which this package does not ship")


def get_activation(activation: str, antialias=False, channels=None) -> nn.Module:
    if antialias:
        raise NotImplementedError(_ANTIALIAS_REFUSAL)
    if activation == "snake":
        return SnakeBeta(channels)
    if activation == "elu":
        return nn.ELU()
    if activation == "none":
        return nn.Identity()
    raise ValueError(f"Unknown activation {activation}")


def _act(use_snake):
    return "snake" if use_snake else "elu"


class _Container(_FusedModule):
    pass


class ResidualUnit(_Container):
    def __init__(self, in_channels, out_channels, dilation, use_snake=False, antialias_activation=False):
        super().__init__()
        self.dilation = dilation
        self.layers = nn.Sequential(
            get_activation(_act(use_snake), antialias=antialias_activation, channels=out_channels),
            WNConv1d(in_channels, out_channels, kernel_size=7, dilation=dilation, padding=(dilation * 6) // 2),
            get_activation(_act(use_snake), antialias=antialias_activation, channels=out_channels),
            WNConv1d(out_channels, out_channels, kernel_size=1))


class EncoderBlock(_Container):
    def __init__(self, in_channels, out_channels, stride, use_snake=False, antialias_activation=False):
        super().__init__()
        self.layers = nn.Sequential(
            ResidualUnit(in_channels, in_channels, 1, use_snake=use_snake),
            ResidualUnit(in_channels, in_channels, 3, use_snake=use_snake),
            ResidualUnit(in_channels, in_channels, 9, use_snake=use_snake),
            get_activation(_act(use_snake), antialias=antialias_activation, channels=in_channels),
            WNConv1d(in_channels, out_channels, kernel_size=2 * stride, stride=stride, padding=math.ceil(stride / 2)))


class DecoderBlock(_Container):
    def __init__(self, in_channels, out_channels, stride, use_snake=False, antialias_activation=False,
                 use_nearest_upsample=False):
        super().__init__()
        if use_nearest_upsample:
            # reference :95-100; the native decoder folds the pair into one 3-tap convolution of the low-rate input
            upsample = nn.Sequential(
                nn.Upsample(scale_factor=stride, mode="nearest"),
                WNConv1d(in_channels, out_channels, kernel_size=2 * stride, stride=1, bias=False, padding="same"))
        else:
            upsample = WNConvTranspose1d(in_channels, out_channels, kernel_size=2 * stride, stride=stride,
                                         padding=math.ceil(stride / 2))
        self.layers = nn.Sequential(
            get_activation(_act(use_snake), antialias=antialias_activation, channels=in_channels),
            upsample,
            ResidualUnit(out_channels, out_channels, 1, use_snake=use_snake),
            ResidualUnit(out_channels, out_channels, 3, use_snake=use_snake),
            ResidualUnit(out_channels, out_channels, 9, use_snake=use_snake))


def _check_strides(strides, decoder, nearest=False):
    """A block's conv has kernel 2s, stride s, padding ceil(s/2) (reference :75,86).  Its output has L * s (decoder) or
    L / s (encoder) positions, which forward allocates, only for an even decoder stride and an encoder stride >= 2:
    an odd decoder stride gives L * s - 1, encoder stride 1 gives L + 1.  A nearest-upsampling decoder block (nearest
    x s, then a 'same' conv) gives L * s for every s >= 2."""
    for s in strides:
        if decoder and nearest and s < 2:
            raise NotImplementedError(f"OobleckDecoder: stride {s} is not supported: nearest upsampling needs strides "
                                      ">= 2")
        if decoder and not nearest and (s < 2 or s % 2):
            raise NotImplementedError(f"OobleckDecoder: stride {s} is not supported: strides must be even (a transposed "
                                      "conv with kernel 2s, padding ceil(s/2) gives L * s positions only for even s)")
        if not decoder and s < 2:
            raise NotImplementedError(f"OobleckEncoder: stride {s} is not supported: strides must be >= 2 (a conv with "
                                      "kernel 2s, padding ceil(s/2) gives L / s positions only for s >= 2)")


def check_oobleck_io_channels(c, what):
    """The encoder input / decoder output widths the native Oobleck runs: 1 or 2 audio channels, or the channels x
    bands of a PQMF pretransform when that is a multiple of 8 up to 128 (its first / last conv then runs on tensor
    cores over 16-byte rows)."""
    if not (c in (1, 2) or (c % 8 == 0 and 8 <= c <= 128)):
        raise NotImplementedError(f"Oobleck: {what} = {c} channels is not supported: the encoder input / decoder "
                                  "output must be 1 or 2 channels, or a multiple of 8 up to 128")


def check_time_shard_devices(devices):
    """shard_time's argument, checked as shard_tokens checks a flat list: None, or 1 to 8 CUDA devices (a device may
    repeat); returns the torch.device list, a device without an index taking the current one."""
    if devices is None:
        return None
    devices = list(devices)
    if any(isinstance(dv, (list, tuple)) for dv in devices):
        raise ValueError("shard_time: give a flat list of devices (there is no row layout for the VAE)")
    if not 1 <= len(devices) <= 8:
        raise ValueError(f"shard_time: 1 to 8 devices, got {len(devices)}")
    devices = [torch.device(dv) for dv in devices]
    for dv in devices:
        if dv.type != "cuda":
            raise _native.NativeError(f"shard_time: {dv} is not a CUDA device (this package has no CPU path)")
    return [dv if dv.index is not None else torch.device("cuda", torch.cuda.current_device()) for dv in devices]


class _NativeOobleck(nn.Module):
    """Shared native-handle plumbing of OobleckEncoder / OobleckDecoder."""

    _is_decoder = False

    def _init_native(self, audio_channels, channels, latent_dim, c_mults, strides, final_tanh, operand_dtype,
                     use_snake=True, use_nearest_upsample=False):
        self.__dict__["_h"] = None
        self.__dict__["_dirty"] = True
        self.__dict__["_shard"] = None           # shard_time state: devices, rank handles, group
        self.__dict__["_shard_dirty"] = True
        self.__dict__["_ncfg"] = dict(audio_channels=audio_channels, channels=channels, latent_dim=latent_dim,
                                      c_mults=list(c_mults), strides=list(strides), final_tanh=bool(final_tanh),
                                      operand_dtype=operand_dtype, use_snake=bool(use_snake),
                                      use_nearest_upsample=bool(use_nearest_upsample))
        # also fires when a parent module's load_state_dict recurses into this one (see models/dit.py)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.refresh_native_weights())

    def _apply(self, fn, *a, **k):
        self.__dict__["_dirty"] = True
        self.__dict__["_shard_dirty"] = True
        return super()._apply(fn, *a, **k)

    def refresh_native_weights(self):
        self.__dict__["_dirty"] = True
        self.__dict__["_shard_dirty"] = True

    def __del__(self):
        try:
            self._drop_shards()
        except Exception:
            pass
        h = self.__dict__.get("_h")
        if h is not None:
            try:
                _native.lib().satb_oobleck_destroy(h)
            except Exception:
                pass

    def native_config(self):
        """The SatbOobleckConfig this module creates its native handles with."""
        nc = self.__dict__["_ncfg"]
        cfg = _native.SatbOobleckConfig()
        cfg.in_channels, cfg.channels, cfg.latent_dim = nc["audio_channels"], nc["channels"], nc["latent_dim"]
        cfg.n_stages = len(nc["c_mults"])
        for i, (m, s) in enumerate(zip(nc["c_mults"], nc["strides"])):
            cfg.c_mults[i], cfg.strides[i] = m, s
        cfg.final_tanh = int(nc["final_tanh"])
        cfg.is_decoder = int(self._is_decoder)
        # "fp16" (default) | "bf16" | "fp16x3": split-operand mode, every conv product as (hi, hi) + (lo, hi) + (hi, lo)
        # with x_lo = fp16(x - x_hi): ~fp32 accuracy (the reference runs these convolutions in strict fp32,
        # inference/generation.py:165-166) at ~3x the tensor-core work
        if nc["operand_dtype"] not in ("fp16", "bf16", "fp16x3"):
            raise ValueError(f"operand_dtype must be fp16, bf16 or fp16x3, got {nc['operand_dtype']}")
        cfg.operand_dtype = {"fp16": 0, "bf16": 1, "fp16x3": 2}[nc["operand_dtype"]]
        return cfg

    def _new_handle(self):
        nc = self.__dict__["_ncfg"]
        cfg = self.native_config()
        h = ctypes.c_void_p()
        act = _native.OOB_ACT_SNAKE if nc["use_snake"] else _native.OOB_ACT_ELU
        _native.check(_native.lib().satb_oobleck_create_variant(ctypes.byref(cfg), act, int(nc["use_nearest_upsample"]),
                                                                ctypes.byref(h)))
        return h

    def _upload_weights(self, h, device, copy_to=None):
        """Loads every parameter into handle h and finalizes it, on device's current stream.  copy_to: the device the
        handle lives on, when it is not the parameters' own (a rank of shard_time)."""
        lib = _native.lib()
        st = _native.stream_ptr(device)
        with torch.no_grad():
            for name, t in self.state_dict().items():
                if not t.is_cuda:
                    raise _native.NativeError(f"parameter {name} is on {t.device}: move the model to a CUDA device "
                                              "(this package has no CPU path)")
                src = t.detach().to(torch.float32).contiguous()
                if copy_to is not None:
                    src = src.to(copy_to)
                _native.check(lib.satb_oobleck_load_weight(h, name.encode(), _native.ptr(src), src.numel(), st))
            _native.check(lib.satb_oobleck_finalize(h, st))

    def _handle(self, device):
        if self.__dict__["_h"] is None:
            self.__dict__["_h"] = self._new_handle()
        if self.__dict__["_dirty"]:
            self._upload_weights(self.__dict__["_h"], device)
            self.__dict__["_dirty"] = False
        return self.__dict__["_h"]

    # ------------------------------------------------------------------ time sharding
    def shard_time(self, devices):
        """Run every later call time-sharded over ``devices`` (see ``AudioAutoencoder.shard_time``); ``None`` returns to
        one device."""
        devices = check_time_shard_devices(devices)
        self._drop_shards()
        if devices is not None:
            self.__dict__["_shard"] = dict(devices=devices, handles=None, group=None)
            self.__dict__["_shard_dirty"] = True
        return self

    def _drop_shards(self):
        sh = self.__dict__.get("_shard")
        self.__dict__["_shard"] = None
        if sh is None:
            return
        lib = _native.lib()
        if sh["group"] is not None:
            lib.satb_oobleck_group_destroy(sh["group"])
        for h in sh["handles"] or []:
            lib.satb_oobleck_destroy(h)

    def _shard_group(self, sh):
        """The group, with every rank handle holding the current weights."""
        devs = sh["devices"]
        if sh["handles"] is None:
            sh["handles"] = [self._new_handle() for _ in devs]
        if self.__dict__["_shard_dirty"]:
            for h, dv in zip(sh["handles"], devs):
                with torch.cuda.device(dv):
                    self._upload_weights(h, dv, copy_to=dv)   # finalize synchronizes: the weights are in place
            self.__dict__["_shard_dirty"] = False
        if sh["group"] is None:
            g = ctypes.c_void_p()
            handles = (ctypes.c_void_p * len(devs))(*[h.value for h in sh["handles"]])
            ids = (ctypes.c_int * len(devs))(*[dv.index for dv in devs])
            _native.check(_native.lib().satb_oobleck_group_create(handles, ids, len(devs), ctypes.byref(g)))
            sh["group"] = g
        return sh["group"]

    def _run(self, x, out_len, single, group):
        """x [B, C, T] -> fp32 [B, out channels, out_len] by the single-device entry point, or by the group one when the
        module is time-sharded (and not paused by a chunked path of AudioAutoencoder)."""
        sh = self.__dict__["_shard"]
        lib = _native.lib()
        xin = x.detach().to(torch.float32).contiguous()
        B, _, T = xin.shape
        n = ctypes.c_longlong(T) if not self._is_decoder else T
        if sh is None or self.__dict__.get("_paused"):
            with torch.cuda.device(x.device):        # the native handle / workspaces live on the model's device
                h = self._handle(x.device)
                out = torch.empty(B, self.out_width, out_len, device=x.device, dtype=torch.float32)
                _native.check(getattr(lib, single)(h, _native.ptr(xin), _native.ptr(out), B, n,
                                                   _native.stream_ptr(x.device)))
            return out
        home = sh["devices"][0]
        if x.device != home:
            raise ValueError(f"the time-sharded model's home device is {home}, but the input is on {x.device}")
        g = self._shard_group(sh)
        with torch.cuda.device(home):
            out = torch.empty(B, self.out_width, out_len, device=home, dtype=torch.float32)
            _native.check(getattr(lib, group)(g, _native.ptr(xin), _native.ptr(out), B, n, _native.stream_ptr(home)))
        return out


class OobleckEncoder(_NativeOobleck):
    _is_decoder = False

    def __init__(self, in_channels=2, channels=128, latent_dim=32, c_mults=[1, 2, 4, 8], strides=[2, 4, 8, 8],
                 use_snake=False, antialias_activation=False, operand_dtype="fp16"):
        super().__init__()
        if antialias_activation:
            raise NotImplementedError(_ANTIALIAS_REFUSAL)
        _check_strides(strides, decoder=False)
        check_oobleck_io_channels(in_channels, "OobleckEncoder in_channels")
        self._init_native(in_channels, channels, latent_dim, c_mults, strides, False, operand_dtype, use_snake=use_snake)
        cm = [1] + list(c_mults)
        self.depth = len(cm)
        layers = [WNConv1d(in_channels, cm[0] * channels, kernel_size=7, padding=3)]
        for i in range(self.depth - 1):
            layers.append(EncoderBlock(cm[i] * channels, cm[i + 1] * channels, strides[i], use_snake=use_snake))
        layers += [get_activation(_act(use_snake), channels=cm[-1] * channels),
                   WNConv1d(cm[-1] * channels, latent_dim, kernel_size=3, padding=1)]
        self.layers = nn.Sequential(*layers)
        self.downsampling_ratio = int(math.prod(strides))
        self.latent_dim = latent_dim
        self.out_width = latent_dim

    @torch.no_grad()
    def forward(self, x):
        """audio [B, in_channels, T] -> pre-bottleneck [B, latent_dim, T / prod(strides)]"""
        if not x.is_cuda:
            raise _native.NativeError("OobleckEncoder.forward needs CUDA tensors (no CPU fallback)")
        out = self._run(x, x.shape[-1] // self.downsampling_ratio, "satb_oobleck_encode", "satb_oobleck_group_encode")
        return out.to(x.dtype)


class OobleckDecoder(_NativeOobleck):
    _is_decoder = True

    def __init__(self, out_channels=2, channels=128, latent_dim=32, c_mults=[1, 2, 4, 8], strides=[2, 4, 8, 8],
                 use_snake=False, antialias_activation=False, use_nearest_upsample=False, final_tanh=True,
                 operand_dtype="fp16"):
        super().__init__()
        if antialias_activation:
            raise NotImplementedError(_ANTIALIAS_REFUSAL)
        _check_strides(strides, decoder=True, nearest=use_nearest_upsample)
        check_oobleck_io_channels(out_channels, "OobleckDecoder out_channels")
        self._init_native(out_channels, channels, latent_dim, c_mults, strides, final_tanh, operand_dtype,
                          use_snake=use_snake, use_nearest_upsample=use_nearest_upsample)
        cm = [1] + list(c_mults)
        self.depth = len(cm)
        layers = [WNConv1d(latent_dim, cm[-1] * channels, kernel_size=7, padding=3)]
        for i in range(self.depth - 1, 0, -1):
            layers.append(DecoderBlock(cm[i] * channels, cm[i - 1] * channels, strides[i - 1], use_snake=use_snake,
                                       antialias_activation=antialias_activation,
                                       use_nearest_upsample=use_nearest_upsample))
        layers += [get_activation(_act(use_snake), channels=cm[0] * channels),
                   WNConv1d(cm[0] * channels, out_channels, kernel_size=7, padding=3, bias=False),
                   nn.Tanh() if final_tanh else nn.Identity()]
        self.layers = nn.Sequential(*layers)
        self.upsampling_ratio = int(math.prod(strides))
        self.out_channels = out_channels
        self.out_width = out_channels

    @torch.no_grad()
    def forward(self, z):
        """latents [B, latent_dim, L] -> audio [B, out_channels, L * prod(strides)]"""
        if not z.is_cuda:
            raise _native.NativeError("OobleckDecoder.forward needs CUDA tensors (no CPU fallback)")
        out = self._run(z, z.shape[-1] * self.upsampling_ratio, "satb_oobleck_decode", "satb_oobleck_group_decode")
        return out.to(z.dtype)


def _micro_batches(x, iterate_batch):
    """``iterate_batch`` (bool or int) is the micro-batch size: True -> 1 (reference :318-324)."""
    if not iterate_batch:
        return [x]
    bs = int(iterate_batch)
    return [x[i:i + bs] for i in range(0, x.shape[0], bs)]


class AudioAutoencoder(nn.Module):
    def __init__(self, encoder, decoder, latent_dim, downsampling_ratio, sample_rate, io_channels=2,
                 bottleneck: Bottleneck = None, pretransform=None, in_channels=None, out_channels=None,
                 soft_clip=False):
        super().__init__()
        self.downsampling_ratio = downsampling_ratio
        self.min_length = downsampling_ratio
        self.sample_rate = sample_rate
        self.latent_dim = latent_dim
        self.io_channels = io_channels
        self.in_channels = io_channels if in_channels is None else in_channels
        self.out_channels = io_channels if out_channels is None else out_channels
        self.encoder = encoder
        self.decoder = decoder
        self.bottleneck = bottleneck
        if pretransform is not None:
            if not isinstance(pretransform, PQMFPretransform):
                raise NotImplementedError("nested pretransforms are outside the native hot path")
            # the encoder reads and the decoder writes io_channels * num_bands sub-bands
            check_oobleck_io_channels(self.io_channels * pretransform.pqmf.num_bands,
                                      f"io_channels {self.io_channels} x PQMF num_bands "
                                      f"{pretransform.pqmf.num_bands}")
        self.pretransform = pretransform
        self.soft_clip = soft_clip
        self.is_discrete = bool(self.bottleneck is not None and self.bottleneck.is_discrete)

    # -- plain encode / decode (reference :268-343) --------------------------------------
    def encode(self, audio, return_info=False, skip_pretransform=False, iterate_batch=False, **kwargs):
        if self.pretransform is not None and not skip_pretransform:
            audio = torch.cat([self.pretransform.encode(a) for a in _micro_batches(audio, iterate_batch)], dim=0)
        latents = audio
        if self.encoder is not None:
            latents = torch.cat([self.encoder(a) for a in _micro_batches(audio, iterate_batch)], dim=0)
        info = {}
        if self.bottleneck is not None:
            latents, binfo = self.bottleneck.encode(latents, return_info=True, **kwargs)
            info.update(binfo)
        return (latents, info) if return_info else latents

    def decode(self, latents, iterate_batch=False, **kwargs):
        if self.bottleneck is not None:
            latents = torch.cat([self.bottleneck.decode(l) for l in _micro_batches(latents, iterate_batch)], dim=0)
        decoded = torch.cat([self.decoder(l) for l in _micro_batches(latents, iterate_batch)], dim=0)
        if self.pretransform is not None:
            decoded = torch.cat([self.pretransform.decode(d) for d in _micro_batches(decoded, iterate_batch)], dim=0)
        if self.soft_clip:
            decoded = torch.tanh(decoded)
        return decoded

    # -- time sharding -------------------------------------------------------------------
    def shard_time(self, devices):
        """Run every later unchunked ``encode`` / ``decode`` (``encode_audio`` / ``decode_audio`` with
        ``chunked=False``) time-sharded over ``devices``; ``None`` returns to one device.

        Rank r runs on ``devices[r]``; a device may repeat (several ranks on one GPU run the same schedule, which is how
        it is tested on a single GPU).  The parameters stay on the home device ``devices[0]``, where the calls take their
        inputs and return their outputs; each rank gets its own native Oobleck handle with a copy of the weights,
        refreshed whenever the parameters change.  Each item's latents are split evenly over the ranks
        (``satb_oobleck_group_plan``); every rank decodes (encodes) its range plus a recompute margin of the decoder's
        (encoder's) receptive field on each interior side, and the home device gathers the ranks' own ranges.  The
        result is bit-identical to the single-device call.  A rank range shorter than the margin, or more ranks than
        latents, is refused at call time.  Ranks on distinct GPUs need peer-to-peer access with the home device.

        The chunked paths and ``reconstruct_audio(chunked=True)`` run on the home device: their chunks are already the
        split.  A PQMF pretransform runs on the home device around the sharded Oobleck.  Sharding the DiT of a
        diffusion model (``shard_tokens``) leaves its pretransform on one device; call this on it to shard the VAE too."""
        devices = check_time_shard_devices(devices)
        for m in (self.encoder, self.decoder):
            if isinstance(m, _NativeOobleck):
                m.shard_time(devices)
        return self

    @contextlib.contextmanager
    def _on_home_device(self):
        """The chunked paths run their chunks unsharded."""
        mods = [m for m in (self.encoder, self.decoder) if isinstance(m, _NativeOobleck)]
        prev = [m.__dict__.get("_paused") for m in mods]
        for m in mods:
            m.__dict__["_paused"] = True
        try:
            yield
        finally:
            for m, p in zip(mods, prev):
                m.__dict__["_paused"] = p

    # -- chunked paths (reference :410-645) ----------------------------------------------
    @staticmethod
    def _chunk_starts(total, chunk, hop, extra=0):
        n_chunk = int(math.ceil((total - chunk) / hop)) + 1
        pad_len = chunk + hop * (n_chunk - 1 + extra) - total
        return n_chunk, pad_len

    @staticmethod
    def _crossfade_sum(pieces, n_chunk, hop, chunk, overlap, total_len, win):
        """Overlap-add chunk outputs [b, n_chunk, c, chunk] with a Bartlett fade on shared edges."""
        b, _, c, _ = pieces.shape
        out = torch.zeros((b, c, total_len), device=pieces.device)
        for i in range(n_chunk):
            piece = pieces[:, i]
            if i != 0:
                piece[:, :, :overlap] *= win[None, None, :overlap]
            if i != n_chunk - 1:
                piece[:, :, -overlap:] *= win[None, None, -overlap:]
            out[..., i * hop: i * hop + chunk] += piece
        return out

    def _run_chunks(self, chunks, fn, max_batch_size):
        with self._on_home_device():
            outs = [fn(chunks[i:i + max_batch_size]) for i in range(0, chunks.shape[0], max_batch_size)]
        return torch.cat(outs, dim=0)

    def encode_audio(self, audio, chunked=False, chunk_size=128, overlap=4, max_batch_size=1, **kwargs):
        bs, n_ch, sample_length = audio.shape
        ratio = self.downsampling_ratio
        assert n_ch == self.in_channels
        assert sample_length % ratio == 0, "The audio length must be a multiple of compression ratio."
        if not chunked:
            return self.encode(audio, **kwargs)
        latent_length = sample_length // ratio
        hop_l = chunk_size - overlap
        win = torch.bartlett_window(overlap * 2, device=audio.device)
        chunk_s, hop_s = chunk_size * ratio, hop_l * ratio
        n_chunk, pad_len = self._chunk_starts(sample_length, chunk_s, hop_s)
        audio = F.pad(audio, (0, pad_len))                                   # zero padding
        chunks = torch.stack([audio[..., i * hop_s: i * hop_s + chunk_s] for i in range(n_chunk)], dim=1)
        zs = self._run_chunks(chunks.reshape(bs * n_chunk, n_ch, chunk_s), self.encode, max_batch_size)
        zs = zs.reshape(bs, n_chunk, zs.shape[1], zs.shape[2])
        latents = self._crossfade_sum(zs, n_chunk, hop_l, chunk_size, overlap, audio.shape[-1] // ratio, win)
        return latents[..., :latent_length]

    def decode_audio(self, latents, chunked=False, chunk_size=128, overlap=4, max_batch_size=1, **kwargs):
        bs, latent_dim, latent_length = latents.shape
        ratio = self.downsampling_ratio
        assert latent_dim == self.latent_dim
        if not chunked:
            return self.decode(latents, **kwargs)
        hop = chunk_size - overlap
        win = torch.bartlett_window(overlap * ratio * 2, device=latents.device)
        n_chunk, pad_len = self._chunk_starts(latent_length, chunk_size, hop)
        latents = F.pad(latents, (0, pad_len), mode="reflect")              # reflect padding
        chunks = torch.stack([latents[..., i * hop: i * hop + chunk_size] for i in range(n_chunk)], dim=1)
        xs = self._run_chunks(chunks.reshape(bs * n_chunk, latent_dim, chunk_size), self.decode, max_batch_size)
        xs = xs.reshape(bs, n_chunk, xs.shape[1], xs.shape[2])
        audio = self._crossfade_sum(xs, n_chunk, hop * ratio, chunk_size * ratio, overlap * ratio,
                                    latents.shape[-1] * ratio, win)
        return audio[..., :latent_length * ratio]

    @torch.no_grad()
    def reconstruct_audio(self, audio, chunked=True, chunk_size=128, overlap=4, max_batch_size=1, **kwargs):
        bs, n_ch, sample_length = audio.shape
        ratio = self.downsampling_ratio
        assert n_ch == self.in_channels
        if not chunked:
            return self.decode(self.encode(audio, **kwargs), **kwargs)
        win = torch.bartlett_window(overlap * ratio * 2, device=audio.device)
        chunk_s, overlap_s = chunk_size * ratio, overlap * ratio
        hop_s = chunk_s - overlap_s
        # the reference pads one hop more here than in encode_audio (:607 vs :455)
        n_chunk, pad_len = self._chunk_starts(sample_length, chunk_s, hop_s, extra=1)
        audio = F.pad(audio, (0, pad_len))
        chunks = torch.stack([audio[..., i * hop_s: i * hop_s + chunk_s] for i in range(n_chunk)], dim=1)
        xs = self._run_chunks(chunks.reshape(bs * n_chunk, n_ch, chunk_s), lambda c: self.decode(self.encode(c)),
                              max_batch_size)
        xs = xs.reshape(bs, n_chunk, xs.shape[1], xs.shape[2])
        rec = self._crossfade_sum(xs, n_chunk, hop_s, chunk_s, overlap_s, audio.shape[-1], win)
        return rec[..., :sample_length]


# ---------------------------------------------------------------------------------- factories
def create_encoder_from_config(encoder_config: tp.Dict[str, tp.Any]):
    if encoder_config["type"] != "oobleck":
        raise NotImplementedError(f"encoder '{encoder_config['type']}' is outside the native hot path (oobleck only)")
    encoder = OobleckEncoder(**encoder_config["config"])
    if not encoder_config.get("requires_grad", True):
        for p in encoder.parameters():
            p.requires_grad = False
    return encoder


def create_decoder_from_config(decoder_config: tp.Dict[str, tp.Any]):
    if decoder_config["type"] != "oobleck":
        raise NotImplementedError(f"decoder '{decoder_config['type']}' is outside the native hot path (oobleck only)")
    decoder = OobleckDecoder(**decoder_config["config"])
    if not decoder_config.get("requires_grad", True):
        for p in decoder.parameters():
            p.requires_grad = False
    return decoder


def create_autoencoder_from_config(config: tp.Dict[str, tp.Any]):
    ae = config["model"]
    bottleneck = ae.get("bottleneck")
    pretransform = ae.get("pretransform")
    if pretransform:
        pretransform = create_pretransform_from_config(pretransform, config["sample_rate"])
    return AudioAutoencoder(
        create_encoder_from_config(ae["encoder"]), create_decoder_from_config(ae["decoder"]),
        io_channels=ae["io_channels"], latent_dim=ae["latent_dim"], downsampling_ratio=ae["downsampling_ratio"],
        sample_rate=config["sample_rate"], bottleneck=create_bottleneck_from_config(bottleneck) if bottleneck else None,
        pretransform=pretransform, in_channels=ae.get("in_channels"), out_channels=ae.get("out_channels"),
        soft_clip=ae["decoder"].get("soft_clip", False))


# ---------------------------------------------------------------------------------- diffusion autoencoder
class DiffusionAutoencoder(AudioAutoencoder):
    """reference models/autoencoders.py:648-690: an (optional) Oobleck encoder and bottleneck, and a DiT decoder that
    samples the pretransform's input (raw audio, PQMF sub-bands or an Oobleck autoencoder's latents) from noise, with
    the upsampled latents as its input-concat conditioning.  ``encode`` is the inherited one.  State-dict keys are the
    reference's: ``encoder.*``, ``diffusion.model.*``, and the bottleneck's and pretransform's.

    The pretransform may be None, a ``PQMFPretransform`` or an ``AutoencoderPretransform``; the DiT then diffuses the
    signal that pretransform decodes, so its io_channels are the audio channels, the channels x bands, or the inner
    autoencoder's latent_dim."""

    def __init__(self, diffusion, diffusion_downsampling_ratio, *args, decoder=None, pretransform=None, **kwargs):
        if decoder is not None:
            raise NotImplementedError(_DIFFAE_DECODER_REFUSAL)
        # AudioAutoencoder accepts a PQMF pretransform only, and checks its width as the input of an Oobleck encoder
        # over channels x bands; here the pretransform wraps the DiT's signal instead, so it is attached afterwards
        super().__init__(*args, decoder=None, pretransform=None, **kwargs)
        if pretransform is not None and not isinstance(pretransform, (PQMFPretransform, AutoencoderPretransform)):
            raise NotImplementedError("DiffusionAutoencoder: the pretransform must be pqmf or an Oobleck autoencoder")
        self.pretransform = pretransform
        dit = getattr(diffusion, "model", None)
        if dit is not None and hasattr(dit, "input_concat_dim"):
            concat = self.latent_dim + getattr(self.bottleneck, "noise_augment_dim", 0)
            if dit.io_channels != self.io_channels or dit.input_concat_dim != concat:
                raise ValueError(f"DiffusionAutoencoder: the DiT has io_channels {dit.io_channels} and input_concat_dim "
                                 f"{dit.input_concat_dim}; the model needs {self.io_channels} and {concat} (latent_dim "
                                 "plus the bottleneck's noise channels)")
        self.diffusion = diffusion
        self.min_length = self.downsampling_ratio * diffusion_downsampling_ratio
        if self.encoder is not None:
            # shrink the initial encoder parameters to avoid saturated latents (reference :661-665)
            with torch.no_grad():
                for param in self.encoder.parameters():
                    param *= 0.5
            self.encoder.refresh_native_weights()

    def decode(self, latents, steps=100, noise=None, **kwargs):
        """latents [B, latent_dim, n] -> bottleneck decode, nearest upsample to n * downsampling_ratio, ``steps``
        v-diffusion steps of the DiT from ``noise`` [B, io_channels, n * downsampling_ratio] (default: a torch.randn
        draw on the latents' device, as the reference draws it), then the pretransform's decode."""
        from ..inference.sampling import sample
        upsampled_length = latents.shape[2] * self.downsampling_ratio
        if self.bottleneck is not None:
            latents = self.bottleneck.decode(latents)
        if latents.shape[2] != upsampled_length:
            latents = F.interpolate(latents, size=upsampled_length, mode="nearest")
        shape = (latents.shape[0], self.io_channels, upsampled_length)
        if noise is None:
            noise = torch.randn(*shape, device=latents.device)
        elif tuple(noise.shape) != shape:
            raise ValueError(f"noise has shape {tuple(noise.shape)}, the decode needs {shape}")
        decoded = sample(self.diffusion, noise, steps, 0, input_concat_cond=latents)
        if self.pretransform is not None:
            with torch.no_grad():
                decoded = self.pretransform.decode(decoded)
        return decoded


_DIFFAE_DECODER_REFUSAL = (
    "DiffusionAutoencoder with a 'decoder' is not supported: the reference's decode passes the latents to "
    "self.decode itself in that case (models/autoencoders.py:673-674), which recurses without end, so there is no "
    "behaviour to reproduce")


def create_diffAE_from_config(config: tp.Dict[str, tp.Any]):
    """reference models/autoencoders.py:790-847 with a DiT diffusion block (``DiTWrapper``, diffusion downsampling 1)."""
    from .diffusion import DiTWrapper
    diffae = config["model"]
    if "decoder" in diffae:
        raise NotImplementedError(_DIFFAE_DECODER_REFUSAL)
    kind = diffae["diffusion"]["type"]
    if kind in ("DAU1d", "adp_1d"):
        raise NotImplementedError(f"diffusion block '{kind}' is not supported: the ADP U-Nets are outside this "
                                  "package (DESIGN.md section 7); the diffusion block must be 'dit'")
    if kind != "dit":
        raise NotImplementedError(f"No such model type: '{kind}'")
    encoder = create_encoder_from_config(diffae["encoder"]) if "encoder" in diffae else None
    diffusion = DiTWrapper(**diffae["diffusion"]["config"])
    bottleneck = diffae.get("bottleneck")
    pretransform = diffae.get("pretransform")
    if pretransform:
        pretransform = create_pretransform_from_config(pretransform, config["sample_rate"])
    return DiffusionAutoencoder(
        encoder=encoder, diffusion=diffusion, io_channels=diffae["io_channels"], sample_rate=config["sample_rate"],
        latent_dim=diffae["latent_dim"], downsampling_ratio=diffae["downsampling_ratio"], diffusion_downsampling_ratio=1,
        bottleneck=create_bottleneck_from_config(bottleneck) if bottleneck else None, pretransform=pretransform or None)
