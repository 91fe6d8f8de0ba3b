"""Native T5 encoder: Hugging Face ``T5EncoderModel.forward`` (transformers ``models/t5/modeling_t5.py``) on the
library's sm_90a kernels (``csrc/t5.cu``), for ``T5Conditioner(native=True)``.

Prompts are packed: only the valid (unmasked) tokens of every prompt are computed, and the padded positions of the
output are exact zeros.  The residual stream is fp32 and the GEMM operands fp16 (the reference's dtype) or bf16.  In
fp16 the 16-bit RMSNorm and feed-forward activations saturate at +-65504 instead of overflowing to infinity.

Built from the T5Config fields it uses; refused with ``NotImplementedError`` before any CUDA call: ``d_kv`` other than
64 or 128, ``feed_forward_proj`` other than ``relu`` / ``gated-gelu``, ``d_model`` not a multiple of 128 or above 4096,
``d_ff`` not a multiple of 32, prompts longer than 512 tokens and masks that are not right-padded prefixes.  Token ids
outside ``[0, vocab_size)`` raise ``ValueError``.
"""
import ctypes
import math
import typing as tp

import torch

from .. import _native
from .._native import NativeError

MAX_LENGTH = 512          # longest prompt an encode takes
BUCKET_SPAN = 2 * MAX_LENGTH - 1   # relative positions -511 .. 511
_FF = {"relu": _native.T5_FF_RELU, "gated-gelu": _native.T5_FF_GATED_GELU}
_DTYPES = {"fp16": 0, "bf16": 1}


def relative_position_buckets(relative_position: torch.Tensor, num_buckets: int = 32,
                              max_distance: int = 128) -> torch.Tensor:
    """T5Attention._relative_position_bucket with bidirectional=True (modeling_t5.py:189-234), the same torch integer
    and float32 log operations in the same order, so the same buckets bit for bit."""
    relative_buckets = 0
    num_buckets //= 2
    relative_buckets += (relative_position > 0).to(torch.long) * num_buckets
    relative_position = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    relative_position_if_large = max_exact + (
        torch.log(relative_position.float() / max_exact)
        / math.log(max_distance / max_exact)
        * (num_buckets - max_exact)
    ).to(torch.long)
    relative_position_if_large = torch.min(
        relative_position_if_large, torch.full_like(relative_position_if_large, num_buckets - 1))
    relative_buckets += torch.where(is_small, relative_position, relative_position_if_large)
    return relative_buckets


def bucket_table(num_buckets: int, max_distance: int) -> torch.Tensor:
    """int32 [1023]: the bucket of relative position k - 511 at index k (the table satb_t5_set_buckets takes)."""
    rel = torch.arange(-(MAX_LENGTH - 1), MAX_LENGTH, dtype=torch.long)
    return relative_position_buckets(rel, num_buckets, max_distance).to(torch.int32)


def check_config(d_model: int, d_kv: int, d_ff: int, feed_forward_proj: str, operand_dtype: str) -> None:
    if d_kv not in (64, 128):
        raise NotImplementedError(f"native T5: d_kv {d_kv} is not supported (64 or 128)")
    if feed_forward_proj not in _FF:
        raise NotImplementedError(f"native T5: feed_forward_proj '{feed_forward_proj}' is not supported "
                                  f"({sorted(_FF)})")
    if d_model % 128 != 0 or not 128 <= d_model <= 4096:
        raise NotImplementedError(f"native T5: d_model {d_model} must be a multiple of 128, at most 4096")
    if d_ff % 32 != 0 or d_ff < 32:
        raise NotImplementedError(f"native T5: d_ff {d_ff} must be a positive multiple of 32")
    if operand_dtype not in _DTYPES:
        raise ValueError(f"operand_dtype must be one of {sorted(_DTYPES)}")


def prompt_lengths(input_ids: torch.Tensor, attention_mask: torch.Tensor, vocab_size: int) -> torch.Tensor:
    """The length of every prompt (int32, on the host) after the checks of T5Encoder.forward: at most 512 tokens,
    masks that are right-padded prefixes, ids inside the vocabulary.  Runs on the tensors' own device."""
    if input_ids.dim() != 2 or attention_mask.shape != input_ids.shape:
        raise ValueError("input_ids and attention_mask must both be [batch, length]")
    B, L = input_ids.shape
    if L > MAX_LENGTH:
        raise NotImplementedError(f"native T5: prompts of {L} tokens exceed {MAX_LENGTH}")
    m = attention_mask.to(torch.bool)
    lengths = m.sum(dim=1)
    prefix = torch.arange(L, device=m.device)[None, :] < lengths[:, None]
    if not torch.equal(m, prefix):
        raise NotImplementedError("native T5: attention masks must be right-padded prefixes (ones, then zeros)")
    if input_ids.dtype.is_floating_point or input_ids.dtype == torch.bool:
        raise ValueError("input_ids must be an integer tensor")
    if B * L > 0 and (int(input_ids.min()) < 0 or int(input_ids.max()) >= vocab_size):
        raise ValueError(f"token ids must lie in [0, {vocab_size})")
    return lengths.to(torch.int32).cpu()


class T5Encoder:
    """``forward(input_ids, attention_mask) -> [B, L, d_model]`` fp32 (``[B, L, out_dim]`` with a projection from
    ``set_proj_out``), exact zeros at padded positions.  Weights: ``load_state_dict`` with a ``T5EncoderModel`` state
    dict (HF keys).  The handle lives on the CUDA device the weights are loaded to."""

    def __init__(self, vocab_size: int, d_model: int, d_kv: int, num_heads: int, d_ff: int, num_layers: int,
                 relative_attention_num_buckets: int = 32, relative_attention_max_distance: int = 128,
                 feed_forward_proj: str = "relu", layer_norm_epsilon: float = 1e-6, operand_dtype: str = "fp16"):
        check_config(d_model, d_kv, d_ff, feed_forward_proj, operand_dtype)
        self.vocab_size, self.d_model, self.d_kv, self.num_heads = vocab_size, d_model, d_kv, num_heads
        self.d_ff, self.num_layers, self.feed_forward_proj = d_ff, num_layers, feed_forward_proj
        self.num_buckets, self.max_distance = relative_attention_num_buckets, relative_attention_max_distance
        self.layer_norm_epsilon, self.operand_dtype = layer_norm_epsilon, operand_dtype
        self.out_dim = d_model
        self.device = None
        self._h = None

    @classmethod
    def from_config(cls, config, operand_dtype: str = "fp16") -> "T5Encoder":
        """From a transformers T5Config (or a dict with its fields)."""
        get = (lambda k, d=None: config.get(k, d)) if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
        return cls(vocab_size=get("vocab_size"), d_model=get("d_model"), d_kv=get("d_kv"), num_heads=get("num_heads"),
                   d_ff=get("d_ff"), num_layers=get("num_layers"),
                   relative_attention_num_buckets=get("relative_attention_num_buckets", 32),
                   relative_attention_max_distance=get("relative_attention_max_distance", 128),
                   feed_forward_proj=get("feed_forward_proj", "relu"),
                   layer_norm_epsilon=get("layer_norm_epsilon", 1e-6), operand_dtype=operand_dtype)

    def _cfg(self):
        return _native.SatbT5Config(
            vocab_size=self.vocab_size, d_model=self.d_model, d_kv=self.d_kv, num_heads=self.num_heads, d_ff=self.d_ff,
            num_layers=self.num_layers, relative_attention_num_buckets=self.num_buckets,
            relative_attention_max_distance=self.max_distance, feed_forward_proj=_FF[self.feed_forward_proj],
            layer_norm_epsilon=self.layer_norm_epsilon, operand_dtype=_DTYPES[self.operand_dtype])

    def load_state_dict(self, state_dict: tp.Mapping[str, torch.Tensor], device="cuda") -> "T5Encoder":
        """Every tensor of a T5EncoderModel state dict (any dtype and device) goes to ``device`` as fp32 and into the
        handle; keys the encoder does not use (``encoder.embed_tokens.weight`` duplicates ``shared.weight``) are
        skipped.  Replaces the weights of an earlier call."""
        device = torch.device(device)
        if device.type != "cuda":
            raise NativeError("T5Encoder runs on a CUDA device only (no CPU fallback)")
        lib = _native.lib()
        with torch.cuda.device(device):
            self.close()
            h = ctypes.c_void_p()
            _native.check(lib.satb_t5_create(ctypes.byref(self._cfg()), ctypes.byref(h)))
            self._h, self.device = h, device
            stream = _native.stream_ptr(device)
            for k, v in state_dict.items():
                if k == "encoder.embed_tokens.weight" and "shared.weight" in state_dict:
                    continue
                if ".relative_attention_bias." in k and not k.startswith("encoder.block.0."):
                    continue
                t = v.detach().to(device=device, dtype=torch.float32).contiguous()
                _native.check(lib.satb_t5_load_weight(h, k.encode(), _native.dev_f32(t, k), t.numel(), stream))
                torch.cuda.current_stream(device).synchronize()
            b = bucket_table(self.num_buckets, self.max_distance).contiguous()
            _native.check(lib.satb_t5_set_buckets(h, ctypes.c_void_p(b.data_ptr()), b.numel()))
            _native.check(lib.satb_t5_finalize(h, stream))
        self.out_dim = self.d_model
        return self

    def set_proj_out(self, weight: torch.Tensor, bias: torch.Tensor) -> None:
        """An nn.Linear(d_model, out_dim) run on the final hidden states inside the encode (the conditioner's
        proj_out); its output width must be a multiple of 8."""
        if self._h is None:
            raise NativeError("load the encoder's weights first")
        w = weight.detach().to(device=self.device, dtype=torch.float32).contiguous()
        b = bias.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if w.shape != (b.numel(), self.d_model):
            raise ValueError("proj_out weight must be [out_dim, d_model] with a bias of out_dim")
        with torch.cuda.device(self.device):
            _native.check(_native.lib().satb_t5_set_proj_out(self._h, _native.dev_f32(w), _native.dev_f32(b),
                                                             w.shape[0], _native.stream_ptr(self.device)))
            torch.cuda.current_stream(self.device).synchronize()
        self.out_dim = w.shape[0]

    def forward(self, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        if self._h is None:
            raise NativeError("load the encoder's weights first")
        for name, t in (("input_ids", input_ids), ("attention_mask", attention_mask)):
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise NativeError(f"{name} must be a CUDA tensor: this package runs on the GPU only (no CPU fallback)")
        lengths = prompt_lengths(input_ids, attention_mask, self.vocab_size)
        B, L = input_ids.shape
        with torch.cuda.device(self.device):
            ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
            out = torch.empty(B, L, self.out_dim, device=self.device, dtype=torch.float32)
            if B * L > 0:
                _native.check(_native.lib().satb_t5_encode(
                    self._h, ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(lengths.data_ptr()), B, L,
                    ctypes.c_void_p(out.data_ptr()), _native.stream_ptr(self.device)))
        return out

    __call__ = forward

    def close(self) -> None:
        if self._h is not None:
            _native.lib().satb_t5_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
