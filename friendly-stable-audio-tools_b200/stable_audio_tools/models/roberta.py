"""Native RoBERTa encoder: Hugging Face ``RobertaModel(output_hidden_states=True).hidden_states[feature_layer_ix]``
(transformers ``models/roberta/modeling_roberta.py``) on the library's sm_90a kernels (``csrc/roberta.cu``), for
``CLAPTextConditioner``.

Only the layers up to the requested hidden state run: ``n = feature_layer_ix mod (num_hidden_layers + 1)`` of them,
index 0 being the embedding output.  Every position is computed, padded ones included; keys are limited to each
prompt's valid prefix, as HF's additive mask does for right-padded masks.  The residual stream is fp32 and the GEMM
operands fp16 (default) or bf16.

Built from the RobertaConfig fields it uses; refused with ``NotImplementedError`` before any CUDA call: a head dim
(hidden_size / num_attention_heads) other than 64, hidden_size not a multiple of 128 or above 1024, intermediate_size
not a multiple of 32, ``hidden_act`` other than ``gelu``, ``position_embedding_type`` other than ``absolute``, prompts
longer than 512 tokens and masks that are not right-padded prefixes of length >= 1.  Token ids outside
``[0, vocab_size)`` raise ``ValueError``.
"""
import ctypes
import typing as tp

import torch

from .. import _native
from .._native import NativeError

MAX_LENGTH = 512          # longest prompt an encode takes
_DTYPES = {"fp16": 0, "bf16": 1}
# keys of a RobertaModel state dict the encoder has no use for: the pooler, and the buffers older checkpoints carry
_UNUSED = ("pooler.", "embeddings.position_ids", "embeddings.token_type_ids")


def layers_to_run(num_hidden_layers: int, feature_layer_ix: int) -> int:
    """The n with hidden_states[feature_layer_ix] == hidden_states[n] for a tuple of num_hidden_layers + 1 entries."""
    if not -(num_hidden_layers + 1) <= feature_layer_ix <= num_hidden_layers:
        raise ValueError(f"feature_layer_ix {feature_layer_ix} is outside the {num_hidden_layers + 1} hidden states")
    return feature_layer_ix % (num_hidden_layers + 1)


def check_config(hidden_size: int, num_attention_heads: int, intermediate_size: int, hidden_act: str = "gelu",
                 position_embedding_type: str = "absolute", operand_dtype: str = "fp16") -> None:
    if num_attention_heads < 1 or hidden_size != 64 * num_attention_heads:
        raise NotImplementedError(f"native RoBERTa: head dim {hidden_size}/{num_attention_heads} is not supported (64)")
    if hidden_size % 128 != 0 or not 128 <= hidden_size <= 1024:
        raise NotImplementedError(f"native RoBERTa: hidden_size {hidden_size} must be a multiple of 128, at most 1024")
    if intermediate_size % 32 != 0 or intermediate_size < 32:
        raise NotImplementedError(f"native RoBERTa: intermediate_size {intermediate_size} must be a positive multiple "
                                  "of 32")
    if hidden_act != "gelu":
        raise NotImplementedError(f"native RoBERTa: hidden_act '{hidden_act}' is not supported ('gelu')")
    if position_embedding_type != "absolute":
        raise NotImplementedError(f"native RoBERTa: position_embedding_type '{position_embedding_type}' is not "
                                  "supported ('absolute')")
    if operand_dtype not in _DTYPES:
        raise ValueError(f"operand_dtype must be one of {sorted(_DTYPES)}")


def prompt_lengths(input_ids: torch.Tensor, attention_mask: torch.Tensor, vocab_size: int) -> torch.Tensor:
    """The length of every prompt (int32, on the host) after the checks of RobertaEncoder.forward: at most 512 tokens,
    masks that are right-padded prefixes of at least one token, ids inside the vocabulary."""
    if input_ids.dim() != 2 or attention_mask.shape != input_ids.shape:
        raise ValueError("input_ids and attention_mask must both be [batch, length]")
    B, L = input_ids.shape
    if L > MAX_LENGTH:
        raise NotImplementedError(f"native RoBERTa: prompts of {L} tokens exceed {MAX_LENGTH}")
    m = attention_mask.to(torch.bool)
    lengths = m.sum(dim=1)
    prefix = torch.arange(L, device=m.device)[None, :] < lengths[:, None]
    if not torch.equal(m, prefix):
        raise NotImplementedError("native RoBERTa: attention masks must be right-padded prefixes (ones, then zeros)")
    if B * L > 0 and int(lengths.min()) < 1:
        raise NotImplementedError("native RoBERTa: every prompt needs at least one unmasked token")
    if input_ids.dtype.is_floating_point or input_ids.dtype == torch.bool:
        raise ValueError("input_ids must be an integer tensor")
    if B * L > 0 and (int(input_ids.min()) < 0 or int(input_ids.max()) >= vocab_size):
        raise ValueError(f"token ids must lie in [0, {vocab_size})")
    return lengths.to(torch.int32).cpu()


class RobertaEncoder:
    """``forward(input_ids, attention_mask) -> [B, L, hidden_size]`` fp32 (``[B, L, out_dim]`` with a projection from
    ``set_proj_out``): hidden state ``feature_layer_ix`` at every position.  Weights: ``load_state_dict`` with a
    ``RobertaModel`` state dict (HF keys).  The handle lives on the CUDA device the weights are loaded to."""

    def __init__(self, vocab_size: int, hidden_size: int, num_hidden_layers: int, num_attention_heads: int,
                 intermediate_size: int, max_position_embeddings: int = 514, type_vocab_size: int = 1,
                 pad_token_id: int = 1, layer_norm_eps: float = 1e-5, hidden_act: str = "gelu",
                 position_embedding_type: str = "absolute", feature_layer_ix: int = -1, operand_dtype: str = "fp16"):
        check_config(hidden_size, num_attention_heads, intermediate_size, hidden_act, position_embedding_type,
                     operand_dtype)
        self.n_layers = layers_to_run(num_hidden_layers, feature_layer_ix)
        self.vocab_size, self.hidden_size, self.num_heads = vocab_size, hidden_size, num_attention_heads
        self.intermediate_size, self.num_hidden_layers = intermediate_size, num_hidden_layers
        self.max_position_embeddings, self.type_vocab_size = max_position_embeddings, type_vocab_size
        self.pad_token_id, self.layer_norm_eps, self.operand_dtype = pad_token_id, layer_norm_eps, operand_dtype
        self.feature_layer_ix = feature_layer_ix
        if max_position_embeddings <= pad_token_id + 1:
            raise NotImplementedError("native RoBERTa: max_position_embeddings leaves no room for a position id")
        self.out_dim = hidden_size
        self.device = None
        self._h = None

    @classmethod
    def from_config(cls, config, feature_layer_ix: int = -1, operand_dtype: str = "fp16") -> "RobertaEncoder":
        """From a transformers RobertaConfig (or a dict with its fields)."""
        get = (lambda k, d=None: config.get(k, d)) if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
        return cls(vocab_size=get("vocab_size"), hidden_size=get("hidden_size"),
                   num_hidden_layers=get("num_hidden_layers"), num_attention_heads=get("num_attention_heads"),
                   intermediate_size=get("intermediate_size"),
                   max_position_embeddings=get("max_position_embeddings", 514),
                   type_vocab_size=get("type_vocab_size", 1), pad_token_id=get("pad_token_id", 1),
                   layer_norm_eps=get("layer_norm_eps", 1e-5), hidden_act=get("hidden_act", "gelu"),
                   position_embedding_type=get("position_embedding_type", "absolute") or "absolute",
                   feature_layer_ix=feature_layer_ix, operand_dtype=operand_dtype)

    def _cfg(self):
        return _native.SatbRobertaConfig(
            vocab_size=self.vocab_size, hidden_size=self.hidden_size, num_heads=self.num_heads,
            intermediate_size=self.intermediate_size, num_layers=self.n_layers,
            max_position_embeddings=self.max_position_embeddings, type_vocab_size=self.type_vocab_size,
            pad_token_id=self.pad_token_id, layer_norm_eps=self.layer_norm_eps,
            operand_dtype=_DTYPES[self.operand_dtype])

    def _used(self, key: str) -> bool:
        if key.startswith(_UNUSED):
            return False
        if key.startswith("encoder.layer."):
            return int(key.split(".")[2]) < self.n_layers
        return True

    def load_state_dict(self, state_dict: tp.Mapping[str, torch.Tensor], device="cuda") -> "RobertaEncoder":
        """The tensors of a RobertaModel state dict (any dtype and device) that the requested hidden state depends on go
        to ``device`` as fp32 and into the handle; the pooler and the layers past the cut are skipped.  Replaces the
        weights of an earlier call."""
        device = torch.device(device)
        if device.type != "cuda":
            raise NativeError("RobertaEncoder runs on a CUDA device only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        lib = _native.lib()
        with torch.cuda.device(device):
            self.close()
            h = ctypes.c_void_p()
            _native.check(lib.satb_roberta_create(ctypes.byref(self._cfg()), ctypes.byref(h)))
            self._h, self.device = h, device
            stream = _native.stream_ptr(device)
            for k, v in state_dict.items():
                if not self._used(k):
                    continue
                t = v.detach().to(device=device, dtype=torch.float32).contiguous()
                _native.check(lib.satb_roberta_load_weight(h, k.encode(), _native.dev_f32(t, k), t.numel(), stream))
                torch.cuda.current_stream(device).synchronize()
            _native.check(lib.satb_roberta_finalize(h, stream))
        self.out_dim = self.hidden_size
        return self

    def set_proj_out(self, weight: torch.Tensor, bias: torch.Tensor) -> None:
        """An nn.Linear(hidden_size, out_dim) run on the hidden state inside the encode (the conditioner's proj_out);
        its output width must be a multiple of 8."""
        if self._h is None:
            raise NativeError("load the encoder's weights first")
        w = weight.detach().to(device=self.device, dtype=torch.float32).contiguous()
        b = bias.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if w.shape != (b.numel(), self.hidden_size):
            raise ValueError("proj_out weight must be [out_dim, hidden_size] with a bias of out_dim")
        with torch.cuda.device(self.device):
            _native.check(_native.lib().satb_roberta_set_proj_out(self._h, _native.dev_f32(w), _native.dev_f32(b),
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
        if L + self.pad_token_id >= self.max_position_embeddings:
            raise NotImplementedError(f"native RoBERTa: {L} tokens need position ids past max_position_embeddings "
                                      f"{self.max_position_embeddings}")
        with torch.cuda.device(self.device):
            ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
            out = torch.empty(B, L, self.out_dim, device=self.device, dtype=torch.float32)
            if B * L > 0:
                _native.check(_native.lib().satb_roberta_encode(
                    self._h, ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(lengths.data_ptr()), B, L,
                    ctypes.c_void_p(out.data_ptr()), _native.stream_ptr(self.device)))
        return out

    __call__ = forward

    def close(self) -> None:
        if self._h is not None:
            _native.lib().satb_roberta_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
