"""Conditioners used by the Stable Audio text-to-audio configs (SURVEY.md 8f "next" row).

They run once per generation, not per denoise step, so they stay plain PyTorch modules:
``NumberConditioner`` (learned Fourier features of a normalised scalar, reference
``models/conditioners.py:64-102`` + ``models/adp.py:680-701,1495-1512``), ``IntConditioner``
(:39-61), ``T5Conditioner`` (frozen fp16 HF T5 encoder, padded to ``max_length``, masked
positions zeroed, :261-346) and ``MultiConditioner`` (:505-549); state-dict keys match the
reference (``conditioner.conditioners.<id>.embedder.embedding.0.weights`` ...).  The T5 encoder
needs the HF model files locally or a network, exactly like the reference.  ``T5Conditioner(native=True)`` (a JSON
conditioner "config" may carry it) runs the same weights on the native packed encoder (models/t5.py) instead of HF's
eager fp16 module.  ``CLAPTextConditioner`` (:105-192, ``"clap_text"``) returns hidden states of CLAP's RoBERTa
text branch computed by the native encoder (models/roberta.py); it needs the roberta-base tokenizer files locally.
"""
import logging
import math
import typing as tp
import warnings

import torch
from torch import nn


class Conditioner(nn.Module):
    def __init__(self, dim: int, output_dim: int, project_out: bool = False):
        super().__init__()
        self.dim, self.output_dim = dim, output_dim
        self.proj_out = nn.Linear(dim, output_dim) if (dim != output_dim or project_out) else nn.Identity()

    def set_device(self, device) -> None:
        raise NotImplementedError()


class LearnedPositionalEmbedding(nn.Module):
    """[x, sin(2 pi x w), cos(2 pi x w)] with learned frequencies w (continuous inputs)."""

    def __init__(self, dim: int):
        super().__init__()
        assert dim % 2 == 0
        self.weights = nn.Parameter(torch.randn(dim // 2))

    def forward(self, x):
        x = x[:, None]
        freqs = x * self.weights[None, :] * 2 * math.pi
        return torch.cat((x, freqs.sin(), freqs.cos()), dim=-1)


class NumberEmbedder(nn.Module):
    def __init__(self, features: int, dim: int = 256):
        super().__init__()
        self.features = features
        self.embedding = nn.Sequential(LearnedPositionalEmbedding(dim), nn.Linear(dim + 1, features))

    def forward(self, x):
        if not torch.is_tensor(x):
            x = torch.tensor(x, device=next(self.embedding.parameters()).device)
        shape = x.shape
        return self.embedding(x.reshape(-1)).view(*shape, self.features)


class NumberConditioner(Conditioner):
    """floats -> clamp to [min_val, max_val] -> normalise to [0, 1] -> NumberEmbedder -> [B, 1, dim]."""

    def __init__(self, output_dim: int, min_val: float = 0, max_val: float = 1):
        super().__init__(output_dim, output_dim)
        self.min_val, self.max_val = min_val, max_val
        self.embedder = NumberEmbedder(features=output_dim)
        self.device = next(self.embedder.parameters()).device

    def set_device(self, device):
        self.to(device)
        self.device = device

    def forward(self, floats: tp.List[float]):
        p = next(self.embedder.parameters())
        self.device = p.device
        x = torch.tensor([float(v) for v in floats]).to(self.device).clamp(self.min_val, self.max_val)
        x = ((x - self.min_val) / (self.max_val - self.min_val)).to(p.dtype)
        emb = self.embedder(x).unsqueeze(1)
        return [emb, torch.ones(emb.shape[0], 1).to(self.device)]


class IntConditioner(Conditioner):
    def __init__(self, output_dim: int, min_val: int = 0, max_val: int = 512):
        super().__init__(output_dim, output_dim)
        self.min_val, self.max_val = min_val, max_val
        self.int_embedder = nn.Embedding(max_val - min_val + 1, output_dim).requires_grad_(True)
        self.device = next(self.int_embedder.parameters()).device

    def set_device(self, device):
        self.to(device)
        self.device = device

    def forward(self, ints: tp.List[int]):
        self.device = next(self.int_embedder.parameters()).device
        idx = torch.tensor(ints).to(self.device).clamp(self.min_val, self.max_val)
        emb = self.int_embedder(idx).unsqueeze(1)
        return [emb, torch.ones(emb.shape[0], 1).to(self.device)]


class T5Conditioner(Conditioner):
    T5_MODEL_DIMS = {"t5-small": 512, "t5-base": 768, "t5-large": 1024, "t5-3b": 1024, "t5-11b": 1024,
                     "google/flan-t5-small": 512, "google/flan-t5-base": 768, "google/flan-t5-large": 1024,
                     "google/flan-t5-xl": 2048, "google/flan-t5-xxl": 4096}

    def __init__(self, output_dim: int, t5_model_name: str = "t5-base", max_length: int = 128,
                 enable_grad: bool = False, project_out: bool = False, native: bool = False):
        """native=True: the encoder runs on the native kernels (models/t5.py), inference only.  The HF model is still
        loaded (and cast to fp16) exactly as with native=False; its weights are handed to the native encoder by
        set_device, and the HF module itself stays on the CPU.  proj_out and the mask multiply run inside the native
        encode."""
        assert t5_model_name in self.T5_MODEL_DIMS, f"Unknown T5 model name: {t5_model_name}"
        if native and enable_grad:
            raise NotImplementedError("T5Conditioner: native=True is inference only (enable_grad=True is refused)")
        if native and max_length > 512:
            raise NotImplementedError(f"T5Conditioner: the native encoder takes max_length <= 512, not {max_length}")
        super().__init__(self.T5_MODEL_DIMS[t5_model_name], output_dim, project_out=project_out)
        from transformers import AutoTokenizer, T5EncoderModel
        self.max_length, self.enable_grad, self.device = max_length, enable_grad, "cpu"
        self.native = native
        prev = logging.root.manager.disable
        logging.disable(logging.ERROR)
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                self.tokenizer = AutoTokenizer.from_pretrained(t5_model_name)
                model = T5EncoderModel.from_pretrained(t5_model_name).train(enable_grad).requires_grad_(enable_grad)
                model = model.to(torch.float16)
        finally:
            logging.disable(prev)
        if enable_grad:
            self.model = model
        else:
            self.__dict__["model"] = model     # frozen: kept out of the state dict like the reference
        if native:
            from .t5 import T5Encoder
            self.__dict__["native_encoder"] = T5Encoder.from_config(model.config, operand_dtype="fp16")

    def set_device(self, device):
        self.to(device)
        if self.native:
            self._load_native(device)
        else:
            self.model.to(device)
        self.device = device

    def _load_native(self, device):
        """Loads the HF module's (fp16) weights into the native encoder on `device` (once per device), and proj_out."""
        from .._native import NativeError
        enc = self.__dict__["native_encoder"]
        device = torch.device(device)
        if device.type != "cuda":
            raise NativeError("T5Conditioner(native=True) runs on a CUDA device only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if enc.device != device:
            enc.load_state_dict(self.model.state_dict(), device=device)
        if isinstance(self.proj_out, nn.Linear):   # its current parameters (a state dict may have been loaded since)
            enc.set_proj_out(self.proj_out.weight, self.proj_out.bias)

    def forward(self, texts: tp.List[str]):
        enc = self.tokenizer(texts, truncation=True, max_length=self.max_length, padding="max_length",
                             return_tensors="pt")
        ids = enc["input_ids"].to(self.device)
        mask = enc["attention_mask"].to(self.device).to(torch.bool)
        if self.native:
            self._load_native(self.device)
            with torch.no_grad():
                return self.__dict__["native_encoder"](ids, mask), mask
        self.model.eval()
        with torch.set_grad_enabled(self.enable_grad):
            emb = self.model(input_ids=ids, attention_mask=mask)["last_hidden_state"]
        emb = self.proj_out(emb.float()) * mask.unsqueeze(-1).float()
        return emb, mask


def _clap_text_branch(clap_ckpt_path: str) -> tp.Dict[str, torch.Tensor]:
    """The ``text_branch.*`` entries of a CLAP checkpoint, prefix removed, read as laion_clap's
    ``clap_module.factory.load_state_dict`` reads it: ``torch.load``, the ``"state_dict"`` entry if there is one, and
    a leading ``module.`` stripped from every key."""
    ckpt = torch.load(clap_ckpt_path, map_location="cpu", weights_only=False)
    sd = ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt
    if next(iter(sd.items()))[0].startswith("module"):
        sd = {k[7:]: v for k, v in sd.items()}
    pre = "text_branch."
    return {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}


class CLAPTextConditioner(Conditioner):
    """CLAP text features (the reference's ``use_text_features=True`` path): hidden state ``feature_layer_ix`` of
    CLAP's RoBERTa text branch at every one of the 77 token positions, then ``proj_out``, with the tokenizer's
    attention mask.  Padded positions keep their features, as in the reference.  The encoder runs on the native
    kernels (models/roberta.py) with fp16 operands, inference only; the text branch's weights stay out of the state
    dict, only ``proj_out`` is in it.

    The text branch is roberta-base (every laion_clap checkpoint); its depth, vocabulary, FF width and position table
    are read from the checkpoint's shapes.  ``audio_model_type`` and ``enable_fusion`` only shape CLAP's audio branch,
    which the reference deletes, so they are accepted and ignored.  Refused: ``use_text_features=False`` (the pooled
    embedding goes through laion_clap's own ``text_projection`` head) and ``finetune=True``."""

    MAX_LENGTH = 77   # laion_clap's tokenizer: padding="max_length", truncation=True, max_length=77

    def __init__(self, output_dim: int, clap_ckpt_path: str, use_text_features=False, feature_layer_ix: int = -1,
                 audio_model_type="HTSAT-base", enable_fusion=True, project_out: bool = False, finetune: bool = False):
        if not use_text_features:
            raise NotImplementedError("CLAPTextConditioner: use_text_features=False (the pooled CLAP text embedding) "
                                      "goes through laion_clap's text_projection head, which this build does not run")
        if finetune:
            raise NotImplementedError("CLAPTextConditioner: the native text encoder is inference only "
                                      "(finetune=True is refused)")
        super().__init__(768, output_dim, project_out=project_out)
        from transformers import RobertaTokenizer
        from .roberta import RobertaEncoder
        self.use_text_features, self.feature_layer_ix, self.finetune = use_text_features, feature_layer_ix, finetune
        self.device = "cpu"
        prev = logging.root.manager.disable
        logging.disable(logging.ERROR)
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                self.tokenizer = RobertaTokenizer.from_pretrained("roberta-base")
        finally:
            logging.disable(prev)
        sd = _clap_text_branch(clap_ckpt_path)
        if not sd:
            raise ValueError(f"{clap_ckpt_path} holds no text_branch.* weights")
        D = sd["embeddings.word_embeddings.weight"].shape[1]
        if D != self.dim:
            raise NotImplementedError(f"CLAPTextConditioner: the text branch is {D} wide; CLAP's RoBERTa is 768")
        cfg = dict(vocab_size=sd["embeddings.word_embeddings.weight"].shape[0], hidden_size=D,
                   num_hidden_layers=1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layer.")),
                   num_attention_heads=D // 64, intermediate_size=sd["encoder.layer.0.intermediate.dense.weight"].shape[0],
                   max_position_embeddings=sd["embeddings.position_embeddings.weight"].shape[0],
                   type_vocab_size=sd["embeddings.token_type_embeddings.weight"].shape[0], pad_token_id=1,
                   layer_norm_eps=1e-5, hidden_act="gelu")
        self.__dict__["text_branch_state"] = sd       # frozen: kept out of the state dict like the reference
        self.__dict__["native_encoder"] = RobertaEncoder.from_config(cfg, feature_layer_ix=feature_layer_ix)

    def set_device(self, device):
        self.to(device)
        self._load_native(device)
        self.device = device

    def _load_native(self, device):
        """Loads the text branch into the native encoder on `device` (once per device), and proj_out."""
        from .._native import NativeError
        enc = self.__dict__["native_encoder"]
        device = torch.device(device)
        if device.type != "cuda":
            raise NativeError("CLAPTextConditioner runs on a CUDA device only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if enc.device != device:
            enc.load_state_dict(self.__dict__["text_branch_state"], device=device)
        if isinstance(self.proj_out, nn.Linear):   # its current parameters (a state dict may have been loaded since)
            enc.set_proj_out(self.proj_out.weight, self.proj_out.bias)

    def forward(self, texts: tp.List[str]):
        # the reference tokenizes a single prompt together with "" (laion_clap's tokenizer squeezes a batch of one)
        batch = [texts[0], ""] if len(texts) == 1 else list(texts)
        enc = self.tokenizer(batch, padding="max_length", truncation=True, max_length=self.MAX_LENGTH,
                             return_tensors="pt")
        ids = enc["input_ids"][:len(texts)].to(self.device)
        mask = enc["attention_mask"][:len(texts)].to(self.device)
        self._load_native(self.device)
        with torch.no_grad():
            return [self.__dict__["native_encoder"](ids, mask), mask]


class MultiConditioner(nn.Module):
    """Applies one conditioner per key of the per-item metadata dicts."""

    def __init__(self, conditioners: tp.Dict[str, Conditioner], default_keys: tp.Dict[str, str] = {}):
        super().__init__()
        self.conditioners = nn.ModuleDict(conditioners)
        self.default_keys = default_keys

    def set_device(self, device):
        for m in self.conditioners.values():
            m.set_device(device)

    def forward(self, batch_metadata: tp.List[tp.Dict[str, tp.Any]]):
        out = {}
        for key, cond in self.conditioners.items():
            ck, inputs = key, []
            for item in batch_metadata:
                if ck not in item:
                    if ck in self.default_keys:
                        ck = self.default_keys[ck]
                    else:
                        raise ValueError(f"Conditioner key {ck} not found in batch metadata")
                v = item[ck]
                inputs.append(v[0] if isinstance(v, (list, tuple)) and len(v) == 1 else v)
            out[key] = cond(inputs)
        return out


_TYPES = {"t5": T5Conditioner, "clap_text": CLAPTextConditioner, "number": NumberConditioner, "int": IntConditioner}


def create_multi_conditioner_from_conditioning_config(config: tp.Dict[str, tp.Any]) -> MultiConditioner:
    conditioners = {}
    for info in config["configs"]:
        kind = info["type"]
        if kind not in _TYPES:
            raise NotImplementedError(f"conditioner type '{kind}' is outside this build's scope "
                                      f"(available: {sorted(_TYPES)})")
        conditioners[info["id"]] = _TYPES[kind](**{"output_dim": config["cond_dim"], **info["config"]})
    return MultiConditioner(conditioners, default_keys=config.get("default_keys", {}))
