"""DiffusionTransformer: the reference's module interface over the native DiT kernels.

Interface parity with reference ``models/dit.py:14-364`` (constructor kwargs, submodule
and parameter names, ``forward`` signature and CFG semantics); the arithmetic runs in
``libsatb200.so`` (``satb_dit_*`` in include/satb200.h):

* step-invariant conditioning work (``to_cond_embed``, ``to_global_embed``, every layer's
  cross-attention k/v; dit.py:149-154, transformer.py:425) is hoisted into
  ``satb_dit_prepare_cond`` and cached while the same conditioning tensors are passed;
* one ``forward`` = one ``satb_dit_forward`` call: batched CFG rows (cond first, uncond
  second, dit.py:270-320), 24 blocks, CFG combine / rescale (dit.py:338-347);
* rows whose context is all-zero (the uncond half without a negative prompt) skip
  cross-attention: the branch is bias-free, so its output is exactly 0 (SURVEY.md H5);
* ``conformer=True`` models run the conformer branch of every block natively
  (``satb_dit_set_conformer``, csrc/conformer.cu), with 16-bit GEMM operands in every ``operand_dtype``;
* ``ff_kwargs`` (any ``mult``, ``no_bias``, ``glu=False``, ``use_conv`` with an odd ``conv_kernel_size``) select the
  native feed-forward variant (``satb_dit_set_feedforward``); its token convolutions run as k-tap GEMMs over each
  item, with 16-bit operands in every ``operand_dtype``;
* ``ff_out_dtype="fp8"`` (with ``operand_dtype="fp8"``) runs every block's FF-out GEMM on e4m3 operands, its
  activations with one scale per (token, 128 inner columns) written by FF-in's epilogue (``satb_dit_set_ff_out_fp8``);
* ``rotary_pos_emb=False``, ``use_sinusoidal_emb`` and ``use_abs_pos_emb`` select the native positional options
  (``satb_dit_set_positions``); the embedding is added to every row, prepended ones included, in project_in's epilogue;
* any ``io_channels`` and ``input_concat_dim`` (an inpainting DiT's latent + 1 mask channel, PQMF sub-bands, raw audio):
  the library pads project_in's K to a multiple of 8 and project_out's N to a multiple of 32 with zero weights;
* ``shard_tokens(devices)`` splits every call's tokens over several ranks (``satb_dit_group_*``): each rank holds a full
  copy of the weights and a contiguous range of every item's tokens, and gathers every rank's self-attention K / V once
  per layer, so one prompt can use several GPUs; with ``cuda_graph`` the whole sharded call is replayed from one
  multi-device CUDA graph the library captures and owns (``satb_dit_group_graph_forward``);
* ``shard_tokens([[...], [...]])`` also splits every CFG call by guidance half (``satb_dit_group_create_cfg``): row 0
  runs the conditional rows and row 1 the unconditional ones, each token-sharded over its own devices, and the halves
  meet once per call, in the combine.

There is no eager / CPU fallback: tensors must live on a CUDA device.
"""
import ctypes
import typing as tp

import torch
from torch import nn

from .. import _native
from .blocks import FourierFeatures
from .transformer import SUPPORTED_HEAD_DIMS, ContinuousTransformer, check_head_dim

# operand_dtype -> SatbDitConfig.operand_dtype.  "fp16" (default) and "bf16": 16-bit operands for every tensor-core
# contraction.  "fp8": e4m3 operands with power-of-two row scales for the self-attention QKV, cross-attention q and
# feed-forward input GEMMs (the three Linear layers fed by a LayerNorm), fp16 everywhere else - the GEMMs of the
# conformer branch included; a precision choice with its own tolerance (DESIGN.md section 5), not a second path to the
# fp16 result.
OPERAND_DTYPES = {"fp16": 0, "bf16": 1, "fp8": 2}
# attention_dtype: None (default) keeps the 16-bit self-attention of the operand mode.  "fp8": self-attention on e4m3
# q, k, v and probabilities with power-of-two scales (satb_dit_set_attention_fp8), head dim 64 only, with any
# operand_dtype; cross-attention stays 16-bit.  A precision choice with its own tolerance (DESIGN.md section 5).
ATTENTION_DTYPES = (None, "fp8")
# ff_out_dtype: None (default) keeps the feed-forward output GEMM (ff.ff.2) at fp16 operands in the "fp8" operand mode.
# "fp8" (operand_dtype="fp8" only; satb_dit_set_ff_out_fp8): its activations are e4m3 with one power-of-two scale per
# (token, 128 inner columns), written by FF-in's epilogue, and its weight e4m3 with one scale per output row.  Linear
# feed-forwards whose inner width (padded to 64) is a multiple of 128.  A precision choice with its own tolerance
# (DESIGN.md section 5).
FF_OUT_DTYPES = (None, "fp8")


class DiffusionTransformer(nn.Module):
    def __init__(self,
                 io_channels: int = 32,
                 patch_size: int = 1,
                 embed_dim: int = 768,
                 cond_token_dim: int = 0,
                 project_cond_tokens: bool = True,
                 global_cond_dim: int = 0,
                 project_global_cond: bool = True,
                 input_concat_dim: int = 0,
                 prepend_cond_dim: int = 0,
                 depth: int = 12,
                 num_heads: int = 8,
                 transformer_type: str = "x-transformers",
                 global_cond_type: str = "prepend",
                 operand_dtype: str = "fp16",
                 attention_dtype=None,
                 ff_out_dtype=None,
                 **kwargs):
        super().__init__()
        if transformer_type != "continuous_transformer":
            raise NotImplementedError("only transformer_type='continuous_transformer' is on the native hot path "
                                      "(the reference's x-transformers branch needs an un-vendored dependency)")
        if prepend_cond_dim > 0 and global_cond_type != "prepend":
            # (the reference itself mis-handles this pair: prepend_length is only set in "prepend" mode, dit.py:185-197,
            # so its output keeps the prepended positions - L + n_prepend columns, a shape no sampler can consume)
            raise NotImplementedError("prepend_cond with global_cond_type='adaLN' is not on the native hot path")
        if num_heads < 1 or embed_dim % num_heads != 0:
            raise NotImplementedError(f"embed_dim {embed_dim} is not a multiple of num_heads {num_heads}: the native "
                                      f"path needs a head dim of {', '.join(map(str, SUPPORTED_HEAD_DIMS))}")
        check_head_dim(embed_dim // num_heads, bool(kwargs.get("attn_kwargs", {}).get("qk_norm", False)))
        if patch_size < 1:
            raise ValueError("patch_size must be >= 1")
        # any width runs natively (project_in's K and project_out's N are zero-padded inside the library); these are
        # the only widths it refuses
        if io_channels < 1:
            raise ValueError(f"io_channels must be >= 1, got {io_channels}")
        if input_concat_dim < 0:
            raise ValueError(f"input_concat_dim must be >= 0, got {input_concat_dim}")
        # the native LayerNorm keeps a row in registers, and the conditioning MLPs stage their input rows in shared
        # memory four floats at a time (satb_dit_create refuses the same)
        if embed_dim > 2048:
            raise NotImplementedError(f"embed_dim {embed_dim} is above 2048, the widest the native path runs")
        for name, dim in (("global_cond_dim", global_cond_dim), ("prepend_cond_dim", prepend_cond_dim)):
            if dim < 0 or dim % 4 != 0 or dim > 6400:
                raise NotImplementedError(f"{name} {dim}: the native path needs a multiple of 4, at most 6400")
        if global_cond_type not in ("prepend", "adaLN"):
            raise ValueError(f"unknown global_cond_type {global_cond_type}")
        if operand_dtype not in OPERAND_DTYPES:
            raise ValueError(f"operand_dtype must be one of {', '.join(OPERAND_DTYPES)}, got {operand_dtype!r}")
        if attention_dtype not in ATTENTION_DTYPES:
            raise ValueError(f"attention_dtype must be None or 'fp8', got {attention_dtype!r}")
        if attention_dtype == "fp8" and embed_dim // num_heads != 64:
            raise NotImplementedError(f"attention_dtype='fp8' needs head dim 64 (got {embed_dim // num_heads})")
        if ff_out_dtype not in FF_OUT_DTYPES:
            raise ValueError(f"ff_out_dtype must be None or 'fp8', got {ff_out_dtype!r}")
        if ff_out_dtype == "fp8" and operand_dtype != "fp8":
            raise ValueError(f"ff_out_dtype='fp8' extends operand_dtype='fp8' (got operand_dtype={operand_dtype!r})")
        self.patch_size = patch_size
        self.cond_token_dim = cond_token_dim
        self.input_concat_dim = input_concat_dim
        self.prepend_cond_dim = prepend_cond_dim
        self.io_channels = io_channels
        self.embed_dim = embed_dim
        self.depth = depth
        self.num_heads = num_heads
        self.global_cond_dim = global_cond_dim
        self.project_cond_tokens = project_cond_tokens
        self.project_global_cond = project_global_cond
        self.transformer_type = transformer_type
        self.global_cond_type = global_cond_type
        self.operand_dtype = operand_dtype
        self.attention_dtype = attention_dtype
        self.ff_out_dtype = ff_out_dtype
        self.qk_norm = bool(kwargs.get("attn_kwargs", {}).get("qk_norm", False))
        # conformer=True (ContinuousTransformer kwarg): every block adds the conformer branch (satb_dit_set_conformer)
        self.conformer = bool(kwargs.get("conformer", False))

        feat_dim = 256
        self.timestep_features = FourierFeatures(1, feat_dim)
        self.to_timestep_embed = nn.Sequential(nn.Linear(feat_dim, embed_dim, bias=True), nn.SiLU(),
                                               nn.Linear(embed_dim, embed_dim, bias=True))
        cond_embed_dim = 0
        if cond_token_dim > 0:
            cond_embed_dim = embed_dim if project_cond_tokens else cond_token_dim
            self.to_cond_embed = nn.Sequential(nn.Linear(cond_token_dim, cond_embed_dim, bias=False), nn.SiLU(),
                                               nn.Linear(cond_embed_dim, cond_embed_dim, bias=False))
        if global_cond_dim > 0:
            glob_embed_dim = embed_dim if project_global_cond else global_cond_dim
            self.to_global_embed = nn.Sequential(nn.Linear(global_cond_dim, glob_embed_dim, bias=False), nn.SiLU(),
                                                 nn.Linear(glob_embed_dim, glob_embed_dim, bias=False))
        if prepend_cond_dim > 0:                                   # dit.py:75-81
            self.to_prepend_embed = nn.Sequential(nn.Linear(prepend_cond_dim, embed_dim, bias=False), nn.SiLU(),
                                                  nn.Linear(embed_dim, embed_dim, bias=False))
        dim_in = io_channels + input_concat_dim                    # dit.py:38
        self.transformer = ContinuousTransformer(
            dim=embed_dim, depth=depth, dim_heads=embed_dim // num_heads, dim_in=dim_in * patch_size,
            dim_out=io_channels * patch_size, cross_attend=cond_token_dim > 0, cond_token_dim=cond_embed_dim,
            global_cond_dim=embed_dim if global_cond_type == "adaLN" else None, **kwargs)
        self.preprocess_conv = nn.Conv1d(dim_in, dim_in, 1, bias=False)
        nn.init.zeros_(self.preprocess_conv.weight)
        self.postprocess_conv = nn.Conv1d(io_channels, io_channels, 1, bias=False)
        nn.init.zeros_(self.postprocess_conv.weight)
        # ff_kwargs (ContinuousTransformer -> TransformerBlock -> FeedForward): the native feed-forward variant, handed
        # to satb_dit_set_feedforward only when it differs from the default SwiGLU (mult 4, biased, Linear)
        ff = self.transformer.layers[0].ff if depth > 0 else None
        self.ff_spec = ff.native_spec() if ff is not None else (4 * embed_dim, 1, 0, 1)
        if ff_out_dtype == "fp8":
            inner, _, conv_k, _ = self.ff_spec
            if conv_k > 0:
                raise NotImplementedError("ff_out_dtype='fp8' is not supported with use_conv feed-forwards (their FF-out "
                                          "is a token convolution)")
            padded = -(-inner // 64) * 64     # the native inner width (zero-padded to a multiple of 64)
            if padded % 128 != 0:
                raise NotImplementedError(f"ff_out_dtype='fp8' needs a feed-forward inner width that is a multiple of "
                                          f"128, the FP8 GEMM's k-block (got {inner}, padded to {padded})")
        # positions (ContinuousTransformer kwargs): the satb_dit_set_positions arguments (rotary, pos_type, abs_max_len),
        # handed over only when they differ from the default (rotary, no embedding)
        tr = self.transformer
        self.pos_spec = (int(tr.rotary_pos_emb is not None), {None: 0, "sinusoidal": 1, "abs": 2}[tr.pos_type],
                         tr.pos_emb.max_seq_len if tr.pos_type == "abs" else 0)

        # native state (not part of the state dict)
        self.__dict__["_h"] = None
        self.__dict__["_weights_dirty"] = True
        self.__dict__["_cond_key"] = None
        self.__dict__["_keepalive"] = None
        self.__dict__["_neg_masked"] = None
        self.__dict__["_graph"] = None
        self.__dict__["_shard"] = None           # shard_tokens state: devices, rank handles, group, streams
        self.__dict__["_shard_dirty"] = True
        # cuda_graph = True: one denoiser call = ONE CUDA-graph launch (the ~280 kernel launches of a forward are
        # captured once per (shape, guidance, conditioning) and replayed).  The returned tensor is then a static
        # buffer that the NEXT call overwrites - fine for the samplers, which consume it at once; off by default.
        # A token-sharded model (shard_tokens) replays every rank's launches, the K/V gathers and the copies of the
        # ranks' slices in and out from one multi-device graph the library captures and invalidates itself.
        self.cuda_graph = False
        # nn.Module.load_state_dict on a PARENT (ConditionedDiffusionModelWrapper, DiTWrapper, copy_state_dict(model, sd))
        # recurses through _load_from_state_dict and never calls a child's load_state_dict override; the post hook
        # below is run for every module of the recursion, so the native copy is refreshed whichever way the
        # parameters were (re)loaded.
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.refresh_native_weights())

    # ------------------------------------------------------------------ native plumbing
    def _apply(self, fn, *a, **k):
        self.__dict__["_weights_dirty"] = True
        self.__dict__["_shard_dirty"] = True
        self._drop_shard_graph()
        return super()._apply(fn, *a, **k)

    def refresh_native_weights(self):
        """Call after mutating parameters in place (``load_state_dict`` / ``.to()`` do it for you)."""
        self.__dict__["_weights_dirty"] = True
        self.__dict__["_shard_dirty"] = True
        self._drop_shard_graph()

    def __del__(self):
        try:
            self._drop_shards()
        except Exception:
            pass
        h = self.__dict__.get("_h")
        if h is not None:
            try:
                _native.lib().satb_dit_destroy(h)
            except Exception:
                pass

    def native_config(self):
        """The SatbDitConfig this module creates its native handle with.

        patch_size p > 1 (dit.py:206-207,221-222): tokens are groups of p positions with features (c p).  The native
        model simply sees io_channels * p channels and L / p positions; forward() does the two rearranges, and the 1x1
        pre/post convs (which act per position on the un-patched signal) are handed over as kron(W, I_p) so that the
        native fold into project_in/out stays generic."""
        return _native.SatbDitConfig(
            io_channels=self.io_channels * self.patch_size, embed_dim=self.embed_dim, depth=self.depth, num_heads=self.num_heads,
            cond_token_dim=self.cond_token_dim, global_cond_dim=self.global_cond_dim,
            project_cond_tokens=int(self.project_cond_tokens), project_global_cond=int(self.project_global_cond),
            global_cond_type=1 if self.global_cond_type == "adaLN" else 0, patch_size=1,
            operand_dtype=OPERAND_DTYPES[self.operand_dtype], qk_norm=int(self.qk_norm),
            input_concat_dim=self.input_concat_dim * self.patch_size, prepend_cond_dim=self.prepend_cond_dim)

    def _new_handle(self):
        """A native handle of this model's config and options, with no weights yet."""
        lib = _native.lib()
        cfg = self.native_config()
        h = ctypes.c_void_p()
        _native.check(lib.satb_dit_create(ctypes.byref(cfg), ctypes.byref(h)))
        options = []
        if self.conformer:
            options.append(lambda: lib.satb_dit_set_conformer(h, 1))
        if self.attention_dtype == "fp8":
            options.append(lambda: lib.satb_dit_set_attention_fp8(h, 1))
        if self.ff_spec != (4 * self.embed_dim, 1, 0, 1):
            options.append(lambda: lib.satb_dit_set_feedforward(h, *self.ff_spec))
        if self.ff_out_dtype == "fp8":                # after the feed-forward variant, whose inner width it checks
            options.append(lambda: lib.satb_dit_set_ff_out_fp8(h, 1))
        if self.pos_spec != (1, 0, 0):
            options.append(lambda: lib.satb_dit_set_positions(h, *self.pos_spec))
        for set_option in options:
            rc = set_option()
            if rc != 0:
                msg = lib.satb_last_error()
                lib.satb_dit_destroy(h)
                raise _native.NativeError(f"satb200 error {rc}: {msg.decode() if msg else '?'}")
        return h

    def _upload_weights(self, h, device, copy_to=None):
        """Loads every parameter into handle h and finalizes it, on device's current stream.  copy_to: the device the
        handle lives on, when it is not the parameters' own (a rank of shard_tokens)."""
        lib = _native.lib()
        st = _native.stream_ptr(device)
        with torch.no_grad():
            weights = list(self.state_dict().items())
            if self.transformer.pos_type == "sinusoidal":
                # a non-persistent buffer, so not in the state dict: handed over as the module holds it (the native
                # table uses these very values rather than recomputing the powers)
                weights.append(("transformer.pos_emb.inv_freq", self.transformer.pos_emb.inv_freq))
            for name, t in weights:
                if name.endswith("rotary_pos_emb.scale") or t is None:
                    continue
                if not t.is_cuda:
                    raise _native.NativeError(
                        f"parameter {name} is on {t.device}: move the model to a CUDA device "
                        "(this package has no CPU path)")
                src = t.detach().to(torch.float32).contiguous()
                if copy_to is not None:
                    src = src.to(copy_to)
                if self.patch_size > 1 and name in ("preprocess_conv.weight", "postprocess_conv.weight"):
                    eye = torch.eye(self.patch_size, device=src.device, dtype=src.dtype)
                    src = torch.kron(src[:, :, 0], eye).unsqueeze(-1).contiguous()
                _native.check(lib.satb_dit_load_weight(h, name.encode(), _native.ptr(src), src.numel(), st))
            _native.check(lib.satb_dit_finalize(h, st))

    def _handle(self, device):
        if self.__dict__["_h"] is None:
            self.__dict__["_h"] = self._new_handle()
        if self.__dict__["_weights_dirty"]:
            self._upload_weights(self.__dict__["_h"], device)
            self.__dict__["_weights_dirty"] = False
            self.__dict__["_cond_key"] = None
            self.__dict__["_graph"] = None
        return self.__dict__["_h"]

    @staticmethod
    def _tkey(t):
        return None if t is None else (t.data_ptr(), t._version, tuple(t.shape), str(t.dtype))

    def _prepare(self, h, cross, neg, glob, use_cfg, device, B, prepend=None):
        key = (self._tkey(cross), self._tkey(neg), self._tkey(glob), bool(use_cfg), B, self._tkey(prepend))
        if key == self.__dict__["_cond_key"]:
            return
        self._prepare_native(h, cross, neg, glob, use_cfg, device, B, prepend)
        self.__dict__["_cond_key"] = key
        self.__dict__["_keepalive"] = (cross, neg, glob, prepend)   # keep the keyed storage alive

    def _prepare_native(self, h, cross, neg, glob, use_cfg, device, B, prepend, copy_to=None):
        f32 = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()
        if copy_to is not None:
            f32 = lambda t: None if t is None else t.detach().to(device=copy_to, dtype=torch.float32).contiguous()
        c, n, g, pc = f32(cross), f32(neg), f32(glob), f32(prepend)
        for name, tt in (("cross_attn_cond", c), ("negative_cross_attn_cond", n), ("global_embed", g),
                         ("prepend_cond", pc)):
            if tt is not None and tt.shape[0] != B:
                raise ValueError(f"{name} batch {tt.shape[0]} != input batch {B}")
        Mctx = c.shape[1] if c is not None else 0
        if pc is not None and pc.shape[2] != self.prepend_cond_dim:
            raise ValueError(f"prepend_cond width {pc.shape[2]} != prepend_cond_dim {self.prepend_cond_dim}")
        _native.check(_native.lib().satb_dit_set_prepend_cond(h, _native.ptr(pc), B, pc.shape[1] if pc is not None else 0,
                                                              _native.stream_ptr(device)))
        _native.check(_native.lib().satb_dit_prepare_cond(h, _native.ptr(c), _native.ptr(n), _native.ptr(g), B, Mctx,
                                                          1 if use_cfg else 0, _native.stream_ptr(device)))

    # ------------------------------------------------------------------ token sharding
    def shard_tokens(self, devices):
        """Run every later call token-sharded over ``devices`` (context parallel); ``None`` returns to one device.

        Rank r runs on ``devices[r]``; a device may repeat (several ranks on one GPU run the same sharded schedule, which
        is how it is tested on a single GPU).  The parameters stay on the home device ``devices[0]``, where ``forward``
        takes its inputs and returns its output; each rank gets its own native handle with a copy of the weights,
        refreshed whenever the parameters change.  ``forward`` splits each item's tokens by the library's plan
        (``satb_dit_group_plan``: the prepended tokens on rank 0, boundaries on multiples of 128 tokens), runs all ranks
        with one K/V gather per layer, and concatenates the ranks' outputs on the home device.  Samplers and the VAE run
        unchanged on the home device.

        Refused with NotImplementedError: conformer blocks and ``use_conv`` feed-forwards (their token convolutions
        would need the neighbouring ranks' tokens), ``attention_dtype="fp8"`` (its V channel scales span all of an
        item's tokens) and, at call time, ``return_info``.  Ranks on distinct GPUs need peer-to-peer access between them.

        Two rows, ``[[a, b], [c, d]]``, split each classifier-free-guidance call by half as well (CFG split): row 0 runs
        the conditional rows and row 1 the unconditional rows, each token-sharded over its own devices by the same plan,
        and row 0 combines the two halves' outputs, the only exchange between the rows.  The rows have equal lengths of
        1 to 8 devices; the home device is ``devices[0][0]``.  A call without CFG (``cfg_scale == 1``, or neither
        cross-attention nor prepend conditioning) runs on row 0 only, as ``shard_tokens(row 0)`` would.  The refusals
        above apply only when a row has more than one device: ``[[a], [b]]`` runs every model option.

        With ``cuda_graph`` off, each call enqueues every rank's launches eagerly.  With it on (the multistep SDE samplers
        and the v-diffusion ``sample`` switch it on), each call is one launch of a multi-device CUDA graph
        (``satb_dit_group_graph_forward``): it copies the ranks' slices of the input in, runs the sharded forward and
        copies the slices of the output back, and returns a static buffer on the home device that the next call
        overwrites.  The library captures it on the first call and again whenever the shape, the guidance scalars, the
        conditioning, the weights or a workspace change, and orders it against eager sharded calls itself."""
        cfg_split = False
        if devices is not None:
            devices = list(devices)
            nested = [isinstance(dv, (list, tuple)) for dv in devices]
            if any(nested):
                if not all(nested):
                    raise ValueError("shard_tokens: give a flat list of devices or two rows of devices, not a mix")
                if len(devices) != 2:
                    raise ValueError(f"shard_tokens: a CFG split takes two rows of devices (conditional, unconditional), "
                                     f"got {len(devices)}")
                rows = [list(row) for row in devices]
                if any(isinstance(dv, (list, tuple)) for row in rows for dv in row):
                    raise ValueError("shard_tokens: each row is a list of devices (no deeper nesting)")
                if len(rows[0]) != len(rows[1]):
                    raise ValueError(f"shard_tokens: the two rows need the same length, got {len(rows[0])} and "
                                     f"{len(rows[1])}")
                if not 1 <= len(rows[0]) <= 8:
                    raise ValueError(f"shard_tokens: 1 to 8 devices per row, got {len(rows[0])}")
                cfg_split = True
                world = len(rows[0])
                devices = rows[0] + rows[1]
            else:
                world = len(devices)
            if world > 1 or not cfg_split:      # a CFG row of one device holds every token
                if self.conformer:
                    raise NotImplementedError("shard_tokens: conformer blocks are not supported (their depthwise "
                                              "convolution needs the neighbouring ranks' tokens)")
                if self.ff_spec[2] > 0:
                    raise NotImplementedError("shard_tokens: use_conv feed-forwards are not supported (their token "
                                              "convolution needs the neighbouring ranks' tokens)")
                if self.attention_dtype == "fp8":
                    raise NotImplementedError("shard_tokens: attention_dtype='fp8' is not supported (its V channel "
                                              "scales span all of an item's tokens)")
            devices = [torch.device(dv) for dv in devices]
            if not 1 <= world <= 8:
                raise ValueError(f"shard_tokens: 1 to 8 devices, got {len(devices)}")
            for dv in devices:
                if dv.type != "cuda":
                    raise _native.NativeError(f"shard_tokens: {dv} is not a CUDA device (this package has no CPU path)")
            devices = [dv if dv.index is not None else torch.device("cuda", torch.cuda.current_device()) for dv in devices]
        self._drop_shards()
        if devices is not None:
            self.__dict__["_shard"] = dict(devices=devices, world=world, cfg_split=cfg_split, handles=None, group=None,
                                           streams=None, cond_key=None, keepalive=None, graph_io=None)
            self.__dict__["_shard_dirty"] = True
        return self

    def _drop_shards(self):
        sh = self.__dict__.get("_shard")
        self.__dict__["_shard"] = None
        if sh is None:
            return
        lib = _native.lib()
        if sh["group"] is not None:
            lib.satb_dit_group_destroy(sh["group"])
        for h in sh["handles"] or []:
            lib.satb_dit_destroy(h)

    def _drop_shard_graph(self):
        """Drops the sharded model's captured graph and its static buffers; the next graph call captures again."""
        sh = self.__dict__.get("_shard")
        if sh is None:
            return
        if sh["group"] is not None:
            _native.check(_native.lib().satb_dit_group_graph_reset(sh["group"]))
        sh["graph_io"] = None

    def shard_graph_stats(self):
        """(captures, replays, kernel launches of the current graph) of the sharded model's group, or None when the
        model is not sharded or its group does not exist yet."""
        sh = self.__dict__.get("_shard")
        if sh is None or sh["group"] is None:
            return None
        c, r, n = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_ulonglong()
        _native.check(_native.lib().satb_dit_group_graph_stats(sh["group"], ctypes.byref(c), ctypes.byref(r),
                                                               ctypes.byref(n)))
        return c.value, r.value, n.value

    def _shard_group(self, sh):
        lib = _native.lib()
        devs = sh["devices"]
        if sh["group"] is not None and not self.__dict__["_shard_dirty"]:
            return sh["group"]
        if sh["group"] is not None:
            lib.satb_dit_group_destroy(sh["group"])
            sh["group"] = None
            sh["graph_io"] = None
        if sh["handles"] is None:
            sh["handles"] = []
            for _ in devs:
                sh["handles"].append(self._new_handle())
        for h, dv in zip(sh["handles"], devs):
            with torch.cuda.device(dv):
                self._upload_weights(h, dv, copy_to=dv)
        g = ctypes.c_void_p()
        handles = (ctypes.c_void_p * len(devs))(*[h.value for h in sh["handles"]])
        ids = (ctypes.c_int * len(devs))(*[dv.index for dv in devs])
        create = lib.satb_dit_group_create_cfg if sh["cfg_split"] else lib.satb_dit_group_create
        _native.check(create(handles, ids, sh["world"], ctypes.byref(g)))
        sh["group"] = g
        if sh["streams"] is None:
            sh["streams"] = [torch.cuda.Stream(device=dv) for dv in devs]
        sh["cond_key"] = None
        self.__dict__["_shard_dirty"] = False
        return g

    def _sharded_prepare(self, sh, x, cross, neg, glob, prepend, use_cfg):
        """The group, with every rank handle's conditioning prepared for this call."""
        devs = sh["devices"]
        home = devs[0]
        if x.device != home:
            raise ValueError(f"the token-sharded model's home device is {home}, but x is on {x.device}")
        g = self._shard_group(sh)
        B = x.shape[0]
        key = (self._tkey(cross), self._tkey(neg), self._tkey(glob), bool(use_cfg), B, self._tkey(prepend))
        if key != sh["cond_key"]:
            for h, dv in zip(sh["handles"], devs):
                with torch.cuda.device(dv):
                    self._prepare_native(h, cross, neg, glob, use_cfg, dv, B, prepend, copy_to=dv)
            sh["cond_key"] = key
            sh["keepalive"] = (cross, neg, glob, prepend)
        return g

    def _sharded_forward(self, sh, x, t, cross, neg, glob, prepend, use_cfg, cfg_scale, scale_phi):
        lib = _native.lib()
        devs = sh["devices"]
        home = devs[0]
        g = self._sharded_prepare(sh, x, cross, neg, glob, prepend, use_cfg)
        B, _, L = x.shape
        P = 0 if self.global_cond_type == "adaLN" else 1 + (prepend.shape[1] if prepend is not None else 0)
        W = sh["world"]
        tb = _native.group_plan(W, P, L)
        # the ranks this call runs: both rows of a CFG split under CFG, else row 0; row 0 writes the output
        run = devs if sh["cfg_split"] and use_cfg else devs[:W]
        xin = x.detach().to(torch.float32)
        tin = t.detach().to(torch.float32).contiguous()
        xs, ts, outs = [], [], []
        for r, dv in enumerate(run):
            lo, hi = max(tb[r % W] - P, 0), tb[r % W + 1] - P  # this rank's latent tokens
            with torch.cuda.device(dv):
                xs.append(xin[:, :, lo:hi].to(dv).contiguous())
                ts.append(tin.to(dv))
                if r < W:
                    outs.append(torch.empty(B, self.io_channels * self.patch_size, hi - lo, device=dv,
                                            dtype=torch.float32))
                sh["streams"][r].wait_stream(torch.cuda.current_stream(dv))
        ptrs = lambda ts_: (ctypes.c_void_p * len(devs))(*[q.data_ptr() for q in ts_])
        streams = (ctypes.c_void_p * len(devs))(*[s_.cuda_stream for s_ in sh["streams"]])
        _native.check(lib.satb_dit_group_forward(g, ptrs(xs), ptrs(ts), ptrs(outs), B, L, float(cfg_scale),
                                                 float(scale_phi), streams))
        for r, dv in enumerate(run):
            torch.cuda.current_stream(dv).wait_stream(sh["streams"][r])
        return torch.cat([o.to(home) for o in outs], dim=2)

    def _sharded_graph_forward(self, sh, x, t, cross, neg, glob, prepend, use_cfg, cfg_scale, scale_phi):
        """The sharded call as one launch of the group's multi-device CUDA graph (satb_dit_group_graph_forward).  The
        library captures it, with one eager warm-up call in front, whenever the key (static buffers, shape, guidance)
        or any rank handle's weights, conditioning or workspaces changed, and orders it against eager sharded calls.
        x, t and the output are static home-device buffers per (B, C, L); the returned tensor is overwritten by the
        next call."""
        devs = sh["devices"]
        home = devs[0]
        g = self._sharded_prepare(sh, x, cross, neg, glob, prepend, use_cfg)
        B, C, L = x.shape
        io = sh["graph_io"]
        if io is None or io["key"] != (B, C, L):
            io = dict(key=(B, C, L), x=torch.empty(B, C, L, device=home, dtype=torch.float32),
                      t=torch.empty(B, device=home, dtype=torch.float32),
                      out=torch.empty(B, self.io_channels * self.patch_size, L, device=home, dtype=torch.float32))
            sh["graph_io"] = io
        io["x"].copy_(x)
        io["t"].copy_(t)
        cur = torch.cuda.current_stream(home)
        others = {dv for dv in devs if dv != home}
        for dv in others:                     # the ranks' conditioning was prepared on their devices' current streams
            cur.wait_stream(torch.cuda.current_stream(dv))
        streams = (ctypes.c_void_p * len(devs))(*[s_.cuda_stream for s_ in sh["streams"]])
        with torch.cuda.device(home):
            _native.check(_native.lib().satb_dit_group_graph_forward(
                g, _native.ptr(io["x"]), _native.ptr(io["t"]), _native.ptr(io["out"]), B, L, float(cfg_scale),
                float(scale_phi), streams, ctypes.c_void_p(cur.cuda_stream)))
        for dv in others:                     # later work there (new conditioning) must not overtake the graph
            torch.cuda.current_stream(dv).wait_stream(cur)
        return io["out"]

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, t, cross_attn_cond=None, cross_attn_cond_mask=None, negative_cross_attn_cond=None,
                negative_cross_attn_mask=None, input_concat_cond=None, global_embed=None, prepend_cond=None,
                prepend_cond_mask=None, cfg_scale=1.0, cfg_dropout_prob=0.0, causal=False, scale_phi=0.0, mask=None,
                return_info=False, **kwargs):
        if causal:
            raise AssertionError("Causal mode is not supported for DiffusionTransformer")
        if return_info and self.__dict__["_shard"] is not None:
            raise NotImplementedError("return_info is not supported by the token-sharded forward (shard_tokens): "
                                      "call shard_tokens(None) first")
        if prepend_cond is not None and self.prepend_cond_dim == 0:
            raise ValueError("prepend_cond given to a model built with prepend_cond_dim=0")
        if (input_concat_cond is None) != (self.input_concat_dim == 0):
            raise ValueError("input_concat_cond must be given exactly when the model has input_concat_dim > 0 "
                             f"(input_concat_dim={self.input_concat_dim})")
        if self.training and cfg_dropout_prob > 0.0:
            raise NotImplementedError("training-time CFG dropout is outside the inference hot path")
        if self.transformer.pos_type == "abs":
            # AbsolutePositionalEmbedding's assertion (transformer.py:61-63) over the tokens after the prepend concat
            n_seq = x.shape[2] // self.patch_size
            if self.global_cond_type == "prepend":
                n_seq += 1 + (prepend_cond.shape[1] if prepend_cond is not None else 0)
            max_len = self.transformer.pos_emb.max_seq_len
            assert n_seq <= max_len, (f"you are passing in a sequence length of {n_seq} but your absolute positional "
                                      f"embedding has a max sequence length of {max_len}")
        if not x.is_cuda:
            raise _native.NativeError("DiffusionTransformer.forward needs CUDA tensors (no CPU fallback)")
        # masks are accepted and ignored exactly like the reference (dit.py:250-252,
        # transformer.py:787-802 never forwards them to the layers)
        if cross_attn_cond is not None and self.cond_token_dim == 0:
            cross_attn_cond = None
        use_cfg = cfg_scale != 1.0 and (cross_attn_cond is not None or prepend_cond is not None)   # dit.py:270
        if input_concat_cond is not None:
            # dit.py:163-168: nearest-neighbour resize to the latent length, channel concat in front of the 1x1
            # pre-conv (which the native finalize folds into project_in over all io + concat channels); the CFG
            # halves share it (dit.py:281-284), as they share x
            if input_concat_cond.shape[2] != x.shape[2]:
                input_concat_cond = torch.nn.functional.interpolate(input_concat_cond, (x.shape[2],), mode="nearest")
            x = torch.cat([x, input_concat_cond.to(x.dtype)], dim=1)
        neg = None
        if use_cfg and negative_cross_attn_cond is not None:
            neg = negative_cross_attn_cond
            if negative_cross_attn_mask is not None:
                # masked once per (cond, mask) pair: the cache holds the raw tensors themselves (identity and
                # version are compared, never a recycled data_ptr), so a later call with another negative prompt
                # that the allocator placed at the same address cannot hit it
                prev = self.__dict__.get("_neg_masked")
                if (prev is not None and prev[0] is negative_cross_attn_cond and prev[1] is negative_cross_attn_mask
                        and prev[2] == (negative_cross_attn_cond._version, negative_cross_attn_mask._version)):
                    neg = prev[3]
                else:
                    neg = torch.where(negative_cross_attn_mask.to(torch.bool).unsqueeze(2), neg, torch.zeros_like(neg))
                    self.__dict__["_neg_masked"] = (negative_cross_attn_cond, negative_cross_attn_mask,
                                                    (negative_cross_attn_cond._version,
                                                     negative_cross_attn_mask._version), neg)
        p = self.patch_size
        if p > 1:
            if x.shape[2] % p != 0:
                raise ValueError(f"sequence length {x.shape[2]} is not a multiple of patch_size {p}")
            if use_cfg and scale_phi != 0.0:
                # the std rescale (dit.py:342-345) is over the un-patched channels: take the combined and the
                # conditional outputs from two native calls and rescale here (device tensors, torch elementwise)
                kw = dict(cross_attn_cond=cross_attn_cond, cross_attn_cond_mask=cross_attn_cond_mask,
                          negative_cross_attn_cond=negative_cross_attn_cond,
                          negative_cross_attn_mask=negative_cross_attn_mask, global_embed=global_embed,
                          prepend_cond=prepend_cond)
                if input_concat_cond is not None:                  # x already carries it: split it off again
                    kw["input_concat_cond"] = x[:, self.io_channels:]
                    x = x[:, :self.io_channels]
                cfg_out = self.forward(x, t, cfg_scale=cfg_scale, scale_phi=0.0, **kw)
                cond_out = self.forward(x, t, cfg_scale=1.0, scale_phi=0.0, **kw)
                rescaled = cfg_out * (cond_out.std(dim=1, keepdim=True) / cfg_out.std(dim=1, keepdim=True))
                out = scale_phi * rescaled + (1 - scale_phi) * cfg_out
                return (out, {"hidden_states": []}) if return_info else out
            b_, c_, l_ = x.shape
            x = x.reshape(b_, c_, l_ // p, p).transpose(2, 3).reshape(b_, c_ * p, l_ // p)   # channel = c * p + pi
        sh = self.__dict__["_shard"]
        if sh is not None:
            run = self._sharded_forward
            if self.cuda_graph and not torch.cuda.is_current_stream_capturing():
                run = self._sharded_graph_forward
            return self._unpatch(run(sh, x, t, cross_attn_cond, neg, global_embed, prepend_cond, use_cfg, cfg_scale,
                                     scale_phi)).to(x.dtype)
        # handles, workspaces and TMA descriptors live on the model's device: make it current for the native calls
        # (generate_diffusion_cond(device='cuda:1') with current device 0 must work)
        with torch.cuda.device(x.device):
            h = self._handle(x.device)
            B, C, L = x.shape
            self._prepare(h, cross_attn_cond, neg, global_embed, use_cfg, x.device, B, prepend_cond)
            xin = x.detach().to(torch.float32).contiguous()
            tin = t.detach().to(torch.float32).contiguous()
            out = torch.empty(B, self.io_channels * p, L, device=x.device, dtype=torch.float32)
            st = _native.stream_ptr(x.device)
            if return_info:
                P = 0 if self.global_cond_type == "adaLN" else 1 + (prepend_cond.shape[1] if prepend_cond is not None else 0)
                rows = (2 * B if use_cfg else B) * (L + P)
                hidden = torch.empty(rows, self.embed_dim, device=x.device, dtype=torch.float32)
                _native.check(_native.lib().satb_dit_forward_debug(h, _native.ptr(xin), _native.ptr(tin), _native.ptr(out),
                                                                   _native.ptr(hidden), B, L, float(cfg_scale),
                                                                   float(scale_phi), st))
                info = {"hidden_states": [hidden.view(-1, L + P, self.embed_dim)]}
                return self._unpatch(out).to(x.dtype), info
            if self.cuda_graph and not torch.cuda.is_current_stream_capturing():
                out = self._graph_forward(h, xin, tin, B, L, float(cfg_scale), float(scale_phi), x.device)
                return self._unpatch(out).to(x.dtype)
            self.__dict__["_graph"] = None       # an eager call may regrow workspaces the captured graph points into
            _native.check(_native.lib().satb_dit_forward(h, _native.ptr(xin), _native.ptr(tin), _native.ptr(out), B, L,
                                                         float(cfg_scale), float(scale_phi), st))
            return self._unpatch(out).to(x.dtype)

    def _graph_forward(self, h, xin, tin, B, L, cfg_scale, scale_phi, device):
        """satb_dit_forward through a captured CUDA graph (SURVEY.md 8f-1): the C entry point enqueues on the stream it
        is given and neither allocates nor synchronises once the workspace exists, so the whole forward - ~280
        launches with their programmatic-dependent-launch edges - is captured once and replayed with two small
        device copies (x, t) in front."""
        lib = _native.lib()
        key = (B, L, cfg_scale, scale_phi, self.__dict__["_cond_key"], device.index)
        g = self.__dict__["_graph"]
        if g is None or g["key"] != key:
            sx, st_ = torch.empty_like(xin), torch.empty_like(tin)
            so = torch.empty(B, self.io_channels * self.patch_size, L, device=xin.device, dtype=torch.float32)
            sx.copy_(xin)
            st_.copy_(tin)

            def run():
                _native.check(lib.satb_dit_forward(h, _native.ptr(sx), _native.ptr(st_), _native.ptr(so), B, L, cfg_scale,
                                                   scale_phi, _native.stream_ptr(device)))
            side = torch.cuda.Stream(device=device)
            side.wait_stream(torch.cuda.current_stream(device))
            with torch.cuda.stream(side):        # warm-up outside the capture: workspace, tensor maps, attributes
                run()
                run()
            torch.cuda.current_stream(device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = _native.launch_count()
            with torch.cuda.graph(graph):
                run()
            g = dict(key=key, graph=graph, x=sx, t=st_, out=so, launches=_native.launch_count() - n0)
            self.__dict__["_graph"] = g
        g["x"].copy_(xin, non_blocking=True)
        g["t"].copy_(tin, non_blocking=True)
        g["graph"].replay()
        lib.satb_add_launch_count(g["launches"])
        return g["out"]

    def _unpatch(self, out):
        p = self.patch_size
        if p == 1:
            return out
        b, cp, tt = out.shape                                     # "b (c p) t -> b c (t p)"
        return out.reshape(b, cp // p, p, tt).transpose(2, 3).reshape(b, cp // p, tt * p)
