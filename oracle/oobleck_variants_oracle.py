"""CPU restatement of the reference Oobleck VAE's other block options: ELU activations (``use_snake=False``) and
nearest-neighbour upsampling (``use_nearest_upsample=True``, decoder only), reference models/autoencoders.py:29-194.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Built on ``oobleck_oracle`` without changing it, as
``conformer_oracle`` is on ``dit_oracle``: the same weight-norm fold, the same operand rounding switch
(``oobleck_oracle.operand_rounding``) and the same synthetic-weight generator; a config without the two options gives
``oobleck_oracle``'s results.

Under operand rounding the nearest-upsample conv is computed the way the native decoder does it: the weight-normed
kernel W [cout, cin, 2s] is folded into a 3-tap kernel of the low-rate input (``nearest_fold``, summed in float64 and
rounded once to float32), which is then rounded to the operand type.  In plain fp32 the oracle follows the reference:
``F.interpolate`` then ``F.conv1d(padding='same')``.
"""
import math

import torch
import torch.nn.functional as F

from . import oobleck_oracle as oo


def elu(x):
    """nn.ELU() (alpha 1): x > 0 ? x : exp(x) - 1."""
    return F.elu(x)


def _act(x, sd, pfx, use_snake):
    return oo.snake_beta(x, sd[pfx + "alpha"], sd[pfx + "beta"]) if use_snake else elu(x)


def nearest_fold(w, s):
    """W [cout, cin, 2s] of the conv after a nearest x s upsample -> [3, s, cout, cin]: tap o + 1 (o = -1, 0, 1) of
    phase p holds sum over k with floor((p + k - s + 1) / s) = o of W[:, :, k].  Output position s m + p of
    conv_same(upsample(x)) is sum_o W'[o + 1, p] x[m + o] (x zero outside [0, L)).  Summed in float64."""
    cout, cin, k = w.shape
    assert k == 2 * s
    out = torch.zeros(3, s, cout, cin, dtype=torch.float64, device=w.device)
    wd = w.double()
    for p in range(s):
        for kk in range(k):
            o = (p + kk - s + 1) // s
            out[o + 1, p] += wd[:, :, kk]
    return out


def nearest_conv_folded(x, wf):
    """x [B, cin, L], wf [3, s, cout, cin] -> [B, cout, L * s] through the 3-tap form."""
    _, s, cout, cin = wf.shape
    wc = wf.permute(1, 2, 3, 0).reshape(s * cout, cin, 3)       # channel p * cout + co, taps o = -1, 0, 1
    y = F.conv1d(x, wc.to(x.dtype), padding=1)                   # [B, s * cout, L]
    B, _, L = y.shape
    return y.view(B, s, cout, L).permute(0, 2, 3, 1).reshape(B, cout, L * s)


def _nearest_upsample_conv(x, sd, pfx, s):
    w = oo.fold_weight_norm(sd[pfx + "weight_g"], sd[pfx + "weight_v"])
    if oo._OPERAND_DTYPE is None:
        return F.conv1d(F.interpolate(x, scale_factor=s, mode="nearest"), w, padding="same")
    wf = oo._rnd(nearest_fold(w, s).float())
    return nearest_conv_folded(oo._rnd(x), wf)


def residual_unit(x, sd, pfx, dilation, use_snake=True):
    y = _act(x, sd, pfx + "layers.0.", use_snake)
    y = oo._wn_conv(y, sd, pfx + "layers.1.", dilation=dilation, padding=(dilation * 6) // 2)
    y = _act(y, sd, pfx + "layers.2.", use_snake)
    y = oo._wn_conv(y, sd, pfx + "layers.3.")
    return x + y


def oobleck_decoder(z, sd, cfg):
    """models/autoencoders.py:156-194 with DecoderBlock :88-116, every option but antialias_activation."""
    use_snake, nearest = cfg.get("use_snake", False), cfg.get("use_nearest_upsample", False)
    c_mults = [1] + list(cfg["c_mults"])
    strides = list(cfg["strides"])
    x = oo._wn_conv(z, sd, "layers.0.", padding=3)
    li = 1
    for i in range(len(c_mults) - 1, 0, -1):
        s = strides[i - 1]
        p = f"layers.{li}."
        x = _act(x, sd, p + "layers.0.", use_snake)
        if nearest:
            x = _nearest_upsample_conv(x, sd, p + "layers.1.1.", s)
        else:
            x = oo._wn_convT(x, sd, p + "layers.1.", stride=s, padding=math.ceil(s / 2))
        for j, d in enumerate((1, 3, 9)):
            x = residual_unit(x, sd, f"{p}layers.{2 + j}.", d, use_snake)
        li += 1
    x = _act(x, sd, f"layers.{li}.", use_snake)
    x = oo._wn_conv(x, sd, f"layers.{li + 1}.", padding=3)
    if cfg.get("final_tanh", True):
        x = torch.tanh(x)
    return x


def oobleck_encoder(a, sd, cfg):
    """models/autoencoders.py:119-153 with EncoderBlock :71-85, either activation."""
    use_snake = cfg.get("use_snake", False)
    c_mults = [1] + list(cfg["c_mults"])
    strides = list(cfg["strides"])
    x = oo._wn_conv(a, sd, "layers.0.", padding=3)
    li = 1
    for i in range(len(c_mults) - 1):
        s = strides[i]
        p = f"layers.{li}."
        for j, d in enumerate((1, 3, 9)):
            x = residual_unit(x, sd, f"{p}layers.{j}.", d, use_snake)
        x = _act(x, sd, p + "layers.3.", use_snake)
        x = oo._wn_conv(x, sd, p + "layers.4.", stride=s, padding=math.ceil(s / 2))
        li += 1
    x = _act(x, sd, f"layers.{li}.", use_snake)
    return oo._wn_conv(x, sd, f"layers.{li + 1}.", padding=1)


# ---------------------------------------------------------------------------------------------------- weights
def _drop_snake(shapes):
    return {k: v for k, v in shapes.items() if not k.endswith(("alpha", "beta"))}


def decoder_param_shapes(cfg):
    """The reference OobleckDecoder's state-dict shapes for cfg's options: no alpha / beta keys with ELU; with nearest
    upsampling each block's conv is "layers.{b}.layers.1.1." (Conv1d [cout, cin, 2s], no bias)."""
    shapes = oo.decoder_param_shapes(cfg)
    if cfg.get("use_nearest_upsample", False):
        out = {}
        for k, v in shapes.items():
            pfx = next((p for p in oo.decoder_transposed_prefixes(cfg) if k.startswith(p) and k.count(".") == 4), None)
            if pfx is None:
                out[k] = v
            elif k.endswith("weight_g"):
                cin, cout, kk = shapes[pfx + "weight_v"]
                out[pfx + "1.weight_g"] = (cout, 1, 1)
                out[pfx + "1.weight_v"] = (cout, cin, kk)
        shapes = out
    return shapes if cfg.get("use_snake", False) else _drop_snake(shapes)


def encoder_param_shapes(cfg):
    shapes = oo.encoder_param_shapes(cfg)
    return shapes if cfg.get("use_snake", False) else _drop_snake(shapes)


def make_decoder_weights(cfg, seed=0):
    """oobleck_oracle's synthetic weights over decoder_param_shapes(cfg) (ConvTranspose1d fan-in for transposed
    blocks; the nearest conv counts as a Conv1d)."""
    tr = () if cfg.get("use_nearest_upsample", False) else oo.decoder_transposed_prefixes(cfg)
    return oo.make_oobleck_weights(decoder_param_shapes(cfg), seed=seed, transposed=tr)


def make_encoder_weights(cfg, seed=0):
    return oo.make_oobleck_weights(encoder_param_shapes(cfg), seed=seed)
