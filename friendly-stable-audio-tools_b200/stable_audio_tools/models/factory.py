"""JSON config -> module tree (interface parity with reference ``models/factory.py:4-50``)."""
import json


def create_model_from_config(model_config):
    model_type = model_config["model_type"]
    if model_type == "autoencoder":
        from .autoencoders import create_autoencoder_from_config
        return create_autoencoder_from_config(model_config)
    if model_type in ("diffusion_cond", "diffusion_cond_inpaint", "diffusion_prior"):
        from .diffusion import create_diffusion_cond_from_config
        return create_diffusion_cond_from_config(model_config)
    if model_type == "diffusion_autoencoder":
        from .autoencoders import create_diffAE_from_config
        return create_diffAE_from_config(model_config)
    raise NotImplementedError(
        f"model_type '{model_type}' is outside the H100-native hot path (supported: autoencoder, diffusion_cond, "
        "diffusion_cond_inpaint, diffusion_prior, diffusion_autoencoder)")


def create_model_from_config_path(model_config_path):
    with open(model_config_path) as f:
        return create_model_from_config(json.load(f))


def create_pretransform_from_config(pretransform_config, sample_rate):
    kind = pretransform_config["type"]
    if kind == "autoencoder":
        from .autoencoders import create_autoencoder_from_config
        from .pretransforms import AutoencoderPretransform
        # the autoencoder factory wants a top-level config carrying the sample rate
        autoencoder = create_autoencoder_from_config({"sample_rate": sample_rate, "model": pretransform_config["config"]})
        pretransform = AutoencoderPretransform(
            autoencoder, scale=pretransform_config.get("scale", 1.0),
            model_half=pretransform_config.get("model_half", False),
            iterate_batch=pretransform_config.get("iterate_batch", False),
            chunked=pretransform_config.get("chunked", False))
    elif kind == "pqmf":
        from .pretransforms import PQMFPretransform
        pretransform = PQMFPretransform(**pretransform_config["config"])
    else:
        # wavelet needs pywt; dac_pretrained and audiocraft_pretrained need the dac / audiocraft packages and their
        # downloaded checkpoints.  None of them is shipped with this package.
        raise NotImplementedError(f"pretransform '{kind}' is outside the native hot path (autoencoder and pqmf only)")
    enable_grad = pretransform_config.get("enable_grad", False)
    pretransform.enable_grad = enable_grad
    pretransform.eval().requires_grad_(enable_grad)
    return pretransform


def create_bottleneck_from_config(bottleneck_config):
    kind = bottleneck_config["type"]
    if kind == "vae":
        from .bottleneck import VAEBottleneck
        bottleneck = VAEBottleneck()
    elif kind == "tanh":
        from .bottleneck import TanhBottleneck
        bottleneck = TanhBottleneck()
    elif kind == "l2_norm":
        from .bottleneck import L2Bottleneck
        bottleneck = L2Bottleneck()
    elif kind == "wasserstein":
        from .bottleneck import WassersteinBottleneck
        bottleneck = WassersteinBottleneck(**bottleneck_config.get("config", {}))
    else:
        raise NotImplementedError(f"bottleneck '{kind}' is outside the native hot path "
                                  "(vae / tanh / l2_norm / wasserstein only)")
    if not bottleneck_config.get("requires_grad", True):
        for p in bottleneck.parameters():
            p.requires_grad = False
    return bottleneck
