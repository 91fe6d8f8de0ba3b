"""H100-native drop-in for the Stable Audio denoising hot path.

Same import surface as the reference package for that path
(reference ``stable_audio_tools/__init__.py:1-2``): model construction from the
reference's JSON configs, and the pretrained-model loader.  The arithmetic lives in
``libsatb200.so`` (hand-written sm_90a CUDA behind the C ABI of ``include/satb200.h``).
"""
from .models.factory import create_model_from_config, create_model_from_config_path
from .models.pretrained import get_pretrained_model

__all__ = ["create_model_from_config", "create_model_from_config_path", "get_pretrained_model"]
