"""Model package of the H100-native drop-in: only the factory functions are re-exported here."""
from . import factory as _factory

create_model_from_config = _factory.create_model_from_config
create_model_from_config_path = _factory.create_model_from_config_path

__all__ = ("create_model_from_config", "create_model_from_config_path")
