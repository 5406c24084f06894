"""regtr_b200 -- H100-native (sm_90a) implementation of the RegTR correspondence-prediction
hot path behind the reference's nn.Module API.  See DESIGN.md / INTEGRATION.md."""
from .config import Cfg, get_config, load_config  # noqa: F401

__all__ = ['Cfg', 'get_config', 'load_config', 'RegTR']


def __getattr__(name):
    if name == 'RegTR':
        from .regtr import RegTR
        return RegTR
    raise AttributeError(name)
