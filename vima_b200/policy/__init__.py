"""Policy classes behind the reference's `vima.policy` names (reference: vima/policy/__init__.py:1-4): the VIMA policy and
its three baselines, all running on the sm_90a kernels of libvima_b200.so."""
from . import vima_flamingo_policy as _flamingo
from . import vima_gato_policy as _gato
from . import vima_gpt_policy as _gpt
from . import vima_policy as _vima

VIMAPolicy = _vima.VIMAPolicy
VIMAGatoPolicy = _gato.VIMAGatoPolicy
VIMAGPTPolicy = _gpt.VIMAGPTPolicy
VIMAFlamingoPolicy = _flamingo.VIMAFlamingoPolicy

__all__ = ["VIMAPolicy", "VIMAGatoPolicy", "VIMAFlamingoPolicy", "VIMAGPTPolicy"]
