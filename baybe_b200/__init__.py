"""baybe_b200 -- H100-native (sm_90a) GP-posterior + acquisition scoring engine that drops in
behind BayBE's Surrogate / AcquisitionFunction / Recommender surfaces for purely discrete
search spaces.  See DESIGN.md; the C ABI is declared in include/baybe_b200.h."""

__version__ = "0.1.0"

from baybe_b200 import engine  # noqa: F401  (registers the torch.library ops)
from baybe_b200.engine import AcqConfig, DeviceGP, sobol_normal_samples  # noqa: F401
