"""MCMC: vectorised-chain HMC / NUTS kernels, warm-up adaptation, diagnostics."""
from .api import MCMC  # noqa: F401
from .nuts import HMC, NUTS  # noqa: F401
from .potential import (GlmPotential, HierNormalPotential, LogisticPotential, NativePotential,  # noqa: F401
                        TracePotential)
