"""pyro_b200 -- native CUDA numerics behind Pyro's two hot paths, for the H100.

The Trace_ELBO SVI step and the NUTS/HMC leapfrog of pyro-ppl/pyro 1.9.1, re-built on
hand-written sm_90a CUDA kernels behind a C ABI (include/pyro_b200.h).  The Python here is the
host-side mirror of the reference's interface for those paths (same names, arguments and error
behaviour: ``sample/param/plate``, ``poutine``, ``distributions``, ``infer.SVI/Trace_ELBO/MCMC/NUTS``,
``optim.ClippedAdam``), so model and guide code written for Pyro runs unchanged with
``import pyro_b200 as pyro``.  See DESIGN.md for the path, INTEGRATION.md for the binding a
Pyro maintainer would add.
"""
from . import distributions, poutine  # noqa: F401
from .params import clear_param_store, get_param_store  # noqa: F401
from .primitives import deterministic, factor, param, plate, sample  # noqa: F401
from .util import set_rng_seed  # noqa: F401
from . import infer, optim  # noqa: F401,E402

__version__ = "0.1.0"
