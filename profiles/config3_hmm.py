"""BASELINE config 3 (GaussianHMM, H = 512 hidden dims, O = 4, T = 10 000, SVI on one GPU):
`SVI.step` with learnable parameters for the five parts, empty guide, Trace_ELBO, ClippedAdam
(structure of profiler/gaussianhmm.py:12-56 and pyro/contrib/timeseries/lgssm.py:72-95), plus the bare
log_prob forward / forward+backward.  The steady-state path (time-invariant parameters: covariance
recursion until convergence, then a blocked linear scan of the means) is the default; the step-by-step
recursion is timed at a shorter T for comparison.
usage: python profiles/config3_hmm.py [T] [H]"""
import json
import os
import sys
import time

import torch
from torch.distributions import constraints

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer import SVI, Trace_ELBO  # noqa: E402
from pyro_b200.optim import ClippedAdam  # noqa: E402

T = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
H = int(sys.argv[2]) if len(sys.argv) > 2 else 512
O = 4
dev = torch.device("cuda", 0)
torch.manual_seed(0)
data = torch.randn(T, O, device=dev)
F0 = 0.5 * torch.randn(H, H, device=dev) / H ** 0.5        # spectral radius ~0.5: a stable filter
H0 = torch.randn(H, O, device=dev)
t0s = (torch.randn(H, device=dev) * 0.1).exp()
o0s = (torch.randn(O, device=dev) * 0.1).exp()


def model(x, steady=True):
    F = pyro.param("trans_matrix", lambda: F0.clone())
    Hm = pyro.param("obs_matrix", lambda: H0.clone())
    tsc = pyro.param("trans_scale", lambda: t0s.clone(), constraint=constraints.positive)
    osc = pyro.param("obs_scale", lambda: o0s.clone(), constraint=constraints.positive)
    isc = pyro.param("init_scale", lambda: torch.ones(H, device=dev), constraint=constraints.positive)
    z = torch.zeros(H, device=dev)
    hmm = dist.GaussianHMM(dist.Normal(z, isc).to_event(1), F, dist.Normal(z, tsc).to_event(1), Hm,
                           dist.Normal(torch.zeros(O, device=dev), osc).to_event(1), duration=x.shape[0],
                           steady_state=steady)
    pyro.sample("obs", hmm, obs=x)


def guide(x, steady=True):
    pass


def sync_time(fn, reps):
    fn()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / reps, out


pyro.clear_param_store()
svi = SVI(model, guide, ClippedAdam({"lr": 1e-3}), Trace_ELBO())
dt, loss = sync_time(lambda: svi.step(data), 5)
print(json.dumps({"config": "GaussianHMM SVI step", "H": H, "O": O, "T": T, "path": "steady-state scan",
                  "ms_per_step": round(dt * 1e3, 2), "steps_per_sec": round(1 / dt, 2), "loss": round(float(loss), 2),
                  "mem_GB": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2)}))
Ts = min(T, 1000)
pyro.clear_param_store()
svi2 = SVI(model, guide, ClippedAdam({"lr": 1e-3}), Trace_ELBO())
dt2, loss2 = sync_time(lambda: svi2.step(data[:Ts], False), 1)
print(json.dumps({"config": "GaussianHMM SVI step", "H": H, "O": O, "T": Ts, "path": "step-by-step recursion",
                  "ms_per_step": round(dt2 * 1e3, 2), "ms_per_step_scaled_to_T": round(dt2 * 1e3 * T / Ts, 1),
                  "loss": round(float(loss2), 2)}))
