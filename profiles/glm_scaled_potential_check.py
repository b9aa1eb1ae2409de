"""GPU check of the regression potential with a latent weight scale (GlmPotential, b2_glm_potential) on
horseshoe logistic regression, ``tau ~ HalfCauchy(1)``, ``lam ~ HalfCauchy(1)[D]``, ``w ~ Normal(0, tau * lam)``,
``b ~ Normal(0, 10)``, ``y ~ Bernoulli(logits = X @ w + b)``:
  * device time of one potential evaluation (U and dU/dz for all chains) at N = 1e6, D = 32 for C = 8, 64, 128
    chains: the latent-scale GlmPotential, the constant-scale GlmPotential of the same likelihood
    (tests/models.py::logistic_model) and TracePotential of the horseshoe model, alternating (timed as in
    glm_nuts_check.py: CUDA events around graph replays, L2 flushed between replays);
  * NUTS chain-leapfrogs per second on the horseshoe model at N = 1e6 (8 chains, tree depth capped at 6 so the
    traced run stays short), GlmPotential and TracePotential runs alternating.
The card's name, power limit and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_scaled_potential_check.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from glm_nuts_check import data, models, timer  # noqa: E402
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer import MCMC, NUTS  # noqa: E402
from pyro_b200.infer.mcmc import GlmPotential, TracePotential  # noqa: E402
from pyro_b200.infer.mcmc.compile import recognise  # noqa: E402


def horseshoe_model(X, y):
    D = X.shape[-1]
    tau = pyro.sample("tau", dist.HalfCauchy(X.new_ones(())))
    lam = pyro.sample("lam", dist.HalfCauchy(X.new_ones(D)).to_event(1))
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), tau.unsqueeze(-1) * lam).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
    with pyro.plate("data", X.shape[0]):
        logits = (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b
        pyro.sample("y", dist.Bernoulli(logits=logits), obs=y)


def potential_times(dev, reps):
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    X, y = data(1_000_000, 32, None, dev)
    scaled = recognise(horseshoe_model, (X, y))
    const = recognise(models.logistic_model, (X, y))
    assert isinstance(scaled, GlmPotential) and scaled.weight_scale is not None
    assert isinstance(const, GlmPotential) and const.weight_scale is None
    for C in (8, 64, 128):
        z = 0.1 * torch.randn(C, scaled.dim, device=dev)
        zc = z[:, scaled.sites["w"][0].start:scaled.sites["b"][0].stop].contiguous()   # [w, b]
        trace = TracePotential(horseshoe_model, (X, y), num_chains=C)
        t_s, m_s, (Us, _) = timer(scaled, z, flush)
        t_c, m_c, _ = timer(const, zc, flush)
        t_t, m_t, (Ut, _) = timer(trace, z, flush)
        du = float(((Us - Ut).abs() / Ut.abs().clamp(min=1)).max())
        a, b, c = [], [], []
        for _ in range(reps):   # alternate the three potentials
            a.append(t_s())
            b.append(t_c())
            c.append(t_t())
        for v in (a, b, c):
            v.sort()
        med = [v[len(v) // 2] for v in (a, b, c)]
        print("horseshoe C=%3d  latent scale %8.1f us (%s)  constant scale %8.1f us (%s)  TracePotential %9.1f us "
              "(%s)  latent - constant %+.1f us  trace / latent x%.1f  [min %.1f / %.1f / %.1f]  max rel |dU| %.1e"
              % (C, med[0], m_s, med[1], m_c, med[2], m_t, med[0] - med[1], med[2] / med[0], a[0], b[0], c[0], du))
        del trace
    del flush


def nuts_rate(compile_model, X, y, steps):
    kernel = NUTS(horseshoe_model, max_tree_depth=6)
    kernel.compile_model = compile_model
    mc = MCMC(kernel, num_samples=steps, warmup_steps=steps, num_chains=8, seed=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mc.run(X, y)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    leaps = kernel.leapfrog_count()
    return leaps / dt, type(kernel.potential).__name__, leaps


def main():
    quick = "--quick" in sys.argv
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    potential_times(dev, 5 if quick else 20)
    X, y = data(1_000_000, 32, None, dev)
    steps = 5 if quick else 15
    for rnd in range(1 if quick else 2):    # alternate the two routes
        for compile_model in (True, False):
            rate, name, leaps = nuts_rate(compile_model, X, y, steps)
            print("NUTS horseshoe N=1e6 C=8 round %d: %-15s %9.0f chain-leapfrogs/s (%d chain-leapfrogs)"
                  % (rnd, name, rate, leaps))


if __name__ == "__main__":
    main()
