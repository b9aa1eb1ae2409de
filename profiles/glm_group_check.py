"""GPU check of multilevel regression on GlmPotential (b2_glm_potential): a varying intercept by group,
``y ~ Bernoulli(logits = X @ w + b + alpha[g])`` or ``Poisson(rate = exp(X @ w + b + alpha[g]))`` with
``alpha ~ Normal(0, s_a)[G]``, ``s_a ~ HalfNormal(1)``:
  * device time of one potential evaluation (U and dU/dz for all chains) at N = 1e5 and 1e6, D = 16, G = 48, C = 64:
    GlmPotential with the group effect, TracePotential of the same model, and (Poisson) the plain GlmPotential of a
    real [N, 64] X, whose contraction has the same width without the group columns (timed as in glm_nuts_check.py:
    CUDA events around graph replays, L2 flushed between replays, the potentials alternating);
  * the group kernel's own device time (torch.profiler, a separate pass) and its algorithmic HBM bytes (X, y and
    the 4-byte group index; W and the partials are negligible) over that time, as a share of the H100 SXM's 3.35 TB/s;
  * NUTS chain-leapfrogs per second on the multilevel logistic model (N = 1e4, D = 8, G = 20, 8 chains),
    GlmPotential and TracePotential runs alternating.
The card's name, power limit and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_group_check.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from glm_nuts_check import timer  # noqa: E402
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer import MCMC, NUTS  # noqa: E402
from pyro_b200.infer.mcmc import GlmPotential, TracePotential  # noqa: E402
from pyro_b200.infer.mcmc.compile import recognise  # noqa: E402

HBM_PEAK = 3.35e12


def lin(X, w, b):
    return (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b


def multilevel(kind, G):
    def model(X, g, y):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        s_a = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
        alpha = pyro.sample("alpha", dist.Normal(X.new_zeros(G), s_a.unsqueeze(-1)).to_event(1))
        alpha = alpha.squeeze(-2) if alpha.dim() > 1 else alpha
        with pyro.plate("data", X.shape[0]):
            eta = lin(X, w, b) + alpha[..., g]
            d = dist.Bernoulli(logits=eta) if kind == "Bernoulli" else dist.Poisson(torch.exp(eta))
            pyro.sample("y", d, obs=y)
    return model


def plain_poisson(X, y):
    w = pyro.sample("w", dist.Normal(X.new_zeros(X.shape[-1]), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Poisson(torch.exp(lin(X, w, b))), obs=y)


def data(kind, n, D, G, dev):
    gen = torch.Generator(device=dev).manual_seed(0)
    X = torch.randn(n, D, generator=gen, device=dev)
    g = torch.randint(0, G, (n,), generator=gen, device=dev)
    eta = X @ (torch.randn(D, generator=gen, device=dev) / D ** 0.5) * 0.5 + 0.5 * torch.randn(
        G, generator=gen, device=dev)[g]
    y = (torch.rand(n, generator=gen, device=dev) < torch.sigmoid(eta)).float() if kind == "Bernoulli" \
        else torch.poisson(torch.exp(eta), generator=gen)
    return X, g, y


def kernel_us(pot, z, reps=20):
    """Mean device time of the group kernel over `reps` eager evaluations, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    pot.value_and_grad(z)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pot.value_and_grad(z)
        torch.cuda.synchronize()
    ts = [e.device_time_total for e in prof.key_averages() if "group_tc_kernel" in e.key]
    return sum(ts) / reps if ts else float("nan")


def potential_times(dev, reps):
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    D, G, C = 16, 48, 64
    for kind in ("Bernoulli", "Poisson"):
        for n in (100_000, 1_000_000):
            X, g, y = data(kind, n, D, G, dev)
            model = multilevel(kind, G)
            grp = recognise(model, (X, g, y))
            assert isinstance(grp, GlmPotential) and grp.group_effect is not None, kind
            z = 0.1 * torch.randn(C, grp.dim, device=dev)
            trace = TracePotential(model, (X, g, y), num_chains=C)
            pots = [("GlmPotential+groups", grp, z), ("TracePotential", trace, z)]
            if kind == "Poisson":
                X64 = torch.randn(n, D + G, device=dev)
                wide = recognise(plain_poisson, (X64, y))
                assert isinstance(wide, GlmPotential) and wide.group_effect is None
                pots.append(("GlmPotential X[N,64]", wide, 0.1 * torch.randn(C, wide.dim, device=dev)))
            timers = [(name,) + timer(p, zz, flush) for name, p, zz in pots]
            Ug, Ut = timers[0][3][0], timers[1][3][0]
            du = float(((Ug - Ut).abs() / Ut.abs().clamp(min=1)).max())
            t = {name: [] for name, *_ in timers}
            for _ in range(reps):   # alternate the potentials
                for name, once, _, _ in timers:
                    t[name].append(once())
            med = {name: sorted(v)[len(v) // 2] for name, v in t.items()}
            line = "  ".join("%s %9.1f us (%s)" % (name, med[name], mode) for name, _, mode, _ in timers)
            print("%-9s N=%7d D=%d G=%d C=%d  %s  trace / groups x%.1f  max rel |dU| %.1e"
                  % (kind, n, D, G, C, line, med["TracePotential"] / med["GlmPotential+groups"], du))
            k_us = kernel_us(grp, z)
            nbytes = n * D * 4 + n * 4 + n * 4       # X, y, group index
            print("%-9s N=%7d  group kernel %.1f us (profiler)  algorithmic bytes %.1f MB  %.0f GB/s  %.1f%% of "
                  "3.35 TB/s" % (kind, n, k_us, nbytes / 1e6, nbytes / k_us / 1e3, 100 * nbytes / k_us / 1e-6 /
                                 HBM_PEAK))
            del trace, timers, pots
    del flush


def nuts_rate(compile_model, X, g, y, steps):
    kernel = NUTS(multilevel("Bernoulli", 20))
    kernel.compile_model = compile_model
    mc = MCMC(kernel, num_samples=steps, warmup_steps=steps, num_chains=8, seed=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mc.run(X, g, y)
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
    X, g, y = data("Bernoulli", 10_000, 8, 20, dev)
    steps = 20 if quick else 100
    for rnd in range(1 if quick else 2):    # alternate the two routes
        for compile_model in (True, False):
            rate, name, leaps = nuts_rate(compile_model, X, g, y, steps)
            print("NUTS multilevel logistic N=1e4 D=8 G=20 C=8 round %d: %-15s %9.0f chain-leapfrogs/s "
                  "(%d chain-leapfrogs)" % (rnd, name, rate, leaps))


if __name__ == "__main__":
    main()
