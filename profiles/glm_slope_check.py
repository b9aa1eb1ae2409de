"""GPU check of multilevel regression with varying slopes on GlmPotential (b2_glm_potential, S slopes):
``y ~ Bernoulli(logits = X @ w + b + alpha[g] + beta[g] * X[:, 0])``, ``alpha ~ Normal(0, s_a)[G]``,
``beta ~ Normal(0, s_b)[G]``, latent HalfNormal scales:
  * device time of one potential evaluation (U and dU/dz for all chains) at N = 1e5 and 1e6, D = 16, G = 32, S = 1
    (80 columns), C = 64: the slope potential, TracePotential of the same model, and the intercept-only group
    potential at G = 64, whose contraction has the same width (CUDA events around graph replays, L2 flushed between
    replays, the potentials alternating, as in glm_nuts_check.py);
  * NUTS chain-leapfrogs per second on a radon-shaped model (N = 919, D = 2, G = 50, the slope on the floor column,
    both blocks non-centred, latent sigma, 8 chains), GlmPotential and TracePotential runs alternating.
``--dump PATH`` instead writes U and dU/dz of fixed intercept-only (S = 0) group potentials to PATH, so that two
builds can be compared bitwise; ``--root DIR`` imports pyro_b200 from DIR.
The card's name, power limit and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_slope_check.py [--quick] [--dump PATH] [--root DIR]"""
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
if "--root" in sys.argv:
    sys.path.insert(0, os.path.abspath(sys.argv[sys.argv.index("--root") + 1]))
sys.path.insert(1, HERE)
import torch  # noqa: E402

from glm_nuts_check import timer  # noqa: E402
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer import MCMC, NUTS  # noqa: E402
from pyro_b200.infer.mcmc import GlmPotential, TracePotential  # noqa: E402
from pyro_b200.infer.mcmc.compile import recognise  # noqa: E402


def lin(X, w, b):
    return (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b


def chains(t):
    return t.squeeze(-2) if t.dim() > 1 else t


def multilevel(kind, G, slope, noncentred=False):
    """A varying intercept, and with ``slope`` a varying slope on column 0 of X."""
    def model(X, g, y):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5))) if kind == "Normal" else None
        eta = lin(X, w, b)
        for name in ("a", "b") if slope else ("a",):
            s = pyro.sample("s_" + name, dist.HalfNormal(X.new_full((), 1.0)))
            if noncentred:
                e = pyro.sample("eta_" + name, dist.Normal(X.new_zeros(G), 1.0).to_event(1))
                t = chains(s.unsqueeze(-1) * e)
            else:
                t = chains(pyro.sample("t_" + name, dist.Normal(X.new_zeros(G), s.unsqueeze(-1)).to_event(1)))
            eta = eta + (t[..., g] if name == "a" else t[..., g] * X[:, 1 if kind == "Normal" else 0])
        with pyro.plate("data", X.shape[0]):
            if kind == "Bernoulli":
                d = dist.Bernoulli(logits=eta)
            elif kind == "Poisson":
                d = dist.Poisson(torch.exp(eta))
            else:
                d = dist.Normal(eta, sigma)
            pyro.sample("y", d, obs=y)
    return model


def data(kind, n, D, G, dev, seed=0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn(n, D, generator=gen, device=dev)
    g = torch.randint(0, G, (n,), generator=gen, device=dev)
    eta = X @ (torch.randn(D, generator=gen, device=dev) / D ** 0.5) * 0.5 + 0.5 * torch.randn(
        G, generator=gen, device=dev)[g] + 0.3 * torch.randn(G, generator=gen, device=dev)[g] * X[:, 0]
    if kind == "Bernoulli":
        y = (torch.rand(n, generator=gen, device=dev) < torch.sigmoid(eta)).float()
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta.clamp(max=4.0)), generator=gen)
    else:
        y = eta + 0.6 * torch.randn(n, generator=gen, device=dev)
    return X, g, y


def dump(path, dev):
    """U and dU/dz of S = 0 group potentials at a few shapes, every kind the seeds reach, C = 1, 64 and 65."""
    out = {}
    for kind in ("Bernoulli", "Poisson", "Normal"):
        for n, D, G in ((70_001, 16, 48), (1_000_000, 16, 48), (10_003, 3, 28)):
            X, g, y = data(kind, n, D, G, dev, seed=n + D)
            pot = recognise(multilevel(kind, G, slope=False, noncentred=kind == "Normal"), (X, g, y))
            assert isinstance(pot, GlmPotential) and pot.group_effect is not None, kind
            for C in (1, 64, 65):
                gen = torch.Generator(device=dev).manual_seed(C)
                z = 0.1 * torch.randn(C, pot.dim, generator=gen, device=dev)
                U, Gr = pot.value_and_grad(z)
                out["%s n=%d D=%d G=%d C=%d" % (kind, n, D, G, C)] = (U.cpu(), Gr.cpu())
    torch.save(out, path)
    print("dumped %d S = 0 potential evaluations to %s" % (len(out), path))


def potential_times(dev, reps):
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    D, G, C = 16, 32, 64
    for n in (100_000, 1_000_000):
        X, g, y = data("Bernoulli", n, D, G, dev)
        model = multilevel("Bernoulli", G, slope=True)
        slope = recognise(model, (X, g, y))
        assert isinstance(slope, GlmPotential) and slope.group_effect.S == 1
        z = 0.1 * torch.randn(C, slope.dim, device=dev)
        trace = TracePotential(model, (X, g, y), num_chains=C)
        g64 = torch.randint(0, 2 * G, (n,), device=dev)
        wide = recognise(multilevel("Bernoulli", 2 * G, slope=False), (X, g64, y))
        assert isinstance(wide, GlmPotential) and wide.group_effect.S == 0
        pots = [("slope S=1 G=32", slope, z), ("TracePotential", trace, z),
                ("intercept G=64", wide, 0.1 * torch.randn(C, wide.dim, device=dev))]
        timers = [(name,) + timer(p, zz, flush) for name, p, zz in pots]
        Ug, Ut = timers[0][3][0], timers[1][3][0]
        du = float(((Ug - Ut).abs() / Ut.abs().clamp(min=1)).max())
        t = {name: [] for name, *_ in timers}
        for _ in range(reps):   # alternate the potentials
            for name, once, _, _ in timers:
                t[name].append(once())
        med = {name: sorted(v)[len(v) // 2] for name, v in t.items()}
        line = "  ".join("%s %9.1f us (%s)" % (name, med[name], mode) for name, _, mode, _ in timers)
        print("Bernoulli N=%7d D=%d G=%d S=1 C=%d  %s  trace / slope x%.1f  slope / intercept-64 %.2f  "
              "max rel |dU| vs trace %.1e" % (n, D, G, C, line, med["TracePotential"] / med["slope S=1 G=32"],
                                               med["slope S=1 G=32"] / med["intercept G=64"], du))
        del trace, timers, pots
    del flush


def nuts_rate(compile_model, X, g, y, steps):
    kernel = NUTS(multilevel("Normal", 50, slope=True, noncentred=True))
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
    dev = torch.device("cuda")
    if "--dump" in sys.argv:
        dump(sys.argv[sys.argv.index("--dump") + 1], dev)
        return
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    potential_times(dev, 5 if quick else 20)
    X, g, y = data("Normal", 919, 2, 50, dev, seed=22)
    X[:, 1] = (X[:, 1] > 0.5).float()   # the floor column
    steps = 20 if quick else 100
    for rnd in range(1 if quick else 2):    # alternate the two routes
        for compile_model in (True, False):
            rate, name, leaps = nuts_rate(compile_model, X, g, y, steps)
            print("NUTS radon-shaped N=919 D=2 G=50 S=1 C=8 round %d: %-15s %9.0f chain-leapfrogs/s "
                  "(%d chain-leapfrogs)" % (rnd, name, rate, leaps))


if __name__ == "__main__":
    main()
