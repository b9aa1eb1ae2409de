"""GPU check of GlmPotential past 128 columns, where the group effect is gathered per row and its gradient summed over
each group's rows (the rows sorted by group):
  * parity of U and dU/dz against fp64 for each model below (max |dU| / max(1, |U|), max |dgrad| / max |grad|);
  * radon shape (N = 919, D = 2, G = 85, S = 1, uneven county sizes, linear regression), C = 8 and 64: microseconds
    per value_and_grad, GlmPotential against TracePotential;
  * N = 1e6, D = 16, C = 64, logistic regression: the plain model, G = 1 000 with S = 1 and G = 10 000 with S = 3,
    which shows what the group term costs over the X pass;
  * the two models on either side of the route boundary at the same N: D = 16, G = 37, S = 2 (127 columns, one-hot)
    and D = 16, G = 38, S = 2 (130 columns, gathered);
  * the same at N = 1e6 for linear regression, whose plain D = 16 model runs the same X-split tensor-core pipeline as
    the gathered kernel (the plain logistic model at D = 16 runs the fp32 SIMT kernel instead);
  * where the time of each gathered evaluation goes: device time per kernel (torch.profiler, eager calls).
Times are CUDA events around graph replays with L2 flushed, median of `reps`, the models alternating.  The card's
name, power limit and SM clock are printed with the numbers.
Usage: python profiles/glm_many_groups_check.py [--quick]"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(1, HERE)
import torch  # noqa: E402

from glm_nuts_check import timer  # noqa: E402
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer.mcmc import GlmPotential, TracePotential  # noqa: E402
from pyro_b200.infer.mcmc.compile import recognise  # noqa: E402


def chains(t):
    return t.squeeze(-2) if t.dim() > 1 else t


def multilevel(kind, G, S):
    """w, b, a non-centred varying intercept and S centred varying slopes on columns 1 .. S of X (HalfNormal
    scales); G = 0: the plain regression."""
    def model(X, g, y):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        eta = (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b
        if G:
            s = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
            e = pyro.sample("eta_a", dist.Normal(X.new_zeros(G), 1.0).to_event(1))
            eta = eta + chains(s.unsqueeze(-1) * e)[..., g]
            for k in range(1, S + 1):
                sk = pyro.sample("s_%d" % k, dist.HalfNormal(X.new_full((), 0.5)))
                bk = chains(pyro.sample("beta_%d" % k, dist.Normal(X.new_zeros(G), sk.unsqueeze(-1)).to_event(1)))
                eta = eta + bk[..., g] * X[:, k]
        sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5))) if kind == "Normal" else None
        with pyro.plate("data", X.shape[0]):
            if kind == "Normal":
                pyro.sample("y", dist.Normal(eta, sigma), obs=y)
            else:
                pyro.sample("y", dist.Bernoulli(logits=eta), obs=y)
    return model


def data(kind, n, D, G, dev, seed, uneven=False):
    gen = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=gen)
    if uneven:
        probs = torch.rand(max(G, 1), generator=gen) ** 3 + 0.01
        g = torch.multinomial(probs, n, replacement=True, generator=gen)
    else:
        g = torch.randint(0, max(G, 1), (n,), generator=gen)
    g = g.sort().values
    eta = X @ (torch.randn(D, generator=gen) / D ** 0.5) + 0.5 * torch.randn(max(G, 1), generator=gen)[g]
    y = eta + 0.6 * torch.randn(n, generator=gen) if kind == "Normal" else (torch.rand(n, generator=gen)
                                                                             < torch.sigmoid(eta)).float()
    return X.to(dev), g.to(dev), y.to(dev)


def parity(pot, model, args, z):
    """max |U - U64| / max(1, |U64|) and max |grad - grad64| / max |grad64| against TracePotential in fp64"""
    U, G = pot.value_and_grad(z)
    tp = TracePotential(model, tuple(a.double() if a.is_floating_point() else a for a in args),
                        num_chains=z.shape[0])
    zd = z.double()
    Ur, Gr = tp.value_and_grad(zd)
    return (float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1)).max()),
            float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max())))


def kernel_times(pot, z, reps=5):
    """[(kernel name, mean device us per evaluation)] of eager evaluations"""
    from torch.profiler import ProfilerActivity, profile
    pot.value_and_grad(z)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pot.value_and_grad(z)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            out[e.name] = out.get(e.name, 0.0) + e.device_time / reps
    return sorted(out.items(), key=lambda kv: -kv[1])


def main():
    dev = torch.device("cuda")
    quick = "--quick" in sys.argv
    reps = 5 if quick else 21
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    # radon shape
    model = multilevel("Normal", 85, 1)
    X, g, y = data("Normal", 919, 2, 85, dev, 1, uneven=True)
    glm = recognise(model, (X, g, y))
    assert isinstance(glm, GlmPotential) and glm.group_effect.sorted == 1
    for C in (8, 64):
        z = 0.3 * torch.randn(C, glm.dim, device=dev)
        eu, eg = parity(glm, model, (X, g, y), z)
        tg, _, _ = timer(glm, z, flush)
        tt, mt, _ = timer(TracePotential(model, (X, g, y), num_chains=C), z, flush)
        a, b = [], []
        for _ in range(reps):                 # alternating
            a.append(tg())
            b.append(tt())
        a.sort()
        b.sort()
        print("radon N=919 D=2 G=85 S=1 C=%d: GlmPotential %.1f us, TracePotential %.1f us (%s); "
              "vs fp64 U %.1e grad %.1e" % (C, a[reps // 2], b[reps // 2], mt, eu, eg))
    # N = 1e6: the plain model against the gathered ones; the two sides of the route boundary
    n = 200_000 if quick else 1_000_000
    cases = [("Bernoulli", "plain", 16, 0, 0), ("Bernoulli", "G=1000 S=1", 16, 1000, 1),
             ("Bernoulli", "G=10000 S=3", 16, 10000, 3), ("Bernoulli", "G=37 S=2 (127 cols, one-hot)", 16, 37, 2),
             ("Bernoulli", "G=38 S=2 (130 cols, gathered)", 16, 38, 2), ("Normal", "plain", 16, 0, 0),
             ("Normal", "G=1000 S=1", 16, 1000, 1), ("Normal", "G=10000 S=3", 16, 10000, 3)]
    timers = []
    for kind, label, D, G, S in cases:
        label = ("logistic " if kind == "Bernoulli" else "linear   ") + label
        model = multilevel(kind, G, S)
        X, g, y = data(kind, n, D, G, dev, 2)
        pot = recognise(model, (X, g, y))
        assert isinstance(pot, GlmPotential), label
        z = 0.1 * torch.randn(64, pot.dim, device=dev)
        eu, eg = parity(pot, model, (X, g, y), z)
        t, mode, _ = timer(pot, z, flush)
        # the potential and its data stay alive: the captured graph reads their device memory
        timers.append((label, t, mode, eu, eg, (pot, X, g, y), z))
    res = {label: [] for label, *_ in timers}
    for _ in range(reps):
        for label, t, *_ in timers:
            res[label].append(t())
    for label, _, mode, eu, eg, _, _ in timers:
        v = sorted(res[label])[reps // 2]
        print("N=%d D=16 C=64 %-40s %8.1f us (%s); vs fp64 U %.1e grad %.1e" % (n, label, v, mode, eu, eg))
    for label, _, _, _, _, (pot, *_), z in timers:
        print("kernels of %s:" % label)
        for name, us in kernel_times(pot, z):
            print("    %8.1f us  %s" % (us, name[:110]))


if __name__ == "__main__":
    main()
