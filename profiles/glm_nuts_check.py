"""GPU check of the regression potential for HMC / NUTS (GlmPotential, b2_glm_potential) against the traced
potential (TracePotential) on the same models, in alternating runs:
  * device time of one potential evaluation (U and dU/dz for all chains) at N = 1e6, D = 32 for C = 8, 64, 128
    chains, logistic regression with an intercept and softmax regression with K = 10 (CUDA events around
    graph replays, L2 flushed between replays; a potential that cannot be captured is timed eagerly and
    reported as such);
  * NUTS chain-leapfrogs per second on tests/models.py::logistic_model at N = 1e6 (8 chains, tree depth
    capped at 6 so the traced run stays short).
The card's name, power limit and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_nuts_check.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import models  # noqa: E402
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.infer import MCMC, NUTS  # noqa: E402
from pyro_b200.infer.mcmc import GlmPotential, TracePotential  # noqa: E402
from pyro_b200.infer.mcmc.compile import recognise  # noqa: E402


def softmax_model(X, y, K):
    D = X.shape[-1]
    W = pyro.sample("W", dist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
    b = pyro.sample("b", dist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1))
    with pyro.plate("data", X.shape[0]):
        Wm = W.squeeze(-3) if W.dim() > 2 else W
        pyro.sample("y", dist.Categorical(logits=X @ Wm.mT + b), obs=y)


def data(n, D, K, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    X = torch.randn(n, D, generator=g, device=dev)
    if K is None:
        w = torch.randn(D, generator=g, device=dev) / D ** 0.5
        return X, (torch.rand(n, generator=g, device=dev) < torch.sigmoid(X @ w + 0.3)).float()
    W = torch.randn(K, D, generator=g, device=dev) / D ** 0.5
    return X, torch.multinomial(torch.softmax(X @ W.mT, -1), 1, generator=g).squeeze(-1)


def timer(pot, z, flush):
    """Returns (a function timing one evaluation in microseconds, "graph" | "eager (...)", the outputs)."""
    zbuf = z.clone()
    out = pot.value_and_grad(zbuf)
    torch.cuda.synchronize()
    mode = "graph"
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            pot.value_and_grad(zbuf)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = pot.value_and_grad(zbuf)
        run = g.replay
    except Exception as e:  # noqa: BLE001 -- the traced potential need not be capturable
        torch.cuda.synchronize()
        mode = "eager (%s)" % type(e).__name__
        run = lambda: pot.value_and_grad(zbuf)  # noqa: E731

    def once():
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3
    for _ in range(3):
        once()
    return once, mode, out


def potential_times(dev, reps):
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    n, D = 1_000_000, 32
    for label, K in (("logistic", None), ("softmax K=10", 10)):
        X, y = data(n, D, K, dev)
        model, args = (models.logistic_model, (X, y)) if K is None else (softmax_model, (X, y, K))
        glm = recognise(model, args)
        assert isinstance(glm, GlmPotential), label
        for C in (8, 64, 128):
            z = 0.1 * torch.randn(C, glm.dim, device=dev)
            trace = TracePotential(model, args, num_chains=C)
            t_glm, m_glm, (Ug, Gg) = timer(glm, z, flush)
            t_tr, m_tr, (Ut, Gt) = timer(trace, z, flush)
            du = float(((Ug - Ut).abs() / Ut.abs().clamp(min=1)).max())
            a, b = [], []
            for _ in range(reps):   # alternate the two potentials
                a.append(t_glm())
                b.append(t_tr())
            a.sort()
            b.sort()
            print("%-13s C=%3d  GlmPotential %8.1f us (%s)  TracePotential %9.1f us (%s)  x%.1f  "
                  "[min %.1f / %.1f]  max rel |dU| %.1e"
                  % (label, C, a[len(a) // 2], m_glm, b[len(b) // 2], m_tr, b[len(b) // 2] / a[len(a) // 2],
                     a[0], b[0], du))
            del trace
    del flush


def nuts_rate(dev, compile_model, X, y, steps):
    kernel = NUTS(models.logistic_model, max_tree_depth=6)
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
            rate, name, leaps = nuts_rate(dev, compile_model, X, y, steps)
            print("NUTS logistic_model N=1e6 C=8 round %d: %-15s %9.0f chain-leapfrogs/s (%d chain-leapfrogs)"
                  % (rnd, name, rate, leaps))


if __name__ == "__main__":
    main()
