"""GPU check of multilevel regression under SVI past 128 columns (b2_glm_group_gather_sum, rows sorted by group):
``y ~ Bernoulli(logits = eta)`` and ``y ~ Normal(eta, sigma)`` with ``eta = X @ w + b + alpha[g] + SUM_k beta_k[g] *
X[:, c_k]`` at N = 1e6, D = 16, P = 16 and 64 particles, in four shapes:
  G = 1 000, S = 1 and G = 10 000, S = 3 (gathered); G = 37, S = 2 (127 columns, one-hot: b2_glm_group_slope_sum) and
  G = 38, S = 2 (130 columns, gathered), either side of the route boundary.
  * device time of the site's value and all its gradients: the fused call against the materialised site (cuBLAS
    ``W @ X.T``, the ``[P, N]`` gathers, products and adds, the site kernel and autograd's backward), the route
    LAZY_LINEAR = False takes.  CUDA events around CUDA-graph replays with L2 flushed before each replay; median of
    20 replays per window, the two routes alternating over 5 windows;
  * one graph-captured ``SVI.step`` (JitTrace_ELBO, ClippedAdam) of the unchanged model on the lazy route against
    ``LAZY_LINEAR = False``, in alternating runs;
  * in a separate run, the per-kernel split of the gathered call from torch.profiler (G = 10 000, S = 3, P = 64).
The card's name, power limit and current and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_many_groups_svi_check.py [--quick]"""
import ctypes
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyro_b200 as pyro  # noqa: E402
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200 import _native as N  # noqa: E402
from pyro_b200.infer import SVI, JitTrace_ELBO  # noqa: E402
from pyro_b200.infer import elbo as elbo_mod  # noqa: E402
from pyro_b200.optim import ClippedAdam  # noqa: E402

DEV = "cuda"
COLS = (2, 0, 5)
KINDS = {"Bernoulli": N.GLM_BERNOULLI, "Normal": N.GLM_NORMAL}
SHAPES = [(1000, 1), (10000, 3), (37, 2), (38, 2)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def data(kind, n, D, G, S, P):
    """Sorted rows of the model, and one particle set of its parameters."""
    gen = torch.Generator().manual_seed(0)
    X = torch.randn(n, D, generator=gen)
    g = torch.sort(torch.randint(0, G, (n,), generator=gen)).values
    eta = X @ (0.3 * torch.randn(D, generator=gen) / D ** 0.5) + 0.5 * torch.randn(G, generator=gen)[g]
    for k in range(S):
        eta = eta + 0.3 * torch.randn(G, generator=gen)[g] * X[:, COLS[k]]
    y = torch.bernoulli(torch.sigmoid(eta), generator=gen) if kind == "Bernoulli" else eta + 0.6 * torch.randn(n)
    W = 0.1 * torch.randn(P, D, generator=gen)
    T = [(0.5 if k == 0 else 0.3) * torch.randn(P, G, generator=gen) for k in range(1 + S)]
    b = 0.1 * torch.randn(P, generator=gen)
    sigma = 0.6 + 0.1 * torch.rand(P, generator=gen)
    return [t.to(DEV) for t in (X, g, y, W, b, sigma)], [t.to(DEV) for t in T]


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    return gr.replay


def timed(run, flush, reps):
    out = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3)
    return statistics.median(out)


def fused_call(kind, n, D, G, S, P):
    """The fused site call (gathered past 128 columns, one-hot below) as a closure, and its route's name."""
    (X, g, y, W, b, sigma), T = data(kind, n, D, G, S, P)
    code = KINDS[kind]
    g32 = g.to(torch.int32)
    dev = torch.device(DEV)
    total, db, dsig = torch.empty((), device=DEV), torch.empty(P, device=DEV), torch.empty(P, device=DEV)
    sl = N.b2_glm_slope_tables(S)
    for k in range(S):
        sl.col[k], sl.beta[k], sl.beta_stride[k] = COLS[k], T[k + 1].data_ptr(), G
    sg = sigma.data_ptr() if kind == "Normal" else None
    if D + G * (1 + S) > 128:
        ws = N.workspace(dev, int(N.lib().b2_glm_group_gather_sum_workspace(code, n, D, G, S, P)), tag="gather_check")
        dW, dT = torch.empty(P, D, device=DEV), torch.empty(1 + S, P, G, device=DEV)

        def run():
            N.check(N.lib().b2_glm_group_gather_sum(
                code, X.data_ptr(), y.data_ptr(), sg, 1, g32.data_ptr(), G, W.data_ptr(), D, T[0].data_ptr(), G,
                ctypes.byref(sl), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, None, total.data_ptr(), dW.data_ptr(),
                db.data_ptr(), dsig.data_ptr(), dT.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr()),
                "b2_glm_group_gather_sum")
        return run, "gathered", (X, g, y, W, b, sigma, T)
    ws = N.workspace(dev, int(N.lib().b2_glm_group_slope_sum_workspace(code, n, D, G, S, P)), tag="slope_check")
    dWAB = torch.empty(P, D + G * (1 + S), device=DEV)

    def run():
        N.check(N.lib().b2_glm_group_slope_sum(
            code, X.data_ptr(), y.data_ptr(), None, 0, sg, 1, g32.data_ptr(), G, W.data_ptr(), D, T[0].data_ptr(), G,
            ctypes.byref(sl), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, None, total.data_ptr(), dWAB.data_ptr(),
            db.data_ptr(), dsig.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr()), "b2_glm_group_slope_sum")
    return run, "one-hot", (X, g, y, W, b, sigma, T)


def site_times(kind, n, D, G, S, P, reps):
    run, route, (X, g, y, W, b, sigma, T) = fused_call(kind, n, D, G, S, P)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    Wr, br, sr = (t.clone().requires_grad_(True) for t in (W, b, sigma))
    Tr = [t.clone().requires_grad_(True) for t in T]
    yP = y.expand(P, n)

    def materialised():
        eta = Wr @ X.T + br[:, None] + Tr[0][..., g]
        for k in range(S):
            eta = eta + Tr[k + 1][..., g] * X[:, COLS[k]]
        d = dist.Bernoulli(logits=eta) if kind == "Bernoulli" else dist.Normal(eta, sr[:, None])
        s = d._fused_sum(yP, None, 1.0, 1.0, 1.0)
        torch.autograd.grad(s, [Wr, br] + Tr + ([sr] if kind == "Normal" else []))

    runs = {"fused " + route: graphed(run), "materialised": graphed(materialised)}
    res = {k: [] for k in runs}
    for _ in range(5):                      # alternating windows
        for k, r in runs.items():
            res[k].append(timed(r, flush, reps))
    return {k: statistics.median(v) for k, v in res.items()}


def make_model(kind, G, S):
    def model(X, g, y):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
        sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.0))) if kind == "Normal" else None
        alpha = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
        betas = [pyro.sample("beta%d" % k, dist.Normal(X.new_zeros(G), 0.3).to_event(1)) for k in range(S)]
        with pyro.plate("data", X.shape[0]):
            eta = w.squeeze(-2) @ X.T + b + alpha.squeeze(-2)[..., g]
            for k, be in enumerate(betas):
                eta = eta + be.squeeze(-2)[..., g] * X[:, COLS[k]]
            d = dist.Bernoulli(logits=eta) if kind == "Bernoulli" else dist.Normal(eta, sigma)
            pyro.sample("y", d, obs=y)

    def guide(X, g, y):
        D = X.shape[-1]
        sites = [("w", (D,)), ("b", ()), ("alpha", (G,))] + [("beta%d" % k, (G,)) for k in range(S)]
        for name, shape in sites + ([("sigma", ())] if kind == "Normal" else []):
            loc = pyro.param(name + "_loc", X.new_zeros(shape))
            scale = pyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=dist.constraints.positive)
            if name == "sigma":
                pyro.sample(name, dist.LogNormal(loc, scale))
            else:
                d = dist.Normal(loc, scale)
                pyro.sample(name, d.to_event(1) if shape else d)
    return model, guide


def step_time(kind, G, S, X, g, y, P, lazy, steps):
    model, guide = make_model(kind, G, S)
    elbo_mod.LAZY_LINEAR = lazy
    pyro.clear_param_store()
    calls = []
    real = dist._GlmGatherFn.apply
    dist._GlmGatherFn.apply = lambda *a: calls.append(1) or real(*a)
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        for _ in range(5):
            svi.step(X, g, y)
        torch.cuda.synchronize()
        assert bool(calls) == lazy, "the lazy route made no gathered call" if lazy else "a fused call without the seam"
        t0 = time.perf_counter()
        for _ in range(steps):
            svi.step(X, g, y)
        torch.cuda.synchronize()
    finally:
        dist._GlmGatherFn.apply = real
        elbo_mod.LAZY_LINEAR = True
    return (time.perf_counter() - t0) / steps * 1e6


def kernel_split(kind, n, D, G, S, P):
    from torch.profiler import ProfilerActivity, profile
    run, _, _ = fused_call(kind, n, D, G, S, P)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            run()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if e.count and t:
            rows.append((e.key, e.count, t))
    return rows


def main():
    quick = "--quick" in sys.argv
    n, D = 1_000_000, 16
    print("card (name, power limit, SM clock, max SM clock):", card())
    for kind in KINDS:
        for G, S in SHAPES:
            for P in (16, 64):
                t = site_times(kind, n, D, G, S, P, 10 if quick else 20)
                print("site value + gradients, %s N=%d D=%d G=%d S=%d (%d columns) P=%d: %s" % (
                    kind, n, D, G, S, D + G * (1 + S), P, ", ".join("%s %.1f us" % kv for kv in t.items())))
    G, S = 1000, 1
    for kind in KINDS:
        (X, g, y, *_), _ = data(kind, n, D, G, S, 1)
        for P in (16, 64):
            lz, mt = [], []
            for _ in range(2 if quick else 4):
                lz.append(step_time(kind, G, S, X, g, y, P, True, 10 if quick else 30))
                mt.append(step_time(kind, G, S, X, g, y, P, False, 10 if quick else 30))
            print("graph-captured SVI.step, %s N=%d D=%d G=%d S=%d P=%d: lazy %.1f us, LAZY_LINEAR=False %.1f us "
                  "(medians of %d alternating runs)" % (kind, n, D, G, S, P, statistics.median(lz),
                                                        statistics.median(mt), len(lz)))
    for kind in KINDS:
        print("per-kernel device time of the gathered call (torch.profiler, mean of 10), %s N=%d D=%d G=10000 S=3 "
              "P=64:" % (kind, n, D))
        for name, count, t in kernel_split(kind, n, D, 10000, 3, 64):
            print("  %8.1f us  x%-3d %s" % (t / count, count, name[:110]))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
