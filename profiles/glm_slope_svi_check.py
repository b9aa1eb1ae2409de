"""GPU check of varying slopes under SVI (b2_glm_group_slope_sum):
``y ~ Bernoulli(logits = X @ w + b + alpha[g] + beta[g] * X[:, 2])`` at N = 1e6, D = 16, G = 32, S = 1 (80 columns),
P = 16 and 64 particles:
  * device time of the site's value and all its gradients: the fused call (pack, slope kernel, finish) with X split
    (B2_FLAG_GLM_3XTF32) and at default precision (X rounded to TF32), against
      (a) the materialised site (cuBLAS ``W @ X.T``, the ``[P, N]`` gathers of alpha and beta, the product with the
          covariate, the adds, the Bernoulli site kernel and autograd's backward), the route LAZY_LINEAR = False takes;
      (b) the intercept-only fused call (b2_glm_group_sum) at G = 64, which has the same 80 columns.
    CUDA events around CUDA-graph replays with L2 flushed before each replay; median of 20 replays per window, the
    routes alternating over 5 windows;
  * (c) one graph-captured ``SVI.step`` (JitTrace_ELBO, ClippedAdam) of the unchanged model on the lazy route against
    ``LAZY_LINEAR = False``, in alternating runs (N = 1e6 takes the default precision).
The card's name, power limit and current and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_slope_svi_check.py [--quick]"""
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
COL = 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def data(n, D, G, P):
    gen = torch.Generator().manual_seed(0)
    X = torch.randn(n, D, generator=gen)
    g = torch.randint(0, G, (n,), generator=gen)
    eta = X @ (0.3 * torch.randn(D, generator=gen) / D ** 0.5) + 0.5 * torch.randn(G, generator=gen)[g]
    eta = eta + 0.3 * torch.randn(G, generator=gen)[g] * X[:, COL]
    y = torch.bernoulli(torch.sigmoid(eta), generator=gen)
    W = 0.1 * torch.randn(P, D, generator=gen)
    A = 0.5 * torch.randn(P, G, generator=gen)
    B = 0.3 * torch.randn(P, G, generator=gen)
    b = 0.1 * torch.randn(P, generator=gen)
    return [t.to(DEV) for t in (X, g, y, W, A, B, b)]


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


def site_times(n, D, G, P, reps):
    X, g, y, W, A, B, b = data(n, D, G, P)
    g32 = g.to(torch.int32)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    dev = torch.device(DEV)
    ws = N.workspace(dev, int(N.lib().b2_glm_group_slope_sum_workspace(N.GLM_BERNOULLI, n, D, G, 1, P)),
                     tag="glm_slope_check")
    total = torch.empty((), device=DEV)
    dWAB, db = torch.empty(P, D + 2 * G, device=DEV), torch.empty(P, device=DEV)
    sl = N.b2_glm_slope_tables(1)
    sl.col[0], sl.beta[0], sl.beta_stride[0] = COL, B.data_ptr(), G

    def fused(flags):
        def run():
            N.check(N.lib().b2_glm_group_slope_sum(
                N.GLM_BERNOULLI, X.data_ptr(), y.data_ptr(), None, 0, None, 0, g32.data_ptr(), G, W.data_ptr(), D,
                A.data_ptr(), G, ctypes.byref(sl), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, flags, None,
                total.data_ptr(), dWAB.data_ptr(), db.data_ptr(), None, ws.data_ptr(), ws.numel(), N.stream_ptr()),
                "b2_glm_group_slope_sum")
        return run

    # (b) the intercept-only call at the same width: G2 = 2 G groups
    G2 = 2 * G
    g2 = torch.randint(0, G2, (n,), generator=torch.Generator().manual_seed(1)).to(DEV).to(torch.int32)
    A2 = 0.5 * torch.randn(P, G2, device=DEV)
    ws2 = N.workspace(dev, int(N.lib().b2_glm_group_sum_workspace(N.GLM_BERNOULLI, n, D, G2, P)),
                      tag="glm_slope_check_group")
    dWA2 = torch.empty(P, D + G2, device=DEV)

    def intercept_only():
        N.check(N.lib().b2_glm_group_sum(
            N.GLM_BERNOULLI, X.data_ptr(), y.data_ptr(), None, 0, None, 0, g2.data_ptr(), G2, W.data_ptr(), D,
            A2.data_ptr(), G2, b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, None, total.data_ptr(), dWA2.data_ptr(),
            db.data_ptr(), None, ws2.data_ptr(), ws2.numel(), N.stream_ptr()), "b2_glm_group_sum")

    Wr, Ar, Br, br = (t.clone().requires_grad_(True) for t in (W, A, B, b))
    yP = y.expand(P, n)

    def materialised():
        eta = Wr @ X.T + br[:, None] + Ar[..., g] + Br[..., g] * X[:, COL]
        s = dist.Bernoulli(logits=eta)._fused_sum(yP, None, 1.0, 1.0, 1.0)
        torch.autograd.grad(s, [Wr, Ar, Br, br])

    runs = {"fused split X": graphed(fused(N.B2_FLAG_GLM_3XTF32)), "fused default": graphed(fused(0)),
            "(b) intercept-only G=%d default" % G2: graphed(intercept_only), "(a) materialised": graphed(materialised)}
    res = {k: [] for k in runs}
    for _ in range(5):                      # alternating windows
        for k, r in runs.items():
            res[k].append(timed(r, flush, reps))
    return {k: statistics.median(v) for k, v in res.items()}


def model(X, g, y):
    D, G = X.shape[-1], 32
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
    alpha = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
    beta = pyro.sample("beta", dist.Normal(X.new_zeros(G), 0.3).to_event(1))
    with pyro.plate("data", X.shape[0]):
        eta = w.squeeze(-2) @ X.T + b + alpha.squeeze(-2)[..., g] + beta.squeeze(-2)[..., g] * X[:, COL]
        pyro.sample("y", dist.Bernoulli(logits=eta), obs=y)


def guide(X, g, y):
    D, G = X.shape[-1], 32
    for name, shape in (("w", (D,)), ("b", ()), ("alpha", (G,)), ("beta", (G,))):
        loc = pyro.param(name + "_loc", X.new_zeros(shape))
        scale = pyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=dist.constraints.positive)
        d = dist.Normal(loc, scale)
        pyro.sample(name, d.to_event(1) if shape else d)


def step_time(X, g, y, P, lazy, steps):
    elbo_mod.LAZY_LINEAR = lazy
    pyro.clear_param_store()
    calls = []
    real = dist._GlmSlopeFn.apply
    dist._GlmSlopeFn.apply = lambda *a: calls.append(1) or real(*a)
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        for _ in range(5):
            svi.step(X, g, y)
        torch.cuda.synchronize()
        assert bool(calls) == lazy, "the lazy route made no fused call" if lazy else "a fused call without the seam"
        t0 = time.perf_counter()
        for _ in range(steps):
            svi.step(X, g, y)
        torch.cuda.synchronize()
    finally:
        dist._GlmSlopeFn.apply = real
        elbo_mod.LAZY_LINEAR = True
    return (time.perf_counter() - t0) / steps * 1e6


def main():
    quick = "--quick" in sys.argv
    n, D, G = 1_000_000, 16, 32
    print("card (name, power limit, SM clock, max SM clock):", card())
    for P in (16, 64):
        t = site_times(n, D, G, P, 10 if quick else 20)
        print("site value + gradients, N=%d D=%d G=%d S=1 P=%d: %s" % (
            n, D, G, P, ", ".join("%s %.1f us" % kv for kv in t.items())))
    X, g, y, *_ = data(n, D, G, 1)
    for P in (16, 64):
        lz, mt = [], []
        for _ in range(2 if quick else 4):
            lz.append(step_time(X, g, y, P, True, 20 if quick else 50))
            mt.append(step_time(X, g, y, P, False, 20 if quick else 50))
        print("(c) graph-captured SVI.step, N=%d D=%d G=%d S=1 P=%d: lazy %.1f us, LAZY_LINEAR=False %.1f us (medians "
              "of %d alternating runs)" % (n, D, G, P, statistics.median(lz), statistics.median(mt), len(lz)))
    print("card after the runs:", card())


if __name__ == "__main__":
    main()
