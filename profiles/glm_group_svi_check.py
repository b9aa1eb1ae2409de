"""GPU check of multilevel regression under SVI (b2_glm_group_sum): ``y ~ Bernoulli(logits = X @ w + b + alpha[g])``
at N = 1e6, D = 16, G = 48, P = 16 and 64 particles:
  * device time of the site's value and gradients: the fused call (pack, group kernel, finish) with X split
    (B2_FLAG_GLM_3XTF32) and at default precision (X rounded to TF32), against the materialised site (cuBLAS
    ``W @ X.T``, the ``[P, N]`` gather of alpha, the add, the Bernoulli site kernel and autograd's backward).  CUDA
    events around CUDA-graph replays with L2 flushed between replays; the routes alternate;
  * one graph-captured ``SVI.step`` (JitTrace_ELBO, ClippedAdam) of the unchanged model on the lazy route against
    ``LAZY_LINEAR = False``, in alternating runs (N = 1e6 takes the default precision).
The card's name, power limit and maximum SM clock are printed with the numbers.
Usage: python profiles/glm_group_svi_check.py [--quick]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def data(n, D, G, P):
    gen = torch.Generator().manual_seed(0)
    X = torch.randn(n, D, generator=gen)
    g = torch.randint(0, G, (n,), generator=gen)
    eta = X @ (0.3 * torch.randn(D, generator=gen) / D ** 0.5) + 0.5 * torch.randn(G, generator=gen)[g]
    y = torch.bernoulli(torch.sigmoid(eta), generator=gen)
    W = 0.1 * torch.randn(P, D, generator=gen)
    A = 0.5 * torch.randn(P, G, generator=gen)
    b = 0.1 * torch.randn(P, generator=gen)
    return [t.to(DEV) for t in (X, g, y, W, A, b)]


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
    X, g, y, W, A, b = data(n, D, G, P)
    g32 = g.to(torch.int32)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_group_sum_workspace(N.GLM_BERNOULLI, n, D, G, P)),
                     tag="glm_group_check")
    total = torch.empty((), device=DEV)
    dWA, db = torch.empty(P, D + G, device=DEV), torch.empty(P, device=DEV)

    def fused(flags):
        def run():
            N.check(N.lib().b2_glm_group_sum(
                N.GLM_BERNOULLI, X.data_ptr(), y.data_ptr(), None, 0, None, 0, g32.data_ptr(), G, W.data_ptr(), D,
                A.data_ptr(), G, b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, flags, None, total.data_ptr(),
                dWA.data_ptr(), db.data_ptr(), None, ws.data_ptr(), ws.numel(), N.stream_ptr()), "b2_glm_group_sum")
        return run

    Wr, Ar, br = (t.clone().requires_grad_(True) for t in (W, A, b))
    yP = y.expand(P, n)

    def materialised():
        eta = Wr @ X.T + br[:, None] + Ar[..., g]
        s = dist.Bernoulli(logits=eta)._fused_sum(yP, None, 1.0, 1.0, 1.0)
        torch.autograd.grad(s, [Wr, Ar, br])

    runs = {"fused split X": graphed(fused(N.B2_FLAG_GLM_3XTF32)), "fused default": graphed(fused(0)),
            "materialised": graphed(materialised)}
    res = {k: [] for k in runs}
    for _ in range(5):                      # alternating windows
        for k, r in runs.items():
            res[k].append(timed(r, flush, reps))
    return {k: statistics.median(v) for k, v in res.items()}


def model(X, g, y):
    D, G = X.shape[-1], 48
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
    a = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=w.squeeze(-2) @ X.T + b + a.squeeze(-2)[..., g]), obs=y)


def guide(X, g, y):
    D, G = X.shape[-1], 48
    for name, shape in (("w", (D,)), ("b", ()), ("alpha", (G,))):
        loc = pyro.param(name + "_loc", X.new_zeros(shape))
        scale = pyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=dist.constraints.positive)
        d = dist.Normal(loc, scale)
        pyro.sample(name, d.to_event(1) if shape else d)


def step_time(X, g, y, P, lazy, steps):
    elbo_mod.LAZY_LINEAR = lazy
    pyro.clear_param_store()
    svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
              JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
    for _ in range(5):
        svi.step(X, g, y)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        svi.step(X, g, y)
    torch.cuda.synchronize()
    elbo_mod.LAZY_LINEAR = True
    return (time.perf_counter() - t0) / steps * 1e6


def main():
    quick = "--quick" in sys.argv
    n, D, G = 1_000_000, 16, 48
    print("card (name, power limit, max SM clock):", card())
    for P in (16, 64):
        t = site_times(n, D, G, P, 10 if quick else 30)
        print("site value + gradients, N=%d D=%d G=%d P=%d: %s" % (
            n, D, G, P, ", ".join("%s %.1f us" % kv for kv in t.items())))
    X, g, y, *_ = data(n, D, G, 1)
    for P in (16, 64):
        lz, mt = [], []
        for _ in range(2 if quick else 4):
            lz.append(step_time(X, g, y, P, True, 20 if quick else 50))
            mt.append(step_time(X, g, y, P, False, 20 if quick else 50))
        print("graph-captured SVI.step, N=%d D=%d G=%d P=%d: lazy %.1f us, LAZY_LINEAR=False %.1f us (medians of %d "
              "alternating runs)" % (n, D, G, P, statistics.median(lz), statistics.median(mt), len(lz)))


if __name__ == "__main__":
    main()
