"""GPU check of the Poisson-regression likelihood kernel (b2_glm_poisson_log_rate, glm_poisson_tc.cu), at
N = 1e6, P = 64:
  - kernel + finish device time (CUDA events around graph replays, L2 flushed before each, median of 25) at
    D in {10, 32, 64, 100, 128}, beside the logistic-regression kernel at the same D, and the materialised site
    it replaces (cuBLAS log-rate, exp, the generic Poisson site kernel, autograd), timed the same way;
  - one graph-captured SVI.step (JitTrace_ELBO, 16 vectorised particles) of the unchanged Poisson model at D = 32,
    fused against LAZY_LINEAR = False, in alternating runs;
  - GlmPotential evaluations at C = 8 / 64 / 128 chains against TracePotential;
  - NUTS chain-leapfrogs per second on the Poisson model at N = 1e6, D = 32, 8 chains, on GlmPotential and on
    TracePotential (compile_model = False), alternating.
The card's name and power limit are printed with the figures.
Usage: python profiles/glm_poisson_check.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pyro_b200 import _native as N  # noqa: E402

QUICK = "--quick" in sys.argv
DS = [10, 32] if QUICK else [10, 32, 64, 100, 128]
REPS = 25


def kernel_call(entry, wsfn, X, y, W, b):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev))
    ws = N.workspace(dev, int(getattr(N.lib(), wsfn)(n, D, P)), tag="glm_poisson_check")

    def call():
        total, sum_p, dW, db = out
        N.check(getattr(N.lib(), entry)(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, sum_p.data_ptr(),
            total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)), entry)
    return call, out


def materialised(X, y, W, b):
    """The site as it runs without the kernel: [P, N] log-rate and rate, the generic Poisson kernel, autograd."""
    import pyro_b200.distributions as dist
    Wr, br = W.clone().requires_grad_(True), b.clone().requires_grad_(True)

    def call():
        rate = torch.exp(Wr @ X.t() + br[:, None])
        total = dist.Poisson(rate)._fused_sum(y, None, 1.0, 1.0, 1.0, True)
        return torch.autograd.grad(total, [Wr, br])
    return call


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def timed(fn, flush, reps=REPS):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def site(dev, D, flush):
    from oracle import dists as od
    n, P = 1000000, 64
    g = torch.Generator(device=dev).manual_seed(D)
    X = torch.randn(n, D, device=dev, generator=g)
    wt = 0.3 * torch.randn(D, device=dev, generator=g) / D ** 0.5
    y = torch.poisson(torch.exp(X @ wt + 0.5), generator=g)
    yb = (y > 1).float()
    W = (0.05 * torch.randn(P, D, device=dev, generator=g) / D ** 0.5 + wt).contiguous()
    b = 0.5 + 0.05 * torch.randn(P, device=dev, generator=g)
    Wd, bd = W.double().requires_grad_(True), b.double().requires_grad_(True)
    s_ref = od.poisson(y.double(), torch.exp(Wd @ X.double().t() + bd[:, None])).sum(1)
    gW, gb = torch.autograd.grad(s_ref.sum(), [Wd, bd])
    call, out = kernel_call("b2_glm_poisson_log_rate", "b2_glm_poisson_workspace", X, y, W, b)
    bcall, _ = kernel_call("b2_glm_bernoulli_logits", "b2_glm_workspace", X, yb, W, b)
    call()
    torch.cuda.synchronize()
    _, sum_p, dW, db = out
    es = float(((sum_p.double() - s_ref.detach()).abs() / s_ref.detach().abs()).max())
    ew = float((dW.double() - gW).abs().max()) / float(gW.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    fused = timed(graphed(call), flush)
    bern = timed(graphed(bcall), flush)
    mat = timed(graphed(materialised(X, y, W, b)), flush)
    print("D=%3d  poisson %6.0f us (%.0f-%.0f)  bernoulli %6.0f us  materialised %7.0f us (%.0f-%.0f)  "
          "err sum %.1e dW %.1e db %.1e" % (D, fused[0], fused[1], fused[2], bern[0], mat[0], mat[1], mat[2],
                                            es, ew, eb), flush=True)


def svi_steps(dev):
    import pyro_b200 as pyro
    from pyro_b200.infer import SVI, JitTrace_ELBO
    from pyro_b200.infer import elbo as elbo_mod
    from pyro_b200.optim import ClippedAdam
    from test_glm_poisson import poisson_guide, poisson_model
    n, D, P = 1000000, 32, 16
    g = torch.Generator(device=dev).manual_seed(0)
    X = torch.randn(n, D, device=dev, generator=g)
    y = torch.poisson(torch.exp(X @ (0.3 * torch.randn(D, device=dev, generator=g) / D ** 0.5) + 0.5),
                      generator=g)
    res = {True: [], False: []}
    steps = 5 if QUICK else 20
    for rnd in range(2 if QUICK else 3):
        for lazy in (True, False):
            elbo_mod.LAZY_LINEAR = lazy
            pyro.clear_param_store()
            svi = SVI(poisson_model, poisson_guide, ClippedAdam({"lr": 0.001}),
                      JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
            for _ in range(3):
                svi.step(X, y)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                svi.step(X, y)
            torch.cuda.synchronize()
            res[lazy].append((time.perf_counter() - t0) / steps * 1e3)
    elbo_mod.LAZY_LINEAR = True
    print("SVI.step (graph-captured, D=32, N=1e6, 16 particles): fused %s ms, LAZY_LINEAR=False %s ms"
          % (["%.3f" % t for t in res[True]], ["%.3f" % t for t in res[False]]), flush=True)


def potentials(dev):
    from test_glm_poisson import _direct_potential, _trace_model
    from pyro_b200.infer.mcmc import TracePotential
    n, D = 1000000, 32
    g = torch.Generator(device=dev).manual_seed(1)
    X = torch.randn(n, D, device=dev, generator=g)
    y = torch.poisson(torch.exp(X @ (0.3 * torch.randn(D, device=dev, generator=g) / D ** 0.5) + 0.5),
                      generator=g)
    pot = _direct_potential(X, y, True)
    for C in (8, 64, 128):
        z = 0.05 * torch.randn(C, pot.dim, device=dev, generator=g)
        tp = TracePotential(_trace_model(True), (X, y), num_chains=C)
        out = []
        for fn in (pot.value_and_grad, tp.value_and_grad):
            for _ in range(3):
                fn(z)
            torch.cuda.synchronize()
            reps = 20
            t0 = time.perf_counter()
            for _ in range(reps):
                fn(z)
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) / reps * 1e3)
        print("potential C=%3d: GlmPotential %.3f ms  TracePotential %.3f ms" % (C, out[0], out[1]), flush=True)


def nuts(dev):
    from test_glm_poisson import poisson_model
    from pyro_b200.infer import MCMC, NUTS
    n, D = 1000000, 32
    g = torch.Generator(device=dev).manual_seed(2)
    X = torch.randn(n, D, device=dev, generator=g)
    y = torch.poisson(torch.exp(X @ (0.3 * torch.randn(D, device=dev, generator=g) / D ** 0.5) + 0.5),
                      generator=g)
    steps = 20 if QUICK else 50
    for rnd in range(2):
        for compile_model in (True, False):       # GlmPotential / TracePotential, alternating
            kernel = NUTS(poisson_model, max_tree_depth=6)
            kernel.compile_model = compile_model
            mc = MCMC(kernel, num_samples=steps, warmup_steps=steps, num_chains=8, seed=0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mc.run(X, y)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            leaps = int(kernel.leapfrog_count())
            print("NUTS Poisson N=1e6 D=32 8 chains, max_tree_depth 6, %d + %d transitions: %s, %d chain-leapfrogs "
                  "in %.2f s = %.0f /s" % (steps, steps, type(kernel.potential).__name__, leaps, dt, leaps / dt),
                  flush=True)

def main():
    if not torch.cuda.is_available():
        raise SystemExit("glm_poisson_check.py needs a CUDA device")
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)   # 64 MB > L2
    for D in DS:
        site(dev, D, flush)
    svi_steps(dev)
    potentials(dev)
    nuts(dev)


if __name__ == "__main__":
    main()
