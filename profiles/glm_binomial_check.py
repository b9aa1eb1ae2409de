"""GPU check of the Binomial-regression likelihood kernel (b2_glm_binomial_logits, glm_binomial_tc.cu), at
N = 1e6, P = 64:
  - kernel + finish device time (CUDA events around graph replays, L2 flushed before each, median of 25) at
    D in {10, 32, 64, 100, 128}, with one trial count (100) and with per-row counts drawn from 0..200, beside the
    Poisson-regression kernel at the same D and the materialised site it replaces (cuBLAS logits, the generic
    Binomial site kernel, autograd), timed the same way; errors against fp64;
  - one graph-captured SVI.step (JitTrace_ELBO, 16 vectorised particles) of the unchanged Binomial model at D = 32,
    fused against LAZY_LINEAR = False, in alternating runs;
  - GlmPotential evaluations at C = 8 / 64 / 128 chains against TracePotential;
  - NUTS chain-leapfrogs per second on the Binomial model at N = 1e6, D = 32, 8 chains, on GlmPotential and on
    TracePotential (compile_model = False), alternating.
The card's name and power limit are printed with the figures.
Usage: python profiles/glm_binomial_check.py [--quick]"""
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


def data(dev, n, D, trials, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn(n, D, device=dev, generator=g)
    wt = 0.5 * torch.randn(D, device=dev, generator=g) / D ** 0.5
    m = (torch.randint(0, 201, (n,), device=dev, generator=g).float() if trials == "rows"
         else torch.full((1,), float(trials), device=dev))
    y = torch.binomial(m.expand(n).contiguous(), torch.sigmoid(X @ wt), generator=g)
    return X, y, m, wt, g


def binomial_call(X, y, m, W, b):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev))
    ws = N.workspace(dev, int(N.lib().b2_glm_binomial_workspace(n, D, P)), tag="glm_binomial_check")
    per_row = 1 if m.numel() == n else 0

    def call():
        total, sum_p, dW, db = out
        N.check(N.lib().b2_glm_binomial_logits(
            X.data_ptr(), y.data_ptr(), m.data_ptr(), per_row, W.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0,
            sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(),
            N.stream_ptr(dev)), "b2_glm_binomial_logits")
    return call, out


def poisson_call(X, y, W, b):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev))
    ws = N.workspace(dev, int(N.lib().b2_glm_poisson_workspace(n, D, P)), tag="glm_poisson_check")

    def call():
        total, sum_p, dW, db = out
        N.check(N.lib().b2_glm_poisson_log_rate(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, sum_p.data_ptr(),
            total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
            "b2_glm_poisson_log_rate")
    return call


def materialised(X, y, m, W, b):
    """The site as it runs without the kernel: [P, N] logits, the generic Binomial site kernel, autograd."""
    import pyro_b200.distributions as dist
    Wr, br = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    tc = m if m.numel() > 1 else m.reshape(())

    def call():
        logits = Wr @ X.t() + br[:, None]
        total = dist.Binomial(tc, logits=logits)._fused_sum(y, None, 1.0, 1.0, 1.0, True)
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


def site(dev, D, trials, flush):
    from test_glm_binomial import binomial_lp
    n, P = 1000000, 64
    X, y, m, wt, g = data(dev, n, D, trials, D)
    W = (0.05 * torch.randn(P, D, device=dev, generator=g) / D ** 0.5 + wt).contiguous()
    b = 0.1 * torch.randn(P, device=dev, generator=g)
    Wd, bd = W.double().requires_grad_(True), b.double().requires_grad_(True)
    s_ref = binomial_lp(y.double(), m.double().expand(n), Wd @ X.double().t() + bd[:, None]).sum(1)
    gW, gb = torch.autograd.grad(s_ref.sum(), [Wd, bd])
    call, out = binomial_call(X, y, m, W, b)
    call()
    torch.cuda.synchronize()
    _, sum_p, dW, db = out
    es = float(((sum_p.double() - s_ref.detach()).abs() / s_ref.detach().abs()).max())
    ew = float((dW.double() - gW).abs().max()) / float(gW.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    fused = timed(graphed(call), flush)
    pois = timed(graphed(poisson_call(X, torch.poisson(torch.full_like(y, 2.0)), W, b)), flush)
    mat = timed(graphed(materialised(X, y, m, W, b)), flush)
    print("D=%3d trials=%-4s binomial %6.0f us (%.0f-%.0f)  poisson %6.0f us  materialised %7.0f us (%.0f-%.0f)  "
          "err sum %.1e dW %.1e db %.1e" % (D, trials, fused[0], fused[1], fused[2], pois[0], mat[0], mat[1], mat[2],
                                            es, ew, eb), flush=True)


def svi_steps(dev):
    import pyro_b200 as pyro
    from pyro_b200.infer import SVI, JitTrace_ELBO
    from pyro_b200.infer import elbo as elbo_mod
    from pyro_b200.optim import ClippedAdam
    from test_glm_binomial import binomial_guide, binomial_model
    n, D, P = 1000000, 32, 16
    X, y, m, _, _ = data(dev, n, D, "rows", 0)
    res = {True: [], False: []}
    steps = 5 if QUICK else 20
    for rnd in range(2 if QUICK else 3):
        for lazy in (True, False):
            elbo_mod.LAZY_LINEAR = lazy
            pyro.clear_param_store()
            svi = SVI(binomial_model, binomial_guide, ClippedAdam({"lr": 0.001}),
                      JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
            for _ in range(3):
                svi.step(X, y, m)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                svi.step(X, y, m)
            torch.cuda.synchronize()
            res[lazy].append((time.perf_counter() - t0) / steps * 1e3)
    elbo_mod.LAZY_LINEAR = True
    print("SVI.step (graph-captured, D=32, N=1e6, per-row trials, 16 particles): fused %s ms, LAZY_LINEAR=False %s ms"
          % (["%.3f" % t for t in res[True]], ["%.3f" % t for t in res[False]]), flush=True)


def potentials(dev):
    from test_glm_binomial import _direct_potential, binomial_model
    from pyro_b200.infer.mcmc import TracePotential
    n, D = 1000000, 32
    X, y, m, _, g = data(dev, n, D, "rows", 1)
    pot = _direct_potential(X, y, m, True)
    for C in (8, 64, 128):
        z = 0.05 * torch.randn(C, pot.dim, device=dev, generator=g)
        tp = TracePotential(binomial_model, (X, y, m), num_chains=C)
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
    from test_glm_binomial import binomial_model
    from pyro_b200.infer import MCMC, NUTS
    n, D = 1000000, 32
    X, y, m, _, _ = data(dev, n, D, "rows", 2)
    steps = 20 if QUICK else 50
    for rnd in range(2):
        for compile_model in (True, False):       # GlmPotential / TracePotential, alternating
            kernel = NUTS(binomial_model, max_tree_depth=6)
            kernel.compile_model = compile_model
            mc = MCMC(kernel, num_samples=steps, warmup_steps=steps, num_chains=8, seed=0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mc.run(X, y, m)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            leaps = int(kernel.leapfrog_count())
            print("NUTS Binomial N=1e6 D=32 8 chains, max_tree_depth 6, %d + %d transitions: %s, %d chain-leapfrogs "
                  "in %.2f s = %.0f /s" % (steps, steps, type(kernel.potential).__name__, leaps, dt, leaps / dt),
                  flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("glm_binomial_check.py needs a CUDA device")
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)   # 64 MB > L2
    for D in DS:
        for trials in (100, "rows"):
            site(dev, D, trials, flush)
    svi_steps(dev)
    potentials(dev)
    nuts(dev)


if __name__ == "__main__":
    main()
