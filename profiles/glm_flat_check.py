"""GPU check of the logistic-regression likelihood kernel for feature counts without a kernel of their own
(b2_glm_bernoulli_logits, glm_flat_tc.cu), at N = 1e6, P = 64:
  - kernel + finish device time (CUDA events around graph replays, L2 flushed between replays, median of 25),
    beside D = 16 (fp32 SIMT kernel) and D = 32 (glm_tc.cu), which show what the bulk-copy load path costs;
  - the materialised site the kernel replaces (cuBLAS logits, the generic Bernoulli site kernel, autograd
    for dW and db), timed the same way but eagerly;
  - errors of sum_p, dW and db against fp64;
  - one graph-captured SVI.step of the unchanged `logistic_model` at D = 100 against LAZY_LINEAR = False,
    in alternating runs.
Usage: python profiles/glm_flat_check.py [--quick]"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pyro_b200 import _native as N  # noqa: E402

DS = [10, 15, 16, 28, 31, 32, 33, 54, 64, 100, 123, 128]
REPS = 25


def run(X, y, W, b, flags=0):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev))
    ws = N.workspace(dev, int(N.lib().b2_glm_workspace(n, D, P)), tag="glm_flat_check")

    def call():
        total, sum_p, dW, db = out
        N.check(N.lib().b2_glm_bernoulli_logits(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, flags,
            sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(),
            N.stream_ptr(dev)), "b2_glm_bernoulli_logits")
    return call, out


def materialised(X, y, W, b):
    """The site as it runs without the kernel: [P, N] logits, the generic Bernoulli site kernel, autograd."""
    import pyro_b200.distributions as dist
    Wr, br = W.clone().requires_grad_(True), b.clone().requires_grad_(True)

    def call():
        logits = Wr @ X.t() + br[:, None]
        total = dist.Bernoulli(logits=logits)._fused_sum(y, None, 1.0, 1.0, 1.0, True)
        return torch.autograd.grad(total, [Wr, br])
    return call


def timed(fn, flush):
    ts = []
    for _ in range(REPS):
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
    n, P = 1000000, 64
    g = torch.Generator(device=dev).manual_seed(D)
    X = torch.randn(n, D, device=dev, generator=g)
    wt = torch.randn(D, device=dev, generator=g) / D ** 0.5
    y = (torch.rand(n, device=dev, generator=g) < torch.sigmoid(X @ wt + 0.5)).float()
    W = (0.3 * torch.randn(P, D, device=dev, generator=g) / D ** 0.5 + wt).contiguous()
    b = 0.5 + 0.2 * torch.randn(P, device=dev, generator=g)
    # fp64 reference
    Wd, bd = W.double().requires_grad_(True), b.double().requires_grad_(True)
    lg = Wd @ X.double().t() + bd[:, None]
    s_ref = (y.double() * lg - torch.nn.functional.softplus(lg)).sum(1)
    gW, gb = torch.autograd.grad(s_ref.sum(), [Wd, bd])
    s_ref = s_ref.detach()
    del lg
    call, (total, sum_p, dW, db) = run(X, y, W, b)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e_sum = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    e_dw = float((dW.double() - gW).abs().max() / gW.abs().max())
    e_db = float((db.double() - gb).abs().max() / gb.abs().max())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    t_k = timed(graph.replay, flush)
    mat = materialised(X, y, W, b)
    for _ in range(2):
        mat()
    t_m = timed(mat, flush)
    kern = "SIMT fp32" if D in (4, 8, 16) else "glm_tc" if D == 32 else "flat_tc"
    print("D=%3d %-9s kernel+finish %7.1f us (min %.1f max %.1f) | materialised %8.1f us (min %.1f max %.1f)"
          " | %.2fx | rel err sum_p %.1e dW %.1e db %.1e"
          % (D, kern, t_k[0], t_k[1], t_k[2], t_m[0], t_m[1], t_m[2], t_m[0] / t_k[0], e_sum, e_dw, e_db))
    return e_sum < 2e-5 and e_dw < 2e-4 and e_db < 2e-4


def svi_steps(dev, reps, steps):
    import models
    import pyro_b200 as pyro
    from pyro_b200.infer import SVI, JitTrace_ELBO
    from pyro_b200.infer import elbo as elbo_mod
    from pyro_b200.optim import ClippedAdam

    n, D, P = 1000000, 100, 64
    torch.manual_seed(0)
    X = torch.randn(n, D, device=dev)
    y = (torch.rand(n, device=dev) < torch.sigmoid(X[:, 0] - 0.5 * X[:, 1])).float()

    def one(lazy):
        elbo_mod.LAZY_LINEAR = lazy
        pyro.clear_param_store()
        svi = SVI(models.logistic_model, models.logistic_guide, ClippedAdam({"lr": 0.01}),
                  JitTrace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        for _ in range(3):             # eager step, capture, first replay
            loss = svi.step(X, y)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            loss = svi.step(X, y)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3, loss

    res = {True: [], False: []}
    try:
        for _ in range(reps):
            for lazy in (True, False):
                ms, loss = one(lazy)
                res[lazy].append(ms)
                print("SVI step D=100 graph-captured %-12s %.3f ms  loss %.6e"
                      % ("fused" if lazy else "materialised", ms, loss))
    finally:
        elbo_mod.LAZY_LINEAR = True
    print("SVI step fused %s ms, materialised %s ms"
          % (["%.3f" % v for v in res[True]], ["%.3f" % v for v in res[False]]))


def main():
    quick = "--quick" in sys.argv
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ok = True
    for D in (DS[:3] if quick else DS):
        ok = site(dev, D, flush) and ok
    svi_steps(dev, 1 if quick else 3, 10 if quick else 30)
    print("GLM_FLAT_CHECK", "OK" if ok else "FAIL", time.strftime("%H:%M:%S"))


if __name__ == "__main__":
    main()
