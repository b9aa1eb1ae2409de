"""GPU check of the linear-regression likelihood kernel (b2_glm_normal_loc, glm_normal_tc.cu), at N = 1e6, P = 64:
  - kernel + finish device time (CUDA events around graph replays, L2 flushed before each, median of 25) at
    D in {10, 32, 64, 100, 128}, beside the logistic-regression kernel at the same D with B2_FLAG_GLM_3XTF32 (the
    same three-product GEMM 1), and the materialised site it replaces (cuBLAS loc, the generic Normal site
    kernel, autograd for dW, db and dsigma), timed the same way;
  - errors against fp64 at sigma* = 0.5, 0.05 and 0.005 (y = X w* + 3 + sigma* eps, rms(X w*) = 1);
  - one graph-captured SVI.step (JitTrace_ELBO, 64 vectorised particles, latent sigma) of the unchanged model at
    D = 32, fused against LAZY_LINEAR = False, in alternating runs;
  - GlmPotential evaluations at C = 8 / 64 / 128 chains against TracePotential (HalfNormal sigma prior);
  - NUTS chain-leapfrogs per second on the model at N = 1e6, D = 32, 8 chains, on GlmPotential and on
    TracePotential (compile_model = False), alternating.
The card's name and power limit are printed with the figures.
Usage: python profiles/glm_normal_check.py [--quick]"""
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


def normal_call(X, y, W, b, sig):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev), torch.empty(P, device=dev))
    ws = N.workspace(dev, int(N.lib().b2_glm_normal_workspace(n, D, P)), tag="glm_normal_check")

    def call():
        total, sum_p, dW, db, ds = out
        N.check(N.lib().b2_glm_normal_loc(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), sig.data_ptr(), 1, n, D, P, 1.0, 1.0, 1.0, 0,
            sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(), ds.data_ptr(), ws.data_ptr(),
            ws.numel(), N.stream_ptr(dev)), "b2_glm_normal_loc")
    return call, out


def bernoulli_call(X, y, W, b):
    n, D = X.shape
    P = W.shape[0]
    dev = X.device
    out = (torch.empty((), device=dev), torch.empty(P, device=dev), torch.empty(P, D, device=dev),
           torch.empty(P, device=dev))
    ws = N.workspace(dev, int(N.lib().b2_glm_workspace(n, D, P)), tag="glm_normal_check_b")

    def call():
        total, sum_p, dW, db = out
        N.check(N.lib().b2_glm_bernoulli_logits(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, N.B2_FLAG_GLM_3XTF32,
            sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(),
            N.stream_ptr(dev)), "b2_glm_bernoulli_logits")
    return call


def materialised(X, y, W, b, sig):
    """The site as it runs without the kernel: the [P, N] loc, the generic Normal site kernel, autograd."""
    import pyro_b200.distributions as dist
    Wr, br, sr = W.clone().requires_grad_(True), b.clone().requires_grad_(True), sig.clone().requires_grad_(True)

    def call():
        loc = Wr @ X.t() + br[:, None]
        total = dist.Normal(loc, sr[:, None])._fused_sum(y, None, 1.0, 1.0, 1.0, True)
        return torch.autograd.grad(total, [Wr, br, sr])
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


def problem(dev, D, sigma_star):
    n, P = 1000000, 64
    g = torch.Generator(device=dev).manual_seed(D)
    X = torch.randn(n, D, device=dev, generator=g)
    wt = torch.randn(D, device=dev, generator=g)
    wt = wt / wt.norm()
    y = X @ wt + 3.0 + sigma_star * torch.randn(n, device=dev, generator=g)
    W = (0.05 * torch.randn(P, D, device=dev, generator=g) / D ** 0.5 + wt).contiguous()
    b = 3.0 + 0.05 * torch.randn(P, device=dev, generator=g)
    sig = sigma_star * torch.exp(0.1 * torch.randn(P, device=dev, generator=g))
    return X, y, W, b, sig


def errors(X, y, W, b, sig):
    from oracle import dists as od
    Wd, bd, sd = W.double().requires_grad_(True), b.double().requires_grad_(True), sig.double().requires_grad_(True)
    s_ref = od.normal(y.double(), Wd @ X.double().t() + bd[:, None], sd[:, None]).sum(1)
    gW, gb, gs = torch.autograd.grad(s_ref.sum(), [Wd, bd, sd])
    s_ref = s_ref.detach()
    call, out = normal_call(X, y, W, b, sig)
    call()
    torch.cuda.synchronize()
    _, sum_p, dW, db, ds = out
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    ew = float((dW.double() - gW).abs().max()) / float(gW.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    eds = float((ds.double() - gs).abs().max()) / float((X.shape[0] / sig.double()).max())
    return es, ew, eb, eds


def site(dev, D, flush):
    X, y, W, b, sig = problem(dev, D, 0.5)
    yb = (y > 3.0).float()
    call, _ = normal_call(X, y, W, b, sig)
    fused = timed(graphed(call), flush)
    bern = timed(graphed(bernoulli_call(X, yb, W, b)), flush)
    mat = timed(graphed(materialised(X, y, W, b, sig)), flush)
    print("D=%3d  normal %6.0f us (%.0f-%.0f)  bernoulli 3xTF32 %6.0f us  materialised %7.0f us (%.0f-%.0f)"
          % (D, fused[0], fused[1], fused[2], bern[0], mat[0], mat[1], mat[2]), flush=True)
    for s in (0.5, 0.05, 0.005):
        es, ew, eb, eds = errors(*problem(dev, D, s))
        print("       sigma*=%-6g err sum %.1e dW %.1e db %.1e dsigma %.1e" % (s, es, ew, eb, eds), flush=True)


def svi_steps(dev):
    import pyro_b200 as pyro
    from pyro_b200.infer import SVI, JitTrace_ELBO
    from pyro_b200.infer import elbo as elbo_mod
    from pyro_b200.optim import ClippedAdam
    from test_glm_normal import _guide, _model
    n, D, P = 1000000, 32, 64
    X, y, _, _, _ = problem(dev, D, 0.5)
    res = {True: [], False: []}
    steps = 5 if QUICK else 20
    for rnd in range(2 if QUICK else 3):
        for lazy in (True, False):
            elbo_mod.LAZY_LINEAR = lazy
            pyro.clear_param_store()
            svi = SVI(_model("latent"), _guide("latent"), ClippedAdam({"lr": 0.001}),
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
    print("SVI.step (graph-captured, latent sigma, D=32, N=1e6, %d particles): fused %s ms, LAZY_LINEAR=False %s ms"
          % (P, ["%.3f" % t for t in res[True]], ["%.3f" % t for t in res[False]]), flush=True)


def potentials(dev):
    from test_glm_normal import _nuts_model
    from pyro_b200.infer.mcmc import TracePotential
    from pyro_b200.infer.mcmc.compile import recognise
    X, y, W, _, _ = problem(dev, 32, 0.5)
    model = _nuts_model("HalfNormal")
    pot = recognise(model, (X, y))
    g = torch.Generator(device=dev).manual_seed(1)
    for C in (8, 64, 128):
        z = 0.05 * torch.randn(C, pot.dim, device=dev, generator=g)
        z[:, :32] += W[0]
        tp = TracePotential(model, (X, y), num_chains=C)
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
        print("potential C=%3d: %s %.3f ms  TracePotential %.3f ms" % (C, type(pot).__name__, out[0], out[1]),
              flush=True)


def nuts(dev):
    from test_glm_normal import _nuts_model
    from pyro_b200.infer import MCMC, NUTS
    X, y, _, _, _ = problem(dev, 32, 0.5)
    steps = 20 if QUICK else 50
    for rnd in range(2):
        for compile_model in (True, False):       # GlmPotential / TracePotential, alternating
            kernel = NUTS(_nuts_model("HalfNormal"), max_tree_depth=6)
            kernel.compile_model = compile_model
            mc = MCMC(kernel, num_samples=steps, warmup_steps=steps, num_chains=8, seed=0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mc.run(X, y)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            leaps = int(kernel.leapfrog_count())
            print("NUTS linear regression N=1e6 D=32 8 chains, max_tree_depth 6, %d + %d transitions: %s, %d "
                  "chain-leapfrogs in %.2f s = %.0f /s" % (steps, steps, type(kernel.potential).__name__, leaps, dt,
                                                         leaps / dt), flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("glm_normal_check.py needs a CUDA device")
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
