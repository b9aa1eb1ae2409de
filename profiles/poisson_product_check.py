"""GPU check of the fused Poisson factorisation likelihood (b2_poisson_product), the bottom layer of BASELINE
config 5: errors against an fp64 torch evaluation and kernel + finish device time (CUDA events around graph
replays, L2 flushed between replays) at P = 32 and P = 256, N = 320, K = 15, J = 4096, against the kernel's
data-sheet floors; one observation site (value and both factor gradients, graph-captured) on the fused and
the materialised path for K = 1, 4, 8, 15; then the config-5 SVI step (sparse gamma DEF, TraceMeanField_ELBO) on the fused path against
the materialised path (LAZY_LINEAR = False), alternating in one process, eager and graph-captured, with the
peak memory of each.
Usage: python profiles/poisson_product_check.py [--quick]
       python profiles/poisson_product_check.py --profile P     (torch.profiler table of one step, both paths)"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pyro_b200 import _native as N  # noqa: E402

# H100 SXM data sheet (700 W card): HBM3 bandwidth, dense TF32 tensor rate, MUFU ops/clk/SM x SMs x boost clock
HBM_BPS = 3.35e12
TF32_FLOPS = 495e12
MUFU_OPS = 16 * 132 * 1.98e9
n_, K_, J_ = 320, 15, 4096


def data(P, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.poisson(torch.distributions.Gamma(0.5, 0.5).sample((n_, J_)) * 2.0, generator=g).to(dev)
    A = torch.distributions.Gamma(0.3, 0.3).sample((P, n_, K_)).to(dev)
    B = torch.distributions.Gamma(0.3, 0.3).sample((P, K_, J_)).to(dev)
    return A, B, x


def run(A, B, x):
    P, n, K = A.shape
    J = B.shape[-1]
    dev = A.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    sum_p = torch.empty(P, dtype=torch.float32, device=dev)
    dA, dB = torch.empty_like(A), torch.empty_like(B)
    ws = N.workspace(dev, int(N.lib().b2_poisson_product_workspace(n, K, J, P)), tag="pp_check")

    def call():
        N.check(N.lib().b2_poisson_product(
            A.data_ptr(), B.data_ptr(), x.data_ptr(), n, K, J, P, 1.0, 1.0, 1.0, 0, sum_p.data_ptr(),
            total.data_ptr(), dA.data_ptr(), dB.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
            "b2_poisson_product")
    return call, (sum_p, dA, dB)


def accuracy(P, dev):
    A, B, x = data(P, dev)
    call, (sum_p, dA, dB) = run(A, B, x)
    call()
    torch.cuda.synchronize()
    es, eA, eB = 0.0, 0.0, 0.0
    for s in range(0, P, 16):
        A64 = A[s:s + 16].double().requires_grad_()
        B64 = B[s:s + 16].double().requires_grad_()
        rate = A64 @ B64
        xd = x.double()
        sp = (torch.xlogy(xd, rate) - rate - torch.lgamma(xd + 1)).sum((-1, -2))
        sp.sum().backward()
        es = max(es, float(((sum_p[s:s + 16].double() - sp.detach()).abs() / sp.detach().abs()).max()))
        for got, ref, name in ((dA[s:s + 16], A64.grad, "A"), (dB[s:s + 16], B64.grad, "B")):
            e = float(((got.double() - ref).abs().flatten(1).amax(1) / ref.abs().flatten(1).amax(1)).max())
            if name == "A":
                eA = max(eA, e)
            else:
                eB = max(eB, e)
    print("ERR P=%d N=%d K=%d J=%d: sum_p %.2e rel, dA %.2e, dB %.2e of the particle's max |grad|"
          % (P, n_, K_, J_, es, eA, eB))
    return es < 2e-6 and eA < 2e-4 and eB < 2e-4


def floors(P):
    terms = P * n_ * J_
    hbm = (P * (n_ * K_ + K_ * J_) * 4 * 2 + n_ * J_ * 4) / HBM_BPS   # factors read, gradients written, x once
    mufu = 2 * terms / MUFU_OPS                                        # lg2 + rcp per term
    tensor = 2 * 16 * terms * (3 + 2) / TF32_FLOPS                     # GEMM 1 x 3 (split) + two gradient GEMMs, K -> 16
    return hbm, mufu, tensor


def kernel_time(P, dev):
    A, B, x = data(P, dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    call, _ = run(A, B, x)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    ts = []
    for _ in range(20):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    med = ts[len(ts) // 2]
    hbm, mufu, tensor = floors(P)
    print("TIME kernel + finish P=%d N=%d K=%d J=%d: median %.1f us (min %.1f, max %.1f)"
          % (P, n_, K_, J_, med, ts[0], ts[-1]))
    print("     floors (H100 SXM data sheet): HBM %.1f us, MUFU %.1f us, TF32 tensor %.1f us -> %.2fx the largest"
          % (hbm * 1e6, mufu * 1e6, tensor * 1e6, med / (max(hbm, mufu, tensor) * 1e6)))


def site_time(P, K, dev, reps=20):
    """One observation site (value + both factor gradients) on the fused path and on the materialised path
    (bmm, generic Poisson kernel, autograd), each captured in a CUDA graph; median replay time in us."""
    import pyro_b200.distributions as dist
    from pyro_b200.lazy import SiteValue
    g = torch.Generator().manual_seed(1)
    x = torch.poisson(torch._standard_gamma(torch.full((n_, J_), 0.5), generator=g) * 4.0, generator=g).to(dev)
    A = (torch._standard_gamma(torch.full((P, n_, K), 0.3), generator=g) / 0.3).to(dev).requires_grad_()
    B = (torch._standard_gamma(torch.full((P, K, J_), 0.3), generator=g) / 0.3).to(dev).requires_grad_()
    out = {}
    for lazy in (True, False):
        def step():
            rate = SiteValue.wrap(A) @ SiteValue.wrap(B) if lazy else A @ B
            dist.Poisson(rate).to_event(1)._fused_sum(x, None, 1.0, 1.0, 1.0, True).backward()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                A.grad = B.grad = None
                step()
        torch.cuda.current_stream().wait_stream(s)
        A.grad = B.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts.sort()
        out[lazy] = ts[len(ts) // 2]
        A.grad = B.grad = None
        del graph
    print("SITE P=%d N=%d K=%d J=%d: fused %.1f us, materialised %.1f us (%.2fx)"
          % (P, n_, K, J_, out[True], out[False], out[False] / out[True]))


def make_svi(P, graph, dev):
    import models
    import pyro_b200 as pyro
    from pyro_b200.infer import SVI, TraceMeanField_ELBO
    from pyro_b200.optim import AdagradRMSProp
    torch.manual_seed(0)
    x = torch.poisson(torch.distributions.Gamma(0.5, 0.5).sample((n_, J_)) * 2.0).to(dev)
    pyro.clear_param_store()
    m = models.SparseGammaDEF(J_, (100, 40, K_), device=dev, dtype=torch.float32)
    elbo = TraceMeanField_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1)
    elbo.capture_graph = graph
    return SVI(m.model, m.guide, AdagradRMSProp({"eta": 4.5, "t": 0.1}), elbo), x


def svi_steps(P, dev, reps, steps=10):
    from pyro_b200.infer import elbo as elbo_mod
    res = {}
    try:
        for rep in range(reps):
            for graph in (False, True):
                for lazy in ((True, False) if rep % 2 == 0 else (False, True)):   # alternate which runs first
                    elbo_mod.LAZY_LINEAR = lazy
                    svi, x = make_svi(P, graph, dev)
                    for _ in range(4):
                        loss = svi.step(x)
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats(dev)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        loss = svi.step(x)
                    e1.record()
                    e1.synchronize()
                    ms = e0.elapsed_time(e1) / steps
                    peak = torch.cuda.max_memory_allocated(dev) / 1e9
                    key = ("graph" if graph else "eager", "fused" if lazy else "materialised")
                    res.setdefault(key, []).append(ms)
                    print("SVI P=%d %-5s %-12s %.3f ms/step  peak %.2f GB  loss %.6e" % (P, key[0], key[1], ms, peak, loss))
                    del svi
                    torch.cuda.empty_cache()
    finally:
        elbo_mod.LAZY_LINEAR = True
    for k, v in sorted(res.items()):
        print("SVI P=%d %s %s: %s ms" % (P, k[0], k[1], ["%.3f" % t for t in v]))


def profile(P, dev):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile
    from pyro_b200.infer import elbo as elbo_mod
    for lazy in (False, True):
        elbo_mod.LAZY_LINEAR = lazy
        svi, x = make_svi(P, False, dev)
        for _ in range(3):
            svi.step(x)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            svi.step(x)
            torch.cuda.synchronize()
        print("PROFILE P=%d %s" % (P, "fused" if lazy else "materialised"))
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12, max_name_column_width=60))
    elbo_mod.LAZY_LINEAR = True


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    if "--profile" in sys.argv:
        profile(int(sys.argv[sys.argv.index("--profile") + 1]), dev)
        return
    quick = "--quick" in sys.argv
    ok = True
    for P in (32, 256):
        ok = accuracy(P, dev) and ok
        kernel_time(P, dev)
    for P in (32, 256):
        for K in (1, 4, 8, 15):
            site_time(P, K, dev)
    for P in (32, 256):
        svi_steps(P, dev, 1 if quick else 4)
    print("POISSON_PRODUCT_CHECK", "OK" if ok else "FAIL", time.strftime("%H:%M:%S"))


if __name__ == "__main__":
    main()
