"""GPU check of the fused softmax-regression likelihood (b2_glm_categorical_logits): accuracy against an fp64
torch evaluation for several (N, P, K); kernel device time at N = 1e6, D = 32, P = 64, K = 10 (CUDA events
around graph replays, L2 flushed between replays) against its data-sheet floors; and one SVI step of the
softmax model on the fused path against the materialised path (LAZY_LINEAR = False), in alternating runs.
Usage: python profiles/glm_categorical_check.py [--quick]"""
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


def run(X, y, W, b):
    n, D = X.shape
    P, K, _ = W.shape
    dev = X.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    sum_p = torch.empty(P, dtype=torch.float32, device=dev)
    dW = torch.empty(P, K, D, dtype=torch.float32, device=dev)
    db = torch.empty(P, K, dtype=torch.float32, device=dev)
    ws = N.workspace(dev, int(N.lib().b2_glm_categorical_workspace(n, D, K, P)), tag="glm_cat_check")

    def call():
        N.check(N.lib().b2_glm_categorical_logits(
            X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr() if b is not None else None,
            n, D, K, P, 1.0, 1.0, 1.0, 0, sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(),
            db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)), "b2_glm_categorical_logits")
    return call, (total, sum_p, dW, db)


def reference(X, y, W, b):
    """fp64 per-particle sums, dW, db, one particle at a time (a [P, N, K] fp64 tensor would not fit)."""
    Xd = X.double()
    P, K, _ = W.shape
    s = torch.empty(P, dtype=torch.float64, device=X.device)
    gW = torch.empty(W.shape, dtype=torch.float64, device=X.device)
    gb = torch.empty(P, K, dtype=torch.float64, device=X.device)
    onehot = torch.nn.functional.one_hot(y, K).double()
    for p in range(P):
        lg = Xd @ W[p].double().t() + (b[p].double() if b is not None else 0.0)
        s[p] = (lg.gather(1, y[:, None]).squeeze(1) - lg.logsumexp(-1)).sum()
        g = onehot - torch.softmax(lg, -1)
        gW[p] = g.t() @ Xd
        gb[p] = g.sum(0)
    return s, gW, gb


def floors(n, P, K):
    kp = 2 if K <= 2 else 4 if K <= 4 else 8 if K <= 8 else 16
    hbm = (n * 32 * 4 + n * 8) / HBM_BPS
    # the epilogue issues per padded logit one ex2 plus, per thread and (particle, row), one rcp and one lg2:
    # 2 ops per padded logit for KP = 16 (a thread's two rows belong to one particle), 3 for KP <= 8
    mufu = P * n * kp * (2 if kp == 16 else 3) / MUFU_OPS
    # GEMM 1 (W hi + lo) and GEMM 2 ([X | 1], 40 columns) over P * Kp rows
    tensor = (2 * 2 * P * kp * n * 32 + 2 * P * kp * n * 40) / TF32_FLOPS
    return hbm, mufu, tensor


def accuracy(dev, quick):
    ok = True
    cases = [(300, 7, 3, True), (8191, 65, 16, False), (70001, 16, 10, True), (1000000, 64, 10, True),
             (1000000, 64, 2, True), (1000000, 64, 16, False)]
    if quick:
        cases = cases[:3]
    for n, P, K, bias in cases:
        X = torch.randn(n, 32, device=dev)
        Wt = torch.randn(K, 32, device=dev) / 32 ** 0.5
        y = torch.distributions.Categorical(logits=X @ Wt.t()).sample()
        W = (Wt + 0.3 * torch.randn(P, K, 32, device=dev)).contiguous()
        b = 0.2 * torch.randn(P, K, device=dev) if bias else None
        s_ref, gW, gb = reference(X, y, W, b)
        call, (total, sum_p, dW, db) = run(X, y, W, b)
        call()
        torch.cuda.synchronize()
        e_sum = float(((sum_p.double() - s_ref).abs() / s_ref.abs().clamp_min(1.0)).max())
        e_tot = float((total.double() - s_ref.sum()).abs() / s_ref.sum().abs())
        e_dw = float((dW.double() - gW).abs().max() / gW.abs().max().clamp_min(1.0))
        e_db = float((db.double() - gb).abs().max() / gb.abs().max().clamp_min(1.0))
        print("CASE n=%d P=%d K=%d bias=%d rel err: sum_p %.2e total %.2e dW %.2e db %.2e"
              % (n, P, K, bias, e_sum, e_tot, e_dw, e_db))
        if not (e_sum < 2e-5 and e_dw < 2e-4 and e_db < 2e-4):
            print("   ^^^ OUT OF TOLERANCE")
            ok = False
    return ok


def kernel_time(dev):
    n, P, K = 1000000, 64, 10
    X = torch.randn(n, 32, device=dev)
    y = torch.randint(0, K, (n,), device=dev)
    W = 0.3 * torch.randn(P, K, 32, device=dev)
    b = torch.randn(P, K, device=dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    call, _ = run(X, y, W, b)
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
    hbm, mufu, tensor = floors(n, P, K)
    print("TIME kernel + finish N=1e6 D=32 P=64 K=10: median %.1f us (min %.1f, max %.1f)" % (med, ts[0], ts[-1]))
    print("     floors (H100 SXM data sheet): HBM %.1f us, MUFU %.1f us, TF32 tensor %.1f us -> %.2fx the largest"
          % (hbm * 1e6, mufu * 1e6, tensor * 1e6, med / (max(hbm, mufu, tensor) * 1e6)))


def svi_steps(dev, reps):
    import models
    import pyro_b200 as pyro
    import pyro_b200.distributions as dist
    from pyro_b200.infer import SVI, Trace_ELBO
    from pyro_b200.infer import elbo as elbo_mod
    from pyro_b200.optim import ClippedAdam
    from test_glm_categorical import softmax_guide, softmax_model

    n, D, P, K = 1000000, 32, 64, 10
    torch.manual_seed(0)
    X = torch.randn(n, D, device=dev)
    y = torch.distributions.Categorical(logits=X @ (torch.randn(K, D, device=dev) / D ** 0.5).t()).sample()
    eW, eb = torch.randn(P, 1, K, D, device=dev), torch.randn(P, 1, K, device=dev)

    def guide(*args):
        with models.InjectNoise({"W": eW, "b": eb}):
            softmax_guide(*args)

    calls = []
    real = dist._GlmCategoricalFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)
    dist._GlmCategoricalFn.apply = spy

    def one(lazy, steps):
        elbo_mod.LAZY_LINEAR = lazy
        pyro.clear_param_store()
        svi = SVI(softmax_model, guide, ClippedAdam({"lr": 0.01}),
                  Trace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        loss = svi.step(X, y, K)   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            loss = svi.step(X, y, K)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3, loss

    res = {True: [], False: []}
    try:
        for _ in range(reps):
            for lazy in (True, False):
                ms, loss = one(lazy, 5)
                res[lazy].append(ms)
                print("SVI step %-12s %.2f ms  loss %.6e" % ("fused" if lazy else "materialised", ms, loss))
    finally:
        dist._GlmCategoricalFn.apply = real
        elbo_mod.LAZY_LINEAR = True
    print("SVI fused kernel calls: %d" % len(calls))
    print("SVI step fused %s ms, materialised %s ms" % (["%.2f" % v for v in res[True]], ["%.2f" % v for v in res[False]]))


def main():
    quick = "--quick" in sys.argv
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU", q.stdout.strip())
    torch.manual_seed(0)
    ok = accuracy(dev, quick)
    kernel_time(dev)
    svi_steps(dev, 1 if quick else 3)
    print("GLM_CATEGORICAL_CHECK", "OK" if ok else "FAIL", time.strftime("%H:%M:%S"))


if __name__ == "__main__":
    main()
