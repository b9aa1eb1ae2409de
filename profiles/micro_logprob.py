"""Micro-benchmark of the fused log_prob(+score) kernels per family (SURVEY.md 8d "micro log_prob"):
elementwise-stored operands, M = 2^26 elements (event families: rows x K), device time from a
CUDA-graph replay between CUDA events, L2 flushed between replays.  Prints achieved GB/s on the
ALGORITHMIC bytes (operands once at stored shape; + gradient outputs when requested) and the
fraction of the measured HBM copy peak."""
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyro_b200.distributions as dist  # noqa: E402
from pyro_b200.optim import ClippedAdam  # noqa: E402
import pyro_b200 as pyro  # noqa: E402

RESULTS = {}
VERBOSE = True
ONLY = None


def run(verbose=True, only=None):
    """Run the table; returns {row name: {ms, GBps, frac, algorithmic_bytes}} (bench.py puts it under
    ``variants.micro`` so the driver re-measures it every round).  ``only``: regular expression selecting rows."""
    global VERBOSE, ONLY
    VERBOSE = verbose
    ONLY = re.compile(only) if only else None
    RESULTS.clear()
    _run()
    return dict(RESULTS)


def _run():
    global flush, peak
    dev = "cuda"
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0  # H100 SXM data sheet
    M = 1 << 26
    torch.manual_seed(0)
    flush = torch.empty(64 * 1024 * 1024, device=dev)


    def timed(name, fn, nbytes, reps=5):
        if ONLY is not None and not ONLY.search(name):
            return
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fn()
        ts = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); graph.replay(); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = min(ts)
        gbs = nbytes / ms / 1e6
        RESULTS[name] = {"ms": round(ms, 4), "GBps": round(gbs, 1), "frac": round(gbs / peak, 3),
                         "algorithmic_bytes": int(nbytes)}
        if VERBOSE:
            print("%-44s %8.3f ms %8.1f GB/s  %5.1f%% of %.0f" % (name, ms, gbs, 100 * gbs / peak, peak))


    x = torch.randn(M, device=dev)
    loc = torch.randn(M, device=dev)
    pos = torch.rand(M, device=dev) * 2 + 0.5
    pos2 = torch.rand(M, device=dev) * 2 + 0.5
    unit = torch.rand(M, device=dev).clamp(0.01, 0.99)
    cnt = torch.poisson(pos * 2)
    bern = (unit > 0.5).float()
    fams = [
        ("Normal(loc,scale)", lambda g: dist.Normal(loc.requires_grad_(g), pos), x, 12),
        ("Cauchy(loc,scale)", lambda g: dist.Cauchy(loc.requires_grad_(g), pos), x, 12),
        ("HalfCauchy(scale)", lambda g: dist.HalfCauchy(pos.requires_grad_(g)), x.abs(), 8),
        ("Exponential(rate)", lambda g: dist.Exponential(pos.requires_grad_(g)), x.abs(), 8),
        ("Bernoulli(logits)", lambda g: dist.Bernoulli(logits=loc.requires_grad_(g)), bern, 8),
        ("Poisson(rate)", lambda g: dist.Poisson(pos.requires_grad_(g)), cnt, 8),
        ("Gamma(conc,rate)", lambda g: dist.Gamma(pos.requires_grad_(g), pos2), x.abs() + 0.01, 12),
        ("Beta(c1,c0)", lambda g: dist.Beta(pos.requires_grad_(g), pos2), unit, 12),
        ("LogNormal(loc,scale)", lambda g: dist.LogNormal(loc.requires_grad_(g), pos), x.abs() + 0.01, 12),
    ]
    for name, mk, val, bpe in fams:
        timed(name + " sum", lambda: mk(False)._fused_sum(val, None, 1.0, 1.0, 1.0, True), M * bpe)
        timed(name + " sum + d/dparam0 (full)", lambda: mk(True)._fused_sum(val, None, 1.0, 1.0, 1.0, True), M * (bpe + 4))
        loc.requires_grad_(False); pos.requires_grad_(False)
    # materialised log_prob (drop-in API) and its backward
    timed("Normal log_prob materialised", lambda: dist.Normal(loc, pos).log_prob(x), M * 16)
    # event families
    for K in (8, 64, 1024):
        rows = M // K
        conc = torch.rand(rows, K, device=dev) * 2 + 0.3
        v = torch.distributions.Dirichlet(torch.ones(K, device=dev)).sample((1024,)).repeat(rows // 1024, 1).clamp(min=1e-6)
        timed("Dirichlet K=%d log_prob" % K, lambda: dist.Dirichlet(conc).log_prob(v), rows * (8 * K + 4))
        logits = torch.randn(rows, K, device=dev)
        idx = torch.randint(0, K, (rows,), device=dev)
        timed("Categorical K=%d log_prob" % K, lambda: dist.Categorical(logits=logits).log_prob(idx), rows * (4 * K + 12))
    for n in (2, 8, 32):
        rows = (1 << 25) // (n * n)
        A = torch.randn(rows, n, n, device=dev)
        # cholesky returns column-major matrices; the kernels want row-major events (a one-off copy here, not timed)
        L = torch.linalg.cholesky(A @ A.transpose(-1, -2) + n * torch.eye(n, device=dev)).contiguous()
        assert L.stride()[-1] == 1
        mu, xv = torch.randn(rows, n, device=dev), torch.randn(rows, n, device=dev)
        timed("MVN n=%d log_prob (per-row scale_tril)" % n, lambda: dist.MultivariateNormal(mu, scale_tril=L).log_prob(xv),
              rows * (4 * n * n + 8 * n + 4))
    # optimiser: 28 B / element (+4 for the fused zeroing)
    p = torch.randn(M, device=dev, requires_grad=True)
    p.grad = torch.randn(M, device=dev)
    pyro.get_param_store()._param_to_name[p] = "p"
    opt = ClippedAdam({"lr": 1e-3})
    opt([p])
    timed("ClippedAdam fused (p,g,m,v; zero g)", lambda: opt([p]), M * 32)


if __name__ == "__main__":
    run(True, only=sys.argv[1] if len(sys.argv) > 1 else None)
