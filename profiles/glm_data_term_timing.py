"""Device time of the Poisson and Binomial likelihood calls (kernel + finish) at N = 1e6, P = 64, the cases whose data
term (SUM lgamma(y + 1), SUM log C(m, y)) each CTA sums in fp64 and folds into its lp partials, with the logistic
call beside them.  CUDA events around 20 back-to-back calls, median of 15 windows, after a warm-up; X (128 MB at
D = 32) does not fit in L2, so no flush is needed.  One JSON line per configuration, with the card's name.

    python profiles/glm_data_term_timing.py [path/to/libpyro_b200.so]

The optional library path times another build of the same C ABI (a parent commit's, say) with the same script, so
that two builds can be compared in alternating runs on one machine."""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyro_b200 import _native as N  # noqa: E402

if len(sys.argv) > 1:
    N.LIB_PATH = os.path.abspath(sys.argv[1])
DEV = torch.device("cuda")
n, P = 1_000_000, 64


def timed(call, windows=15, per=20):
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(per):
            call()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / per)
    return statistics.median(ts), min(ts)


def setup(D, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=g)
    wt = 0.3 * torch.randn(D, generator=g) / D ** 0.5
    W = wt + 0.01 * torch.randn(P, D, generator=g)
    return X, wt, W


def main():
    L = N.lib()
    st = N.stream_ptr(DEV)
    name = torch.cuda.get_device_name()
    for D in (10, 32):
        X, wt, W = setup(D, D)
        l = X @ wt
        Xg, Wg = X.to(DEV), W.to(DEV)
        out = [torch.empty(P, device=DEV), torch.empty((), device=DEV), torch.empty(P, D, device=DEV),
               torch.empty(P, device=DEV)]
        ptrs = [t.data_ptr() for t in out]
        cases = []
        for level in (0.0, 4.6):
            y = torch.poisson(torch.exp(l + level)).to(DEV)
            b = torch.full((P,), level, device=DEV)
            ws = N.workspace(DEV, int(L.b2_glm_poisson_workspace(n, D, P)), tag="timing")
            cases.append(("poisson level %.1f" % level, lambda y=y, b=b, ws=ws: L.b2_glm_poisson_log_rate(
                Xg.data_ptr(), y.data_ptr(), Wg.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, *ptrs,
                ws.data_ptr(), ws.numel(), st)))
        for m in (10, 1000, "rows"):
            mt = (torch.randint(1, 1001, (n,)).float() if m == "rows" else torch.full((1,), float(m))).to(DEV)
            mm = mt if m == "rows" else mt.expand(n)
            y = torch.binomial(mm.cpu().expand(n).contiguous(), torch.sigmoid(l)).to(DEV)
            b = torch.zeros(P, device=DEV)
            ws = N.workspace(DEV, int(L.b2_glm_binomial_workspace(n, D, P)), tag="timing")
            cases.append(("binomial m=%s" % m, lambda y=y, b=b, ws=ws, mt=mt, r=int(m == "rows"):
                          L.b2_glm_binomial_logits(Xg.data_ptr(), y.data_ptr(), mt.data_ptr(), r, Wg.data_ptr(),
                                                   b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, *ptrs, ws.data_ptr(),
                                                   ws.numel(), st)))
        y = torch.bernoulli(torch.sigmoid(l)).to(DEV)
        b = torch.zeros(P, device=DEV)
        ws = N.workspace(DEV, int(L.b2_glm_workspace(n, D, P)), tag="timing")
        cases.append(("bernoulli", lambda y=y, b=b, ws=ws: L.b2_glm_bernoulli_logits(
            Xg.data_ptr(), y.data_ptr(), Wg.data_ptr(), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, 0, *ptrs,
            ws.data_ptr(), ws.numel(), st)))
        for label, call in cases:
            N.check(call(), label)
            med, best = timed(call)
            print(json.dumps({"lib": N.LIB_PATH, "case": label, "D": D, "us_median": round(med, 2),
                              "us_min": round(best, 2), "gpu": name}))


if __name__ == "__main__":
    main()
