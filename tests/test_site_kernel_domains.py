"""The site and event scoring kernels (``b2_site_score``, ``b2_event_score``) across each family's parameter
domain and on every kernel path the host selector can take, against the fp64 oracle (oracle/dists.py).

Reference.  Inputs are rounded to the kernel dtype first; the oracle formula is then evaluated on those rounded
inputs in fp64 on the CPU, with autograd for the gradients.

Tolerance rule.  With r the fp64 reference and k the kernel result:
  * fp64:  |k - r| <= 1e-12 * max(1, |r|) + kappa * 2^-52 * S
  * fp32:  |k - r| <= max(1e-5 * max(1, |r|), kappa * 2^-23 * S), with 2e-4 in place of 1e-5 for gradients
S is the sum of the magnitudes of the formula's terms, computed in fp64 (for a gradient: the sum of the magnitudes
of the terms' partial derivatives), so an ill-conditioned point is held to what the dtype can represent there
instead of being waved through.  kappa is one constant per family (``KAPPA``).  Finiteness must match: the kernel
is +-inf or NaN exactly where the reference is, except where torch's own fp32 evaluation of the oracle overflows
in the same direction.  Failure messages report torch fp32's error next to the kernel's.

One convention differs from torch: the kernels differentiate xlogy(a, y) = a*log(y) analytically, so d/da is
log(y) everywhere, while torch's xlogy backward returns 0 where a == 0 and y <= 0 (a Poisson count of 0 at rate
0: the kernel's value gradient is -inf there).  The reference takes the analytic derivative, and
``test_xlogy_coefficient_gradient_is_analytic`` pins both.

The CPU tier runs the same grids through the host build of the element functors (tests/hostcheck.py); the
``gpu`` tier runs them through the kernels, one shape per kernel path, and ``test_kernel_routing`` proves with
the profiler that those shapes reach the kernels they are meant for.
"""
import math
from unittest import mock

import numpy as np
import pytest
import torch

from conftest import EMULATE, device
from oracle import dists as odists

DEV = device()
F32_TINY = float(np.finfo(np.float32).tiny)

# ---------------------------------------------------------------------------------------------------------------
# reference: fp64 oracle with autograd
# ---------------------------------------------------------------------------------------------------------------
_torch_xlogy = torch.xlogy


class _XlogyAnalytic(torch.autograd.Function):
    """torch.xlogy with d/da = log(y) everywhere (torch's backward returns 0 where a == 0 and y <= 0)."""

    @staticmethod
    def forward(ctx, a, y):
        ctx.save_for_backward(a, y)
        return _torch_xlogy(a, y)

    @staticmethod
    def backward(ctx, g):
        a, y = ctx.saved_tensors
        return g * torch.log(y), g * a / y


_torch_digamma = torch.digamma


class _DigammaAccurate(torch.autograd.Function):
    """torch.digamma whose backward is scipy's trigamma (torch's fp64 polygamma(1) is only ~1e-9 accurate)."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return _torch_digamma(x)

    @staticmethod
    def backward(ctx, g):
        from scipy.special import polygamma
        (x,) = ctx.saved_tensors
        return g * torch.as_tensor(polygamma(1, x.detach().double().numpy()), dtype=x.dtype)


def _xlogy(a, y):
    a, y = torch.broadcast_tensors(torch.as_tensor(a, dtype=y.dtype), y)
    return _XlogyAnalytic.apply(a, y)


def _sp(l):
    return torch.logaddexp(l, torch.zeros_like(l))


def _probs_logits(p):
    eps = torch.finfo(p.dtype).eps
    pc = p.clamp(min=eps, max=1 - eps)
    return torch.log(pc) - torch.log1p(-pc)


def _lg(v):
    return torch.lgamma(v)


# terms of each formula (their sum is the log density), used for the condition measure S
def _terms_binomial(k, n, l):
    with torch.no_grad():
        lb = [_lg(n + 1), -_lg(k + 1), -_lg(n - k + 1)]
    return [k * l, -n * _sp(l)] + lb


TERMS = {
    0: lambda x, m, s: [-((x - m) ** 2) / (2 * s * s), -s.log(), torch.full_like(x, -odists.LOG_SQRT_2PI)],
    1: lambda x, l: [x * l, -_sp(l)],
    2: lambda x, a, b: [_xlogy(a, b), _xlogy(a - 1, x), -b * x, -_lg(a)],
    3: lambda x, c1, c0: [_xlogy(c1 - 1, x), _xlogy(c0 - 1, 1 - x), _lg(c1 + c0), -_lg(c1), -_lg(c0)],
    4: lambda x, r: [_xlogy(x, r), -r, -_lg(x + 1)],
    5: lambda x, m, s: [torch.full_like(x, -math.log(math.pi)), -s.log(), -(((x - m) / s) ** 2).log1p()],
    6: lambda x, s: [torch.full_like(x, math.log(2 / math.pi)), -s.log(), -((x / s) ** 2).log1p()],
    7: lambda x, r: [r.log(), -r * x],
    # log x is a rounded intermediate: (log x - loc)^2 enters S expanded, so its cancellation is measured
    8: lambda x, m, s: [-(x.log() ** 2) / (2 * s * s), x.log() * m / (s * s), -(m * m) / (2 * s * s), -s.log(),
                        torch.full_like(x, -odists.LOG_SQRT_2PI), -x.log()],
    9: lambda x, s: [-(x * x) / (2 * s * s), -s.log(), torch.full_like(x, math.log(2) - odists.LOG_SQRT_2PI)],
    10: lambda x, p: [x * _probs_logits(p), -_sp(_probs_logits(p))],
    11: lambda x, lo, hi: [-torch.log(hi - lo)],
    12: lambda x, mp, sp, mq, sq: [0.5 * (sp / sq) ** 2, 0.5 * ((mp - mq) / sq) ** 2, torch.full_like(mp, -0.5),
                                   -torch.log(sp / sq)],
    13: lambda x, ap, bp, aq, bq: [aq * (bp / bq).log(), _lg(aq), -_lg(ap), (ap - aq) * torch.digamma(ap),
                                   (bq - bp) * (ap / bp)],
    16: _terms_binomial,
    17: lambda k, n, p: _terms_binomial(k, n, _probs_logits(p)),
}
# partial derivatives that the oracle's own autograd graph forms by cancellation, added to S of a gradient: the
# fp64 reference carries their rounding (KL Gamma's d/d rate_p sums -conc_p/rate_p and (rate_q - rate_p) *
# conc_p/rate_p^2)
EXTRA_SG = {13: lambda ap, bp, aq, bq: {2: 2 * (ap / bp).abs() + (bq * ap / (bp * bp)).abs(),
                                         1: ((bq - bp) / bp).abs()}}
# the probs families clamp to the kernel dtype's eps (torch's clamp_probs uses the eps of the probs' dtype)
PROBS_SLOT = {10: 0, 17: 1}
HAS_VALUE = {f: f not in (12, 13) for f in TERMS}
NPARAMS = {f: odists.ELEMENTWISE[f][1] for f in TERMS}
KAPPA = {f: 32 for f in TERMS}


def _oracle(fam):
    return odists.ELEMENTWISE[fam][0]


def _leaves(arrs, shape, dtype):
    return [None if a is None else
            torch.tensor(np.broadcast_to(a, shape), dtype=dtype).requires_grad_(True) for a in arrs]


def _grads(out, leaves):
    want = [t for t in leaves if t is not None]
    gs = list(torch.autograd.grad(out.sum(), want, allow_unused=True, retain_graph=True))
    res = []
    for t in leaves:
        if t is None:
            res.append(None)
            continue
        g = gs.pop(0)
        res.append(np.zeros(t.shape) if g is None else g.detach().double().numpy())
    return res


def reference(fam, x, params, shape, kdtype=np.float64):
    """fp64 oracle on the (already rounded) inputs, broadcast to ``shape``: lp, per-element gradients of
    [value, *params], their condition measures S, and torch fp32's own lp and gradients."""
    fn0 = _oracle(fam)
    fn = fn0
    if fam in PROBS_SLOT and kdtype == np.float32:
        e = float(np.finfo(np.float32).eps)

        def fn(x_, *p):
            p = list(p)
            p[PROBS_SLOT[fam]] = p[PROBS_SLOT[fam]].clamp(min=e, max=1 - e)
            return fn0(x_, *p)
    out = {}
    with mock.patch.object(torch, "xlogy", _xlogy), mock.patch.object(torch, "digamma", _DigammaAccurate.apply):
        for dt, key in ((torch.float64, "r"), (torch.float32, "t32")):
            leaves = _leaves([x if HAS_VALUE[fam] else None] + list(params), shape, dt)
            xin = leaves[0] if HAS_VALUE[fam] else None
            lp = fn(xin, *leaves[1:]).expand(shape)
            out[key] = (lp.detach().double().numpy(), _grads(lp, leaves))
        leaves = _leaves([x if HAS_VALUE[fam] else torch.zeros(())] + list(params), shape, torch.float64)
        tl = list(leaves)
        if fam in PROBS_SLOT and kdtype == np.float32:
            e = float(np.finfo(np.float32).eps)
            tl[1 + PROBS_SLOT[fam]] = tl[1 + PROBS_SLOT[fam]].clamp(min=e, max=1 - e)
        terms = [t.expand(shape) for t in TERMS[fam](*tl)]
        s_lp = sum(t.detach().abs() for t in terms).numpy()
        s_g = [np.zeros(shape) for _ in leaves]
        for t in terms:
            if not t.requires_grad:
                continue
            for i, g in enumerate(_grads(t, leaves)):
                s_g[i] = s_g[i] + np.abs(np.nan_to_num(g, nan=0.0, posinf=np.inf, neginf=np.inf))
        if fam in EXTRA_SG:
            for i, v in EXTRA_SG[fam](*[t.detach() for t in tl[1:]]).items():
                s_g[i] = s_g[i] + v.numpy()
    if not HAS_VALUE[fam]:
        out["r"][1][0] = np.zeros(shape)
        out["t32"][1][0] = np.zeros(shape)
    return {"lp": out["r"][0], "g": out["r"][1], "lp32": out["t32"][0], "g32": out["t32"][1],
            "s_lp": s_lp, "s_g": s_g}


def tolerance(ref, S, dtype, kappa, grad):
    a = np.abs(np.nan_to_num(ref, nan=0.0, posinf=0.0, neginf=0.0))
    S = np.nan_to_num(S, nan=0.0, posinf=np.inf)
    if dtype == np.float64:
        return 1e-12 * np.maximum(1, a) + kappa * 2.0 ** -52 * S
    return np.maximum((2e-4 if grad else 1e-5) * np.maximum(1, a), kappa * 2.0 ** -23 * S)


def check(what, got, ref, S, ref32, dtype, kappa, grad, inputs=None, exact_zero=None):
    """The tolerance rule on arrays of one shape; ``exact_zero`` marks entries that must be exactly 0."""
    got = np.asarray(got, np.float64)
    ref = np.broadcast_to(np.asarray(ref, np.float64), got.shape)
    ref32 = np.broadcast_to(np.asarray(ref32, np.float64), got.shape)
    S = np.broadcast_to(np.asarray(S, np.float64), got.shape)
    msgs = []
    if exact_zero is not None:
        nz = exact_zero & (got != 0)
        if nz.any():
            msgs.append("%d masked-out entries are not exactly 0 (first %r)" % (nz.sum(), got[nz][:3]))
        live = ~exact_zero
    else:
        live = np.ones(got.shape, bool)
    fr, fk = np.isfinite(ref), np.isfinite(got)
    overflow_like_torch = fr & ~fk & (ref32 == got)
    bad_fin = live & (fr != fk) & ~overflow_like_torch
    both_nf = live & ~fr & ~fk
    bad_nf = both_nf & ~((np.isnan(ref) & np.isnan(got)) | (ref == got))
    tol = tolerance(ref, S, dtype, kappa, grad)
    both = live & fr & fk
    err = np.where(both, np.abs(got - ref), 0.0)
    bad_val = both & (err > tol)
    for name, bad in (("finiteness", bad_fin | bad_nf), ("value", bad_val)):
        if not bad.any():
            continue
        idx = np.argwhere(bad)
        worst = tuple(idx[np.argmax((err / np.where(tol > 0, tol, 1))[bad])]) if name == "value" else tuple(idx[0])
        e32 = abs(ref32[worst] - ref[worst])
        inp = "" if inputs is None else " inputs=%s" % [float(np.broadcast_to(a, got.shape)[worst])
                                                         for a in inputs if a is not None]
        msgs.append("%s: %d bad %s; worst at %s: kernel %.9g ref %.9g (err %.3g, tol %.3g, torch fp32 err %.3g)%s"
                    % (what, bad.sum(), name, worst, got[worst], ref[worst], abs(got[worst] - ref[worst]),
                       tol[worst], e32, inp))
    return msgs


# ---------------------------------------------------------------------------------------------------------------
# domains: random log-uniform draws plus listed edge values, joint edges first
# ---------------------------------------------------------------------------------------------------------------
def _logu(rng, lo, hi, n):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n))


def _sgn(rng, n):
    return np.where(rng.random(n) < 0.5, -1.0, 1.0)


def _f32_around(v):
    c = np.float32(v)
    return [float(np.nextafter(c, np.float32(0))), float(c), float(np.nextafter(c, np.float32(np.inf)))]


def _fill(rng, n, edges, rand):
    """edges: list of tuples (one value per operand); rand(rng, m) -> tuple of arrays.  Edges first, then draws."""
    cols = list(zip(*edges)) if edges else None
    m = n - (len(edges) if edges else 0)
    r = rand(rng, max(m, 0))
    out = []
    for i, col in enumerate(r):
        e = np.asarray(cols[i], np.float64) if cols else np.zeros(0)
        out.append(np.concatenate([e, np.asarray(col, np.float64)])[:n])
    return out


def _normal_like(rng, m, positive=False):
    loc = np.where(rng.random(m) < 0.2, 0.0, _sgn(rng, m) * _logu(rng, 1e-3, 1e3, m))
    scale = _logu(rng, 1e-6, 1e6, m)
    u = _sgn(rng, m) * _logu(rng, 1e-3, 1e3, m)
    if positive:
        loc = np.zeros(m)
    return loc + u * scale, loc, scale


def grid(fam, n, dtype, seed=0):
    """(value, [params]) in fp64, one entry per element; value None for the KL families."""
    rng = np.random.default_rng(seed + 101 * fam)
    eps = float(np.finfo(dtype).eps)
    if fam == 0:
        edges = [(0.0, 0.0, 1e-6), (1e-3, 0.0, 1e-6), (1e9, 0.0, 1e6), (-1e9, 0.0, 1e6), (1.0, 1.0, 1.0),
                 (1e3 + 1e-3, 1e3, 1e-6)]
        x, loc, s = _fill(rng, n, edges, lambda r, m: _normal_like(r, m))
        return x, [loc, s]
    if fam == 1:
        l_e = [0.0, 100.0, -100.0, 88.0, -88.0, 20.0, -20.0, 1e-4]
        edges = [(y, l) for l in l_e for y in (0.0, 1.0)]
        return tuple_xp(_fill(rng, n, edges, lambda r, m: (r.integers(0, 2, m).astype(float),
                                                            _sgn(r, m) * _logu(r, 1e-4, 100, m))))
    if fam in (10, 17):
        pe = [0.0, eps / 4, eps / 2, eps, 2 * eps, 0.5, 1 - 2 * eps, 1 - eps, 1 - eps / 2, 1.0]

        def rp(r, m):
            lo = _logu(r, 1e-9, 0.5, m)
            return np.where(r.random(m) < 0.5, lo, 1 - lo)
        if fam == 10:
            edges = [(y, p) for p in pe for y in (0.0, 1.0)]
            return tuple_xp(_fill(rng, n, edges, lambda r, m: (r.integers(0, 2, m).astype(float), rp(r, m))))
        edges = [(k, 10.0, p) for p in pe for k in (0.0, 3.0, 10.0)]
        return tuple_xp(_fill(rng, n, edges, lambda r, m: _binom_counts(r, m) + (rp(r, m),)))
    if fam == 2:
        a_e = _f32_around(1e-30) + _f32_around(1e30) + [1e-6, 1e7, 1.0, 0.5, 3.999999, 4.0, 4.000001]
        edges = [(x, a, b) for a in a_e for (x, b) in ((1.3, 0.7), (1e-20, 1e-6), (1e6, 1e6), (1.0, 1.0))]
        edges += [(0.0, 1.0, 2.0)]
        return tuple_xp(_fill(rng, n, edges, lambda r, m: (_logu(r, 1e-20, 1e6, m), _logu(r, 1e-6, 1e7, m),
                                                            _logu(r, 1e-6, 1e6, m))))
    if fam == 3:
        c_e = _f32_around(1e-6) + [1e-7, 1e9, 1.0, 0.5, 4.0]
        edges = [(x, c1, c0) for c1 in c_e for c0 in (1e-7, 1.0, 2.5, 1e9) for x in (0.37, 1e-20)]
        edges += [(0.5, a, b) for a, b in ((5e8, 5e8), (4.9999997e8, 5.0000003e8), (5e8, 5.0001e8), (1e9, 1.0))]
        edges += [(1 - 1e-7, 2.0, 3.0), (1 - 6e-8, 0.5, 0.5), (1e-30, 0.5, 0.5)]

        def rb(r, m):
            lo = _logu(r, 1e-20, 0.5, m)
            return np.where(r.random(m) < 0.5, lo, 1 - _logu(r, 6e-8, 0.5, m)), _logu(r, 1e-7, 1e9, m), \
                _logu(r, 1e-7, 1e9, m)
        return tuple_xp(_fill(rng, n, edges, rb))
    if fam == 4:
        edges = [(float(k), r) for k in range(66) for r in (0.7, 40.0)]
        edges += [(0.0, 0.0), (0.0, 1e-6), (1e6, 1e6), (1e6, 1e-6), (2.5, 3.0), (63.5, 60.0), (64.0, 64.0)]

        def rpois(r, m):
            k = np.where(r.random(m) < 0.5, r.integers(0, 70, m).astype(float), np.round(_logu(r, 1, 1e6, m)))
            k = np.where(r.random(m) < 0.15, _logu(r, 1e-3, 1e3, m), k)   # non-integer counts
            return k, _logu(r, 1e-6, 1e6, m)
        return tuple_xp(_fill(rng, n, edges, rpois))
    if fam == 16:
        edges = [(k, nn, l) for nn, k in ((0.0, 0.0), (10.0, 0.0), (10.0, 10.0), (100.0, 37.0), (127.0, 64.0),
                                          (126.0, 63.0), (64.0, 1.0), (1e6, 0.0), (1e6, 1e6), (1e6, 1e6 - 63),
                                          (1e6, 1e6 - 64), (1e6, 5e5))
                 for l in (0.0, 3.0, -3.0, 100.0, -100.0)]
        return tuple_xp(_fill(rng, n, edges, lambda r, m: _binom_counts(r, m) + (_sgn(r, m) * _logu(r, 1e-4, 100, m),)))
    if fam in (5, 6):
        def rc(r, m):
            loc = np.zeros(m) if fam == 6 else np.where(r.random(m) < 0.2, 0.0, _sgn(r, m) * _logu(r, 1e-3, 1e3, m))
            s = _logu(r, 1e-6, 1e6, m)
            u = _logu(r, 1e-3, 1e19, m) * (np.abs(_sgn(r, m)) if fam == 6 else _sgn(r, m))
            x = loc + u * s
            if fam == 6:
                x = np.where(r.random(m) < 0.05, -x, x)
                return x, s
            return x, loc, s
        if fam == 6:
            edges = [(0.0, 1.0), (-1.0, 1.0), (-1e-30, 1e-6), (1e25, 1e6), (1e13, 1e-6)]
        else:
            edges = [(0.0, 0.0, 1.0), (1e25, 0.0, 1e6), (-1e13, 0.0, 1e-6), (1e3, 1e3, 1e-6)]
        return tuple_xp(_fill(rng, n, edges, rc))
    if fam == 7:
        edges = [(0.0, 1e-6), (0.0, 1e6), (1e6, 1e6), (1e-6, 1e-6), (-1.0, 2.0)]
        return tuple_xp(_fill(rng, n, edges, lambda r, m: (_logu(r, 1e-6, 1e6, m), _logu(r, 1e-6, 1e6, m))))
    if fam == 8:
        def rln(r, m):
            x = _logu(r, 1e-20, 1e20, m)
            s = _logu(r, 1e-6, 1e6, m)
            u = _sgn(r, m) * _logu(r, 1e-3, 1e3, m)
            loc = np.where(r.random(m) < 0.5, np.log(x) - u * s, r.uniform(-50, 50, m))
            return x, loc, s
        edges = [(1e-20, 0.0, 1.0), (1e20, 0.0, 1e6), (1.0, 0.0, 1e-6), (math.e, 1.0, 1.0)]
        return tuple_xp(_fill(rng, n, edges, rln))
    if fam == 9:
        def rhn(r, m):
            x, _, s = _normal_like(r, m, positive=True)
            x = np.abs(x)
            return np.where(r.random(m) < 0.05, -x, x), s
        edges = [(0.0, 1.0), (-1.0, 1.0), (-1e-30, 1e-6), (1e9, 1e6), (1e-3, 1e-6)]
        return tuple_xp(_fill(rng, n, edges, rhn))
    if fam == 11:
        def ru(r, m):
            lo = _sgn(r, m) * _logu(r, 1e-3, 1e3, m)
            w = _logu(r, 1e-3, 1e3, m) * np.maximum(1.0, np.abs(lo))
            t = r.uniform(-0.2, 1.2, m)
            return lo + t * w, lo, lo + w
        edges = [(1.0, 1.0, 2.0), (2.0, 1.0, 2.0), (0.0, -1.0, 1.0), (-1.0, -1.0, 1.0), (3.0, -1.0, 1.0)]
        x, lo, hi = _fill(rng, n, edges, ru)
        # values on both bounds of the rounded interval
        k = max(n // 20, 1)
        x = x.copy()
        x[len(edges):len(edges) + k] = lo[len(edges):len(edges) + k].astype(dtype)
        x[len(edges) + k:len(edges) + 2 * k] = hi[len(edges) + k:len(edges) + 2 * k].astype(dtype)
        return x, [lo, hi]
    if fam == 12:
        def rkn(r, m):
            return (_sgn(r, m) * _logu(r, 1e-3, 1e3, m), _logu(r, 1e-3, 1e3, m),
                    _sgn(r, m) * _logu(r, 1e-3, 1e3, m), _logu(r, 1e-3, 1e3, m))
        ps = _fill(rng, n, [(0.0, 1.0, 0.0, 1.0), (1e3, 1e-3, -1e3, 1e3), (0.5, 1e3, 0.5, 1e-3)], rkn)
        return None, ps
    if fam == 13:
        def rkg(r, m):
            return (_logu(r, 1e-6, 1e7, m), _logu(r, 1e-6, 1e6, m), _logu(r, 1e-6, 1e7, m), _logu(r, 1e-6, 1e6, m))
        ps = _fill(rng, n, [(1.0, 1.0, 1.0, 1.0), (1e-6, 1.0, 1e7, 1e6), (1e7, 1e6, 1e-6, 1e-6), (4.0, 2.0, 3.999999, 2.0)],
                   rkg)
        return None, ps
    raise KeyError(fam)


def _binom_counts(r, m):
    nn = np.where(r.random(m) < 0.5, r.integers(0, 130, m).astype(float), np.round(_logu(r, 1, 1e6, m)))
    k = np.floor(r.random(m) * (nn + 1))
    k = np.where(r.random(m) < 0.1, np.maximum(nn - 63, 0), k)
    k = np.where(r.random(m) < 0.1, np.maximum(nn - 64, 0), k)
    return k, nn


def tuple_xp(cols):
    return cols[0], list(cols[1:])


def rounded(arrs, dtype):
    return [None if a is None else np.asarray(a, dtype).astype(np.float64) for a in arrs]


ELEM_FAMS = sorted(TERMS)
NAMES = {0: "normal", 1: "bernoulli_logits", 2: "gamma", 3: "beta", 4: "poisson", 5: "cauchy", 6: "halfcauchy",
         7: "exponential", 8: "lognormal", 9: "halfnormal", 10: "bernoulli_probs", 11: "uniform", 12: "kl_normal",
         13: "kl_gamma", 16: "binomial_logits", 17: "binomial_probs"}
DTYPES = [(np.float64, torch.float64), (np.float32, torch.float32)]


# ---------------------------------------------------------------------------------------------------------------
# CPU tier: the host build of the element functors, same grids, same rule
# ---------------------------------------------------------------------------------------------------------------
def _host_eval(fam, x, ps, npdt, grad=True):
    import hostcheck as H
    return H.eval_family(fam, x, ps, npdt, grad=grad)


@pytest.mark.parametrize("npdt", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("fam", ELEM_FAMS, ids=[NAMES[f] for f in ELEM_FAMS])
def test_host_functors_over_domain(fam, npdt):
    n = 3000
    x, ps = grid(fam, n, npdt)
    x, *ps = rounded([x] + ps, npdt)
    ref = reference(fam, x, ps, (n,), npdt)
    lp, dx, dp = _host_eval(fam, x, ps, npdt)
    lpf, _, _ = _host_eval(fam, x, ps, npdt, grad=False)
    inputs = [x] + ps
    msgs = check("lp", lp, ref["lp"], ref["s_lp"], ref["lp32"], npdt, KAPPA[fam], False, inputs)
    msgs += check("lp (forward only)", lpf, ref["lp"], ref["s_lp"], ref["lp32"], npdt, KAPPA[fam], False, inputs)
    if HAS_VALUE[fam]:
        msgs += check("d/dvalue", dx, ref["g"][0], ref["s_g"][0], ref["g32"][0], npdt, KAPPA[fam], True, inputs)
    for k in range(len(ps)):
        msgs += check("d/dp%d" % k, dp[k], ref["g"][1 + k], ref["s_g"][1 + k], ref["g32"][1 + k], npdt,
                      KAPPA[fam], True, inputs)
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("npdt", [np.float64, np.float32], ids=["f64", "f32"])
def test_host_fused_draw_functors(npdt):
    """Families 14 / 15 (the fused reparameterised Normal draw and its backward) over the Normal domain: z is
    loc + eps*scale rounded once, lp is Normal(loc, scale).log_prob of that rounded z, and the backward is
    d/dloc = gz, d/dscale = gz*eps - c/scale."""
    n = 3000
    rng = np.random.default_rng(7)
    _, loc, scale = _normal_like(rng, n)
    eps = rng.standard_normal(n) * _logu(rng, 1e-3, 10, n)
    eps, loc, scale = rounded([eps, loc, scale], npdt)
    lp, z, dp = _host_eval(14, eps, [loc, scale], npdt)
    zr = (loc.astype(npdt) + eps.astype(npdt) * scale.astype(npdt)).astype(np.float64)
    tol = (1e-15 if npdt == np.float64 else 2e-7) * (np.abs(loc) + np.abs(eps * scale))
    assert np.all(np.abs(z - zr) <= tol)
    ref = reference(0, z, [loc, scale], (n,), npdt)
    msgs = check("lp", lp, ref["lp"], ref["s_lp"], ref["lp32"], npdt, KAPPA[0], False)
    assert np.all(dp[0] == 0) and np.all(dp[1] == 0)
    gz = rng.standard_normal(n)
    c = np.full(n, 0.37)
    gz, c = rounded([gz, c], npdt)
    _, _, dp = _host_eval(15, gz, [eps, scale, c], npdt)
    assert np.array_equal(dp[0], gz)
    want = gz * eps - c / scale
    S = np.abs(gz * eps) + np.abs(c / scale)
    msgs += check("d/dscale", dp[1], want, S, want, npdt, KAPPA[0], True)
    assert not msgs, "\n".join(msgs)


def test_oracle_binomial_matches_torch():
    """The Binomial oracle restates pyro/distributions/torch.py:83-101: its value is torch.distributions.Binomial's
    log_prob, and (log_binomial under no_grad) its gradients are k - n*sigmoid(l) and -softplus(l)."""
    rng = np.random.default_rng(3)
    n = torch.tensor(np.round(_logu(rng, 1, 1e4, 200)))
    k = torch.floor(torch.rand(200, dtype=torch.float64) * (n + 1))
    l = torch.tensor(rng.standard_normal(200) * 5, requires_grad=True)
    nn = n.clone().requires_grad_(True)
    lp = odists.binomial_logits(k, nn, l)
    ref = torch.distributions.Binomial(n, logits=l.detach()).log_prob(k)
    assert torch.allclose(lp.detach(), ref, rtol=1e-12, atol=1e-9)
    gl, gn = torch.autograd.grad(lp.sum(), [l, nn])
    assert torch.allclose(gl, k - n * torch.sigmoid(l.detach()), rtol=1e-12, atol=1e-12)
    assert torch.allclose(gn, -torch.nn.functional.softplus(l.detach()), rtol=1e-12, atol=1e-12)
    p = torch.sigmoid(l.detach())
    assert torch.allclose(odists.binomial_probs(k, n, p), ref, rtol=1e-9, atol=1e-7)


def test_xlogy_coefficient_gradient_is_analytic():
    """d/da of xlogy(a, y) is log(y) also at a zero coefficient (Gamma / Beta concentration exactly 1, Poisson
    count 0), as torch's backward gives for y > 0; at a Poisson count of 0 and rate 0 the functor's value gradient
    is log(0) - digamma(1) = -inf, where torch's backward masks the log term to 0."""
    for npdt in (np.float64, np.float32):
        _, _, dp = _host_eval(2, np.array([2.0]), [np.array([1.0]), np.array([3.0])], npdt)
        assert abs(dp[0][0] - (math.log(3.0) + math.log(2.0) + 0.5772156649015329)) < 1e-5
        _, _, dp = _host_eval(3, np.array([0.25]), [np.array([1.0]), np.array([2.0])], npdt)
        assert abs(dp[0][0] - (math.log(0.25) + 1.5)) < 1e-5   # psi(3) - psi(1) = 1.5
        _, dx, _ = _host_eval(4, np.array([0.0, 0.0]), [np.array([3.0, 0.0])], npdt)
        assert abs(dx[0] - (math.log(3.0) + 0.5772156649015329)) < 1e-5 and dx[1] == -np.inf
    a = torch.tensor([1.0, 0.0], dtype=torch.float64, requires_grad=True)
    (g,) = torch.autograd.grad(torch.xlogy(a - torch.tensor([1.0, 0.0], dtype=torch.float64),
                                           torch.tensor([2.0, 0.0], dtype=torch.float64)).sum(), a)
    assert g.tolist() == [math.log(2.0), 0.0]   # torch: analytic for y > 0, masked to 0 at a == 0, y == 0


# ---------------------------------------------------------------------------------------------------------------
# GPU tier: element families on every site kernel path
# ---------------------------------------------------------------------------------------------------------------
# path -> (common shape, layout of the value, layout of each parameter, options)
#   layouts: "full" (stored = common shape), "col" ([C], shared by all rows), "row" ([R, 1]), "off" (a view at an
#   element offset of one, so no operand is 16-byte aligned)
R, C = 16, 1024
PATHS = {
    "small": ((6000,), "full", "full", {}),                  # site_small_kernel, full-shape outputs
    "small_bcast": ((48, 96), "col", "rowlast", {}),         # site_small_kernel, mode-3 stored-shape reductions
    "vec": ((R, C), "full", "full", {}),                     # site_vec_kernel
    "vec_shared_value": ((R, C), "col", "full", {}),         # site_vec_kernel, row-invariant value (run_aux)
    "vec_row_param": ((R, C), "full", "rowlast", {}),        # site_vec_kernel, one scalar parameter per row
    "vec_maskup": ((R, C), "full", "full", {"mask": True}),  # site_vec_kernel<MASKUP>
    "gen": ((R * C + 3,), "off", "off", {}),                 # site_gen_kernel
}


def _layout_array(flat, shape, layout, k=0, nparams=1):
    """Stored array of one operand for a path; values come from the front of its grid column."""
    if layout == "rowlast":
        layout = "row" if k == nparams - 1 else "full"
    if layout == "col":
        if len(shape) == 2 and k == 0:
            return flat[: shape[1]].reshape(shape[1])
        layout = "full"
    if layout == "row":
        return flat[: shape[0]].reshape(shape[0], 1)
    n = int(np.prod(shape))
    return flat[:n].reshape(shape)


def _dev_tensor(a, tdt, layout):
    t = torch.as_tensor(np.ascontiguousarray(a), dtype=tdt)
    if layout == "off":
        buf = torch.empty(t.numel() + 1, dtype=tdt, device=DEV)
        buf[1:] = t.reshape(-1).to(DEV)
        return buf[1:].view(t.shape)
    return t.to(DEV)


def _reduce_to(a, stored_shape, shape):
    """Sum a common-shape array to a stored shape (over the dims where the stored operand is broadcast)."""
    st = (1,) * (len(shape) - len(stored_shape)) + tuple(stored_shape)
    axes = tuple(i for i, (s, c) in enumerate(zip(st, shape)) if s == 1 and c != 1)
    return np.sum(a, axis=axes, keepdims=True).reshape(stored_shape) if axes else a.reshape(stored_shape)


def _gather_fail(msgs, label, new):
    msgs.extend("[%s] %s" % (label, m) for m in new)


def run_element_case(fam, npdt, tdt, path, seed=0):
    from pyro_b200 import _native as N
    from pyro_b200.distributions import _ops
    shape, xl, pl, opts = PATHS[path]
    n = int(np.prod(shape))
    x, ps = grid(fam, n, npdt, seed)
    npar = NPARAMS[fam]
    xs = None
    if HAS_VALUE[fam]:
        xs = _layout_array(np.asarray(x, npdt).astype(np.float64), shape, xl if xl != "off" else "full", 0)
        if xl == "col" and fam in (12, 13):
            xs = None
    pss = [_layout_array(np.asarray(p, npdt).astype(np.float64), shape, pl if pl != "off" else "full", k, npar)
           for k, p in enumerate(ps)]
    ref = reference(fam, xs, pss, shape, npdt)
    rng = np.random.default_rng(seed + 7)
    mask = up = None
    scale, weight, coeff = 0.5, -0.25, -2.0   # powers of two: the scaled results are exact
    if opts.get("mask"):
        mask = rng.random(shape) < 0.7
        up = rng.choice([0.5, 1.0, 2.0, -1.0, -0.25], size=shape)
        # NaN parameters under masked-out entries must not leak into any output
        nanpos = (~mask) & (rng.random(shape) < 0.5)
        pss[0] = np.where(nanpos, np.nan, pss[0])
    layout = "off" if xl == "off" else None
    xt = _dev_tensor(xs, tdt, layout) if xs is not None else None
    pt = [_dev_tensor(p, tdt, layout) for p in pss]
    mt = torch.as_tensor(mask, device=DEV) if mask is not None else None
    ut = torch.as_tensor(up, dtype=tdt, device=DEV) if up is not None else None
    live = mask if mask is not None else np.ones(shape, bool)
    f = weight * scale * (up if up is not None else 1.0)
    kap = KAPPA[fam]
    inputs = [np.broadcast_to(a, shape) for a in ([xs] if xs is not None else []) + pss]
    msgs = []
    want_lp = np.where(live, scale * ref["lp"], 0.0)
    for mode in ("forward", "latent", "observed"):
        grad = mode != "forward"
        need_dv = mode == "latent" and xs is not None
        need_dp = [grad] * npar
        out_sum = torch.zeros((), dtype=tdt, device=DEV)
        lp, gv, gp = _ops.site_score(fam, xt, pt, shape, mask=mt, scale=scale, upstream=ut, weight=weight,
                                     sum_coeff=coeff, want_logprob=True, out_sum=out_sum, need_dvalue=need_dv,
                                     need_dparams=need_dp)
        torch.cuda.synchronize() if DEV == "cuda" else None
        lab = "%s %s %s" % (path, mode, np.dtype(npdt).name)
        lpk = lp.double().cpu().numpy()
        _gather_fail(msgs, lab, check("lp", lpk, want_lp, scale * ref["s_lp"], scale * ref["lp32"], npdt, kap, False,
                                      inputs, exact_zero=~live))
        # fused sum: sum_coeff * sum(mask * scale * lp)
        tot = coeff * float(np.sum(want_lp))
        if np.all(np.isfinite(want_lp)) and np.all(np.isfinite(np.where(live, ref["lp32"], 0.0))):
            stol = float(np.sum(np.where(live, tolerance(ref["lp"], ref["s_lp"], npdt, kap, False), 0))) * abs(
                coeff * scale) + (2.0 ** -20 if npdt == np.float32 else 2.0 ** -45) * abs(coeff) * float(
                np.sum(np.abs(want_lp)))
            got = float(out_sum)
            if not abs(got - tot) <= stol:
                msgs.append("[%s] sum: kernel %.9g ref %.9g tol %.3g" % (lab, got, tot, stol))
        if not grad:
            continue
        slots = ([(0, xs, gv)] if need_dv else []) + [(1 + k, pss[k], gp[k]) for k in range(npar)]
        for i, stored, g in slots:
            name = "d/dvalue" if i == 0 else "d/dp%d" % (i - 1)
            gr = np.where(live, f * ref["g"][i], 0.0)
            g32 = np.where(live, f * ref["g32"][i], 0.0)
            S = np.abs(f) * ref["s_g"][i]
            gk = g.double().cpu().numpy()
            if tuple(np.shape(stored)) == tuple(shape):
                _gather_fail(msgs, lab, check(name, gk, gr, S, g32, npdt, kap, True, inputs, exact_zero=~live))
                continue
            # reduced to the stored shape: compare against the reduced reference where every contribution is
            # finite, within the sum of the per-element tolerances
            tol_e = np.where(live, tolerance(ref["g"][i] * f, S, npdt, kap, True), 0.0)
            rr = _reduce_to(gr, np.shape(stored), shape)
            tr = _reduce_to(tol_e, np.shape(stored), shape) + (2.0 ** -22 if npdt == np.float32 else 2.0 ** -50) * \
                _reduce_to(np.abs(gr), np.shape(stored), shape)
            fin32 = _reduce_to(np.isfinite(g32).astype(float), np.shape(stored), shape) == \
                _reduce_to(np.ones(shape), np.shape(stored), shape)
            finr = np.isfinite(rr)
            ok = np.where(finr & np.isfinite(gk), np.abs(gk - rr) <= tr,
                          (~finr & ~np.isfinite(gk)) | (finr & ~np.isfinite(gk) & ~fin32))
            if not ok.all():
                j = tuple(np.argwhere(~ok)[0])
                msgs.append("[%s] %s (reduced to %s): %d bad; first at %s: kernel %.9g ref %.9g tol %.3g"
                            % (lab, name, np.shape(stored), (~ok).sum(), j, gk[j], rr[j], tr[j]))
    return msgs


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("npdt,tdt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("fam", ELEM_FAMS, ids=[NAMES[f] for f in ELEM_FAMS])
def test_site_kernels_over_domain(fam, npdt, tdt, path):
    """Each element family x dtype x {forward only, latent site (value gradient wanted), observed site} on one
    shape per kernel path: lp, the fused sum (scale, mask, weight, sum_coeff) and every gradient reduced to its
    operand's stored shape, by the tolerance rule of the module docstring."""
    if path == "vec_shared_value" and not HAS_VALUE[fam]:
        pytest.skip("the KL families have no value operand")
    msgs = run_element_case(fam, npdt, tdt, path)
    assert not msgs, "\n".join(msgs[:12])


@pytest.mark.gpu
@pytest.mark.skipif(EMULATE, reason="host stand-ins launch no kernels")
def test_device_f64_agrees_with_host_build():
    """fp64: the kernels and the host build of the same functors agree over every domain within the fp64 rule
    with kappa = 4 (CUDA's fp64 lgamma / log stand in for the host libm's, so ill-conditioned points differ by
    more than a few ulp of the result: 3.8e-7 relative on a Beta lp at large concentrations, measured on an H100)."""
    from pyro_b200.distributions import _ops
    msgs = []
    for fam in ELEM_FAMS:
        n = 3000
        x, ps = grid(fam, n, np.float64)
        ref = reference(fam, x, ps, (n,))
        lp_h, dx_h, dp_h = _host_eval(fam, x, ps, np.float64)
        xt = torch.tensor(x, device=DEV) if x is not None else None
        pt = [torch.tensor(p, device=DEV) for p in ps]
        lp, gv, gp = _ops.site_score(fam, xt, pt, (n,), want_logprob=True, need_dvalue=xt is not None,
                                     need_dparams=[True] * len(ps))
        pairs = [("lp", lp, lp_h, ref["s_lp"], False)] + \
            ([("dx", gv, dx_h, ref["s_g"][0], True)] if xt is not None else []) + \
            [("dp%d" % k, gp[k], dp_h[k], ref["s_g"][1 + k], True) for k in range(len(ps))]
        for name, dev_v, host_v, S, grad in pairs:
            msgs += ["%s %s" % (NAMES[fam], m) for m in
                     check(name, dev_v.cpu().numpy(), host_v, S, host_v, np.float64, 4, grad)]
    assert not msgs, "\n".join(msgs[:12])


# ---------------------------------------------------------------------------------------------------------------
# GPU tier: event families (Dirichlet, Categorical, MVN) on every event kernel path
# ---------------------------------------------------------------------------------------------------------------
def _rows_tensor(a, tdt, offset):
    """[rows, K] operand on the device; offset=True stores it one element past a 16-byte boundary."""
    t = torch.as_tensor(np.ascontiguousarray(a), dtype=tdt)
    if not offset:
        return t.to(DEV)
    buf = torch.empty(t.numel() + 1, dtype=tdt, device=DEV)
    buf[1:] = t.reshape(-1).to(DEV)
    return buf[1:].view(t.shape)


def _event_common(nb, rng, tdt):
    mask = rng.random(nb) < 0.75
    up = rng.choice([0.5, 1.0, 2.0, -1.0], size=nb)
    return mask, up


def categorical_logits(nb, K, rng):
    """Row kinds: plain, -inf in the first 16-byte chunk, -inf in the last chunk, -inf everywhere except the
    chosen class, +-1e30, shifted by 1e4, chosen class at -inf."""
    lg = rng.standard_normal((nb, K)) * 3
    v = rng.integers(0, K, nb)
    kind = np.arange(nb) % 7
    for r in range(nb):
        k = kind[r]
        c = min(4, K - 1)
        if k == 1:
            lg[r, :c] = -np.inf
            v[r] = rng.integers(c, K)
        elif k == 2:
            lg[r, K - c:] = -np.inf
            v[r] = rng.integers(0, K - c)
        elif k == 3:
            lg[r, :] = -np.inf
            lg[r, v[r]] = rng.standard_normal()
        elif k == 4:
            lg[r] = np.where(rng.random(K) < 0.5, 1e30, -1e30)
        elif k == 5:
            lg[r] += 1e4
        elif k == 6 and K > 1:
            lg[r, v[r]] = -np.inf
    return lg, v


def _categorical_ref(lg, v):
    l64 = torch.tensor(lg, dtype=torch.float64, requires_grad=True)
    lp = odists.categorical(torch.tensor(v), l64)
    (g,) = torch.autograd.grad(lp.sum(), l64)
    lse = torch.logsumexp(l64.detach(), -1)
    sm = torch.exp(l64.detach() - lse[:, None])
    onehot = torch.nn.functional.one_hot(torch.tensor(v), lg.shape[1]).double()
    lv = torch.gather(l64.detach(), 1, torch.tensor(v)[:, None])[:, 0]
    s_lp = (lv.abs() + lse.abs()).numpy()
    s_g = (onehot + sm * (l64.detach().abs() + lse.abs()[:, None])).nan_to_num(0.0).numpy()
    return lp.detach().numpy(), g.numpy(), s_lp, s_g


def _dirichlet_inputs(nb, K, rng):
    c = _logu(rng, 1e-4, 1e4, (nb, K))
    # x near the simplex vertices for a third of the rows
    z = rng.standard_normal((nb, K)) * np.where(np.arange(nb) % 3 == 0, 20.0, 1.0)[:, None]
    x = np.exp(z - z.max(1, keepdims=True))
    x = np.maximum(x / x.sum(1, keepdims=True), 1e-30)
    return x, c


def _dirichlet_ref(x, c):
    xt = torch.tensor(x, requires_grad=True)
    ct = torch.tensor(c, requires_grad=True)
    with mock.patch.object(torch, "xlogy", _xlogy):
        lp = odists.dirichlet(xt, ct)
        gx, gc = torch.autograd.grad(lp.sum(), [xt, ct])
    cs = ct.detach().sum(-1)
    t_x = torch.xlogy(ct.detach() - 1, xt.detach()).abs()
    s_lp = (t_x.sum(-1) + torch.lgamma(cs).abs() + torch.lgamma(ct.detach()).abs().sum(-1)
            + torch.digamma(cs).abs() * cs).numpy()   # rounding of the concentration sum enters through psi(sum)
    s_gx = ((ct.detach() - 1).abs() / xt.detach()).numpy()
    s_gc = (xt.detach().log().abs() + torch.digamma(cs).abs()[:, None] + torch.digamma(ct.detach()).abs()
            + (torch.polygamma(1, cs) * cs)[:, None]).numpy()
    return lp.detach().numpy(), gx.numpy(), gc.numpy(), s_lp, s_gx, s_gc


def _mvn_inputs(nb, n, rng):
    d = _logu(rng, 1e-3, 1e3, (nb, n))
    L = np.tril(rng.standard_normal((nb, n, n)) * (0.5 / np.sqrt(n)), -1) * d[:, :, None]
    L[:, np.arange(n), np.arange(n)] = d
    mu = rng.standard_normal((nb, n))
    x = mu + np.einsum("bij,bj->bi", L, rng.standard_normal((nb, n)))
    return x, mu, L


def _mvn_ref(x, mu, L):
    xt, mt, Lt = (torch.tensor(a, requires_grad=True) for a in (x, mu, L))
    lp = odists.mvn_tril(xt, mt, Lt)
    gx, gm, gL = torch.autograd.grad(lp.sum(), [xt, mt, Lt])
    n = x.shape[-1]
    with torch.no_grad():
        Ld = Lt.detach()
        z = torch.linalg.solve_triangular(Ld, (xt - mt).detach().unsqueeze(-1), upper=False).squeeze(-1)
        Li = torch.linalg.inv(Ld).abs()
        # componentwise bound of the substitution: |dz| <= n u |L^-1| (|L| |z| + |x| + |mu|)
        dz = torch.einsum("bij,bj->bi", Li, torch.einsum("bij,bj->bi", Ld.abs(), z.abs()) + xt.detach().abs()
                          + mt.detach().abs()) * n
        s_lp = ((z * z).sum(-1) / 2 + (z.abs() * dz).sum(-1) + Ld.diagonal(dim1=-2, dim2=-1).log().abs().sum(-1)
                + n * 0.92).numpy()
        w = torch.linalg.solve_triangular(Ld.transpose(-1, -2), z.unsqueeze(-1), upper=True).squeeze(-1)
        dw = torch.einsum("bji,bj->bi", Li, dz + torch.einsum("bji,bj->bi", Ld.abs(), w.abs()) * n)
        s_gv = w.abs() + dw
        s_gL = (torch.einsum("bi,bj->bij", s_gv, z.abs() + dz) + torch.diag_embed(1 / Ld.diagonal(dim1=-2, dim2=-1))
                .abs()).numpy()
        s_gv = s_gv.numpy()
    return lp.detach().numpy(), gx.numpy(), gm.numpy(), gL.numpy(), s_lp, s_gv, s_gL


EVENT_KAPPA = {"dirichlet": 32, "categorical": 32, "mvn": 32}

# (family, K, rows, offset): rows on both sides of 1024 and 4096, K on both sides of 32 and of the vector width
CAT_CASES = [(K, nb, off) for K in (3, 4, 8, 17, 32, 40, 64, 1000) for nb in (700, 5000) for off in (False, True)
             if not (K == 1000 and nb == 5000)]
DIR_CASES = [(K, nb, off) for K in (2, 3, 8, 17, 32, 40, 64, 1000) for nb in (700, 5000) for off in (False, True)
             if not (K == 1000 and nb == 5000)]
MVN_CASES = [(n, nb) for n in (1, 2, 4, 5, 8, 9, 32, 33, 128, 129) for nb in ((700, 2000) if n <= 33 else (64,))]


def _event_call(fam_id, value, params, nb, K, tdt, mask, up, need_dv, need_dp):
    from pyro_b200.distributions import _ops
    out_sum = torch.zeros((), dtype=tdt, device=DEV)
    lp, gv, gp = _ops.site_score(fam_id, value, params, (nb,), mask=torch.as_tensor(mask, device=DEV),
                                 scale=0.5, upstream=torch.as_tensor(up, dtype=tdt, device=DEV), weight=-0.25,
                                 sum_coeff=-2.0, want_logprob=True, out_sum=out_sum, need_dvalue=need_dv,
                                 need_dparams=need_dp, event_size=K)
    return lp, out_sum, gv, gp


def _event_checks(lab, npdt, kap, mask, up, lpk, sumk, lp, s_lp, grads):
    msgs = []
    live = mask
    want = np.where(live, 0.5 * lp, 0.0)
    _gather_fail(msgs, lab, check("lp", lpk, want, 0.5 * s_lp, want, npdt, kap, False, exact_zero=~live))
    fin = np.isfinite(want)
    if fin.all():
        tot = -2.0 * want.sum()
        stol = 2 * 0.5 * float(np.sum(np.where(live, tolerance(lp, s_lp, npdt, kap, False), 0))) + \
            (2.0 ** -20 if npdt == np.float32 else 2.0 ** -45) * 2 * float(np.abs(want).sum())
        if not abs(sumk - tot) <= stol:
            msgs.append("[%s] sum: kernel %.9g ref %.9g tol %.3g" % (lab, sumk, tot, stol))
    f = -0.125 * up
    for name, gk, gr, S in grads:
        fb = f.reshape((-1,) + (1,) * (gr.ndim - 1))
        lb = live.reshape(fb.shape)
        gw = np.where(lb, fb * gr, 0.0)
        _gather_fail(msgs, lab, check(name, gk, gw, np.abs(fb) * S, gw, npdt, kap, True,
                                      exact_zero=np.broadcast_to(~lb, gk.shape)))
    return msgs


@pytest.mark.gpu
@pytest.mark.parametrize("npdt,tdt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("K,nb,off", CAT_CASES)
def test_categorical_kernels_over_domain(K, nb, off, npdt, tdt):
    """Categorical(logits) with -inf logits in the first 16-byte chunk, in the last, everywhere but the chosen
    class, +-1e30 and a 1e4 shift, through the group, row-per-thread (scalar and 16-byte) and vec kernels, with
    mask, scale, weight and upstream; S for lp is |logit| + |logsumexp|."""
    from pyro_b200 import _native as N
    rng = np.random.default_rng(K * 7919 + nb + off)
    lg, v = categorical_logits(nb, K, rng)
    lg = lg.astype(npdt).astype(np.float64)
    lp, g, s_lp, s_g = _categorical_ref(lg, v)
    mask, up = _event_common(nb, rng, tdt)
    lt = _rows_tensor(lg, tdt, off)
    vt = torch.as_tensor(v, device=DEV)
    msgs = []
    for grad in (False, True):
        lpk, sk, _, gp = _event_call(N.CATEGORICAL, vt, [lt], nb, K, tdt, mask, up, False, [grad])
        grads = [("d/dlogits", gp[0].double().cpu().numpy(), g, s_g)] if grad else []
        msgs += _event_checks("K=%d rows=%d off=%s grad=%s" % (K, nb, off, grad), npdt, EVENT_KAPPA["categorical"],
                              mask, up, lpk.double().cpu().numpy(), float(sk), lp, s_lp, grads)
    assert not msgs, "\n".join(msgs[:12])


@pytest.mark.gpu
@pytest.mark.parametrize("npdt,tdt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("K,nb,off", DIR_CASES)
def test_dirichlet_kernels_over_domain(K, nb, off, npdt, tdt):
    """Dirichlet with concentrations 1e-4 .. 1e4 and values near the simplex vertices, through the group,
    row-per-thread (scalar and 16-byte) and vec kernels, with mask, scale, weight and upstream."""
    from pyro_b200 import _native as N
    rng = np.random.default_rng(K * 31 + nb + off)
    x, c = _dirichlet_inputs(nb, K, rng)
    x, c = (a.astype(npdt).astype(np.float64) for a in (x, c))
    lp, gx, gc, s_lp, s_gx, s_gc = _dirichlet_ref(x, c)
    mask, up = _event_common(nb, rng, tdt)
    xt, ct = _rows_tensor(x, tdt, off), _rows_tensor(c, tdt, off)
    msgs = []
    for grad in (False, True):
        lpk, sk, gv, gp = _event_call(N.DIRICHLET, xt, [ct], nb, K, tdt, mask, up, grad, [grad])
        grads = [("d/dvalue", gv.double().cpu().numpy(), gx, s_gx),
                 ("d/dconc", gp[0].double().cpu().numpy(), gc, s_gc)] if grad else []
        msgs += _event_checks("K=%d rows=%d off=%s grad=%s" % (K, nb, off, grad), npdt, EVENT_KAPPA["dirichlet"],
                              mask, up, lpk.double().cpu().numpy(), float(sk), lp, s_lp, grads)
    assert not msgs, "\n".join(msgs[:12])


@pytest.mark.gpu
@pytest.mark.parametrize("npdt,tdt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("n,nb", MVN_CASES)
def test_mvn_kernels_over_domain(n, nb, npdt, tdt):
    """MultivariateNormal(loc, scale_tril) with factor diagonals spanning 1e-3 .. 1e3 through the row-per-thread,
    group (G = 2 / 4 / 8 / 32, full and partial) and warp kernels; S bounds the triangular solves componentwise."""
    from pyro_b200 import _native as N
    rng = np.random.default_rng(n * 131 + nb)
    x, mu, L = _mvn_inputs(nb, n, rng)
    x, mu, L = (a.astype(npdt).astype(np.float64) for a in (x, mu, L))
    lp, gx, gm, gL, s_lp, s_gv, s_gL = _mvn_ref(x, mu, L)
    mask, up = _event_common(nb, rng, tdt)
    xt, mt, Lt = (torch.as_tensor(a, dtype=tdt, device=DEV) for a in (x, mu, L))
    msgs = []
    for grad in (False, True):
        lpk, sk, gv, gp = _event_call(N.MVN_TRIL, xt, [mt, Lt], nb, n, tdt, mask, up, grad, [grad, grad])
        grads = [("d/dvalue", gv.double().cpu().numpy(), gx, s_gv), ("d/dloc", gp[0].double().cpu().numpy(), gm, s_gv),
                 ("d/dscale_tril", gp[1].double().cpu().numpy(), gL, s_gL)] if grad else []
        msgs += _event_checks("n=%d rows=%d grad=%s" % (n, nb, grad), npdt, EVENT_KAPPA["mvn"], mask, up,
                              lpk.double().cpu().numpy(), float(sk), lp, s_lp, grads)
    assert not msgs, "\n".join(msgs[:12])


# ---------------------------------------------------------------------------------------------------------------
# routing: the shapes above reach the kernels they are meant for
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(EMULATE, reason="host stand-ins launch no kernels")
def test_kernel_routing():
    """torch.profiler kernel names: every site kernel (small, vec, vec<MASKUP>, gen) and every event kernel (group,
    row-per-thread, vec for Dirichlet / Categorical; row-per-thread, group full / partial and warp for MVN) is
    launched by the shapes the domain tests use."""
    from torch.profiler import ProfilerActivity, profile

    def names(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    def element(path, fam=4, npdt=np.float32, tdt=torch.float32):
        return lambda: run_element_case(fam, npdt, tdt, path)

    expect = {
        "small": "site_small_kernel<4, float, true>", "small_bcast": "site_small_kernel<4, float, true>",
        "vec": "site_vec_kernel<4, float, true, false>", "vec_shared_value": "site_vec_kernel<4, float, true, false>",
        "vec_row_param": "site_vec_kernel<4, float, true, false>",
        "vec_maskup": "site_vec_kernel<4, float, true, true>", "gen": "site_gen_kernel<4, float, true>",
    }
    missing = []
    for path, kname in expect.items():
        got = names(element(path))
        if not any(kname in g for g in got):
            missing.append((path, kname, sorted(set(got))))

    def event(test, *args):
        return lambda: test(*args)

    # The row-per-thread kernels have a scalar and a 16-byte path under ONE kernel name (EventArgs::g_log2 picks the
    # path at run time), so the profiler cannot tell them apart.  The 16-byte path is reached through the selector's
    # rule in b2_event_score instead: K a multiple of the vector width and 16-byte-aligned rows, which the aligned
    # K = 4 (fp64), 8 and 32 cases of test_categorical_kernels_over_domain with 5000 rows satisfy; K = 17 and the
    # offset storage take the scalar path.
    ev_expect = [
        ((test_categorical_kernels_over_domain, 17, 700, False), "categorical_kernel<float"),
        ((test_categorical_kernels_over_domain, 17, 5000, True), "categorical_rowthread_kernel<float"),
        ((test_categorical_kernels_over_domain, 8, 5000, False), "categorical_rowthread_kernel<float"),
        ((test_categorical_kernels_over_domain, 64, 700, False), "categorical_vec_kernel<float"),
        ((test_categorical_kernels_over_domain, 64, 700, True), "categorical_kernel<float"),
        ((test_dirichlet_kernels_over_domain, 17, 700, False), "dirichlet_kernel<float"),
        ((test_dirichlet_kernels_over_domain, 8, 5000, False), "dirichlet_rowthread_kernel<float"),
        ((test_dirichlet_kernels_over_domain, 64, 700, False), "dirichlet_vec_kernel<float"),
        ((test_mvn_kernels_over_domain, 2, 2000), "mvn_rowthread_kernel<float"),
        ((test_mvn_kernels_over_domain, 2, 700), "mvn_group_kernel<float, true, 2, true>"),
        ((test_mvn_kernels_over_domain, 4, 700), "mvn_group_kernel<float, true, 4, true>"),
        ((test_mvn_kernels_over_domain, 5, 700), "mvn_group_kernel<float, true, 8, false>"),
        ((test_mvn_kernels_over_domain, 8, 2000), "mvn_group_kernel<float, true, 8, true>"),
        ((test_mvn_kernels_over_domain, 32, 700), "mvn_group_kernel<float, true, 32, true>"),
        ((test_mvn_kernels_over_domain, 9, 700), "mvn_group_kernel<float, true, 32, false>"),
        ((test_mvn_kernels_over_domain, 33, 64), "mvn_tril_kernel<float, true, 4>"),
    ]
    for (test, *args), kname in ev_expect:
        got = names(event(test, *args, np.float32, torch.float32))
        if not any(kname in g for g in got):
            missing.append((test.__name__, args, kname, sorted(set(got))))
    assert not missing, missing
