"""Varying slopes under SVI: ``X @ w + b + alpha[g] + SUM_k beta_k[g] * X[:, c_k]`` kept lazy by pyro_b200/lazy.py and
scored by ``b2_glm_group_slope_sum``, one pass of the family's fused kernel over
``[X | onehot(g) | X[:, c_1] onehot(g) | ..]`` with d/dalpha and d/dbeta_k from the same contraction, for logistic,
Poisson, linear and Binomial regression.

CPU tier: every spelling of a slope stays lazy and the predictor's ``dense()`` equals the model's eager expression bit
for bit; the near misses materialise exactly; SVI steps of all four families with the kernel seam replaced by an fp64
torch restatement match ``LAZY_LINEAR = False``; an intercept-only model keeps its one ``b2_glm_group_sum`` call; an
out-of-range index raises IndexError before anything reads it; the entry point's argument checks; what ptxas makes of
the slope kernels with X rounded to TF32 and of the pack kernel.
GPU tier: the kernel against fp64 (every kind and count form, S = 1..3, shared and per-particle tables, both
precisions, P = 1, 64, 65, ragged N, widths on each side of 32, 64 and 96 and at 128, a covariate of magnitude 1e3),
determinism, the NaN of an index that reaches the kernel, SVI steps against the materialised path, a captured-graph
step against the eager one, the fallbacks, and ``bind.Trace_ELBO`` with reference Pyro."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from pyro_b200 import _build
from pyro_b200 import _native as N
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO, TraceMeanField_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.lazy import LinearPredictorTensor, SiteValue
from pyro_b200.optim import ClippedAdam
from test_glm_group_svi import KIND_CODE, TRIALS, _likelihood, _Noise, group_guide, group_model

DEV = device()
KINDS = ["Bernoulli", "Poisson", "Normal", "Binomial"]
COLS = (2, 0, 4)


# ---- models ------------------------------------------------------------------------------------------------------
def slope_model(kind, form="centred", S=1, order="intercept_first", side="right", spelling="colon", cols=COLS):
    """Regression of ``kind`` with a varying intercept ``alpha[g]`` and S varying slopes on columns ``cols`` of X:
    ``beta_k ~ Normal(0, 0.3)[G]`` (centred) or ``s_bk * eb_k`` with a latent scale (non-centred).  ``order``: where
    the slopes are added (after the intercept and the bias, in front of ``X @ w``, or between ``X @ w`` and the bias);
    ``side``: the covariate right or left of ``*``; ``spelling``: ``X[:, c]``, ``X[..., c]`` or ``X.select(-1, c)``."""
    def model(X, g, y, m=None, mask=None, G=6):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
        sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.0))) if kind == "Normal" else None
        A = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
        A = A.squeeze(-2) if A.dim() > 1 else A
        terms = []
        for k in range(S):
            if form == "centred":
                B = pyro.sample("beta%d" % k, dist.Normal(X.new_zeros(G), 0.3).to_event(1))
                B = B.squeeze(-2) if B.dim() > 1 else B
                bg = B[..., g]
            else:
                s = pyro.sample("s_b%d" % k, dist.HalfNormal(X.new_full((), 0.5)))
                e = pyro.sample("eb%d" % k, dist.Normal(X.new_zeros(G), 1.0).to_event(1))
                e = e.squeeze(-2) if e.dim() > 1 else e
                bg = s * e[..., g]
            c = cols[k]
            x = {"colon": lambda: X[:, c], "ellipsis": lambda: X[..., c], "select": lambda: X.select(-1, c)}[spelling]()
            terms.append(bg * x if side == "right" else x * bg)
        lin = w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w
        with pyro.plate("data", X.shape[0]):
            if order == "intercept_first":
                eta = lin + b + A[..., g]
                for t in terms:
                    eta = eta + t
            elif order == "slopes_first":
                eta = terms[0] + lin
                for t in terms[1:]:
                    eta = t + eta
                eta = (eta + A[..., g]) + b
            else:
                eta = lin
                for t in terms:
                    eta = eta + t
                eta = A[..., g] + (eta + b)
            d = _likelihood(kind, eta, sigma, m)
            pyro.sample("y", d.mask(mask) if mask is not None else d, obs=y)
    return model


def slope_guide(kind, form="centred", S=1, intercept=True):
    def guide(X, g, y, m=None, mask=None, G=6):
        D = X.shape[-1]
        sites = [("w", (D,)), ("b", ())] + ([("alpha", (G,))] if intercept else [])
        if kind == "Normal":
            sites.append(("sigma", ()))
        for k in range(S):
            sites += [("beta%d" % k, (G,))] if form == "centred" else [("s_b%d" % k, ()), ("eb%d" % k, (G,))]
        for name, shape in sites:
            loc = pyro.param(name + "_loc", X.new_zeros(shape))
            scale = pyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=dist.constraints.positive)
            if name == "sigma" or name.startswith("s_b"):
                pyro.sample(name, dist.LogNormal(loc, scale))
            else:
                d = dist.Normal(loc, scale)
                pyro.sample(name, d.to_event(1) if shape else d)
    return guide


def _data(kind, n, D, G, S=1, seed=0, dev=DEV, cols=COLS, big=None):
    """Data of the slope model; ``big``: the first slope's column of X scaled to that magnitude after y is drawn, so
    the data are those of a model whose weight and slope on that column are ``big`` times smaller."""
    gen = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=gen)
    g = torch.randint(0, G, (n,), generator=gen)
    eta = X @ (0.3 * torch.randn(D, generator=gen) / D ** 0.5) + 0.3 + 0.5 * torch.randn(G, generator=gen)[g]
    for k in range(S):
        eta = eta + 0.3 * torch.randn(G, generator=gen)[g] * X[:, cols[k]]
    if big is not None:
        X[:, cols[0]] *= big
    m = torch.randint(1, 20, (n,), generator=gen).float() if kind == "BinomialRows" else torch.full((n,), TRIALS)
    if kind == "Bernoulli":
        y = torch.bernoulli(torch.sigmoid(eta), generator=gen)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta.clamp(max=8.0)), generator=gen)
    elif kind == "Normal":
        y = eta + 0.6 * torch.randn(n, generator=gen)
    else:
        y = torch.binomial(m, torch.sigmoid(eta), generator=gen)
    return X.to(dev), g.to(dev), y.to(dev), m.to(dev)


# ---- CPU tier: lazy semantics -------------------------------------------------------------------------------------
def _sv(t):
    return SiteValue.wrap(t.clone())


def _mk(P=4, n=50, D=6, G=5):
    torch.manual_seed(0)
    X = torch.randn(n, D)
    g = torch.randint(0, G, (n,))
    return X, g, torch.randn(P, 1, D), torch.randn(P, 1), torch.randn(P, G)


def _tables(P, G, seed):
    """(lazy gather, eager gather) of one table in each accepted form: [P, 1, G] squeezed, [P, G], [G], and the
    non-centred ``s * eta[..., g]`` with a per-particle and a shared scale."""
    gen = torch.Generator().manual_seed(seed)
    T3, T2, T1 = torch.randn(P, 1, G, generator=gen), torch.randn(P, G, generator=gen), torch.randn(G, generator=gen)
    s = torch.rand(P, 1, generator=gen) + 0.5
    T3s, T2s, T1s, ss = _sv(T3), _sv(T2), _sv(T1), _sv(s)
    return [lambda g: (T3s.squeeze(-2)[..., g], T3.squeeze(-2)[..., g]), lambda g: (T2s[..., g], T2[..., g]),
            lambda g: (T1s[g], T1[g]), lambda g: (ss * T2s[..., g], s * T2[..., g]),
            lambda g: (0.7 * T1s[..., g], 0.7 * T1[..., g])]


def _check_lazy(got, want, S, tag):
    assert isinstance(got, LinearPredictorTensor) and isinstance(got.lazy, dist.LinearPredictor), tag
    assert got.lazy.group is not None and len(got.lazy.slopes) == S and got.shape == want.shape, tag
    assert torch.equal(got.dense(), want), tag
    assert torch.equal(torch.exp(got).dense(), torch.exp(want)), tag                       # the Poisson rate
    nd = dist.Normal(got, 0.6)
    assert type(nd).__name__ == "_NormalLinear" and torch.equal(nd.loc, want), tag         # the Normal loc
    bd = dist.Binomial(torch.tensor(TRIALS), logits=got)
    assert type(bd).__name__ == "_BinomialLinear" and torch.equal(bd.logits, want), tag    # the Binomial logits
    assert type(dist.Bernoulli(logits=got)).__name__ == "_BernoulliLinear", tag


def test_every_spelling_stays_lazy_and_dense_equals_the_eager_expression_bitwise():
    X, g, w, b, A = _mk()
    ws, bs, As = _sv(w), _sv(b), _sv(A)
    lin, lin_e = ws.squeeze(-2) @ X.T, w.squeeze(-2) @ X.T
    ag, ag_e = As[..., g], A[..., g]
    cols = {"colon": lambda c: X[:, c], "ellipsis": lambda c: X[..., c], "select": lambda c: X.select(-1, c)}
    n_cases = 0
    for ti, table in enumerate(_tables(4, 5, 1)):
        for spelling, col in cols.items():
            for side in ("right", "left"):
                lz, ref = table(g)
                sl = lz * col(3) if side == "right" else col(3) * lz
                sl_e = ref * X[:, 3] if side == "right" else X[:, 3] * ref
                assert isinstance(sl, LinearPredictorTensor) and isinstance(sl.lazy, dist.SlopeGather)
                assert torch.equal(sl.dense(), sl_e) and torch.equal(sl.eager(), sl_e)
                tag = (ti, spelling, side)
                for j, (got, want) in enumerate([
                        (lin + bs + ag + sl, lin_e + b + ag_e + sl_e), (sl + (lin + bs) + ag, sl_e + (lin_e + b) + ag_e),
                        ((lin + sl) + bs + ag, (lin_e + sl_e) + b + ag_e), (ag + (lin + sl + bs), ag_e + (lin_e + sl_e + b)),
                        (bs + (sl + lin) + ag, b + (sl_e + lin_e) + ag_e), (lin + ag + sl, lin_e + ag_e + sl_e)]):
                    _check_lazy(got, want, 1, tag + (j,))
                    n_cases += 1
    assert n_cases == 5 * 3 * 2 * 6
    # S = 2 and 3: mixed forms and sides, in any order with the intercept
    t = _tables(4, 5, 2)
    s1, e1 = t[0](g)
    s2, e2 = t[2](g)
    s3, e3 = t[3](g)
    got = lin + bs + s1 * X[:, 0] + ag + X[..., 5] * s2
    want = lin_e + b + e1 * X[:, 0] + ag_e + X[..., 5] * e2
    _check_lazy(got, want, 2, "S2")
    got = s3 * X.select(-1, 1) + (lin + s1 * X[:, 0]) + ag + bs + X[:, 4] * s2
    want = e3 * X[:, 1] + (lin_e + e1 * X[:, 0]) + ag_e + b + X[:, 4] * e2
    _check_lazy(got, want, 3, "S3")
    assert [s.col for s in got.lazy.slopes] == [0, 1, 4]
    # a shared weight vector: X @ w [N] with [G] tables
    w1, b1, A1, B1 = torch.randn(6), torch.randn(()), torch.randn(5), torch.randn(5)
    A1s, B1s = _sv(A1), _sv(B1)
    got = X @ _sv(w1) + _sv(b1) + A1s[g] + B1s[g] * X[:, 2]
    _check_lazy(got, X @ w1 + b1 + A1[g] + B1[g] * X[:, 2], 1, "shared")
    assert got.lazy.slopes[0].col == 2


def test_near_misses_materialise_exactly():
    X, g, w, b, A = _mk()
    ws, bs, As = _sv(w), _sv(b), _sv(A)
    lin, lin_e = ws.squeeze(-2) @ X.T, w.squeeze(-2) @ X.T
    base, base_e = lin + bs + As[..., g], lin_e + b + A[..., g]
    B, B6 = torch.randn(4, 5), torch.randn(4, 6)
    Bs, B6s = _sv(B), _sv(B6)
    X2 = X.clone()
    sep = torch.randn(50)
    cases = {  # (got, want): every one a plain tensor equal to the eager expression
        "separate covariate": (Bs[..., g] * sep, B[..., g] * sep),
        "copy of a column": (Bs[..., g] * X[:, 2].clone(), B[..., g] * X[:, 2]),
        "scaled column": (Bs[..., g] * (X[:, 2] * 2), B[..., g] * (X[:, 2] * 2)),
        "column of another tensor": (base + Bs[..., g] * X2[:, 2], base_e + B[..., g] * X2[:, 2]),
        "index of equal values": (base + Bs[..., g.clone()] * X[:, 2], base_e + B[..., g] * X[:, 2]),
        "different G": (base + B6s[..., g] * X[:, 2], base_e + B6[..., g] * X[:, 2]),
        "repeated column": (base + Bs[..., g] * X[:, 2] + Bs[..., g] * X[..., 2],
                            base_e + B[..., g] * X[:, 2] + B[..., g] * X[:, 2]),
        "four slopes": (base + Bs[..., g] * X[:, 0] + Bs[..., g] * X[:, 1] + Bs[..., g] * X[:, 2]
                        + Bs[..., g] * X[:, 3],
                        base_e + B[..., g] * X[:, 0] + B[..., g] * X[:, 1] + B[..., g] * X[:, 2] + B[..., g] * X[:, 3]),
        "slope times a number": (base + (Bs[..., g] * X[:, 2]) * 2.0, base_e + (B[..., g] * X[:, 2]) * 2.0),
        "sum of a slope": ((Bs[..., g] * X[:, 2]).sum(), (B[..., g] * X[:, 2]).sum()),
        "slope plus a gather": (Bs[..., g] * X[:, 2] + As[..., g], B[..., g] * X[:, 2] + A[..., g]),
        "offset after slopes": (base + Bs[..., g] * X[:, 2] + sep, base_e + B[..., g] * X[:, 2] + sep),
        "second intercept": (base + Bs[..., g] * X[:, 2] + As[..., g], base_e + B[..., g] * X[:, 2] + A[..., g]),
    }
    for name, (got, want) in cases.items():
        assert type(got) in (torch.Tensor, SiteValue), (name, type(got))
        if want is not None:
            assert torch.equal(got.as_subclass(torch.Tensor), want), name
    # an index of equal values arriving first, and the intercept's index second
    got = lin + Bs[..., g.clone()] * X[:, 2] + As[..., g]
    assert type(got) is torch.Tensor and torch.equal(got, lin_e + B[..., g] * X[:, 2] + A[..., g])
    # X that requires grad: neither X @ w nor the product is lazy
    Xg = X.clone().requires_grad_(True)
    got = ws.squeeze(-2) @ Xg.T + As[..., g] + Bs[..., g] * Xg[:, 2]
    assert not isinstance(got, LinearPredictorTensor)
    assert torch.equal(got.detach().as_subclass(torch.Tensor), (lin_e + A[..., g] + B[..., g] * X[:, 2]))
    # slopes without an intercept stay lazy until they are scored (the SVI test below shows they then materialise)
    got = lin + bs + Bs[..., g] * X[:, 2]
    assert got.lazy.group is None and len(got.lazy.slopes) == 1
    assert torch.equal(got.dense(), lin_e + b + B[..., g] * X[:, 2])
    with pytest.raises(RuntimeError):
        dist._weights(got.lazy)


# ---- CPU tier: SVI with the kernel seam replaced by an fp64 torch restatement ----------------------------------------
def _fp64_launch(meta, X, y, W, b, A, sigma, *B):
    """What b2_glm_group_slope_sum returns, restated in fp64 with torch.distributions and autograd."""
    scale, weight, coeff, _, kind, idx, trials, per_row, s_stride, cols = meta
    ops = [t.detach().double().requires_grad_(t.requires_grad) if t is not None else None
           for t in (W, b, A, sigma) + B]
    Wd, bd, Ad, sd = ops[:4]
    G = A.shape[-1]
    gi = idx.long()
    with torch.enable_grad():
        eta = Wd @ X.double().T + Ad.reshape(-1, G)[:, gi]
        for Bd, c in zip(ops[4:], cols):
            eta = eta + Bd.reshape(-1, G)[:, gi] * X.double()[:, c]
        if bd is not None:
            eta = eta + bd[:, None]
        yd = y.double()
        if kind == N.GLM_BERNOULLI:
            lp = torch.distributions.Bernoulli(logits=eta).log_prob(yd)
        elif kind == N.GLM_POISSON:
            lp = yd * eta - eta.exp() - torch.lgamma(yd + 1)
        elif kind == N.GLM_NORMAL:
            lp = torch.distributions.Normal(eta, sd.reshape(-1, 1) if s_stride else sd.reshape(())).log_prob(yd)
        else:
            lp = torch.distributions.Binomial(trials.double(), logits=eta).log_prob(yd)
        lps = scale * lp.sum()
        need = [o for o in ops if o is not None and o.requires_grad]
        grads = iter(torch.autograd.grad(lps, need))
    out = [weight * next(grads) if o is not None and o.requires_grad else None for o in ops]
    out = [o.float() if o is not None else None for o in out]
    return ((coeff * lps).detach().float(), None, None) + tuple(out)


def _svi(model, guide, args, steps, lazy, elbo_cls=Trace_ELBO, P=8, seed=0):
    """``steps`` SVI steps with guide noise from seed ``seed`` injected through fixed buffers; returns the losses, the
    parameters, the number of fused slope calls and the metas of the fused group calls."""
    pyro.clear_param_store()
    X, G = args[0], args[5]
    shapes = {"w": (X.shape[1],), "b": (), "sigma": (), "alpha": (G,), "s_a": (), "eta": (G,)}
    for k in range(3):
        shapes.update({"beta%d" % k: (G,), "s_b%d" % k: (), "eb%d" % k: (G,)})
    gen = torch.Generator().manual_seed(seed)
    eps = {k: torch.randn((steps, P, 1) + sh, generator=gen, dtype=X.dtype).to(X.device) for k, sh in shapes.items()}
    bufs = {k: torch.empty_like(v[0]) for k, v in eps.items()}

    def noisy_guide(*a):
        with _Noise(bufs):
            guide(*a)
    calls, group_metas = [], []
    real_s, real_g = dist._GlmSlopeFn.apply, dist._GlmGroupFn.apply
    dist._GlmSlopeFn.apply = lambda *a: calls.append(1) or real_s(*a)
    dist._GlmGroupFn.apply = lambda *a: group_metas.append(a[0]) or real_g(*a)
    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    try:
        svi = SVI(model, noisy_guide, ClippedAdam({"lr": 0.01}),
                  elbo_cls(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        losses = []
        for i in range(steps):
            for k in bufs:
                bufs[k].copy_(eps[k][i])
            losses.append(svi.step(*args))
    finally:
        elbo_mod.LAZY_LINEAR = saved
        dist._GlmSlopeFn.apply, dist._GlmGroupFn.apply = real_s, real_g
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls), group_metas


@pytest.fixture
def fp64_seam():
    """The CPU stand-ins of the native seams, with the slope sum restated in fp64 (and _BernoulliLinear's own
    _fused_sum, which the stand-ins replace by the dense path)."""
    import cpu_emulation
    fused = dist._BernoulliLinear._fused_sum
    with cpu_emulation.enabled():
        dist._BernoulliLinear._fused_sum = fused
        saved = dist._GlmSlopeFn.launch
        dist._GlmSlopeFn.launch = _fp64_launch
        try:
            yield
        finally:
            dist._GlmSlopeFn.launch = saved


def _close(l_f, p_f, l_m, p_m, rel, atol):
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= rel * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=atol, rtol=atol), k


@pytest.mark.parametrize("S", [1, 2, 3])
@pytest.mark.parametrize("form", ["centred", "noncentred"])
@pytest.mark.parametrize("kind", KINDS + ["BinomialRows"])
def test_svi_on_the_lazy_route_matches_materialised_with_the_seam_restated(fp64_seam, kind, form, S):
    fam = "Binomial" if kind == "BinomialRows" else kind
    X, g, y, m = _data(kind, 8192, 5, 7, S=S, seed=3 + S, dev="cpu")
    args = (X, g, y, m, None, 7)
    order = ["intercept_first", "slopes_first", "slope_before_bias"][S - 1]
    model, guide = slope_model(fam, form, S, order, "left" if S == 2 else "right"), slope_guide(fam, form, S)
    l_f, p_f, calls, gm = _svi(model, guide, args, 3, True)
    l_m, p_m, calls_m, gm_m = _svi(model, guide, args, 3, False)
    assert calls == 3 and calls_m == 0 and not gm and not gm_m
    _close(l_f, p_f, l_m, p_m, 1e-5, 1e-5)


def test_intercept_only_model_keeps_its_group_call_and_meta(fp64_seam):
    import test_glm_group_svi as group_test
    X, g, y, m = _data("Normal", 8192, 5, 7, S=0, seed=5, dev="cpu")
    saved = dist._GlmGroupFn.launch
    dist._GlmGroupFn.launch = group_test._fp64_launch
    try:
        _, _, calls, metas = _svi(group_model("Normal"), group_guide("Normal"), (X, g, y, m, None, 7), 2, True)
    finally:
        dist._GlmGroupFn.launch = saved
    assert calls == 0 and len(metas) == 2
    for meta in metas:
        scale, weight, coeff, unit, kind, idx, trials, per_row, s_stride = meta       # the parent's meta, unchanged
        assert kind == N.GLM_NORMAL and idx.dtype == torch.int32 and trials is None and per_row == 0


@pytest.mark.parametrize("case", ["no_intercept", "cols129"])
def test_out_of_scope_predictors_materialise_with_the_seam_restated(fp64_seam, case):
    """A slope without an intercept, and D + G (1 + S) = 129 columns, make no fused call and match exactly."""
    if case == "no_intercept":
        X, g, y, m = _data("Poisson", 8192, 5, 7, seed=6, dev="cpu")

        def model(X, g, y, m=None, mask=None, G=6):
            w = pyro.sample("w", dist.Normal(X.new_zeros(X.shape[-1]), 1.0).to_event(1))
            b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
            B = pyro.sample("beta0", dist.Normal(X.new_zeros(G), 0.3).to_event(1)).squeeze(-2)
            with pyro.plate("data", X.shape[0]):
                pyro.sample("y", dist.Poisson(torch.exp(w.squeeze(-2) @ X.T + b + B[..., g] * X[:, 2])), obs=y)
        args, guide = (X, g, y, m, None, 7), slope_guide("Poisson", "centred", 1, intercept=False)
    else:
        X, g, y, m = _data("Poisson", 8192, 9, 40, S=2, seed=7, dev="cpu")      # 9 + 40 * 3 = 129
        args, guide = (X, g, y, m, None, 40), slope_guide("Poisson", "centred", 2)
        model = slope_model("Poisson", "centred", 2)
    l_f, p_f, calls, gm = _svi(model, guide, args, 2, True, P=4)
    l_m, p_m, _, _ = _svi(model, guide, args, 2, False, P=4)
    assert calls == 0 and not gm
    _close(l_f, p_f, l_m, p_m, 1e-6, 1e-6)


def test_out_of_range_index_raises_before_anything_reads_it(fp64_seam):
    X, g, y, m = _data("Bernoulli", 8192, 5, 7, seed=4, dev="cpu")
    launched = []
    dist._GlmSlopeFn.launch = lambda *a: launched.append(1)

    def refuse(self):
        raise AssertionError("materialised")
    saved = (dist.GroupGather.dense, dist.SlopeGather.dense, dist.LinearPredictor.dense)
    dist.GroupGather.dense = dist.SlopeGather.dense = dist.LinearPredictor.dense = refuse
    try:
        for bad in (-1, 7):
            g2 = g.clone()
            g2[100] = bad
            with pytest.raises(IndexError):
                _svi(slope_model("Bernoulli", S=2), slope_guide("Bernoulli", S=2), (X, g2, y, m, None, 7), 1, True)
    finally:
        dist.GroupGather.dense, dist.SlopeGather.dense, dist.LinearPredictor.dense = saved
    assert not launched


# ---- CPU tier: the entry point's argument checks -------------------------------------------------------------------
def test_slope_sum_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p, q = ctypes.c_void_p(4096), ctypes.c_void_p(4100)
    D, G, P, n = 10, 20, 4, 10000

    def tables(S=2, cols=(3, 7, 0), beta=(4096, 4096, 4096), strides=(G, 0, G)):
        sl = N.b2_glm_slope_tables(S)
        for k in range(3):
            sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], beta[k], strides[k]
        return ctypes.byref(sl)

    def call(kind=N.GLM_POISSON, X=p, y=p, trials=p, per_row=0, sigma=p, s_stride=0, groups=p, nG=G, W=p, w_stride=D,
             A=p, a_stride=G, sl="default", nD=D, flags=0, ws=None, nbytes=0, rows=n):
        sl = tables() if sl == "default" else sl
        return L.b2_glm_group_slope_sum(kind, X, y, trials, per_row, sigma, s_stride, groups, nG, W, w_stride, A,
                                        a_stride, sl, None, rows, nD, P, 1.0, 1.0, 1.0, flags, None, None, None, None,
                                        None, ws, nbytes, None)

    assert call() == -5                                                    # valid: the workspace check is next
    # everything b2_glm_group_sum checks
    for k in ("X", "y", "groups", "W", "A"):
        assert call(**{k: None}) == -4, k
    assert call(kind=N.GLM_BINOMIAL, trials=None) == -4 and call(kind=N.GLM_NORMAL, sigma=None) == -4
    assert call(kind=N.GLM_CATEGORICAL) == -2 and call(kind=7) == -2
    for kind in (N.GLM_BERNOULLI, N.GLM_NORMAL, N.GLM_BINOMIAL):
        assert call(kind=kind) == -5
    assert call(nG=0, a_stride=0) == -2 and call(nD=0, w_stride=0) == -2 and call(rows=0) == -2
    assert call(w_stride=0) == -5 and call(a_stride=0) == -5 and call(w_stride=D - 1) == -2 and call(a_stride=3) == -2
    assert call(X=q) == -2 and call(y=q) == -2 and call(groups=q) == -2
    assert call(kind=N.GLM_BINOMIAL, trials=q, per_row=1) == -2 and call(kind=N.GLM_BINOMIAL, trials=q) == -5
    assert call(kind=N.GLM_BINOMIAL, per_row=2) == -2
    assert call(kind=N.GLM_NORMAL, s_stride=2) == -2 and call(kind=N.GLM_NORMAL, s_stride=1) == -5
    assert call(flags=N.B2_FLAG_GLM_FP32) == -2 and call(rows=1 << 31) == -8
    # the slopes: S, columns, width, tables, strides
    assert call(sl=None) == -4
    assert call(sl=tables(S=0)) == -2 and call(sl=tables(S=4)) == -2
    assert call(sl=tables(S=1, beta=(4096, 0, 0))) == -5 and call(sl=tables(S=1, beta=(0, 4096, 4096))) == -4
    assert call(sl=tables(S=3, beta=(4096, 4096, 0))) == -4
    for cols in ((3, -1, 0), (3, D, 0), (3, 7, 3), (3, 3, 0)):
        assert call(sl=tables(S=3, cols=cols)) == -2, cols
    assert call(sl=tables(S=2, cols=(3, 7, 3))) == -5                 # only the first S columns are read
    assert call(sl=tables(S=3), nG=39, a_stride=0) == -2               # 10 + 39 * 3 > 128
    assert call(sl=tables(S=2, strides=(0, 0, 0)), nG=39, a_stride=0) == -5   # 10 + 39 * 3 = 127
    assert call(sl=tables(S=2, strides=(G - 1, 0, 0))) == -2 and call(sl=tables(S=2, strides=(0, 3, 0))) == -2
    need = int(L.b2_glm_group_slope_sum_workspace(N.GLM_POISSON, n, D, G, 2, P))
    assert need > int(L.b2_glm_group_sum_workspace(N.GLM_POISSON, n, D, G, P))
    assert call(ws=p, nbytes=need - 1) == -5
    assert L.b2_glm_group_slope_sum_workspace(N.GLM_CATEGORICAL, n, D, G, 2, P) == 256
    assert L.b2_glm_group_slope_sum_workspace(N.GLM_POISSON, n, D, 40, 2, P) == 256
    assert L.b2_glm_group_slope_sum_workspace(N.GLM_POISSON, n, D, G, 0, P) == 256
    assert L.b2_glm_group_slope_sum_workspace(N.GLM_POISSON, n, D, G, 4, P) == 256


# ---- CPU tier: what ptxas makes of the slope kernels with X rounded to TF32 -----------------------------------------
RN_SLOPE_KERNELS = ["glm_group_slope_rn_tc_kernelINS_2tc9BernoulliELi%dE" % dc for dc in (1, 2, 3, 4)] + \
                   ["glm_group_slope_rn_tc_kernelINS_2tc7PoissonELi%dE" % dc for dc in (1, 2, 3, 4)] + \
                   ["glm_group_slope_rn_tc_kernelINS_2tc8BinomialILb%dEEELi%dE" % (r, dc) for r in (0, 1)
                    for dc in (2, 3, 4)]


@pytest.fixture(scope="module")
def group_sass(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, cuobjdump = sass_test._tools()
    obj = str(tmp_path_factory.mktemp("glm_group_slope_rn") / "glm_group.o")
    src = os.path.join(_build.CSRC, "glm_group.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


@pytest.mark.parametrize("mangled", RN_SLOPE_KERNELS)
def test_rn_slope_kernel_sass(group_sass, mangled):
    """No C7515/C7520 serialisation note, no spills and no stack frame, and no warpgroup wait or arrive between two
    HGMMA of one contraction (GEMM 1 m64n64k8, GEMM 2 m64n(32 DC + 8)k8)."""
    import test_glm_tc_sass as sass_test
    log, sass = group_sass
    for line in log.splitlines():
        if mangled in line:
            assert "C7515" not in line and "C7520" not in line, line
    props, used = sass_test._ptxas_properties(log, mangled)
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used
    dc = int(re.search(r"Li(\d)E$", mangled).group(1))
    shapes, bad, prev, between = [], [], None, []
    for line in sass_test._sass_function(sass, mangled):
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            if m.group(1) == prev and between:
                bad.append("%s after %s" % (m.group(1), between))
            shapes.append(m.group(1))
            prev, between = m.group(1), []
        elif "WARPGROUP.DEPBAR" in line or "WARPGROUP.ARRIVE" in line:
            between.append(line.split(";")[0].split("*/")[-1].strip())
    assert "64x64x8" in shapes and "64x%dx8" % (32 * dc + 8) in shapes, shapes
    assert not bad, bad


def test_slope_pack_kernel_has_no_stack_frame(group_sass):
    import test_glm_tc_sass as sass_test
    props, used = sass_test._ptxas_properties(group_sass[0], "glm_group_slope_pack_kernel")
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used


# ---- GPU tier: the kernel against fp64 ------------------------------------------------------------------------------
def _launch(kind, X, y, m, g32, W, A, Bs, cols, b, sigma, flags, shared=()):
    n, D = X.shape
    G, S = A.shape[-1], len(Bs)
    P = b.shape[0]
    dev = torch.device(DEV)
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dWAB = torch.empty(P, D + G * (1 + S), device=DEV)
    db = torch.empty(P, device=DEV)
    dsig = torch.empty(P, device=DEV)
    code = KIND_CODE[kind]
    sl = N.b2_glm_slope_tables(S)
    for k in range(S):
        sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], Bs[k].data_ptr(), 0 if "beta" in shared else G
    ws = N.workspace(dev, int(N.lib().b2_glm_group_slope_sum_workspace(code, n, D, G, S, P)), tag="glm_slope_test")
    N.check(N.lib().b2_glm_group_slope_sum(
        code, X.data_ptr(), y.data_ptr(), m.data_ptr() if kind == "BinomialRows" else m[:1].clone().data_ptr(),
        int(kind == "BinomialRows"), sigma.data_ptr(), 1, g32.data_ptr(), G, W.data_ptr(), 0 if "w" in shared else D,
        A.data_ptr(), 0 if "alpha" in shared else G, ctypes.byref(sl), b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, flags,
        sum_p.data_ptr(), total.data_ptr(), dWAB.data_ptr(), db.data_ptr(), dsig.data_ptr(), ws.data_ptr(), ws.numel(),
        N.stream_ptr(dev)), "b2_glm_group_slope_sum")
    torch.cuda.synchronize()
    return sum_p, total, dWAB, db, dsig


def _reference(kind, X, y, m, g, W, A, Bs, cols, b, sigma, P):
    D, G = X.shape[1], A.shape[-1]
    Wd = W.double().expand(P, D).clone().requires_grad_(True)
    Ad = A.double().expand(P, G).clone().requires_grad_(True)
    Bd = [t.double().expand(P, G).clone().requires_grad_(True) for t in Bs]
    bd = b.double().clone().requires_grad_(True)
    sd = sigma.double().clone().requires_grad_(True)
    Xd = X.double()
    eta = Wd @ Xd.T + bd[:, None] + Ad[:, g]
    for t, c in zip(Bd, cols):
        eta = eta + t[:, g] * Xd[:, c]
    yd = y.double()
    if kind == "Bernoulli":
        lp = torch.distributions.Bernoulli(logits=eta).log_prob(yd)
    elif kind == "Poisson":
        lp = yd * eta - eta.exp() - torch.lgamma(yd + 1)
    elif kind == "Normal":
        lp = torch.distributions.Normal(eta, sd[:, None]).log_prob(yd)
    else:
        mm = m.double() if kind == "BinomialRows" else m.double()[:1]
        lp = torch.distributions.Binomial(mm, logits=eta).log_prob(yd)
    s = lp.sum(1)
    grads = torch.autograd.grad(s.sum(), [Wd, Ad, bd, sd] + Bd, allow_unused=True)
    return s.detach(), grads


def _operands(n, D, G, S, P, shared, seed, big=None, cols=None):
    gen = torch.Generator().manual_seed(seed)
    W = 0.3 * torch.randn(1 if "w" in shared else P, D, generator=gen) / D ** 0.5
    if big is not None:
        W[:, cols[0]] /= big          # the weight of the scaled column, as the slope's: logits of the usual size
    W = W.to(DEV)
    A = (0.5 * torch.randn(1 if "alpha" in shared else P, G, generator=gen)).to(DEV)
    Bs = [(0.3 * torch.randn(1 if "beta" in shared else P, G, generator=gen)
           / (big if big and k == 0 else 1.0)).to(DEV) for k in range(S)]
    b = (0.3 + 0.05 * torch.randn(P, generator=gen)).to(DEV)
    sigma = (0.6 + 0.1 * torch.rand(P, generator=gen)).to(DEV)
    return W, A, Bs, b, sigma


# (n, D, G, S, P, shared, precision, covariate magnitude): ragged N from 8192 to 1e6, D + G (1 + S) = 31, 32, 33, 64,
# 65, 96, 97, 128 and 80.  At default precision a slope column is rounded to TF32 like X's own columns, but its
# coefficient (0.3 here) is larger than w's (0.3 / sqrt(D)), so its rounding moves the logits more: 128 columns with
# three slopes take the 2e-6 bound on the sum from 250 000 rows (Poisson at 65 537 rows: 2.2e-6), and split X below.
_CASES = [(8192, 7, 12, 1, 1, "", "split", None), (8193, 8, 12, 1, 64, "w", "split", None),
          (70001, 9, 8, 2, 65, "beta", "default", None), (99999, 16, 16, 2, 64, "", "default", None),
          (250003, 17, 12, 3, 1, "alpha", "default", None), (1_000_000, 16, 20, 3, 65, "", "split", None),
          (1_000_000, 17, 40, 1, 64, "beta", "default", None), (65537, 32, 24, 3, 64, "w,beta", "split", None),
          (250001, 32, 24, 3, 65, "", "default", None),
          (70000, 16, 32, 1, 16, "", "default", 1e3), (70000, 16, 32, 1, 16, "", "split", 1e3)]
_KERNEL_KINDS = ["Bernoulli", "Poisson", "Normal", "Binomial", "BinomialRows"]


def _cols(D, S):
    return [2, 0, D - 1][:S]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _CASES, ids=["%d-D%d-G%d-S%d-P%d-%s-%s-%s" % c for c in _CASES])
@pytest.mark.parametrize("kind", _KERNEL_KINDS)
def test_kernel_against_fp64(kind, case):
    """sum_p within 2e-6 relative; dW, d/dalpha, each d/dbeta_k and db within 2e-4 of their largest entry; two
    launches bitwise equal."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G, S, P, shared, prec, big = case
    cols = _cols(D, S)
    X, g, y, m = _data(kind, n, D, G, S=S, seed=n + D + G, cols=cols, big=big)
    W, A, Bs, b, sigma = _operands(n, D, G, S, P, shared.split(","), P + D + S, big, cols)
    flags = N.B2_FLAG_GLM_3XTF32 if prec == "split" else 0
    g32 = g.to(torch.int32)
    out = _launch(kind, X, y, m, g32, W, A, Bs, cols, b, sigma, flags, shared.split(","))
    sum_p, total, dWAB, db, dsig = out
    s_ref, (gW, gA, gb, gs, *gB) = _reference(kind, X, y, m, g, W, A, Bs, cols, b, sigma, P)

    def rel(got, want):
        return float((got.double() - want).abs().max()) / float(want.abs().max())
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    errs = {"dW": rel(dWAB[:, :D], gW), "dalpha": rel(dWAB[:, D:D + G], gA), "db": rel(db, gb)}
    for k in range(S):
        errs["dbeta%d" % k] = rel(dWAB[:, D + (k + 1) * G:D + (k + 2) * G], gB[k])
    if kind == "Normal":
        errs["dsigma"] = rel(dsig, gs)
    print("\n%s %s: sum %.1e %s" % (kind, case, es, " ".join("%s %.1e" % kv for kv in errs.items())))
    assert es <= 2e-6 and all(e <= 2e-4 for e in errs.values()), (es, errs)
    again = _launch(kind, X, y, m, g32, W, A, Bs, cols, b, sigma, flags, shared.split(","))
    for u, v in zip(out[:4], again):
        assert torch.equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["split", "default"])
def test_out_of_range_index_in_the_kernel_gives_nan(prec):
    """An index that reaches the kernel unchecked makes every particle's sum and every group column (intercept and
    slopes) NaN."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G, S, P = 70000, 16, 16, 2, 8
    X, g, y, m = _data("Bernoulli", n, D, G, S=S, seed=21)
    W, A, Bs, b, sigma = _operands(n, D, G, S, P, [], 22)
    for bad in (-1, G):
        g32 = g.to(torch.int32)
        g32[4321] = bad
        sum_p, _, dWAB, _, _ = _launch("Bernoulli", X, y, m, g32, W, A, Bs, _cols(D, S), b, sigma,
                                       N.B2_FLAG_GLM_3XTF32 if prec == "split" else 0)
        assert bool(torch.isnan(sum_p).all()) and bool(torch.isnan(dWAB[:, D:]).all())


# ---- GPU tier: SVI -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", [("Bernoulli", "centred", 1, "intercept_first", "right", "colon"),
                                  ("Bernoulli", "noncentred", 2, "slopes_first", "left", "select"),
                                  ("Poisson", "centred", 3, "slope_before_bias", "right", "ellipsis"),
                                  ("Poisson", "noncentred", 1, "intercept_first", "left", "colon"),
                                  ("Normal", "centred", 2, "intercept_first", "right", "colon"),
                                  ("Normal", "noncentred", 1, "slopes_first", "right", "ellipsis"),
                                  ("Binomial", "centred", 1, "slope_before_bias", "left", "colon"),
                                  ("Binomial", "noncentred", 3, "intercept_first", "right", "select"),
                                  ("BinomialRows", "centred", 2, "intercept_first", "right", "colon")],
                         ids=lambda c: "-".join(map(str, c)))
def test_svi_matches_materialised(case):
    """Four Trace_ELBO + ClippedAdam steps at N = 70 000, D = 16, G = 24 (up to 112 columns), 16 particles: one fused
    call per step, losses within 2e-5 relative and parameters within 2e-4 of LAZY_LINEAR = False."""
    if EMULATE:
        pytest.skip("kernel test")
    kind, form, S, order, side, spelling = case
    fam = "Binomial" if kind == "BinomialRows" else kind
    X, g, y, m = _data(kind, 70000, 16, 24, S=S, seed=11)
    model, guide = slope_model(fam, form, S, order, side, spelling), slope_guide(fam, form, S)
    l_f, p_f, calls, gm = _svi(model, guide, (X, g, y, m, None, 24), 4, True, P=16)
    l_m, p_m, calls_m, _ = _svi(model, guide, (X, g, y, m, None, 24), 4, False, P=16)
    assert calls == 4 and calls_m == 0 and not gm
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_mean_field_elbo_matches_materialised():
    if EMULATE:
        pytest.skip("kernel test")
    X, g, y, m = _data("Poisson", 70000, 16, 32, S=2, seed=12)
    model, guide = slope_model("Poisson", S=2), slope_guide("Poisson", S=2)
    l_f, p_f, calls, _ = _svi(model, guide, (X, g, y, m, None, 32), 3, True, TraceMeanField_ELBO, P=16)
    l_m, p_m, _, _ = _svi(model, guide, (X, g, y, m, None, 32), 3, False, TraceMeanField_ELBO, P=16)
    assert calls == 3
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Bernoulli", "Normal"])
def test_captured_graph_step_equals_eager(kind):
    """A JitTrace_ELBO (graph-captured) run equals the eager one bit for bit; every fused site is three launches."""
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, g, y, m = _data(kind, 70000, 16, 32, S=2, seed=14)
    model, guide = slope_model(kind, S=2), slope_guide(kind, S=2)
    per_call = []
    real = dist._GlmSlopeFn.launch

    def counted(*a):
        n0 = N.launch_count()
        out = real(*a)
        per_call.append(N.launch_count() - n0)
        return out
    dist._GlmSlopeFn.launch = counted
    try:
        l_e, p_e, n_e, _ = _svi(model, guide, (X, g, y, m, None, 32), 4, True, P=16)
        l_g, p_g, n_g, _ = _svi(model, guide, (X, g, y, m, None, 32), 4, True, JitTrace_ELBO, P=16)
    finally:
        dist._GlmSlopeFn.launch = real
    assert n_e == 4 and n_g >= 1 and per_call and set(per_call) == {3}, per_call
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["N8191", "masked", "fp64", "cols129", "no_tensor_cores"])
def test_fallbacks_match_materialised(case):
    """Sites outside the fused scope make no fused call and match LAZY_LINEAR = False to 1e-6."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G, S = (8191 if case == "N8191" else 9000), (9 if case == "cols129" else 16), (40 if case == "cols129"
                                                                                          else 12), 2
    X, g, y, m = _data("Poisson", n, D, G, S=S, seed=15)
    mask = (torch.rand(n, device=DEV) < 0.7) if case == "masked" else None
    if case == "fp64":
        X, y = X.double(), y.double()
    model = slope_model("Poisson", S=S)
    if case == "no_tensor_cores":
        def model(X, g, y, m=None, mask=None, G=6):
            D = X.shape[-1]
            w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
            b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
            A = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1)).squeeze(-2)
            B0 = pyro.sample("beta0", dist.Normal(X.new_zeros(G), 0.3).to_event(1)).squeeze(-2)
            B1 = pyro.sample("beta1", dist.Normal(X.new_zeros(G), 0.3).to_event(1)).squeeze(-2)
            with pyro.plate("data", X.shape[0]):
                lp = dist.LinearPredictor(X, w, b, tensor_cores=False)
                eta = LinearPredictorTensor(lp) + A[..., g] + B0[..., g] * X[:, 2] + B1[..., g] * X[:, 0]
                pyro.sample("y", dist.Poisson(torch.exp(eta)), obs=y)
    guide = slope_guide("Poisson", S=S)
    l_f, p_f, calls, gm = _svi(model, guide, (X, g, y, m, mask, G), 2, True, P=4)
    l_m, p_m, _, _ = _svi(model, guide, (X, g, y, m, mask, G), 2, False, P=4)
    assert calls == 0 and not gm
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 1e-6 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=1e-6, rtol=1e-6), k


@pytest.mark.gpu
def test_reference_pyro_model_under_bind_matches_materialised():
    """The multilevel logistic model written against the unmodified reference with one varying slope, through
    bind.Trace_ELBO: the kernel scores the site, and three steps match the model whose logits are materialised by
    ``* 1.0``."""
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as rpyro
    import pyro.distributions as rdist
    X, g, y, _ = _data("Bernoulli", 70000, 16, 48, seed=16)

    def run(lazy):
        torch.manual_seed(0)

        def model(X, g, y):
            D = X.shape[-1]
            w = rpyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
            b = rpyro.sample("b", rdist.Normal(X.new_zeros(()), 5.0))
            a = rpyro.sample("alpha", rdist.Normal(X.new_zeros(48), 0.5).to_event(1))
            be = rpyro.sample("beta", rdist.Normal(X.new_zeros(48), 0.3).to_event(1))
            with rpyro.plate("data", X.shape[0]):
                logits = w.squeeze(-2) @ X.T + b + a.squeeze(-2)[..., g] + be.squeeze(-2)[..., g] * X[:, 2]
                rpyro.sample("y", rdist.Bernoulli(logits=logits if lazy else logits * 1.0), obs=y)

        def guide(X, g, y):
            D = X.shape[-1]
            for name, shape in (("w", (D,)), ("b", ()), ("alpha", (48,)), ("beta", (48,))):
                loc = rpyro.param(name + "_loc", X.new_zeros(shape))
                scale = rpyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=rdist.constraints.positive)
                d = rdist.Normal(loc, scale)
                rpyro.sample(name, d.to_event(1) if shape else d)

        rpyro.clear_param_store()
        calls = []
        real = dist._GlmSlopeFn.apply
        dist._GlmSlopeFn.apply = lambda *a: calls.append(1) or real(*a)
        try:
            svi = bind.SVI(model, guide, bind.ClippedAdam({"lr": 0.01}),
                           bind.Trace_ELBO(num_particles=16, vectorize_particles=True, max_plate_nesting=1))
            losses = [svi.step(X, g, y) for _ in range(3)]
        finally:
            dist._GlmSlopeFn.apply = real
        store = rpyro.get_param_store()
        return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls)

    l_f, p_f, calls = run(True)
    l_m, p_m, calls_m = run(False)
    assert calls == 3 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k
