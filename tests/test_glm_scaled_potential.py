"""NUTS / HMC on regression with a latent weight scale: the hierarchical ``w ~ Normal(0, tau)``, ARD
``w ~ Normal(0, lam)`` and horseshoe ``w ~ Normal(0, tau * lam)`` priors, through ``GlmPotential``
(``b2_glm_potential`` with a latent ``scale``).

CPU tier: which models ``recognise`` routes to ``GlmPotential`` (every likelihood kind, every scale form and prior,
scale sites drawn before and after the other sites, linear regression with a latent noise scale too), their z
layout against ``TracePotential``, the near misses that must keep the traced route, and the entry point's argument
checks.  GPU tier: U and dU/dz against an fp64 restatement and against ``TracePotential``, determinism, CUDA-graph
replay, HMC trajectories against the oracle integrator, NUTS posteriors against ``TracePotential`` runs, the routes
``NUTS(model)`` and ``bind.NUTS`` take, and the one native call of a constant weight scale."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from oracle import dists as odists
from oracle import mcmc as omcmc
from pyro_b200 import _native as N
from pyro_b200.infer import HMC, MCMC, NUTS
from pyro_b200.infer.mcmc import GlmPotential, LogisticPotential, TracePotential
from pyro_b200.infer.mcmc.compile import recognise

DEV = device()
KINDS = ["Bernoulli", "Categorical", "Poisson", "Binomial", "Normal"]
FORMS = ["tau", "lam", "tau*lam", "lam*tau"]
PRIORS = ["HalfNormal", "HalfCauchy", "Exponential", "LogNormal"]
K_CAT = 3
TRIALS = 10.0


# ---- models ----------------------------------------------------------------------------------------------------
def _scale_prior(prior, X, shape=(), how="expand"):
    """A positive prior with constant parameters; for a per-coefficient ``shape``, one value repeated, written as
    an expansion or as full parameter tensors."""
    params = {"HalfNormal": (1.5,), "HalfCauchy": (1.0,), "Exponential": (2.0,), "LogNormal": (-0.5, 0.8)}[prior]
    if shape and how == "full":
        d = getattr(dist, prior)(*[X.new_full(shape, p) for p in params])
        return d.to_event(len(shape))
    d = getattr(dist, prior)(*[X.new_full((), p) for p in params])
    return d.expand(shape).to_event(len(shape)) if shape else d


def _wshape(kind, D):
    return (K_CAT, D) if kind == "Categorical" else (D,)


def _eta(kind, X, w, b):
    if kind == "Categorical":
        return X @ (w.squeeze(-3) if w.dim() > 2 else w).mT + b
    return (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b


def _likelihood(kind, eta, sigma):
    if kind == "Bernoulli":
        return dist.Bernoulli(logits=eta)
    if kind == "Categorical":
        return dist.Categorical(logits=eta)
    if kind == "Poisson":
        return dist.Poisson(torch.exp(eta))
    if kind == "Binomial":
        return dist.Binomial(eta.new_full((), TRIALS), logits=eta)
    return dist.Normal(eta, sigma)


def scaled_model(kind, form, prior="HalfCauchy", bias=True, order="scales_first", sigma="const", lam_how="expand",
                 change=None):
    """Regression of ``kind`` with the weight prior Normal(0, S), S = tau, lam, tau * lam or lam * tau (``form``).
    ``order``: "scales_first" draws tau, lam, w, b (, sigma); "bias_first" draws b (, sigma), lam, tau, w.
    ``sigma`` (linear regression): "const" (0.6) or "latent" (HalfNormal(1.5)).  ``change`` makes a near miss."""
    def model(X, y):
        D = X.shape[-1]
        wshape = _wshape(kind, D)
        site = {}

        def draw_bias():
            if bias:
                bshape = (K_CAT,) if kind == "Categorical" else ()
                s_b = X.new_full(bshape, 10.0)
                if change == "bias_scale":
                    s_b = s_b * site["tau"]
                d = dist.Normal(X.new_zeros(bshape), s_b)
                site["b"] = pyro.sample("b", d.to_event(len(bshape)) if bshape else d)
            if kind == "Normal" and sigma == "latent":
                site["sigma"] = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))

        def draw_scales():
            names = ["tau", "lam"] if order == "scales_first" else ["lam", "tau"]
            for name in names:
                if name == "tau" and "tau" in form:
                    p = "Uniform" if change == "uniform" else prior
                    d = dist.Uniform(X.new_zeros(()), X.new_full((), 5.0)) if p == "Uniform" \
                        else _scale_prior(prior, X)
                    site["tau"] = pyro.sample("tau", d)
                if name == "lam" and "lam" in form:
                    lshape = (D,) if change == "lam_shape" else wshape
                    if change == "lam_varying":
                        d = dist.HalfCauchy(torch.linspace(0.5, 1.5, D, dtype=X.dtype).expand(lshape)).to_event(
                            len(lshape))
                    else:
                        d = _scale_prior(prior, X, lshape, lam_how)
                    site["lam"] = pyro.sample("lam", d)
            if change == "extra":
                pyro.sample("extra", dist.HalfNormal(X.new_full((), 1.0)))

        if order == "bias_first" and change != "bias_scale":
            draw_bias()
            draw_scales()
        else:
            draw_scales()
        # S broadcast over the weight's shape: tau carries the chain dims of a scalar site
        tau = site.get("tau")
        if tau is not None:
            tau = tau.reshape(tau.shape + (1,) * len(wshape))
        lam = site.get("lam")
        if form == "tau":
            S = tau ** 2 if change == "square" else tau
        elif form == "lam":
            S = lam
        elif form == "tau*lam":
            S = tau + lam if change == "sum" else tau * lam
        else:
            S = lam * tau
        w = pyro.sample("w", dist.Normal(X.new_zeros(wshape), S).to_event(len(wshape)))
        if order != "bias_first" or change == "bias_scale":
            draw_bias()
        b = site.get("b", 0.0)
        with pyro.plate("data", X.shape[0]):
            eta = _eta(kind, X, w, b)
            if change == "in_likelihood":
                eta = eta * site["tau"].unsqueeze(-1) if site["tau"].dim() else eta * site["tau"]
            s = site.get("sigma", 0.6)
            d = _likelihood(kind, eta, s)
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool, device=X.device))
            pyro.sample("y", d, obs=y)
    return model


def _data(kind, n, D, dtype=torch.float32, dev="cpu", seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn(n, D, generator=g, device=dev, dtype=dtype)
    wt = torch.randn(_wshape(kind, D), generator=g, device=dev, dtype=dtype) / D ** 0.5
    wt = wt * (torch.rand(wt.shape, generator=g, device=dev, dtype=dtype) < 0.5)   # sparse: half the weights zero
    if kind == "Categorical":
        y = torch.multinomial(torch.softmax(X @ wt.mT, -1), 1, generator=g).squeeze(-1)
        return X, y
    eta = X @ wt + 0.3
    u = torch.rand(n, generator=g, device=dev, dtype=dtype)
    if kind == "Bernoulli":
        y = (u < torch.sigmoid(eta)).to(dtype)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta), generator=g)
    elif kind == "Binomial":
        p = torch.sigmoid(eta)
        y = (torch.rand(n, int(TRIALS), generator=g, device=dev, dtype=dtype) < p[:, None]).sum(-1).to(dtype)
    else:
        y = eta + 0.6 * torch.randn(n, generator=g, device=dev, dtype=dtype)
    return X, y


def _recognised(model, *args):
    import cpu_emulation
    with cpu_emulation.enabled():
        return recognise(model, args)


def _check_layout(pot, model, args):
    tp = TracePotential(model, args)
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, transform, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
        assert transform == ("exp" if site in ("tau", "lam", "sigma") else "identity"), site
    z = torch.randn(3, pot.dim)
    got, want = pot.unpack(z), tp.unpack(z)
    assert list(got) == list(want)
    for site in got:
        assert got[site].shape == want[site].shape and torch.allclose(got[site], want[site]), site


# ---- CPU tier: recognition and layout ----------------------------------------------------------------------------
@pytest.mark.parametrize("prior", PRIORS)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
def test_recognises_latent_weight_scales(kind, form, prior):
    X, y = _data(kind, 300, 32 if kind in ("Bernoulli", "Categorical") else 10)
    model = scaled_model(kind, form, prior)
    pot = _recognised(model, X, y)
    assert isinstance(pot, GlmPotential), (kind, form, prior)
    assert pot.tau_site == ("tau" if "tau" in form else None)
    assert pot.lam_site == ("lam" if "lam" in form else None)
    assert pot.sigma_site is None and pot.has_bias
    sc = pot.weight_scale
    code = GlmPotential._SIGMA_PRIORS[prior]
    if pot.tau_site:
        assert sc.tau_off == pot.sites["tau"][0].start and sc.tau_prior == code
    if pot.lam_site:
        assert sc.lam_off == pot.sites["lam"][0].start and sc.lam_prior == code
        assert pot.sites["lam"][2] == _wshape(kind, X.shape[1])
    _check_layout(pot, model, (X, y))


@pytest.mark.parametrize("case", ["bias_first", "lam_full", "normal_sigma_tau", "normal_sigma_horseshoe_bias_first",
                                  "nobias_logistic", "nobias_softmax"])
def test_recognition_variants(case):
    kind, form, kw = {"bias_first": ("Poisson", "tau*lam", dict(order="bias_first")),
                      "lam_full": ("Bernoulli", "lam", dict(lam_how="full")),
                      "normal_sigma_tau": ("Normal", "tau", dict(sigma="latent")),
                      "normal_sigma_horseshoe_bias_first": ("Normal", "lam*tau",
                                                            dict(sigma="latent", order="bias_first")),
                      "nobias_logistic": ("Bernoulli", "tau", dict(bias=False)),
                      "nobias_softmax": ("Categorical", "lam", dict(bias=False))}[case]
    X, y = _data(kind, 300, 32 if kind in ("Bernoulli", "Categorical") else 10)
    model = scaled_model(kind, form, **kw)
    pot = _recognised(model, X, y)
    assert isinstance(pot, GlmPotential), case
    _check_layout(pot, model, (X, y))
    if kw.get("order") == "bias_first":
        assert list(pot.sites)[0] == "b" and list(pot.sites)[-1] == "w"
    if kw.get("sigma") == "latent":
        assert pot.sigma_site == "sigma" and pot.sites["sigma"][1] == "exp"
        assert pot.tau_site == "tau"
    if not kw.get("bias", True):
        assert not pot.has_bias


@pytest.mark.parametrize("change", ["sum", "square", "lam_shape", "lam_varying", "uniform", "in_likelihood",
                                    "bias_scale", "extra", "mask", "fp64"])
def test_near_misses_are_not_recognised(change):
    kind, form = "Bernoulli", "tau*lam"
    if change == "square":
        form = "tau"
    if change == "lam_shape":
        kind, form = "Categorical", "lam"
    if change in ("in_likelihood", "bias_scale", "uniform"):
        form = "tau"
    X, y = _data(kind, 300, 32, dtype=torch.float64 if change == "fp64" else torch.float32)
    model = scaled_model(kind, form, change=None if change == "fp64" else change)
    pot = _recognised(model, X, y)
    assert not isinstance(pot, GlmPotential), change


def test_sigma_used_as_weight_scale_is_not_recognised():
    """A noise scale that is also the weight scale has two roles."""
    def model(X, y):
        D = X.shape[-1]
        s = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), s.unsqueeze(-1)).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        with pyro.plate("data", X.shape[0]):
            pyro.sample("y", dist.Normal(_eta("Normal", X, w, b), s), obs=y)
    X, y = _data("Normal", 300, 10)
    assert not isinstance(_recognised(model, X, y), GlmPotential)


def test_intercept_free_logistic_with_constant_scale_keeps_logistic_potential():
    def model(X, y):
        beta = pyro.sample("beta", dist.Normal(X.new_zeros(X.shape[-1]), X.new_ones(X.shape[-1])))
        logits = (X * beta.unsqueeze(-2)).sum(-1) if beta.dim() > 1 else (X * beta).sum(-1)
        return pyro.sample("y", dist.Bernoulli(logits=logits), obs=y)
    X, y = _data("Bernoulli", 300, 16)
    assert isinstance(_recognised(model, X, y), LogisticPotential)


def test_latent_scale_entry_point_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)
    D = 10

    def regression(kind=N.GLM_POISSON, X=p, y=p, trials=None, per_row=0, n=10000, Dx=D, K=1, bias=1, w_off=1,
                   b_off=D + 1, s_off=-1, s_b=10.0, s_prior=0, sp0=0.0, sp1=0.0, sigma=1.0, tau=(0, 1, 1.0, 1.0),
                   lam=(D + 2, 2, 1.0, 1.0)):
        sc = N.b2_glm_weight_scale()
        sc.tau_off, sc.tau_prior, sc.tau_p0, sc.tau_p1 = tau
        sc.lam_off, sc.lam_prior, sc.lam_p0, sc.lam_p1 = lam
        return N.b2_glm_regression(kind=kind, X=X, y=y, N=n, D=Dx, K=K, trials=trials, trials_per_row=per_row,
                                   has_bias=bias, w_off=w_off, b_off=b_off, s_b=s_b, s_off=s_off, s_prior=s_prior,
                                   sp0=sp0, sp1=sp1, sigma=sigma, scale=ctypes.pointer(sc))

    def call(z=p, Dz=2 * D + 2, null=False, ws=None, nbytes=0, **kw):
        m = None if null else ctypes.byref(regression(**kw))
        return L.b2_glm_potential(m, z, 4, Dz, p, p, ws, nbytes, None)

    # z = [tau, w (10), b, lam (10)]: valid, so the workspace check is next
    assert call() == -5
    assert call(X=None) == -4 and call(y=None) == -4 and call(z=None) == -4 and call(null=True) == -4
    assert call(kind=N.GLM_BINOMIAL) == -4                                   # Binomial needs its trials
    assert call(kind=7) == -2 and call(kind=N.GLM_BERNOULLI) == -2          # Bernoulli: D in {4, 8, 16, 32}
    assert call(Dx=129) == -2 and call(n=0) == -2
    assert call(n=1 << 31) == -8
    # the row: out of it, overlapping, or not exactly the blocks
    assert call(Dz=2 * D + 3) == -2 and call(Dz=2 * D + 1) == -2
    assert call(tau=(1, 1, 1.0, 1.0)) == -2                                  # tau inside w
    assert call(lam=(D + 1, 2, 1.0, 1.0)) == -2                              # lam over b
    assert call(lam=(D + 3, 2, 1.0, 1.0)) == -2                              # lam past the row's end
    assert call(w_off=-1) == -2 and call(b_off=2 * D + 2) == -2
    assert call(tau=(-1, 1, 1.0, 1.0), lam=(-1, 1, 1.0, 1.0)) == -2          # no latent weight scale
    assert call(s_off=2 * D + 2, Dz=2 * D + 3) == -2                         # a noise scale outside linear regression
    # priors: codes in range, positive parameters, a finite LogNormal loc
    assert call(tau=(0, 0, 1.0, 1.0)) == -2 and call(lam=(D + 2, 5, 1.0, 1.0)) == -2
    assert call(tau=(0, N.SIGMA_HALFCAUCHY, 0.0, 1.0)) == -2 and call(lam=(D + 2, N.SIGMA_EXPONENTIAL, -1.0, 1.0)) == -2
    assert call(tau=(0, N.SIGMA_LOGNORMAL, math.inf, 1.0)) == -2 and call(tau=(0, N.SIGMA_LOGNORMAL, 0.0, 0.0)) == -2
    assert call(tau=(0, N.SIGMA_LOGNORMAL, -3.0, 0.5)) == -5
    assert call(s_b=0.0) == -2 and call(bias=0, Dz=2 * D + 1, lam=(D + 1, 2, 1.0, 1.0)) == -5
    # alignment
    assert call(X=q) == -2 and call(y=q) == -2
    assert call(kind=N.GLM_BINOMIAL, trials=q, per_row=1) == -2 and call(kind=N.GLM_BINOMIAL, trials=q) == -5
    assert call(kind=N.GLM_BINOMIAL, trials=p, per_row=2) == -2
    # linear regression: a latent sigma with a valid prior, or a positive constant
    nz = dict(kind=N.GLM_NORMAL, Dz=2 * D + 3, s_off=2 * D + 2)
    assert call(**nz, s_prior=N.SIGMA_HALFNORMAL, sp0=1.0) == -5
    assert call(**nz, s_prior=0, sp0=1.0) == -2 and call(**nz, s_prior=N.SIGMA_HALFNORMAL, sp0=0.0) == -2
    assert call(**dict(nz, s_off=D + 1), s_prior=N.SIGMA_HALFNORMAL, sp0=1.0) == -2   # sigma over b
    assert call(kind=N.GLM_NORMAL, sigma=0.0) == -2 and call(kind=N.GLM_NORMAL, sigma=0.6) == -5
    # softmax: lam is K*D wide
    KD = K_CAT * 32
    assert call(kind=N.GLM_CATEGORICAL, Dx=32, K=K_CAT, Dz=2 * KD + K_CAT + 1, w_off=1, b_off=KD + 1,
                lam=(KD + K_CAT + 1, 2, 1.0, 1.0)) == -5
    assert call(kind=N.GLM_CATEGORICAL, Dx=32, K=K_CAT, Dz=KD + 32 + K_CAT + 1, w_off=1, b_off=KD + 1,
                lam=(KD + K_CAT + 1, 2, 1.0, 1.0)) == -2
    need = int(L.b2_glm_potential_workspace(ctypes.byref(regression()), 4))
    assert need > 256 and call(ws=p, nbytes=need - 1) == -5


# ---- GPU tier ------------------------------------------------------------------------------------------------------
def _prior_lp(prior, v):
    kind, p0, p1 = prior
    zero = torch.zeros((), dtype=v.dtype, device=v.device)
    if kind == "HalfNormal":
        return odists.half_normal(v, zero + p0)
    if kind == "HalfCauchy":
        return odists.half_cauchy(v, zero + p0)
    if kind == "Exponential":
        return odists.exponential(v, zero + p0)
    return odists.log_normal(v, zero + p0, zero + p1)


def _prior_of(pot, part):
    """(kind, p0, p1) of the tau or lam prior the potential was given"""
    inv = {v: k for k, v in GlmPotential._SIGMA_PRIORS.items()}
    sc = pot.weight_scale
    return inv[getattr(sc, part + "_prior")], getattr(sc, part + "_p0"), getattr(sc, part + "_p1")


def _oracle_potential(X, y, pot, kind):
    """fp64 U(z) (pyro/infer/mcmc/util.py:275-286): -(log joint) - SUM of the logs of the positive sites (the
    Jacobians of their exp transforms)."""
    Xd = X.double()
    yd = y if kind == "Categorical" else y.double()

    def U(z):
        zero = torch.zeros((), dtype=z.dtype, device=z.device)
        lp = torch.zeros(z.shape[:-1], dtype=z.dtype, device=z.device)
        vals = {}
        for name, (sl, transform, _) in pot.sites.items():
            u = z[..., sl]
            vals[name] = u.exp() if transform == "exp" else u
            if transform == "exp":
                lp = lp + u.sum(-1)
        w = vals[pot.weight]
        S = zero + 1.0
        if pot.tau_site is not None:
            S = S * vals[pot.tau_site]
            lp = lp + _prior_lp(_prior_of(pot, "tau"), vals[pot.tau_site]).sum(-1)
        if pot.lam_site is not None:
            S = S * vals[pot.lam_site]
            lp = lp + _prior_lp(_prior_of(pot, "lam"), vals[pot.lam_site]).sum(-1)
        lp = lp + odists.normal(w, zero, S).sum(-1)
        bv = 0.0
        if pot.bias is not None:
            bv = vals[pot.bias]
            lp = lp + odists.normal(bv, zero, zero + pot.s_b).sum(-1)
        if kind == "Categorical":
            W = w.reshape(w.shape[:-1] + (pot.K, pot.Dx))
            logits = Xd @ W.mT + (bv.unsqueeze(-2) if pot.bias is not None else 0.0)
            return -(lp + odists.categorical(yd, logits).sum(-1))
        eta = w @ Xd.T + bv
        if kind == "Bernoulli":
            ll = odists.bernoulli_logits(yd, eta)
        elif kind == "Poisson":
            ll = odists.poisson(yd, eta.exp())
        elif kind == "Binomial":
            m = zero + TRIALS
            ll = (torch.lgamma(m + 1) - torch.lgamma(yd + 1) - torch.lgamma(m - yd + 1) + yd * eta
                  - m * F.softplus(eta))
        else:
            if pot.sigma_site is not None:
                s = vals[pot.sigma_site]
                lp = lp + odists.half_normal(s, zero + 1.5).sum(-1)
            else:
                s = zero + pot.sigma
            ll = odists.normal(yd, eta, s)
        return -(lp + ll.sum(-1))
    return U


def _oracle_value_and_grad(U, z, n, K):
    """fp64 U and dU/dz, in chunks of chains that keep the [c, N, K] logits near 1 GB."""
    step = max(1, (1 << 27) // (n * K))
    Us, Gs = [], []
    for i in range(0, z.shape[0], step):
        zc = z[i:i + step].double().detach().requires_grad_(True)
        u = U(zc)
        (g,) = torch.autograd.grad(u.sum(), zc)
        Us.append(u.detach())
        Gs.append(g)
    return torch.cat(Us), torch.cat(Gs)


def _chain_state(pot, C, seed):
    """Chains in the body of the prior: w small, log scales near 0, log sigma near log 0.6."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = 0.3 * torch.randn(C, pot.dim, generator=g)
    if pot.sigma_site is not None:
        z[:, pot.sites[pot.sigma_site][0]] += math.log(0.6)
    return z.to(DEV)


def _gpu_setup(kind, form, n, sigma="const", seed=0):
    D = 32 if kind in ("Bernoulli", "Categorical") else 10
    X, y = _data(kind, n, D, dev=DEV, seed=seed)
    model = scaled_model(kind, form, sigma=sigma)
    pot = recognise(model, (X, y))
    assert isinstance(pot, GlmPotential), (kind, form)
    return X, y, model, pot


@pytest.mark.gpu
@pytest.mark.parametrize("n", [300, 8192, 1_000_000])
@pytest.mark.parametrize("form", ["tau", "lam", "tau*lam"])
@pytest.mark.parametrize("kind", KINDS)
def test_potential_against_fp64_and_trace(kind, form, n):
    """U and dU/dz for C = 1, 8, 130 chains against fp64, bitwise repeatable, and against TracePotential where its
    [C, N, K] logits fit comfortably, within the bounds of the constant-scale potential's tests
    (tests/test_glm_potential.py): U 2e-6 relative to max(1, |U|), the gradient 2e-4 of max |grad| at N = 1e6 and up
    to 64 chains, 5e-4 elsewhere."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, model, pot = _gpu_setup(kind, form, n, sigma="latent" if form == "tau*lam" else "const", seed=n)
    K = pot.K
    U_ref_fn = _oracle_potential(X, y, pot, kind)
    errs = []
    for C in (1, 8, 130):
        z = _chain_state(pot, C, C)
        U, G = pot.value_and_grad(z)
        U2, G2 = pot.value_and_grad(z)
        assert torch.equal(U, U2) and torch.equal(G, G2)
        Ur, Gr = _oracle_value_and_grad(U_ref_fn, z, n, K)
        eu = float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max())
        eg = float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max()))
        et = gt = 0.0
        if C * n * K <= 64 * 70001 * 16:
            tp = TracePotential(model, (X, y), num_chains=C)
            assert list(tp.sites) == list(pot.sites) and tp.dim == pot.dim
            Ut, Gt = tp.value_and_grad(z)
            et = float(((U - Ut).abs() / Ut.abs().clamp(min=1.0)).max())
            gt = float((G - Gt).abs().max()) / max(1.0, float(Gt.abs().max()))
        errs.append((C, eu, eg, et, gt))
    print("\nscaled potential %s %s n=%d: (C, U vs fp64, grad vs fp64, U vs trace, grad vs trace) %s"
          % (kind, form, n, ["%d %.1e %.1e %.1e %.1e" % e for e in errs]))
    for C, eu, eg, et, gt in errs:
        gtol = 2e-4 if n == 1_000_000 and C <= 64 else 5e-4
        assert eu <= 2e-6 and eg <= gtol, (C, eu, eg)
        assert et <= 2e-6 and gt <= 5e-4, (C, et, gt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,form,sigma", [("Bernoulli", "tau*lam", "const"), ("Categorical", "lam", "const"),
                                             ("Normal", "tau*lam", "latent")])
def test_captured_graph_replay_equals_eager(kind, form, sigma):
    if EMULATE:
        pytest.skip("needs CUDA graphs")
    X, y, _, pot = _gpu_setup(kind, form, 70001, sigma=sigma, seed=3)
    z = _chain_state(pot, 64, 0)
    U0, G0 = pot.value_and_grad(z)
    zbuf = torch.zeros_like(z)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pot.value_and_grad(zbuf)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    n0 = N.launch_count()
    with torch.cuda.graph(graph):
        Ug, Gg = pot.value_and_grad(zbuf)
    assert N.launch_count() - n0 == 4   # pack, GLM kernel, GLM finish, potential finish
    zbuf.copy_(z)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(Ug, U0) and torch.equal(Gg, G0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,form", [("Bernoulli", "tau*lam"), ("Poisson", "lam")],
                         ids=["horseshoe-logistic", "ard-poisson"])
def test_hmc_trajectory_matches_oracle_integrator(kind, form):
    """Twenty leapfrog steps of HMC's integrator on GlmPotential from identical (z, r) against
    oracle.mcmc.velocity_verlet on the fp64 potential."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.004
    X, y, _, pot = _gpu_setup(kind, form, n, seed=11)
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = _chain_state(pot, C, 5)
    r0 = torch.randn(C, pot.dim, device=DEV)
    z, r = z0.clone(), r0.clone()
    _, g = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, g, U, _ = kernel._leapfrog(z, r, g, epsv, minv)
    Uo = _oracle_potential(X.cpu(), y.cpu(), pot, kind)
    errs = []
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        errs.append((float((z[c].double().cpu() - zr).abs().max()),
                     float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max())),
                     abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))))
    print("\nhmc trajectory %s %s: (z err, r err, U err) %s" % (kind, form, ["%.1e %.1e %.1e" % e for e in errs]))
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


def _hierarchical_logistic(X, y):
    D = X.shape[-1]
    tau = pyro.sample("tau", dist.HalfNormal(X.new_full((), 1.0)))
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), tau.unsqueeze(-1)).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_eta("Bernoulli", X, w, b)), obs=y)


def _ard_linear(X, y):
    D = X.shape[-1]
    lam = pyro.sample("lam", dist.HalfNormal(X.new_ones(D)).to_event(1))
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), lam).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Normal(_eta("Normal", X, w, b), sigma), obs=y)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["hierarchical_logistic", "ard_linear"])
def test_nuts_posterior_matches_trace_potential(case):
    """NUTS at N = 10^4, D = 8, 8 chains on GlmPotential against a run on TracePotential (compile_model = False) of
    the same model: means within 0.3 posterior standard deviations, standard deviations within 25 %.  The ARD
    model's per-coefficient scales make a funnel for the weights near zero; its trees are capped at depth 6 in both
    runs so that the traced run stays short."""
    if EMULATE:
        pytest.skip("kernel test")
    model, kind = (_hierarchical_logistic, "Bernoulli") if case == "hierarchical_logistic" \
        else (_ard_linear, "Normal")
    D = 8
    X, y = _data(kind, 10_000, D, dev=DEV, seed=21)
    out = {}
    for compile_model in (True, False):
        kernel = NUTS(model, max_tree_depth=6) if kind == "Normal" else NUTS(model)
        kernel.compile_model = compile_model
        mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1 if compile_model else 2)
        mc.run(X, y)
        want = GlmPotential if compile_model else TracePotential
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        s = mc.get_samples()
        width = {"w": D, "lam": D, "b": 1, "tau": 1, "sigma": 1}
        # the positive sites on the log scale, where their posteriors are closer to Normal
        cols = [s[name].reshape(-1, width[name]).double().cpu() for name in sorted(s)]
        out[compile_model] = torch.cat([c.log() if name in ("tau", "lam", "sigma") else c
                                        for name, c in zip(sorted(s), cols)], -1)
    got, ref = out[True], out[False]
    m_, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    print("\nnuts %s: max |mean diff| / sd %.2f, max |sd diff| / sd %.2f"
          % (case, float(((m_ - rm).abs() / rs).max()), float(((sd - rs).abs() / rs).max())))
    assert bool(((m_ - rm).abs() <= 0.3 * rs).all()), float(((m_ - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


@pytest.mark.gpu
def test_routes_taken_by_nuts_model():
    """NUTS(model) builds GlmPotential for latent weight scales of every kind and samples on it."""
    if EMULATE:
        pytest.skip("kernel test")
    for kind, form, sigma in (("Bernoulli", "tau*lam", "const"), ("Categorical", "tau", "const"),
                              ("Poisson", "lam", "const"), ("Binomial", "lam*tau", "const"),
                              ("Normal", "tau*lam", "latent")):
        X, y = _data(kind, 9000, 32 if kind in ("Bernoulli", "Categorical") else 10, dev=DEV, seed=1)
        kernel = NUTS(scaled_model(kind, form, sigma=sigma))
        kernel.setup(5, 4, X, y)
        assert type(kernel.potential) is GlmPotential and kernel.potential.weight_scale is not None, kind
        n0 = N.launch_count()
        kernel.sample()
        assert N.launch_count() - n0 > 0 and kernel.num_leapfrogs > 0


@pytest.mark.gpu
def test_bind_nuts_recognises_reference_pyro_models():
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as ref_pyro
    import pyro.distributions as rdist
    from pyro.infer import MCMC as RefMCMC

    def horseshoe(X, y):
        D = X.shape[-1]
        tau = ref_pyro.sample("tau", rdist.HalfCauchy(X.new_ones(())))
        lam = ref_pyro.sample("lam", rdist.HalfCauchy(X.new_ones(D)).to_event(1))
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), tau.unsqueeze(-1) * lam).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Bernoulli(logits=X @ w + b), obs=y)

    def ard_linear(X, y):
        D = X.shape[-1]
        with ref_pyro.plate("coef", D):
            lam = ref_pyro.sample("lam", rdist.Exponential(X.new_full((), 2.0)))
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), lam).to_event(1))
        sigma = ref_pyro.sample("sigma", rdist.HalfNormal(X.new_full((), 1.5)))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Normal(X @ w, sigma), obs=y)

    Xb, yb = _data("Bernoulli", 4000, 32, dev=DEV, seed=1)
    Xn, yn = _data("Normal", 4000, 10, dev=DEV, seed=2)
    for model, args in ((horseshoe, (Xb, yb)), (ard_linear, (Xn, yn))):
        pot = bind.recognise(model, args, {}, poutine=ref_pyro.poutine)
        assert isinstance(pot, GlmPotential) and pot.weight_scale is not None, model.__name__
        kernel = bind.NUTS(model, num_chains=4, seed=0)
        mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
        mc.run(*args)
        assert isinstance(kernel._kernel.potential, GlmPotential)
        for v in mc.get_samples().values():
            assert bool(torch.isfinite(v).all())


@pytest.mark.gpu
def test_constant_scale_makes_one_call_with_no_scale_or_group(monkeypatch):
    """A constant weight scale makes the one b2_glm_potential call with a null scale, a null group and today's
    scalar arguments."""
    if EMULATE:
        pytest.skip("kernel test")
    import models
    X, y = _data("Bernoulli", 9000, 32, dev=DEV, seed=4)
    pot = recognise(models.logistic_model, (X, y))
    assert isinstance(pot, GlmPotential) and pot.weight_scale is None
    L = N.lib()
    calls = []
    real = L.b2_glm_potential

    def spy(*a):
        m = a[0]._obj
        calls.append((m.kind, m.N, m.D, m.K, m.has_bias, a[2], a[3], m.w_off, m.b_off, m.s_w, m.s_b, bool(m.scale),
                      bool(m.group)))
        return real(*a)

    monkeypatch.setattr(L, "b2_glm_potential", spy)
    z = 0.3 * torch.randn(8, pot.dim, device=DEV)
    U, G = pot.value_and_grad(z)
    torch.cuda.synchronize()
    assert calls == [(N.GLM_BERNOULLI, 9000, 32, 1, 1, 8, 33, 0, 32, 1.0, 10.0, False, False)]
    assert bool(torch.isfinite(U).all())
