"""NUTS / HMC on multilevel regression with varying slopes: ``X @ w + b + alpha[g] + SUM_k beta_k[g] * X[:, c_k]``
through ``GlmPotential`` (``b2_glm_potential`` with ``b2_glm_group_effect.S`` slopes), each slope scored as G
more columns of the fused GLM kernel's contraction, ``x_{c_k} onehot(g)``.

CPU tier: which models ``recognise`` routes to ``GlmPotential`` (every likelihood kind, centred and non-centred slopes,
a constant slope scale or each of the four priors on a latent one, one to three slopes with mixed forms, the ways a
model can write the slope term), their z layout against ``TracePotential``, the near misses that must keep the traced
route, and the entry point's checks of the slope fields.  GPU tier: U and dU/dz against an fp64 restatement and
against ``TracePotential`` (C = 1, 64, 65, ragged N and widths, a covariate of magnitude 1e3), determinism, the NaN of
an out-of-range group index in every block, CUDA-graph replay, an HMC trajectory against the oracle integrator, NUTS
posteriors against ``TracePotential`` runs, and the route ``bind.NUTS`` takes with reference Pyro."""
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
from pyro_b200.infer.mcmc import GlmPotential, TracePotential
from pyro_b200.infer.mcmc.compile import recognise
from test_glm_group_potential import PRIOR_PARAMS, S_B, S_CONST, S_W, TRIALS, _lin, _likelihood, _prior_lp, \
    _recognised, group_sass  # noqa: F401 -- group_sass is a fixture
from test_glm_group_potential import test_group_kernel_sass as _check_group_kernel_sass

DEV = device()
KINDS = ["Bernoulli", "Poisson", "Binomial", "Normal"]
FORMS = ["centred", "noncentred"]
SCALES = ["const", "HalfNormal", "HalfCauchy", "Exponential", "LogNormal"]


def _chains(t):
    """A table with TracePotential's chain dims ([C, 1, G]) as [C, G]; a prototype's [G] as it is."""
    return t.squeeze(-2) if t.dim() > 1 else t


def slope_model(kind, slopes=(("centred", "const", 2),), a_form="centred", a_scale="const", G=6, sigma="const",
                spelling="ellipsis", change=None):
    """Regression of ``kind`` with a varying intercept (``a_form``, ``a_scale``, as in test_glm_group_potential) and
    one varying slope per ``(form, scale, column)`` of ``slopes``: ``beta_k ~ Normal(0, s_k)[G]`` (centred) or
    ``beta_k = s_k * eta_k`` (non-centred), ``s_k`` the constant 0.4 + 0.1 k or a positive site ``s_k`` with prior
    ``scale``, times ``X[:, column]``.  ``spelling`` is how the model writes the slope term; ``change`` makes a near
    miss."""
    def table(X, name, form, scale, const, shared=None):
        """(the [G] table as the likelihood uses it, eta of a non-centred one, the scale as drawn)"""
        if shared is not None:
            s = shared
        elif scale == "const":
            s = X.new_full((), const)
        else:
            s = pyro.sample("s_" + name, getattr(dist, scale)(*[X.new_full((), p) for p in PRIOR_PARAMS[scale]]))
        loc = X.new_zeros(G)
        if change == "mean" and name == "b1":
            loc = loc + 0.5
        if change == "latent_mean" and name == "b1":
            loc = loc + pyro.sample("mu_b1", dist.Normal(X.new_zeros(()), 1.0)).unsqueeze(-1)
        if form == "centred":
            t = pyro.sample("beta_" + name if name != "a" else "alpha", dist.Normal(loc, s.unsqueeze(-1)).to_event(1))
            return _chains(t), None, s
        e = pyro.sample("eta_" + name, dist.Normal(loc, X.new_ones(())).to_event(1))
        return _chains(s.unsqueeze(-1) * e), _chains(e), s

    def model(X, g, y, xs=None):
        D = X.shape[-1]
        site = {}
        site["w"] = pyro.sample("w", dist.Normal(X.new_zeros(D), S_W).to_event(1))
        site["b"] = pyro.sample("b", dist.Normal(X.new_zeros(()), S_B))
        if kind == "Normal" and sigma == "latent":
            site["sigma"] = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
        eta = _lin(X, site["w"], site["b"])
        if change != "no_intercept":
            A, _, sa = table(X, "a", a_form, a_scale, S_CONST)
            eta = eta + A[..., g]
        for k, (form, scale, col) in enumerate(slopes, 1):
            shared = None
            if change == "shared_scale" and k == 1:
                shared = sa
            if change == "scale_is_sigma" and k == 1:
                shared = site["sigma"]
            Bk, ek, sk = table(X, "b%d" % k, form, scale, 0.4 + 0.1 * k, shared)
            x = X[:, col]
            if change == "separate_cov" and k == 1:
                x = xs
            elif change == "square" and k == 1:
                x = x ** 2
            elif change == "plus_one" and k == 1:
                x = x + 1
            gk = (g + 1) % G if change == "other_index" and k == 1 else g
            if spelling == "x_first":
                term = x * Bk[gk]
            elif spelling == "index_select":
                term = Bk.index_select(-1, gk) * X[..., col]
            elif spelling == "scale_after":
                term = sk * ek[..., gk] * x
            else:
                term = Bk[..., gk] * x
            eta = eta + term
        with pyro.plate("data", X.shape[0]):
            d = _likelihood(kind, eta, site.get("sigma", 0.6))
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool, device=X.device))
            pyro.sample("y", d, obs=y)
    return model


def _data(kind, n, D, G, dtype=torch.float32, dev="cpu", seed=0, slopes=(2,), big_col=None):
    """X, the group index (group 1 left empty when G > 2) and y drawn from a model with a varying intercept and
    slopes on the columns ``slopes``; ``big_col`` scales one column of X to magnitude 1e3."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    X = torch.randn(n, D, generator=gen, dtype=dtype)
    if big_col is not None:
        X[:, big_col] = 1e3 + 30.0 * X[:, big_col]
    g = torch.randint(0, G, (n,), generator=gen)
    if G > 2:
        g[g == 1] = 0
    wt = torch.randn(D, generator=gen, dtype=dtype) / D ** 0.5
    eta = X @ wt + 0.3 + 0.5 * torch.randn(G, generator=gen, dtype=dtype)[g]
    for c in slopes:
        scale = 1e-4 if c == big_col else 0.3
        eta = eta + scale * torch.randn(G, generator=gen, dtype=dtype)[g] * X[:, c]
    if big_col is not None:
        eta = eta - wt[big_col] * X[:, big_col]
    if kind == "Bernoulli":
        y = (torch.rand(n, generator=gen, dtype=dtype) < torch.sigmoid(eta)).to(dtype)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta.clamp(max=4.0)), generator=gen)
    elif kind == "Binomial":
        y = (torch.rand(n, int(TRIALS), generator=gen, dtype=dtype) < torch.sigmoid(eta)[:, None]).sum(-1).to(dtype)
    else:
        y = eta + 0.6 * torch.randn(n, generator=gen, dtype=dtype)
    return X.to(dev), g.to(dev), y.to(dev)


def _check_layout(pot, model, args):
    tp = TracePotential(model, args)
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, transform, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
        assert transform == ("exp" if site.startswith("s_") or site == "sigma" else "identity"), site
    z = torch.randn(3, pot.dim)
    got, want = pot.unpack(z), tp.unpack(z)
    for site in got:
        assert got[site].shape == want[site].shape and torch.allclose(got[site], want[site]), site


def _check_slopes(pot, slopes, G):
    ge = pot.group_effect
    assert ge.S == len(slopes) and len(pot.group["slopes"]) == len(slopes)
    for k, (form, scale, col) in enumerate(slopes):
        e, name = ge.slope[k], "b%d" % (k + 1)
        site = ("beta_" if form == "centred" else "eta_") + name
        assert pot.group["slopes"][k]["site"] == site and e.b_off == pot.sites[site][0].start
        assert e.col == col and e.noncentred == (form == "noncentred")
        if scale == "const":
            assert e.s_off == -1 and e.s_const == pytest.approx(0.4 + 0.1 * (k + 1), rel=1e-6)
        else:
            assert e.s_off == pot.sites["s_" + name][0].start and e.s_prior == GlmPotential._SIGMA_PRIORS[scale]
            assert (e.sp0, e.sp1) == pytest.approx((PRIOR_PARAMS[scale] + (1.0,))[:2], rel=1e-6)


# ---- CPU tier: recognition and layout ----------------------------------------------------------------------------
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
def test_recognises_one_slope(kind, form, scale):
    G, slopes = 6, ((form, scale, 2),)
    X, g, y = _data(kind, 300, 5, G)
    model = slope_model(kind, slopes, a_form="noncentred" if form == "centred" else "centred", G=G)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), (kind, form, scale)
    assert pot.group_effect.G == G and pot.weight == "w" and pot.bias == "b"
    _check_slopes(pot, slopes, G)
    assert torch.equal(pot.groups.cpu(), g.to(torch.int32))
    _check_layout(pot, model, (X, g, y))


SETS = {"two": (("centred", "HalfNormal", 0), ("noncentred", "const", 3)),
        "three": (("noncentred", "HalfCauchy", 4), ("centred", "const", 1), ("noncentred", "LogNormal", 2)),
        "three_normal": (("centred", "Exponential", 1), ("noncentred", "HalfNormal", 0), ("centred", "const", 4))}


@pytest.mark.parametrize("case", list(SETS))
def test_recognises_several_slopes(case):
    kind = "Normal" if case == "three_normal" else "Poisson" if case == "two" else "Bernoulli"
    G, slopes = 7, SETS[case]
    X, g, y = _data(kind, 400, 5, G, slopes=[c for _, _, c in slopes])
    model = slope_model(kind, slopes, a_scale="HalfCauchy", G=G, sigma="latent")
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), case
    _check_slopes(pot, slopes, G)
    _check_layout(pot, model, (X, g, y))
    if kind == "Normal":
        assert pot.sigma_site == "sigma"


@pytest.mark.parametrize("spelling", ["x_first", "index_select", "scale_after", "duplicate_column"])
def test_recognition_spellings(spelling):
    G, D = 6, 5
    form = "noncentred" if spelling == "scale_after" else "centred"
    slopes = ((form, "HalfNormal", 3),)
    X, g, y = _data("Bernoulli", 300, D, G, slopes=(3,))
    if spelling == "duplicate_column":     # column 3 repeated as column 1: the lowest is taken
        X[:, 1] = X[:, 3]
    model = slope_model("Bernoulli", slopes, G=G, spelling="ellipsis" if spelling == "duplicate_column" else spelling)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), spelling
    assert pot.group_effect.slope[0].col == (1 if spelling == "duplicate_column" else 3)
    if spelling != "x_first":              # beta[g] gathers along the chain dim of TracePotential's batch
        _check_layout(pot, model, (X, g, y))


@pytest.mark.parametrize("change", ["separate_cov", "square", "plus_one", "other_size", "other_index",
                                    "no_intercept", "shared_scale", "scale_is_sigma", "mean", "latent_mean", "S4",
                                    "width_129", "mvn", "mask", "fp64"])
def test_near_misses_are_not_recognised(change):
    kind, D, G, slopes, kw = "Bernoulli", 5, 6, (("centred", "HalfNormal", 2),), {}
    if change == "shared_scale":
        kw = dict(a_scale="HalfNormal")
    if change == "scale_is_sigma":
        kind, kw = "Normal", dict(sigma="latent")
    if change == "S4":
        slopes = tuple(("centred", "const", c) for c in range(4))
    if change == "width_129":              # 9 + 40 (1 + 2) = 129
        D, G, slopes = 9, 40, (("centred", "const", 1), ("noncentred", "const", 2))
    X, g, y = _data(kind, 300, D, G, dtype=torch.float64 if change == "fp64" else torch.float32)
    args = (X, g, y)
    if change == "separate_cov":
        args = (X, g, y, X[:, 2] + 0.25 * torch.randn(300, generator=torch.Generator().manual_seed(1)))
    if change == "other_size":
        model = _other_size_model
    elif change == "mvn":
        model = _correlated_model
    else:
        model = slope_model(kind, slopes, G=G, change=None if change in ("fp64", "width_129", "S4") else change, **kw)
    assert not isinstance(_recognised(model, *args), GlmPotential), change
    if change == "width_129":              # one column fewer fits
        X, g, y = _data(kind, 300, D - 1, G)
        assert isinstance(_recognised(slope_model(kind, slopes, G=G), X, g, y), GlmPotential)
    if change == "S4":                     # three fit
        assert isinstance(_recognised(slope_model(kind, slopes[:3], G=G), X, g, y), GlmPotential)


def _other_size_model(X, g, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), S_W).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), S_B))
    a = _chains(pyro.sample("alpha", dist.Normal(X.new_zeros(6), 0.7).to_event(1)))
    beta = _chains(pyro.sample("beta_b1", dist.Normal(X.new_zeros(7), 0.5).to_event(1)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_lin(X, w, b) + a[..., g] + beta[..., g] * X[:, 2]), obs=y)


def _correlated_model(X, g, y):
    """[alpha_j, beta_j] ~ MultivariateNormal: a correlated group effect."""
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), S_W).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), S_B))
    cov = torch.tensor([[1.0, 0.3], [0.3, 1.0]])
    ab = pyro.sample("ab", dist.MultivariateNormal(X.new_zeros(6, 2), cov).to_event(1))
    a, beta = ab[..., 0], ab[..., 1]
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_lin(X, w, b) + a[..., g] + beta[..., g] * X[:, 2]), obs=y)


def test_models_without_slopes_keep_their_route():
    """The intercept-only model is tried before slopes: its potential has S = 0."""
    X, g, y = _data("Poisson", 300, 5, 6, slopes=())
    pot = _recognised(slope_model("Poisson", (), a_scale="HalfNormal"), X, g, y)
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == 0 and pot.group["slopes"] == []


def test_slopes_entry_point_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p = ctypes.c_void_p(4096)
    D, G = 10, 20
    # z = [w (10), b, alpha (20), beta_1 (20), log s_1, beta_2 (20)]
    base = dict(Dz=D + 1 + 3 * G + 1, S=2, cols=(3, 7), b_offs=(D + 1 + G, D + 2 + 2 * G), s_offs=(D + 1 + 2 * G, -1),
                nc=(0, 1), priors=(N.SIGMA_HALFNORMAL, 0), p0=(1.0, 0.0), consts=(0.0, 0.5), Dx=D, nG=G)

    def regression(a):
        e = N.b2_glm_group_effect()
        e.groups, e.G, e.a_off, e.noncentred, e.s_off, e.s_const = p, a["nG"], D + 1, 0, -1, 0.7
        e.S = a["S"]
        for k in range(min(a["S"], 2)):
            s = e.slope[k]
            s.col, s.b_off, s.s_off, s.noncentred = a["cols"][k], a["b_offs"][k], a["s_offs"][k], a["nc"][k]
            s.s_prior, s.sp0, s.sp1, s.s_const = a["priors"][k], a["p0"][k], 1.0, a["consts"][k]
        return N.b2_glm_regression(kind=N.GLM_POISSON, X=p, y=p, N=10000, D=a["Dx"], K=1, has_bias=1, w_off=0, b_off=D,
                                   s_w=1.0, s_b=10.0, s_off=-1, sigma=1.0, group=ctypes.pointer(e))

    def call(**kw):
        a = dict(base, **kw)
        return L.b2_glm_potential(ctypes.byref(regression(a)), p, 4, a["Dz"], p, p, None, 0, None)

    def workspace(**kw):
        return L.b2_glm_potential_workspace(ctypes.byref(regression(dict(base, **kw))), 4)

    assert call() == -5                                                     # valid: the workspace check is next
    assert call(S=-1) == -2 and call(S=4) == -2
    assert call(cols=(3, 3)) == -2 and call(cols=(10, 7)) == -2 and call(cols=(-1, 7)) == -2
    assert call(nc=(2, 1)) == -2
    # D + G (1 + S) <= 128: 10 + 39 * 3 = 127 fits and 10 + 40 * 3 = 130 does not
    assert call(nG=39, Dz=D + 1 + 3 * 39 + 1, b_offs=(D + 40, D + 41 + 39), s_offs=(D + 40 + 39, -1)) == -5
    assert call(nG=40, Dz=D + 1 + 3 * 40 + 1, b_offs=(D + 41, D + 42 + 40), s_offs=(D + 41 + 40, -1)) == -2
    # z's row: too wide, too narrow, overlapping blocks, a block past its end
    assert call(Dz=base["Dz"] + 1) == -2 and call(Dz=base["Dz"] - 1) == -2
    assert call(b_offs=(D + 1, D + 2 + 2 * G)) == -2 and call(s_offs=(D, -1)) == -2
    assert call(b_offs=(D + 1 + G, D + 3 + 2 * G)) == -2
    # priors and constant scales
    assert call(priors=(0, 0)) == -2 and call(priors=(5, 0)) == -2 and call(p0=(0.0, 0.0)) == -2
    assert call(consts=(0.0, 0.0)) == -2 and call(consts=(0.0, -1.0)) == -2
    # S = 0 ignores the slope fields
    assert call(S=0, Dz=D + 1 + G, cols=(99, 99)) == -5
    # the workspace counts every group column, G (1 + S)
    assert workspace() > 256
    assert workspace(Dx=12, nG=39) == 256


# ---- CPU tier: what ptxas makes of the slope kernels (glm_flat_pipeline with SLOPES) ----------------------
SLOPE_KERNELS = [("glm_flat_tc", "glm_bernoulli_slope_tc_kernelILi%dE" % dc) for dc in (1, 2, 3, 4)] + \
    [("glm_poisson_tc", "glm_poisson_slope_tc_kernelILi%dE" % dc) for dc in (1, 2, 3, 4)] + \
    [("glm_normal_tc", "glm_normal_slope_tc_kernelILi%dE" % dc) for dc in (1, 2, 3, 4)] + \
    [("glm_binomial_tc", "glm_binomial_slope_tc_kernelILb%dELi%dE" % (r, dc)) for r in (0, 1) for dc in (2, 3, 4)]


@pytest.mark.parametrize("source,mangled", SLOPE_KERNELS)
def test_slope_kernel_sass(group_sass, source, mangled):
    """No C7515/C7520 serialisation note, no spills, and each GEMM one HGMMA chain with one wait."""
    _check_group_kernel_sass(group_sass, source, mangled)


# ---- GPU tier ------------------------------------------------------------------------------------------------------
def _oracle_potential(X, g, y, pot, kind):
    """fp64 U(z) (pyro/infer/mcmc/util.py:275-286) of the group potential with slopes: -(log joint) - SUM of the logs
    of the positive sites.  The sigma prior is the models' HalfNormal(1.5)."""
    Xd, yd = X.double(), y.double()
    inv = {v: k for k, v in GlmPotential._SIGMA_PRIORS.items()}
    ge = pot.group_effect
    blocks = [(pot.group["site"], ge.noncentred, ge.s_off, ge.s_prior, ge.sp0, ge.sp1, ge.s_const, None)]
    blocks += [(sl["site"], e.noncentred, e.s_off, e.s_prior, e.sp0, e.sp1, e.s_const, e.col)
               for sl, e in zip(pot.group["slopes"], ge.slope)]
    site_of = {pot.sites[name][0].start: name for name in pot.sites}

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
        lp = lp + odists.normal(w, zero, zero + pot.s_w).sum(-1)
        lp = lp + odists.normal(vals[pot.bias], zero, zero + pot.s_b).sum(-1)
        eta = w @ Xd.T + vals[pot.bias]
        for site, nc, s_off, s_prior, sp0, sp1, s_const, col in blocks:
            if s_off >= 0:
                s = vals[site_of[s_off]]
                lp = lp + _prior_lp((inv[s_prior], sp0, sp1), s).sum(-1)
            else:
                s = zero + s_const
            a = vals[site]
            if nc:
                lp = lp + odists.normal(a, zero, zero + 1.0).sum(-1)
                a = s * a
            else:
                lp = lp + odists.normal(a, zero, s).sum(-1)
            eta = eta + (a[..., g] if col is None else a[..., g] * Xd[:, col])
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


def _chain_state(pot, C, seed):
    """Chains in the body of the prior: small coefficients, log scales near 0, log sigma near log 0.6; a slope on a
    covariate of magnitude m gets coefficients of about 1 / m."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    z = 0.3 * torch.randn(C, pot.dim, generator=gen)
    z[:, pot.sites[pot.weight][0]] *= min(1.0, (8.0 / pot.Dx) ** 0.5)
    Xmax = pot.X.abs().amax(0).cpu()
    w = pot.sites[pot.weight][0]
    z[:, w] /= Xmax.clamp(min=1.0)
    for sl in pot.group["slopes"]:
        z[:, pot.sites[sl["site"]][0]] /= float(Xmax[sl["col"]].clamp(min=1.0))
    if pot.sigma_site is not None:
        z[:, pot.sites[pot.sigma_site][0]] += math.log(0.6)
    return z.to(DEV)


def _check_against_oracle(model, pot, X, g, y, kind, Cs, seed, label, gtol=5e-4):
    U_ref_fn = _oracle_potential(X, g, y, pot, kind)
    errs = []
    for C in Cs:
        z = _chain_state(pot, C, seed + C)
        U, G = pot.value_and_grad(z)
        U2, G2 = pot.value_and_grad(z)
        assert torch.equal(U, U2) and torch.equal(G, G2)
        zd = z.double().detach().requires_grad_(True)
        Ur = U_ref_fn(zd)
        (Gr,) = torch.autograd.grad(Ur.sum(), zd)
        tp = TracePotential(model, (X, g, y), num_chains=C)
        assert list(tp.sites) == list(pot.sites) and tp.dim == pot.dim
        Ut, Gt = tp.value_and_grad(z)
        errs.append((C, float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max()),
                     float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max())),
                     float(((U - Ut).abs() / Ut.abs().clamp(min=1.0)).max()),
                     float((G - Gt).abs().max()) / max(1.0, float(Gt.abs().max()))))
    print("\nslope potential %s: (C, U vs fp64, grad vs fp64, U vs trace, grad vs trace) %s"
          % (label, ["%d %.1e %.1e %.1e %.1e" % e for e in errs]))
    for C, eu, eg, et, gt in errs:
        assert eu <= 2e-6 and eg <= gtol, (C, eu, eg)
        assert et <= 2e-6 and gt <= gtol, (C, et, gt)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
def test_potential_against_fp64_and_trace(kind, form, scale):
    """U and dU/dz for C = 1, 64, 65 chains against fp64, bitwise repeatable, and against TracePotential: U within
    2e-6 relative to max(1, |U|), the gradient within 5e-4 of max |grad|."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G = 9000, 7, 20
    X, g, y = _data(kind, n, D, G, dev=DEV, seed=n + D, slopes=(2,))
    model = slope_model(kind, ((form, scale, 2),), a_scale="HalfNormal", G=G,
                        sigma="latent" if scale == "HalfCauchy" else "const")
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == 1, (kind, form, scale)
    _check_against_oracle(model, pot, X, g, y, kind, (1, 64, 65), 0, "%s %s %s" % (kind, form, scale))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SETS) + ["big_covariate"])
def test_several_slopes_against_fp64_and_trace(case):
    """S = 2 and 3 with mixed forms, and one slope on a covariate of magnitude 1e3, whose TF32 rounding alone would
    move each logit by about 0.1 * beta: the slope columns are split like X's."""
    if EMULATE:
        pytest.skip("kernel test")
    kind = "Normal" if case == "three_normal" else "Poisson" if case == "two" else "Bernoulli"
    slopes = SETS.get(case, (("centred", "HalfNormal", 3),))
    big = 3 if case == "big_covariate" else None
    X, g, y = _data(kind, 20_000, 6, 24, dev=DEV, seed=7, slopes=[c for _, _, c in slopes], big_col=big)
    model = slope_model(kind, slopes, a_form="noncentred", a_scale="HalfCauchy", G=24, sigma="latent")
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == len(slopes), case
    _check_against_oracle(model, pot, X, g, y, kind, (1, 64, 65), 3, case)


# D + G (1 + S) at 31, 32, 33, 64, 65 and 128
WIDTHS = [(3, 14, 1), (2, 15, 1), (3, 10, 2), (4, 20, 2), (5, 20, 2), (8, 40, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 64, 65, 10_003])
@pytest.mark.parametrize("D,G,S", WIDTHS, ids=["%d+%dx%d" % (d, g, 1 + s) for d, g, s in WIDTHS])
def test_ragged_shapes(D, G, S, n):
    """Every atom count of the kernel, tiles cut anywhere, empty groups; the kind cycles over the four."""
    if EMULATE:
        pytest.skip("kernel test")
    i = WIDTHS.index((D, G, S)) + [1, 63, 64, 65, 10_003].index(n)
    kind, form = KINDS[i % 4], FORMS[(i // 4) % 2]
    slopes = tuple((FORMS[(i + k) % 2], "HalfNormal" if k == 0 else "const", D - 1 - k) for k in range(S))
    X, g, y = _data(kind, n, D, G, dev=DEV, seed=i, slopes=[c for _, _, c in slopes])
    model = slope_model(kind, slopes, a_form=form, a_scale="HalfNormal", G=G)
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == S, (kind, D, G, S, n)
    # GEMM 2 takes the likelihood gradient rounded to TF32: over a handful of rows the rounding does not average out
    _check_against_oracle(model, pot, X, g, y, kind, (1, 65), 1, "%s D=%d G=%d S=%d n=%d" % (kind, D, G, S, n),
                          gtol=5e-4 if n >= 8192 else 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_out_of_range_group_index_gives_nan(kind):
    """A group index outside [0, G) that reaches the kernel makes U and every block's gradient NaN for that call, and
    the next call with valid indices is exact again."""
    if EMULATE:
        pytest.skip("kernel test")
    slopes = (("centred", "HalfCauchy", 1), ("noncentred", "const", 4))
    X, g, y = _data(kind, 5000, 6, 10, dev=DEV, seed=5, slopes=(1, 4))
    pot = recognise(slope_model(kind, slopes, a_scale="HalfCauchy", G=10), (X, g, y))
    z = _chain_state(pot, 8, 0)
    U0, G0 = pot.value_and_grad(z)
    for bad in (10, -1, 1 << 30):
        pot.groups[4321] = bad
        U, G = pot.value_and_grad(z)
        torch.cuda.synchronize()
        assert bool(torch.isnan(U).all()), bad
        for site in ("alpha", "beta_b1", "eta_b2"):
            assert bool(torch.isnan(G[:, pot.sites[site][0]]).all()), (bad, site)
        pot.groups[4321] = int(g[4321])
    U1, G1 = pot.value_and_grad(z)
    assert torch.equal(U1, U0) and torch.equal(G1, G0)


@pytest.mark.gpu
def test_captured_graph_replay_equals_eager():
    if EMULATE:
        pytest.skip("needs CUDA graphs")
    slopes = (("noncentred", "HalfNormal", 3), ("centred", "const", 9))
    X, g, y = _data("Normal", 70001, 16, 32, dev=DEV, seed=3, slopes=(3, 9))
    pot = recognise(slope_model("Normal", slopes, a_scale="HalfNormal", G=32, sigma="latent"), (X, g, y))
    assert pot.group_effect.S == 2
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
def test_hmc_trajectory_matches_oracle_integrator():
    """Twenty leapfrog steps of HMC's integrator on GlmPotential from identical (z, r) against
    oracle.mcmc.velocity_verlet on the fp64 potential."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.004
    slopes = (("noncentred", "HalfCauchy", 2), ("centred", "const", 5))
    X, g, y = _data("Bernoulli", n, 8, 20, dev=DEV, seed=11, slopes=(2, 5))
    pot = recognise(slope_model("Bernoulli", slopes, a_scale="HalfNormal", G=20), (X, g, y))
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = _chain_state(pot, C, 5)
    r0 = torch.randn(C, pot.dim, device=DEV)
    z, r = z0.clone(), r0.clone()
    _, gr = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, gr, U, _ = kernel._leapfrog(z, r, gr, epsv, minv)
    Uo = _oracle_potential(X.cpu(), g.cpu(), y.cpu(), pot, "Bernoulli")
    errs = []
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        errs.append((float((z[c].double().cpu() - zr).abs().max()),
                     float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max())),
                     abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))))
    print("\nhmc trajectory with slopes: (z err, r err, U err) %s" % ["%.1e %.1e %.1e" % e for e in errs])
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


def radon_slope(X, g, y):
    """Varying intercept and varying slope on the floor column (1), both non-centred, latent sigma."""
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
    s_a = pyro.sample("s_a", dist.HalfCauchy(X.new_full((), 1.0)))
    eta_a = pyro.sample("eta_a", dist.Normal(X.new_zeros(50), 1.0).to_event(1))
    s_b = pyro.sample("s_b", dist.HalfCauchy(X.new_full((), 0.5)))
    eta_b = pyro.sample("eta_b", dist.Normal(X.new_zeros(50), 1.0).to_event(1))
    a = _chains(s_a.unsqueeze(-1) * eta_a)
    beta = _chains(s_b.unsqueeze(-1) * eta_b)
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Normal(_lin(X, w, b) + a[..., g] + beta[..., g] * X[:, 1], sigma), obs=y)


def multilevel_logistic_slopes(X, g, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    s_a = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
    alpha = _chains(pyro.sample("alpha", dist.Normal(X.new_zeros(12), s_a.unsqueeze(-1)).to_event(1)))
    s_1 = pyro.sample("s_1", dist.HalfNormal(X.new_full((), 0.5)))
    beta_1 = _chains(pyro.sample("beta_1", dist.Normal(X.new_zeros(12), s_1.unsqueeze(-1)).to_event(1)))
    eta_2 = _chains(pyro.sample("eta_2", dist.Normal(X.new_zeros(12), 1.0).to_event(1)))
    logits = _lin(X, w, b) + alpha[..., g] + beta_1[..., g] * X[:, 0] + 0.3 * eta_2[..., g] * X[:, 3]
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=logits), obs=y)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["radon_slope", "multilevel_logistic_slopes"])
def test_nuts_posterior_matches_trace_potential(case):
    """NUTS with 8 chains on GlmPotential against a run on TracePotential (compile_model = False) of the same model:
    means within 0.3 posterior standard deviations, standard deviations within 25 %.  The radon-shaped model has
    N = 919, D = 2 (a county-level covariate and the floor column), G = 50; the logistic one N = 5000, D = 6, G = 12, S = 2."""
    if EMULATE:
        pytest.skip("kernel test")
    if case == "radon_slope":
        model = radon_slope
        X, g, y = _data("Normal", 919, 2, 50, dev=DEV, seed=22, slopes=(1,))
        X[:, 1] = (X[:, 1] > 0.5).to(X.dtype)   # floor: 0 or 1
    else:
        model, (X, g, y) = multilevel_logistic_slopes, _data("Bernoulli", 5000, 6, 12, dev=DEV, seed=21, slopes=(0, 3))
    out = {}
    for compile_model in (True, False):
        kernel = NUTS(model, max_tree_depth=5)
        kernel.compile_model = compile_model
        mc = MCMC(kernel, num_samples=200, warmup_steps=150, num_chains=8, seed=1 if compile_model else 2)
        mc.run(X, g, y)
        want = GlmPotential if compile_model else TracePotential
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        if compile_model:
            assert kernel.potential.group_effect.S == (1 if case == "radon_slope" else 2)
        s = mc.get_samples()
        cols = [s[name].reshape(s[name].shape[0], -1).double().cpu() for name in sorted(s)]
        out[compile_model] = torch.cat([c.log() if name.startswith("s_") or name == "sigma" else c
                                        for name, c in zip(sorted(s), cols)], -1)
    got, ref = out[True], out[False]
    m_, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    print("\nnuts %s: max |mean diff| / sd %.2f, max |sd diff| / sd %.2f"
          % (case, float(((m_ - rm).abs() / rs).max()), float(((sd - rs).abs() / rs).max())))
    assert bool(((m_ - rm).abs() <= 0.3 * rs).all()), float(((m_ - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


@pytest.mark.gpu
def test_bind_nuts_recognises_reference_pyro_plate_model():
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as ref_pyro
    import pyro.distributions as rdist
    from pyro.infer import MCMC as RefMCMC

    def radon(X, g, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        sigma = ref_pyro.sample("sigma", rdist.HalfNormal(X.new_full((), 1.5)))
        s_a = ref_pyro.sample("s_a", rdist.HalfCauchy(X.new_full((), 1.0)))
        s_b = ref_pyro.sample("s_b", rdist.HalfCauchy(X.new_full((), 0.5)))
        with ref_pyro.plate("county", 50):
            eta_a = ref_pyro.sample("eta_a", rdist.Normal(X.new_zeros(()), 1.0))
            beta = ref_pyro.sample("beta", rdist.Normal(X.new_zeros(()), s_b))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Normal(X @ w + b + s_a * eta_a[g] + beta[g] * X[:, 1], sigma), obs=y)

    args = _data("Normal", 919, 2, 50, dev=DEV, seed=2, slopes=(1,))
    pot = bind.recognise(radon, args, {}, poutine=ref_pyro.poutine)
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == 1
    assert pot.group_effect.slope[0].col == 1 and not pot.group_effect.slope[0].noncentred
    kernel = bind.NUTS(radon, num_chains=4, seed=0)
    mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
    mc.run(*args)
    assert isinstance(kernel._kernel.potential, GlmPotential)
    for v in mc.get_samples().values():
        assert bool(torch.isfinite(v).all())
