"""NUTS / HMC on multilevel regression: a varying intercept by group, ``X @ w + b + alpha[g]``, through
``GlmPotential`` (``b2_glm_potential`` with a group effect), with the group effect scored as G more columns of the
fused GLM kernel's contraction over ``[X | onehot(g)]``.

CPU tier: which models ``recognise`` routes to ``GlmPotential`` (every likelihood kind, centred and non-centred group
effects, a constant group scale or each of the four priors on a latent one, the ways a model can write the gather),
their z layout against ``TracePotential``, the near misses that must keep the traced route, the entry point's
argument checks, and what ptxas makes of the group kernels.  GPU tier: U and dU/dz against an fp64 restatement and
against ``TracePotential`` (ragged N, D + G at every atom boundary, one and two particle slabs), determinism, the NaN
of an out-of-range group index, CUDA-graph replay, HMC trajectories against the oracle integrator, NUTS posteriors
against ``TracePotential`` runs, and the route ``bind.NUTS`` takes with reference Pyro."""
import ctypes
import math
import os
import re
import subprocess

import pytest
import torch
import torch.nn.functional as F

import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from oracle import dists as odists
from oracle import mcmc as omcmc
from pyro_b200 import _build
from pyro_b200 import _native as N
from pyro_b200.infer import HMC, MCMC, NUTS
from pyro_b200.infer.mcmc import GlmPotential, TracePotential
from pyro_b200.infer.mcmc.compile import recognise

DEV = device()
KINDS = ["Bernoulli", "Poisson", "Binomial", "Normal"]
FORMS = ["centred", "noncentred"]
SCALES = ["const", "HalfNormal", "HalfCauchy", "Exponential", "LogNormal"]
PRIOR_PARAMS = {"HalfNormal": (1.5,), "HalfCauchy": (1.0,), "Exponential": (2.0,), "LogNormal": (-0.5, 0.8)}
S_CONST = 0.7
S_W, S_B = 1.0, 10.0
TRIALS = 10.0


# ---- models ----------------------------------------------------------------------------------------------------
def _lin(X, w, b):
    """X @ w + b with w's chain dims (TracePotential's [C, 1, D]) in front of the data dim."""
    return (w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b


def _likelihood(kind, eta, sigma):
    if kind == "Bernoulli":
        return dist.Bernoulli(logits=eta)
    if kind == "Poisson":
        return dist.Poisson(torch.exp(eta))
    if kind == "Binomial":
        return dist.Binomial(eta.new_full((), TRIALS), logits=eta)
    return dist.Normal(eta, sigma)


def group_model(kind, form="centred", scale="const", G=6, bias=True, sigma="const", spelling="ellipsis",
                order="w_first", change=None):
    """Regression of ``kind`` with a varying intercept by group: ``alpha ~ Normal(0, s_a)[G]`` (centred) or
    ``alpha = s_a * eta``, ``eta ~ Normal(0, 1)[G]`` (non-centred); ``s_a`` the constant S_CONST or a positive site
    with prior ``scale``.  ``spelling`` is how the model gathers alpha by group, ``order`` "w_first" (w, b, sigma,
    s_a, alpha) or "group_first" (s_a, alpha, b, w); ``change`` makes a near miss."""
    def model(X, g, y, g2=None):
        D = X.shape[-1]
        site = {}

        def draw_regression():
            s_w = X.new_full((), S_W)
            if change == "tau":
                s_w = pyro.sample("tau", dist.HalfNormal(X.new_full((), 1.0))).unsqueeze(-1)
            site["w"] = pyro.sample("w", dist.Normal(X.new_zeros(D), s_w).to_event(1))
            if bias:
                site["b"] = pyro.sample("b", dist.Normal(X.new_zeros(()), S_B))
            if kind == "Normal" and sigma == "latent":
                site["sigma"] = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))

        def draw_group():
            if change == "sa_is_sigma":
                sa = site["sigma"]
            elif scale == "const":
                sa = X.new_full((), S_CONST)
            else:
                sa = pyro.sample("s_a", getattr(dist, scale)(*[X.new_full((), p) for p in PRIOR_PARAMS[scale]]))
            sa = sa.unsqueeze(-1)          # over the groups, behind the chain dims of a scalar site
            loc = X.new_zeros(G)
            if change == "mean":
                loc = loc + 0.5
            if change == "latent_mean":
                loc = loc + pyro.sample("mu_a", dist.Normal(X.new_zeros(()), 1.0)).unsqueeze(-1)
            if form == "centred":
                site["A"] = pyro.sample("alpha", dist.Normal(loc, sa).to_event(1))
            else:
                site["eta"] = pyro.sample("eta", dist.Normal(loc, X.new_ones(())).to_event(1))
                site["A"] = sa * site["eta"]
            site["sa"] = sa

        if order == "group_first":
            draw_group()
            draw_regression()
        else:
            draw_regression()
            draw_group()
        A = site["A"]
        A = A.squeeze(-2) if A.dim() > 1 else A
        if spelling == "ellipsis":
            ag = A[..., g]
        elif spelling == "getitem":
            ag = A[g]
        elif spelling == "index_select":
            ag = A.index_select(-1, g)
        else:                              # "scale_after": s_a * eta[g]
            e = site["eta"].squeeze(-2) if site["eta"].dim() > 1 else site["eta"]
            sa = site["sa"].squeeze(-2) if site["sa"].dim() > 1 else site["sa"]
            ag = sa * e[..., g]
        if change == "elsewhere":
            ag = ag + 0.1 * g.to(X.dtype)
        if change == "two_index":
            ag = ag + 0.0 * g2.to(X.dtype)
        with pyro.plate("data", X.shape[0]):
            eta = _lin(X, site["w"], site.get("b", 0.0)) + ag
            d = _likelihood(kind, eta, site.get("sigma", 0.6))
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool, device=X.device))
            pyro.sample("y", d, obs=y)
    return model


def _data(kind, n, D, G, dtype=torch.float32, dev="cpu", seed=0):
    """X, the group index (group 1 left empty when G > 2) and y drawn from the model with a group effect."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    X = torch.randn(n, D, generator=gen, dtype=dtype)
    g = torch.randint(0, G, (n,), generator=gen)
    if G > 2:
        g[g == 1] = 0
    wt = torch.randn(D, generator=gen, dtype=dtype) / D ** 0.5
    at = 0.5 * torch.randn(G, generator=gen, dtype=dtype)
    eta = X @ wt + 0.3 + at[g]
    if kind == "Bernoulli":
        y = (torch.rand(n, generator=gen, dtype=dtype) < torch.sigmoid(eta)).to(dtype)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta.clamp(max=4.0)), generator=gen)
    elif kind == "Binomial":
        y = (torch.rand(n, int(TRIALS), generator=gen, dtype=dtype) < torch.sigmoid(eta)[:, None]).sum(-1).to(dtype)
    else:
        y = eta + 0.6 * torch.randn(n, generator=gen, dtype=dtype)
    return X.to(dev), g.to(dev), y.to(dev)


def _recognised(model, *args):
    import cpu_emulation
    with cpu_emulation.enabled():
        return recognise(model, args)


def _check_layout(pot, model, args):
    tp = TracePotential(model, args)
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, transform, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
        assert transform == ("exp" if site in ("s_a", "sigma") else "identity"), site
    z = torch.randn(3, pot.dim)
    got, want = pot.unpack(z), tp.unpack(z)
    for site in got:
        assert got[site].shape == want[site].shape and torch.allclose(got[site], want[site]), site


# ---- CPU tier: recognition and layout ----------------------------------------------------------------------------
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
def test_recognises_group_effects(kind, form, scale):
    G = 6
    X, g, y = _data(kind, 300, 5, G)
    model = group_model(kind, form, scale, G=G)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), (kind, form, scale)
    ge = pot.group_effect
    site = "alpha" if form == "centred" else "eta"
    assert pot.group["site"] == site and ge.G == G and ge.a_off == pot.sites[site][0].start
    assert ge.noncentred == (form == "noncentred") and pot.weight == "w" and pot.bias == "b"
    assert pot.weight_scale is None
    if scale == "const":
        assert ge.s_off == -1 and ge.s_const == pytest.approx(S_CONST, rel=1e-6)
    else:
        assert ge.s_off == pot.sites["s_a"][0].start and ge.s_prior == GlmPotential._SIGMA_PRIORS[scale]
        assert (ge.sp0, ge.sp1) == pytest.approx((PRIOR_PARAMS[scale] + (1.0,))[:2], rel=1e-6)
    assert torch.equal(pot.groups.cpu(), g.to(torch.int32))
    _check_layout(pot, model, (X, g, y))


@pytest.mark.parametrize("case", ["getitem", "index_select", "scale_after", "group_first", "no_intercept",
                                  "normal_latent_sigma", "g_equals_d"])
def test_recognition_variants(case):
    kind, form, kw, D, G = "Bernoulli", "centred", {}, 5, 6
    if case in ("getitem", "index_select"):
        kw = dict(spelling=case)
    elif case == "scale_after":
        form, kw = "noncentred", dict(spelling=case, scale="HalfCauchy")
    elif case == "group_first":
        kind, kw = "Poisson", dict(order="group_first", scale="Exponential")
    elif case == "no_intercept":
        kw = dict(bias=False)
    elif case == "normal_latent_sigma":
        kind, form, kw = "Normal", "noncentred", dict(sigma="latent", scale="HalfNormal")
    else:                                  # the weight and the group effect have the same shape: the probes decide
        kind, D, G = "Binomial", 6, 6
    X, g, y = _data(kind, 300, D, G)
    model = group_model(kind, form, G=G, **kw)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential) and pot.group_effect is not None, case
    if case != "getitem":                  # alpha[g] gathers along the chain dim of TracePotential's batch
        _check_layout(pot, model, (X, g, y))
    assert pot.group["site"] == ("alpha" if form == "centred" else "eta") and pot.weight == "w"
    if case == "group_first":
        assert list(pot.sites)[0] == "s_a" and list(pot.sites)[-1] == "b"
    if case == "no_intercept":
        assert not pot.has_bias
    if case == "normal_latent_sigma":
        assert pot.sigma_site == "sigma" and pot.group["s_site"] == "s_a"


@pytest.mark.parametrize("change", ["two_index", "elsewhere", "mean", "latent_mean", "sa_is_sigma", "tau",
                                    "width_129", "mask", "fp64"])
def test_near_misses_are_not_recognised(change):
    kind, D, G, kw = "Bernoulli", 5, 6, {}
    if change == "sa_is_sigma":
        kind, kw = "Normal", dict(sigma="latent")
    if change == "width_129":
        D, G = 64, 65
    X, g, y = _data(kind, 300, D, G, dtype=torch.float64 if change == "fp64" else torch.float32)
    model = group_model(kind, "centred", G=G, change=None if change in ("fp64", "width_129") else change, **kw)
    args = (X, g, y, g.flip(0)) if change == "two_index" else (X, g, y)
    assert not isinstance(_recognised(model, *args), GlmPotential), change
    if change == "width_129":              # one group fewer fits
        X, g, y = _data(kind, 300, D, G - 1)
        assert isinstance(_recognised(group_model(kind, "centred", G=G - 1), X, g, y), GlmPotential)


def test_models_without_a_group_index_keep_their_route():
    """An int64 [N] argument that no latent uses changes nothing: the model is the plain regression."""
    def model(X, g, y):
        w = pyro.sample("w", dist.Normal(X.new_zeros(X.shape[-1]), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        with pyro.plate("data", X.shape[0]):
            pyro.sample("y", dist.Poisson(torch.exp(_lin(X, w, b))), obs=y)
    X, g, y = _data("Poisson", 300, 5, 6)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential) and pot.group_effect is None


def test_out_of_range_index_is_refused_at_construction():
    X, g, y = _data("Bernoulli", 300, 5, 6)
    pot = _recognised(group_model("Bernoulli", G=6), X, g, y)
    import cpu_emulation
    with cpu_emulation.enabled():
        for bad in (-1, 6):
            g2 = g.clone()
            g2[7] = bad
            with pytest.raises(ValueError):
                GlmPotential(X, y, "Bernoulli", pot.sites, "w", "b", s_w=S_W, s_b=S_B,
                             group=dict(pot.group, index=g2))


def test_group_effect_entry_point_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)
    D, G = 10, 20

    def regression(kind=N.GLM_POISSON, X=p, y=p, trials=None, per_row=0, n=10000, Dx=D, bias=1, w_off=0, b_off=D,
                   s_off=-1, s_w=1.0, s_b=10.0, s_prior=0, sp0=0.0, sp1=0.0, sigma=1.0, groups=p, nG=G, a_off=D + 1,
                   noncentred=0, sa_off=D + G + 1, sa_prior=N.SIGMA_HALFCAUCHY, sa_p0=1.0, sa_p1=1.0, s_const=0.0,
                   tau_off=-1):
        e = N.b2_glm_group_effect()
        e.groups, e.G, e.a_off, e.noncentred = groups, nG, a_off, noncentred
        e.s_off, e.s_prior, e.sp0, e.sp1, e.s_const = sa_off, sa_prior, sa_p0, sa_p1, s_const
        m = N.b2_glm_regression(kind=kind, X=X, y=y, N=n, D=Dx, K=1, trials=trials, trials_per_row=per_row,
                                has_bias=bias, w_off=w_off, b_off=b_off, s_w=s_w, s_b=s_b, s_off=s_off,
                                s_prior=s_prior, sp0=sp0, sp1=sp1, sigma=sigma, group=ctypes.pointer(e))
        if tau_off >= 0:     # a latent weight scale tau
            m.scale = ctypes.pointer(N.b2_glm_weight_scale(tau_off=tau_off, lam_off=-1, tau_prior=1, tau_p0=1.0))
        return m

    def call(z=p, Dz=D + G + 2, null=False, ws=None, nbytes=0, **kw):
        m = None if null else ctypes.byref(regression(**kw))
        return L.b2_glm_potential(m, z, 4, Dz, p, p, ws, nbytes, None)

    def workspace(**kw):
        return L.b2_glm_potential_workspace(ctypes.byref(regression(**kw)), 4)

    # z = [w (10), b, alpha (20), log s_a]: valid, so the workspace check is next
    assert call() == -5
    assert call(X=None) == -4 and call(y=None) == -4 and call(z=None) == -4 and call(null=True) == -4
    assert call(groups=None) == -4 and call(kind=N.GLM_BINOMIAL) == -4
    assert call(kind=N.GLM_CATEGORICAL) == -2 and call(kind=7) == -2
    assert call(kind=N.GLM_BERNOULLI) == -5                                 # any D with a group effect
    assert call(n=0) == -2 and call(n=1 << 31) == -8 and call(Dx=0) == -2
    # D + G <= 128, G >= 1
    assert call(Dx=109, Dz=109 + G + 2, b_off=109, a_off=110, sa_off=130) == -2
    assert call(Dx=108, Dz=108 + G + 2, b_off=108, a_off=109, sa_off=129) == -5
    assert call(nG=0, Dz=D + 2, sa_off=D + 1) == -2
    # the row: out of it, overlapping, or not exactly the blocks
    assert call(Dz=D + G + 3) == -2 and call(Dz=D + G + 1) == -2
    assert call(a_off=D) == -2 and call(a_off=D + 2) == -2                   # alpha over b / past the row's end
    assert call(sa_off=3) == -2 and call(w_off=-1) == -2
    assert call(sa_off=-1, s_const=0.7, Dz=D + G + 1) == -5                  # a constant s_a: no column
    assert call(sa_off=-1, s_const=0.0, Dz=D + G + 1) == -2 and call(sa_off=-1, s_const=-1.0, Dz=D + G + 1) == -2
    assert call(noncentred=1) == -5 and call(noncentred=2) == -2
    assert call(s_off=D + G + 2, Dz=D + G + 3) == -2                         # a noise scale outside linear regression
    # priors: codes in range, positive parameters, a finite LogNormal loc; positive prior scales
    assert call(sa_prior=0) == -2 and call(sa_prior=5) == -2 and call(sa_p0=0.0) == -2
    assert call(sa_prior=N.SIGMA_LOGNORMAL, sa_p0=math.inf) == -2 and call(sa_prior=N.SIGMA_LOGNORMAL, sa_p0=-3.0) == -5
    assert call(s_w=0.0) == -2 and call(s_b=0.0) == -2
    assert call(bias=0, Dz=D + G + 1, a_off=D, sa_off=D + G) == -5
    # alignment of X, y, the group index and per-row trials
    assert call(X=q) == -2 and call(y=q) == -2 and call(groups=q) == -2
    assert call(kind=N.GLM_BINOMIAL, trials=q, per_row=1) == -2 and call(kind=N.GLM_BINOMIAL, trials=q) == -5
    assert call(kind=N.GLM_BINOMIAL, trials=p, per_row=2) == -2
    # linear regression: a latent sigma with a valid prior, or a positive constant
    nz = dict(kind=N.GLM_NORMAL, Dz=D + G + 3, s_off=D + G + 2)
    assert call(**nz, s_prior=N.SIGMA_HALFNORMAL, sp0=1.0) == -5
    assert call(**nz, s_prior=0, sp0=1.0) == -2 and call(**dict(nz, s_off=D + G + 1), s_prior=1, sp0=1.0) == -2
    assert call(kind=N.GLM_NORMAL, sigma=0.0) == -2 and call(kind=N.GLM_NORMAL, sigma=0.6) == -5
    # a group effect with a latent weight scale
    assert call(tau_off=D + G + 2, Dz=D + G + 3) == -2
    need = int(workspace())
    assert need > 256 and call(ws=p, nbytes=need - 1) == -5
    assert workspace(Dx=100, nG=29) == 256
    assert workspace(kind=N.GLM_CATEGORICAL) == 256


# ---- CPU tier: what ptxas makes of the group kernels --------------------------------------------------------------
GROUP_KERNELS = {"glm_flat_tc": ["glm_bernoulli_group_tc_kernelILi%dE" % dc for dc in (1, 2, 3, 4)],
                 "glm_poisson_tc": ["glm_poisson_group_tc_kernelILi%dE" % dc for dc in (1, 2, 3, 4)],
                 "glm_normal_tc": ["glm_normal_group_tc_kernelILi%dE" % dc for dc in (1, 2, 3, 4)],
                 "glm_binomial_tc": ["glm_binomial_group_tc_kernelILb%dELi%dE" % (r, dc)
                                     for r in (0, 1) for dc in (2, 3, 4)]}


@pytest.fixture(scope="module")
def group_sass(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, cuobjdump = sass_test._tools()
    out = {}
    for name in GROUP_KERNELS:
        obj = str(tmp_path_factory.mktemp("glm_group_sass") / (name + ".o"))
        src = os.path.join(_build.CSRC, name + ".cu")
        r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        out[name] = (r.stdout + r.stderr, sass)
    return out


@pytest.mark.parametrize("source,mangled", [(s, m) for s, ms in GROUP_KERNELS.items() for m in ms])
def test_group_kernel_sass(group_sass, source, mangled):
    """No C7515/C7520 serialisation note, no spills, and no warpgroup wait or arrive between two HGMMA of one
    contraction (GEMM 1 m64n64k8, GEMM 2 m64n(32 DC + 8)k8)."""
    import test_glm_tc_sass as sass_test
    log, sass = group_sass[source]
    for line in log.splitlines():
        if mangled in line:
            assert "C7515" not in line and "C7520" not in line, line
    props, used = sass_test._ptxas_properties(log, mangled)
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used
    dc = int(re.search(r"Li(\d)E", mangled).group(1))
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


def _oracle_potential(X, g, y, pot, kind):
    """fp64 U(z) (pyro/infer/mcmc/util.py:275-286): -(log joint) - SUM of the logs of the positive sites (the
    Jacobians of their exp transforms).  The sigma prior is the models' HalfNormal(1.5)."""
    Xd, yd = X.double(), y.double()
    inv = {v: k for k, v in GlmPotential._SIGMA_PRIORS.items()}
    ge = pot.group_effect

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
        eta = w @ Xd.T
        if pot.bias is not None:
            lp = lp + odists.normal(vals[pot.bias], zero, zero + pot.s_b).sum(-1)
            eta = eta + vals[pot.bias]
        if ge.s_off >= 0:
            sa = vals[pot.group["s_site"]]
            lp = lp + _prior_lp((inv[ge.s_prior], ge.sp0, ge.sp1), sa).sum(-1)
        else:
            sa = zero + ge.s_const
        a = vals[pot.group["site"]]
        if ge.noncentred:
            lp = lp + odists.normal(a, zero, zero + 1.0).sum(-1)
            a = sa * a
        else:
            lp = lp + odists.normal(a, zero, sa).sum(-1)
        eta = eta + a[..., g]
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


def _oracle_value_and_grad(U, z):
    zd = z.double().detach().requires_grad_(True)
    u = U(zd)
    (gr,) = torch.autograd.grad(u.sum(), zd)
    return u.detach(), gr


def _chain_state(pot, C, seed):
    """Chains in the body of the prior: small coefficients, log scales near 0, log sigma near log 0.6.  The weights
    shrink with D like the data's, so that the linear predictor stays of order one."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    z = 0.3 * torch.randn(C, pot.dim, generator=gen)
    z[:, pot.sites[pot.weight][0]] *= min(1.0, (8.0 / pot.Dx) ** 0.5)
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
        Ur, Gr = _oracle_value_and_grad(U_ref_fn, z)
        tp = TracePotential(model, (X, g, y), num_chains=C)
        assert list(tp.sites) == list(pot.sites) and tp.dim == pot.dim
        Ut, Gt = tp.value_and_grad(z)
        errs.append((C, float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max()),
                     float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max())),
                     float(((U - Ut).abs() / Ut.abs().clamp(min=1.0)).max()),
                     float((G - Gt).abs().max()) / max(1.0, float(Gt.abs().max()))))
    print("\ngroup potential %s: (C, U vs fp64, grad vs fp64, U vs trace, grad vs trace) %s"
          % (label, ["%d %.1e %.1e %.1e %.1e" % e for e in errs]))
    for C, eu, eg, et, gt in errs:
        assert eu <= 2e-6 and eg <= gtol, (C, eu, eg)
        assert et <= 2e-6 and gt <= gtol, (C, et, gt)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", KINDS)
def test_potential_against_fp64_and_trace(kind, form, scale):
    """U and dU/dz for C = 1, 64, 65 chains against fp64, bitwise repeatable, and against TracePotential, within the
    bounds of the latent-scale potential's tests: U 2e-6 relative to max(1, |U|), the gradient 5e-4 of max |grad|."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G = 3000, 7, 20
    X, g, y = _data(kind, n, D, G, dev=DEV, seed=n + D)
    model = group_model(kind, form, scale, G=G, sigma="latent" if scale == "HalfCauchy" else "const")
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect is not None, (kind, form, scale)
    _check_against_oracle(model, pot, X, g, y, kind, (1, 64, 65), 0, "%s %s %s" % (kind, form, scale))


# D + G just below, at and just above each 32-column atom boundary, and the widest
WIDTHS = [(3, 28), (16, 16), (2, 31), (40, 24), (33, 32), (64, 32), (32, 65), (100, 28)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 64, 65, 10_003])
@pytest.mark.parametrize("D,G", WIDTHS, ids=["%d+%d" % w for w in WIDTHS])
def test_ragged_shapes(D, G, n):
    """Every atom count of the kernel, tiles cut anywhere, empty groups; the kind cycles over the four."""
    if EMULATE:
        pytest.skip("kernel test")
    i = WIDTHS.index((D, G)) + [1, 63, 64, 65, 10_003].index(n)
    kind, form = KINDS[i % 4], FORMS[(i // 4) % 2]
    X, g, y = _data(kind, n, D, G, dev=DEV, seed=i)
    model = group_model(kind, form, "HalfNormal", G=G)
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect is not None, (kind, D, G, n)
    # GEMM 2 takes the likelihood gradient rounded to TF32 (2^-11 relative per row): averaged over thousands of rows
    # the rounding stays within the usual 5e-4, over a handful it need not
    _check_against_oracle(model, pot, X, g, y, kind, (1, 65), 1, "%s %s D=%d G=%d n=%d" % (kind, form, D, G, n),
                          gtol=5e-4 if n >= 8192 else 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_out_of_range_group_index_gives_nan(kind):
    """A group index outside [0, G) that reaches the kernel makes U and the group effect's gradient NaN for that
    call, and the next call with valid indices is exact again."""
    if EMULATE:
        pytest.skip("kernel test")
    X, g, y = _data(kind, 5000, 6, 10, dev=DEV, seed=5)
    pot = recognise(group_model(kind, "centred", "HalfCauchy", G=10), (X, g, y))
    z = _chain_state(pot, 8, 0)
    U0, G0 = pot.value_and_grad(z)
    for bad in (10, -1, 1 << 30):
        pot.groups[4321] = bad
        U, G = pot.value_and_grad(z)
        torch.cuda.synchronize()
        assert bool(torch.isnan(U).all()) and bool(torch.isnan(G[:, pot.sites["alpha"][0]]).all()), bad
        pot.groups[4321] = int(g[4321])
    U1, G1 = pot.value_and_grad(z)
    assert torch.equal(U1, U0) and torch.equal(G1, G0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,form", [("Bernoulli", "centred"), ("Normal", "noncentred")])
def test_captured_graph_replay_equals_eager(kind, form):
    if EMULATE:
        pytest.skip("needs CUDA graphs")
    X, g, y = _data(kind, 70001, 16, 48, dev=DEV, seed=3)
    pot = recognise(group_model(kind, form, "HalfNormal", G=48, sigma="latent"), (X, g, y))
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
@pytest.mark.parametrize("kind,form", [("Bernoulli", "centred"), ("Poisson", "noncentred")])
def test_hmc_trajectory_matches_oracle_integrator(kind, form):
    """Twenty leapfrog steps of HMC's integrator on GlmPotential from identical (z, r) against
    oracle.mcmc.velocity_verlet on the fp64 potential.  U is held to 2e-5 relative for logistic regression and to
    5e-5 for Poisson, whose log-rate terms grow exponentially along the trajectory."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.004
    X, g, y = _data(kind, n, 8, 20, dev=DEV, seed=11)
    pot = recognise(group_model(kind, form, "HalfCauchy", G=20), (X, g, y))
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = _chain_state(pot, C, 5)
    r0 = torch.randn(C, pot.dim, device=DEV)
    z, r = z0.clone(), r0.clone()
    _, gr = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, gr, U, _ = kernel._leapfrog(z, r, gr, epsv, minv)
    Uo = _oracle_potential(X.cpu(), g.cpu(), y.cpu(), pot, kind)
    errs = []
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        errs.append((float((z[c].double().cpu() - zr).abs().max()),
                     float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max())),
                     abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))))
    print("\nhmc trajectory %s %s: (z err, r err, U err) %s" % (kind, form, ["%.1e %.1e %.1e" % e for e in errs]))
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= (2e-5 if kind == "Bernoulli" else 5e-5), (ez, er, eu)


def multilevel_logistic(X, g, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    s_a = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
    alpha = pyro.sample("alpha", dist.Normal(X.new_zeros(20), s_a.unsqueeze(-1)).to_event(1))
    alpha = alpha.squeeze(-2) if alpha.dim() > 1 else alpha
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_lin(X, w, b) + alpha[..., g]), obs=y)


def radon_linear(X, g, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
    s_a = pyro.sample("s_a", dist.HalfCauchy(X.new_full((), 1.0)))
    eta = pyro.sample("eta", dist.Normal(X.new_zeros(85), 1.0).to_event(1))
    alpha = s_a.unsqueeze(-1) * eta
    alpha = alpha.squeeze(-2) if alpha.dim() > 1 else alpha
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Normal(_lin(X, w, b) + alpha[..., g], sigma), obs=y)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["multilevel_logistic", "radon_linear"])
def test_nuts_posterior_matches_trace_potential(case):
    """NUTS with 8 chains on GlmPotential against a run on TracePotential (compile_model = False) of the same model:
    means within 0.3 posterior standard deviations, standard deviations within 25 %.  The multilevel logistic model
    is centred (N = 10^4, D = 8, G = 20), the radon-shaped linear model non-centred with a latent sigma (N = 919,
    D = 2, G = 85)."""
    if EMULATE:
        pytest.skip("kernel test")
    if case == "multilevel_logistic":
        model, (X, g, y) = multilevel_logistic, _data("Bernoulli", 10_000, 8, 20, dev=DEV, seed=21)
    else:
        model, (X, g, y) = radon_linear, _data("Normal", 919, 2, 85, dev=DEV, seed=22)
    out = {}
    for compile_model in (True, False):
        kernel = NUTS(model, max_tree_depth=7)
        kernel.compile_model = compile_model
        mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1 if compile_model else 2)
        mc.run(X, g, y)
        want = GlmPotential if compile_model else TracePotential
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        if compile_model:
            assert kernel.potential.group_effect is not None
        s = mc.get_samples()
        cols = [s[name].reshape(s[name].shape[0], -1).double().cpu() for name in sorted(s)]
        # the positive sites on the log scale, where their posteriors are closer to Normal
        out[compile_model] = torch.cat([c.log() if name in ("s_a", "sigma") else c
                                        for name, c in zip(sorted(s), cols)], -1)
    got, ref = out[True], out[False]
    m_, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    print("\nnuts %s: max |mean diff| / sd %.2f, max |sd diff| / sd %.2f"
          % (case, float(((m_ - rm).abs() / rs).max()), float(((sd - rs).abs() / rs).max())))
    assert bool(((m_ - rm).abs() <= 0.3 * rs).all()), float(((m_ - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


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

    def varying_intercept(X, g, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        s_a = ref_pyro.sample("s_a", rdist.HalfNormal(X.new_full((), 1.0)))
        alpha = ref_pyro.sample("alpha", rdist.Normal(X.new_zeros(12), s_a).to_event(1))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Bernoulli(logits=X @ w + b + alpha[g]), obs=y)

    def radon(X, g, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        sigma = ref_pyro.sample("sigma", rdist.HalfNormal(X.new_full((), 1.5)))
        s_a = ref_pyro.sample("s_a", rdist.HalfCauchy(X.new_full((), 1.0)))
        with ref_pyro.plate("county", 85):
            eta = ref_pyro.sample("eta", rdist.Normal(X.new_zeros(()), 1.0))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Normal(X @ w + b + s_a * eta[g], sigma), obs=y)

    for model, args in ((varying_intercept, _data("Bernoulli", 4000, 8, 12, dev=DEV, seed=1)),
                        (radon, _data("Normal", 919, 2, 85, dev=DEV, seed=2))):
        pot = bind.recognise(model, args, {}, poutine=ref_pyro.poutine)
        assert isinstance(pot, GlmPotential) and pot.group_effect is not None, model.__name__
        kernel = bind.NUTS(model, num_chains=4, seed=0)
        mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
        mc.run(*args)
        assert isinstance(kernel._kernel.potential, GlmPotential)
        for v in mc.get_samples().values():
            assert bool(torch.isfinite(v).all())
