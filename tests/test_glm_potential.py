"""NUTS / HMC on Bayesian logistic and softmax regression through ``GlmPotential`` (``b2_glm_potential``): the
likelihood of every chain from one pass of the fused GLM kernel over X.

CPU tier: which models ``recognise`` routes to ``GlmPotential`` and which keep their routes, and the z layout
(the same as ``TracePotential``'s).  GPU tier: U and dU/dz against an fp64 restatement and against
``TracePotential``, determinism, CUDA-graph replay, an HMC trajectory against the oracle integrator, NUTS
posteriors against the oracle sampler, the routes taken by ``NUTS(model)``, and unmodified Pyro through
``bind``."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import models
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from oracle import dists as odists
from oracle import mcmc as omcmc
from pyro_b200 import _native as N
from pyro_b200 import poutine
from pyro_b200.infer import HMC, MCMC, NUTS
from pyro_b200.infer.mcmc import GlmPotential, LogisticPotential, TracePotential
from pyro_b200.infer.mcmc.compile import recognise

DEV = device()


# ---- models ----------------------------------------------------------------------------------------------
def softmax_model(X, y, K):
    D = X.shape[-1]
    W = pyro.sample("W", dist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
    b = pyro.sample("b", dist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1))
    with pyro.plate("data", X.shape[0]):
        Wm = W.squeeze(-3) if W.dim() > 2 else W
        pyro.sample("y", dist.Categorical(logits=X @ Wm.mT + b), obs=y)


def softmax_model_linear(X, y, K):
    """No bias, the weight drawn first-class as ``Normal(0, 2).expand([K, D])``, logits by ``F.linear``."""
    W = pyro.sample("W", dist.Normal(X.new_zeros(()), 2.0).expand([K, X.shape[-1]]).to_event(2))
    with pyro.plate("data", X.shape[0]):
        logits = F.linear(X, W) if W.dim() == 2 else X @ W.squeeze(-3).mT
        pyro.sample("y", dist.Categorical(logits=logits), obs=y)


def bias_first_model(X, y):
    """Logistic regression with the intercept drawn before the weights (z = [b, w])."""
    b = pyro.sample("b", dist.Normal(X.new_zeros(1), X.new_full((1,), 3.0)).to_event(1))
    w = pyro.sample("w", dist.Normal(X.new_zeros(X.shape[-1]), 0.5).to_event(1))
    with pyro.plate("data", X.shape[0]):
        logits = w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b
        pyro.sample("y", dist.Bernoulli(logits=logits), obs=y)


def _variant(change):
    """logistic_model with one change: the near misses that must not be recognised."""
    def model(X, y):
        D = X.shape[-1]
        loc = X.new_full((D,), 0.5) if change == "loc" else X.new_zeros(D)
        scale = torch.linspace(0.5, 1.5, D, dtype=X.dtype) if change == "scale" else X.new_ones(D)
        w = pyro.sample("w", dist.Normal(loc, scale).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
        if change == "extra":
            pyro.sample("s", dist.Normal(X.new_zeros(()), 1.0))
        with pyro.plate("data", X.shape[0]):
            logits = w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b
            if change == "2b":
                logits = logits + b
            d = dist.Bernoulli(logits=logits)
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool))
            if change == "scale_site":
                with poutine.scale(scale=2.0):
                    pyro.sample("y", d, obs=y)
            else:
                pyro.sample("y", d, obs=y)
    return model


def _data(n, D, K=None, dtype=torch.float32, dev="cpu", seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn(n, D, generator=g, device=dev, dtype=dtype)
    if K is None:
        w = torch.randn(D, generator=g, device=dev, dtype=dtype) / D ** 0.5
        y = (torch.rand(n, generator=g, device=dev, dtype=dtype) < torch.sigmoid(X @ w + 0.3)).to(dtype)
    else:
        W = torch.randn(K, D, generator=g, device=dev, dtype=dtype) / D ** 0.5
        y = torch.multinomial(torch.softmax(X @ W.mT, -1), 1, generator=g).squeeze(-1)
    return X, y


def _recognised(model, *args):
    import cpu_emulation
    with cpu_emulation.enabled():
        return recognise(model, args)


# ---- CPU tier: recognition and layout ---------------------------------------------------------------------
@pytest.mark.parametrize("name", ["logistic_model", "logistic_model_fused", "softmax", "softmax_linear",
                                  "bias_first"])
def test_recognises_regression_models(name):
    K = 5
    if name.startswith("softmax"):
        X, y = _data(300, 32, K)
        model = softmax_model if name == "softmax" else softmax_model_linear
        args = (X, y, K)
    else:
        X, y = _data(300, 16)
        model = {"logistic_model": models.logistic_model, "logistic_model_fused": models.logistic_model_fused,
                 "bias_first": bias_first_model}[name]
        args = (X, y)
    pot = _recognised(model, *args)
    assert isinstance(pot, GlmPotential), name
    # the z layout, site names and value shapes of TracePotential for the same model
    tp = TracePotential(model, args)
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, _, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
    z = torch.randn(3, pot.dim)
    got, want = pot.unpack(z), tp.unpack(z)
    assert list(got) == list(want)
    for site in got:
        assert got[site].shape == want[site].shape and torch.equal(got[site], want[site]), site
    if name == "softmax":
        assert (pot.K, pot.has_bias, pot.s_w, pot.s_b) == (K, True, 1.0, 10.0)
    if name == "softmax_linear":
        assert (pot.K, pot.has_bias, pot.s_w) == (K, False, 2.0)
    if name == "bias_first":
        assert (pot.w_off, pot.b_off, pot.s_w, pot.s_b) == (1, 0, 0.5, 3.0)


@pytest.mark.parametrize("change", ["loc", "scale", "extra", "2b", "mask", "scale_site"])
def test_near_misses_are_not_recognised(change):
    X, y = _data(300, 16)
    pot = _recognised(_variant(change), X, y)
    assert not isinstance(pot, GlmPotential), change


@pytest.mark.parametrize("case", ["fp64", "D33", "K17", "softmax_D16"])
def test_out_of_scope_models_keep_their_route(case):
    if case == "fp64":
        X, y = _data(300, 16, dtype=torch.float64)
        pot = _recognised(models.logistic_model, X, y)
    elif case == "D33":
        X, y = _data(300, 33)
        pot = _recognised(models.logistic_model, X, y)
    else:
        K, D = (17, 32) if case == "K17" else (4, 16)
        X, y = _data(300, D, K)
        pot = _recognised(softmax_model, X, y, K)
    assert pot is None, case


def test_intercept_free_logistic_keeps_logistic_potential():
    X, y = _data(300, 16)
    assert isinstance(_recognised(models.logreg_mcmc_model, X, y), LogisticPotential)


def test_entry_point_validates_arguments_before_any_cuda_call():
    """Logistic, softmax and Poisson regression with a constant weight scale: no pointer is dereferenced and no
    workspace is passed, so every call returns at its first failed check."""
    L = N.lib()
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)

    def call(kind=N.GLM_BERNOULLI, X=p, y=p, n=10000, Dx=16, K=1, bias=1, z=p, C=4, Dz=17, w_off=0, b_off=16,
             s_off=-1, s_w=1.0, s_b=10.0, U=p, g=p, null=False):
        m = N.b2_glm_regression(kind=kind, X=X, y=y, N=n, D=Dx, K=K, has_bias=bias, w_off=w_off, b_off=b_off,
                                s_w=s_w, s_b=s_b, s_off=s_off)
        return L.b2_glm_potential(None if null else ctypes.byref(m), z, C, Dz, U, g, None, 0, None)

    # z = [w (16), b]: valid, so the workspace check is next
    assert call() == -5
    assert call(null=True) == -4 and call(X=None) == -4 and call(y=None) == -4 and call(z=None) == -4
    assert call(U=None) == -4 and call(g=None) == -4
    # kinds and widths: Bernoulli D in {4, 8, 16, 32}, softmax D == 32 and 2 <= K <= 16, Poisson 1 <= D <= 128
    assert call(kind=7) == -2 and call(Dx=10, Dz=11, b_off=10) == -2
    assert call(kind=N.GLM_POISSON, Dx=10, Dz=11, b_off=10) == -5
    assert call(kind=N.GLM_POISSON, Dx=129, Dz=130, b_off=129) == -2
    assert call(kind=N.GLM_CATEGORICAL, Dx=32, K=4, Dz=132, b_off=128) == -5
    assert call(kind=N.GLM_CATEGORICAL, Dx=16, K=4, Dz=68, b_off=64) == -2
    assert call(kind=N.GLM_CATEGORICAL, Dx=32, K=17, Dz=561, b_off=544) == -2
    assert call(n=0) == -2 and call(C=0) == -2
    # the row: out of it, overlapping, or not exactly the blocks
    assert call(Dz=18) == -2 and call(Dz=16) == -2 and call(b_off=15) == -2 and call(w_off=1, b_off=0) == -5
    assert call(w_off=-1) == -2 and call(bias=0, Dz=16) == -5
    assert call(s_off=17, Dz=18) == -2                              # a noise scale outside linear regression
    assert call(s_w=0.0) == -2 and call(s_b=0.0) == -2 and call(bias=0, Dz=16, s_b=0.0) == -5
    # left to the likelihood call, after the workspace check: N (the SIMT Bernoulli kernel takes any) and alignment
    assert call(n=1 << 31) == -5 and call(X=q) == -5 and call(y=q) == -5


# ---- GPU tier ----------------------------------------------------------------------------------------------
def _oracle_potential(X, y, pot):
    """fp64 restatement of U(z) for z [..., Dz] (pyro/infer/mcmc/util.py:275-286 on the regression model):
    -(sum of the Normal prior log densities + the Bernoulli / Categorical log likelihood)."""
    Xd = X.double()
    yd = y.double() if pot.kind == N.GLM_BERNOULLI else y
    weight, bias = pot.weight, pot.bias

    def U(z):
        zero = torch.zeros((), dtype=z.dtype, device=z.device)
        w = z[..., pot.sites[weight][0]]
        lp = odists.normal(w, zero, zero + pot.s_w).sum(-1)
        bv = 0.0
        if bias is not None:
            bv = z[..., pot.sites[bias][0]]
            lp = lp + odists.normal(bv, zero, zero + pot.s_b).sum(-1)
        if pot.kind == N.GLM_BERNOULLI:
            logits = w @ Xd.T + (bv if bias is not None else 0.0)
            lp = lp + odists.bernoulli_logits(yd, logits).sum(-1)
        else:
            W = w.reshape(w.shape[:-1] + (pot.K, pot.Dx))
            logits = Xd @ W.mT + (bv.unsqueeze(-2) if bias is not None else 0.0)
            lp = lp + odists.categorical(yd, logits).sum(-1)
        return -lp
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


# (likelihood, K, bias): Bernoulli with and without an intercept, softmax with K = 2, 10, 16
_KINDS = [("Bernoulli", 1, True), ("Bernoulli", 1, False), ("Categorical", 2, True), ("Categorical", 10, True),
          ("Categorical", 16, False)]


def _direct_potential(kind, K, bias, X, y):
    """GlmPotential built directly (intercept-free Bernoulli is not a recognised route)."""
    D = X.shape[1]
    wshape = (D,) if kind == "Bernoulli" else (K, D)
    nw = K * D
    sites = {"w": (slice(0, nw), "identity", wshape)}
    if bias:
        sites["b"] = (slice(nw, nw + K), "identity", () if kind == "Bernoulli" else (K,))
    return GlmPotential(X, y, kind, sites, "w", "b" if bias else None, s_w=1.0, s_b=10.0)


def _trace_model(kind, K, bias):
    def model(X, y):
        D = X.shape[-1]
        if kind == "Bernoulli":
            w = pyro.sample("w", dist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
            b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0))) if bias else 0.0
            with pyro.plate("data", X.shape[0]):
                pyro.sample("y", dist.Bernoulli(logits=(w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b), obs=y)
        else:
            W = pyro.sample("w", dist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
            b = pyro.sample("b", dist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1)) if bias else 0.0
            with pyro.plate("data", X.shape[0]):
                Wm = W.squeeze(-3) if W.dim() > 2 else W
                pyro.sample("y", dist.Categorical(logits=X @ Wm.mT + b), obs=y)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("n", [300, 8192, 70001, 1_000_000])
@pytest.mark.parametrize("kind,K,bias", _KINDS, ids=["bern-b", "bern", "cat2-b", "cat10-b", "cat16"])
def test_potential_against_fp64_and_trace(kind, K, bias, n):
    """U and dU/dz at identical z for C = 1, 7, 64, 130 chains (one and three particle slabs of the Bernoulli
    kernel, up to 33 class slabs of the softmax kernel) against fp64, bitwise repeatable, and against
    TracePotential in fp32 where its [C, N, K] logits fit comfortably.  Measured on an H100: U within 1.0e-6
    relative of fp64 everywhere; the gradient within 1.9e-4 of max |grad| at N = 300, 4.6e-5 at 8192,
    1.8e-5 at 70001, and at 1e6 5.9e-6 (logistic), 8.8e-5 (softmax, 64 chains) and 2.3e-4 (softmax K = 10,
    130 chains); TracePotential's fp32 gradient is itself up to 2.9e-4 of max |grad| from fp64 at 1e6."""
    if EMULATE:
        pytest.skip("kernel test")
    D = 32
    X, y = _data(n, D, None if kind == "Bernoulli" else K, dev=DEV, seed=n + K)
    pot = _direct_potential(kind, K, bias, X, y)
    U_ref_fn = _oracle_potential(X, y, pot)
    errs = []
    for C in (1, 7, 64, 130):
        g = torch.Generator(device=DEV).manual_seed(C)
        z = 0.3 * torch.randn(C, pot.dim, generator=g, device=DEV)
        U, G = pot.value_and_grad(z)
        U2, G2 = pot.value_and_grad(z)
        assert torch.equal(U, U2) and torch.equal(G, G2)
        Ur, Gr = _oracle_value_and_grad(U_ref_fn, z, n, K)
        eu = float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max())
        eg = float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max()))
        et = gt = 0.0
        if C * n * K <= 64 * 70001 * 16:
            tp = TracePotential(_trace_model(kind, K, bias), (X, y), num_chains=C)
            assert list(tp.sites) == list(pot.sites) and tp.dim == pot.dim
            Ut, Gt = tp.value_and_grad(z)
            et = float(((U - Ut).abs() / Ut.abs().clamp(min=1.0)).max())
            gt = float((G - Gt).abs().max()) / max(1.0, float(Gt.abs().max()))
        errs.append((C, eu, eg, et, gt))
    print("\nglm potential %s K=%d bias=%d n=%d: (C, U vs fp64, grad vs fp64, U vs trace, grad vs trace) %s"
          % (kind, K, bias, n, ["%d %.1e %.1e %.1e %.1e" % e for e in errs]))
    for C, eu, eg, et, gt in errs:
        # gradient: the GLM tests' bounds, 2e-4 of max |grad| at their full size (N = 1e6, 64 particles) and
        # 5e-4 at ragged shapes; g = onehot - softmax enters the gradient contraction rounded to TF32, and fewer
        # CTAs per particle slab (130 chains) accumulate longer fp32 runs
        gtol = 2e-4 if n == 1_000_000 and C <= 64 else 5e-4
        assert eu <= 2e-6 and eg <= gtol, (C, eu, eg)
        assert et <= 2e-6 and gt <= 5e-4, (C, et, gt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,K", [("Bernoulli", 1), ("Categorical", 10)])
def test_captured_graph_replay_equals_eager(kind, K):
    if EMULATE:
        pytest.skip("needs CUDA graphs")
    X, y = _data(70001, 32, None if kind == "Bernoulli" else K, dev=DEV, seed=3)
    pot = _direct_potential(kind, K, True, X, y)
    z = 0.3 * torch.randn(64, pot.dim, device=DEV)
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
@pytest.mark.parametrize("kind,K", [("Bernoulli", 1), ("Categorical", 10)])
def test_hmc_trajectory_matches_oracle_integrator(kind, K):
    """Twenty leapfrog steps of HMC's integrator on GlmPotential from identical (z, r) against
    oracle.mcmc.velocity_verlet on the fp64 potential."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.004
    X, y = _data(n, 32, None if kind == "Bernoulli" else K, dev=DEV, seed=11)
    pot = _direct_potential(kind, K, True, X, y)
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = 0.1 * torch.randn(C, pot.dim, device=DEV)
    r0 = torch.randn(C, pot.dim, device=DEV)
    z, r = z0.clone(), r0.clone()
    _, g = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, g, U, _ = kernel._leapfrog(z, r, g, epsv, minv)
    Uo = _oracle_potential(X.cpu(), y.cpu(), pot)
    errs = []
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        errs.append((float((z[c].double().cpu() - zr).abs().max()),
                     float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max())),
                     abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))))
    print("\nhmc trajectory %s: (z err, r err, U err) %s" % (kind, ["%.1e %.1e %.1e" % e for e in errs]))
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


def _posterior_check(samples, ref, name):
    """Means within 0.3 posterior standard deviations, standard deviations within 25 %."""
    m, s = samples.mean(0), samples.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    assert bool(((m - rm).abs() <= 0.3 * rs).all()), (name, float(((m - rm).abs() / rs).max()))
    assert bool(((s - rs).abs() <= 0.25 * rs).all()), (name, float(((s - rs).abs() / rs).max()))


@pytest.mark.gpu
def test_nuts_logistic_model_posterior():
    """NUTS(logistic_model) at N = 10^4, D = 32, 8 chains, on GlmPotential, against the oracle sampler."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y = _data(10_000, 32, dev=DEV, seed=21)
    kernel = NUTS(models.logistic_model)
    mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1)
    mc.run(X, y)
    assert isinstance(kernel.potential, GlmPotential)
    s = mc.get_samples()
    got = torch.cat([s["w"].reshape(-1, 32), s["b"].reshape(-1, 1)], -1).double().cpu()
    chain = omcmc.NUTSChain(_oracle_potential(X.cpu(), y.cpu(), kernel.potential), 33, seed=2)
    ref, _ = chain.run(torch.zeros(33, dtype=torch.float64), 200, 800)
    _posterior_check(got, ref, "logistic")


@pytest.mark.gpu
def test_nuts_softmax_model_posterior():
    """NUTS on a small softmax regression (N = 200, K = 2, no bias) against the oracle sampler."""
    if EMULATE:
        pytest.skip("kernel test")
    K = 2
    X, y = _data(200, 32, K, dev=DEV, seed=22)
    kernel = NUTS(softmax_model_linear)
    mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1)
    mc.run(X, y, K)
    pot = kernel.potential
    assert isinstance(pot, GlmPotential)
    got = mc.get_samples()["W"].reshape(-1, K * 32).double().cpu()
    chain = omcmc.NUTSChain(_oracle_potential(X.cpu(), y.cpu(), pot), pot.dim, seed=2)
    ref, _ = chain.run(torch.zeros(pot.dim, dtype=torch.float64), 200, 800)
    _posterior_check(got, ref, "softmax")


@pytest.mark.gpu
def test_routes_taken_by_nuts_model():
    """In-scope models build GlmPotential and every evaluation is the four native launches; out-of-scope
    models keep TracePotential / LogisticPotential."""
    if EMULATE:
        pytest.skip("kernel test")
    Xb, yb = _data(9000, 32, dev=DEV, seed=1)
    Xc, yc = _data(9000, 32, 10, dev=DEV, seed=2)
    X33, y33 = _data(9000, 33, 10, dev=DEV, seed=3)
    for model, args, want in ((models.logistic_model, (Xb, yb), GlmPotential),
                              (models.logistic_model_fused, (Xb, yb), GlmPotential),
                              (softmax_model, (Xc, yc, 10), GlmPotential),
                              (softmax_model_linear, (Xc, yc, 10), GlmPotential),
                              (models.logreg_mcmc_model, (Xb, yb), LogisticPotential),
                              (softmax_model, (X33, y33, 10), TracePotential),
                              (models.logistic_model, (Xb.double(), yb.double()), TracePotential)):
        kernel = NUTS(model)
        kernel.setup(5, 4, *args)
        assert type(kernel.potential) is want, (model.__name__, type(kernel.potential).__name__)
        if want is GlmPotential:
            n0 = N.launch_count()
            kernel.sample()
            calls = N.launch_count() - n0
            assert calls > 0 and kernel.num_leapfrogs > 0


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

    def logistic(X, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Bernoulli(logits=X @ w + b), obs=y)

    def softmax(X, y, K):
        D = X.shape[-1]
        W = ref_pyro.sample("W", rdist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Categorical(logits=X @ W.mT + b), obs=y)

    Xb, yb = _data(4000, 32, dev=DEV, seed=1)
    Xc, yc = _data(4000, 32, 4, dev=DEV, seed=2)
    for model, args in ((logistic, (Xb, yb)), (softmax, (Xc, yc, 4))):
        assert isinstance(bind.recognise(model, args, {}, poutine=ref_pyro.poutine), GlmPotential)
        kernel = bind.NUTS(model, num_chains=4, seed=0)
        mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
        mc.run(*args)
        assert isinstance(kernel._kernel.potential, GlmPotential)
        for v in mc.get_samples().values():
            assert bool(torch.isfinite(v).all())
