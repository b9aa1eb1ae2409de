"""Binomial family: the elementwise site kernels (families 16 / 17), the fused Binomial-regression GLM kernels
(glm_binomial_tc.cu), the SVI route (``_BinomialLinear``) and the NUTS route (``GlmPotential`` through
``b2_glm_potential``).

CPU tier: the goldens recorded from the unmodified reference (tests/golden/make_golden_binomial.py), the host-built
functors against them, the lazy-logits routing, recognition, argument checks and the kernels' SASS.  GPU tier: the
kernels against fp64, SVI trajectories against the materialised path, and the potential against fp64.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import hostcheck
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device, load_npz
from oracle import dists as od
from oracle import mcmc as omcmc
from pyro_b200 import _build
from pyro_b200 import _native as N
from pyro_b200 import poutine
from pyro_b200.infer import HMC, MCMC, NUTS, SVI, JitTrace_ELBO, Trace_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.infer.mcmc import GlmPotential, TracePotential
from pyro_b200.lazy import LinearPredictorTensor, SiteValue
from pyro_b200.optim import ClippedAdam

DEV = device()
# (row trials, atoms of 32 columns, split X) -> mangled-name fragment; D = 32 runs the TMA tile pipeline
KERNELS = {(r, "flat", dc, sx): "glm_binomial_flat_tc_kernelILb%dELi%dELb%dE" % (int(r), dc, int(sx))
           for r in (False, True) for dc in (2, 3, 4) for sx in (False, True)}   # D < 32 runs DC = 2
KERNELS.update({(r, "d32", 1, sx): "glm_binomial_tc_kernelILb%dELb%dE" % (int(r), int(sx))
                for r in (False, True) for sx in (False, True)})
IDS = ["%s-%s-DC%d-%s" % ("rows" if r else "const", k, dc, "split_x" if sx else "default")
       for r, k, dc, sx in sorted(KERNELS)]


def binomial_lp(k, n, logits):
    """fp64 restatement of pyro/distributions/torch.py:83-101 at tol = 0; log_binomial is gradient-free there."""
    clamp_by_zero = (logits.clamp(min=0) + logits - logits.clamp(max=0)) / 2   # max(l, 0), gradient 1/2 at 0
    norm = n * (clamp_by_zero + torch.log1p(torch.exp(-logits.abs())))
    with torch.no_grad():
        lb = torch.lgamma(n + 1) - torch.lgamma(k + 1) - torch.lgamma(n + 1 - k)
    return k * logits - norm + lb


# ---- CPU tier: goldens and host-built functors -----------------------------------------------------------------
def _golden(name, kind, tag):
    z = load_npz("binomial.npz")
    return {key: z["%s_%s_%s_%s" % (name, kind, tag, key)] for key in ("n", "k", "p", "lp", "dn", "dp", "dk")}


@pytest.mark.parametrize("name", ["kat", "rand", "edge"])
def test_oracle_against_goldens(name):
    g = _golden(name, "logits", "f64")
    n, k = torch.tensor(g["n"]), torch.tensor(g["k"]).requires_grad_(True)
    l = torch.tensor(g["p"]).requires_grad_(True)
    nn = n.clone().requires_grad_(True)
    lp = binomial_lp(k, nn, l)
    dn, dl, dk = torch.autograd.grad(lp.sum(), [nn, l, k])
    np.testing.assert_allclose(lp.detach().numpy(), g["lp"], rtol=1e-12, atol=1e-12)
    for got, key in ((dn, "dn"), (dl, "dp"), (dk, "dk")):
        np.testing.assert_allclose(got.numpy(), g[key], rtol=1e-12, atol=1e-12, err_msg=key)
    if name == "kat":
        # the reference fixtures are scipy's binom.logpmf
        from scipy import stats
        gp = _golden(name, "probs", "f64")
        np.testing.assert_allclose(gp["lp"], stats.binom.logpmf(gp["k"], gp["n"], gp["p"]), atol=1e-5)


@pytest.mark.parametrize("tag", ["f64", "f32"])
@pytest.mark.parametrize("kind", ["logits", "probs"])
@pytest.mark.parametrize("name", ["kat", "rand", "edge"])
def test_host_functors_against_goldens(name, kind, tag):
    g = _golden(name, kind, tag)
    fam = N.BINOMIAL_LOGITS if kind == "logits" else N.BINOMIAL_PROBS
    dt = np.float64 if tag == "f64" else np.float32
    lp, dx, (dn, dp) = hostcheck.eval_family(fam, g["k"], [g["n"], g["p"]], dtype=dt)
    if tag == "f64":
        rtol, atol = 1e-10, 1e-10
    else:
        # fp32: log C(n, k) of counts up to 200 is a difference of lgamma values near 860 (ulp 6e-5)
        rtol, atol = 2e-5, 2e-3
    np.testing.assert_allclose(lp, g["lp"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(dx, g["dk"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(dn, g["dn"], rtol=rtol, atol=atol)
    # probs gradients grow as 1 / (p (1 - p)) near the ends
    scale = np.maximum(1.0, np.abs(g["dp"]))
    np.testing.assert_array_less(np.abs(dp - g["dp"]) / scale, rtol * 10 + atol)


# ---- CPU tier: the mirror distribution and the lazy logits ----------------------------------------------------
def test_mirror_binomial_shapes_support_and_sampling():
    d = dist.Binomial(10, logits=torch.zeros(3, 4))
    assert tuple(d.batch_shape) == (3, 4) and d.support.upper_bound.item() == 10.0
    s = d.sample((2,))
    assert tuple(s.shape) == (2, 3, 4) and bool((s >= 0).all()) and bool((s <= 10).all())
    d2 = dist.Binomial(torch.tensor([3, 5]), probs=torch.tensor([0.2, 0.9], dtype=torch.float64))
    assert d2.total_count.dtype == torch.float64 and d2.family == N.BINOMIAL_PROBS
    with pytest.raises(NotImplementedError):
        d.rsample()
    with pytest.raises(ValueError):
        dist.Binomial(3, probs=torch.zeros(2), logits=torch.zeros(2))
    assert "Binomial" in dist.__all__


def _lazy(n=9000, D=10, P=4, bias=True):
    torch.manual_seed(0)
    X = torch.randn(n, D)
    w = torch.randn(P, 1, D).as_subclass(SiteValue)
    b = torch.randn(P, 1).as_subclass(SiteValue)
    l = w.squeeze(-2) @ X.T
    return X, (l + b if bias else l)


def test_binomial_of_lazy_logits_builds_the_fused_subclass_in_both_front_ends():
    X, l = _lazy()
    assert isinstance(l, LinearPredictorTensor)
    d = dist.Binomial(10, logits=l)
    assert type(d).__name__ == "_BinomialLinear" and tuple(d.batch_shape) == (4, 9000)
    assert d._dense is None
    # torch's constructor (the reference's Binomial subclasses it): broadcast_all + type_as keep the logits lazy
    trials = torch.randint(0, 20, (9000,)).float()
    for tc in (7, trials):
        td = torch.distributions.Binomial(tc, logits=l, validate_args=True)
        assert isinstance(td.logits, LinearPredictorTensor)
        conv = dist.Binomial(td.total_count, logits=td.__dict__["logits"])
        assert type(conv).__name__ == "_BinomialLinear" and conv._dense is None
        t, per_row = dist._binomial_trials(conv.total_count, conv._lazy)
        assert per_row == (0 if isinstance(tc, int) else 1)
        if per_row:
            assert t.data_ptr() == trials.data_ptr()        # the stored [N] counts, not a [P, N] slice
    # every other use materialises the logits exactly as the model wrote them
    np.testing.assert_array_equal(d.logits.numpy(), l.eager().numpy())


def _route(total_count, value_fn=None, mask=None, dtype=torch.float32, n=9000, D=10, P=4, probs=False,
           offset=False, fail_y=False):
    X, l = _lazy(n, D, P)
    X = X.to(dtype)
    if dtype != torch.float32:
        l = (torch.randn(P, 1, D, dtype=dtype).as_subclass(SiteValue).squeeze(-2) @ X.T
             + torch.randn(P, 1, dtype=dtype).as_subclass(SiteValue))
    if offset:
        l = l + 0.5
    y = torch.zeros(n, dtype=dtype) if value_fn is None else value_fn(n)
    d = dist.Binomial(total_count, probs=torch.sigmoid(l)) if probs else dist.Binomial(total_count, logits=l)
    calls = []
    real_fused, real_mat = dist._GlmBinomialFn.apply, dist._Elementwise._fused_sum
    dist._GlmBinomialFn.apply = lambda *a: calls.append("fused")
    dist._Elementwise._fused_sum = lambda self, *a, **k: calls.append("materialised")
    try:
        d._fused_sum(y, mask, 1.0, 1.0, 1.0)
    finally:
        dist._GlmBinomialFn.apply, dist._Elementwise._fused_sum = real_fused, real_mat
    return calls


@pytest.mark.parametrize("case", ["number", "scalar", "one", "rows", "expanded_scalar"])
def test_in_scope_sites_take_the_kernel(case):
    n = 9000
    tc = {"number": 10, "scalar": torch.tensor(10.0), "one": torch.tensor([10.0]),
          "rows": torch.randint(0, 20, (n,)).float(), "expanded_scalar": torch.tensor(10.0).expand(4, n)}[case]
    assert _route(tc) == ["fused"]


@pytest.mark.parametrize("case", ["offset", "mask", "probs", "per_particle", "fp64", "N8191", "D129", "grad",
                                  "sliced_rows", "y_misaligned"])
def test_near_misses_materialise(case):
    n = 9000
    kw = {}
    tc = 10
    if case == "offset":
        kw["offset"] = True
    elif case == "mask":
        kw["mask"] = torch.ones(n, dtype=torch.bool)
    elif case == "probs":
        kw["probs"] = True
    elif case == "per_particle":
        tc = torch.full((4, 1), 10.0)
    elif case == "fp64":
        kw["dtype"] = torch.float64
        tc = torch.tensor(10.0, dtype=torch.float64)
    elif case == "N8191":
        kw["n"] = 8191
    elif case == "D129":
        kw["D"] = 129
    elif case == "grad":
        tc = torch.tensor(10.0, requires_grad=True)
    elif case == "sliced_rows":
        tc = torch.randint(0, 20, (n + 1,)).float()[1:]
    elif case == "y_misaligned":
        kw["value_fn"] = lambda m: torch.zeros(m + 1)[1:]
    calls = _route(tc, **kw)
    assert calls in ([], ["materialised"]) and "fused" not in calls, (case, calls)


def test_bind_maps_the_reference_binomial():
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference tree not built")
    import pyro.distributions as rd
    X, l = _lazy()
    ref = rd.Binomial(torch.full((9000,), 5.0), logits=l)
    conv = bind.to_b2(ref)
    assert type(conv).__name__ == "_BinomialLinear"
    probs = bind.to_b2(rd.Binomial(5, probs=torch.full((3,), 0.3)))
    assert isinstance(probs, dist.Binomial) and probs.family == N.BINOMIAL_PROBS
    approx = rd.Binomial(5, logits=torch.zeros(3))
    approx.approx_log_prob_tol = 0.1
    assert bind.to_b2(approx) is None


# ---- CPU tier: argument checks --------------------------------------------------------------------------------
def test_binomial_entry_points_validate_arguments_before_any_cuda_call():
    """The pointers are never dereferenced and no workspace is passed: the checks come first."""
    L = N.lib()
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)

    def call(X, y, m, per_row, W, n, D, flags, ws=None, nbytes=0):
        return L.b2_glm_binomial_logits(X, y, m, per_row, W, None, n, D, 8, 1.0, 1.0, 1.0, flags, None, None, None,
                                        None, ws, nbytes, None)

    assert call(None, p, p, 1, p, 10000, 10, 0) == -4                # B2_ERR_NULL
    assert call(p, None, p, 1, p, 10000, 10, 0) == -4
    assert call(p, p, None, 0, p, 10000, 10, 0) == -4
    assert call(p, p, p, 1, None, 10000, 10, 0) == -4
    assert call(p, p, p, 1, p, 0, 10, 0) == -2                       # B2_ERR_BAD_SHAPE
    for D in (0, -1, 129):
        assert call(p, p, p, 1, p, 10000, D, 0) == -2, D
    assert call(p, p, p, 2, p, 10000, 10, 0) == -2                   # trials_per_row not 0 / 1
    assert call(q, p, p, 1, p, 10000, 10, 0) == -2                   # X not 16-byte aligned
    assert call(p, q, p, 1, p, 10000, 10, 0) == -2                   # y not 16-byte aligned
    assert call(p, p, q, 1, p, 10000, 10, 0) == -2                   # per-row trials not 16-byte aligned
    assert call(p, p, p, 1, p, 10000, 32, N.B2_FLAG_GLM_FP32) == -2  # no fp32 SIMT kernel
    assert call(p, p, p, 1, p, 1 << 31, 10, 0) == -8                 # B2_ERR_TOO_LARGE
    for D in (1, 10, 32, 33, 128):                                   # valid: the workspace check is next
        assert call(p, p, q, 0, p, 10000, D, 0) == -5, D             # one count: any alignment
        need = int(L.b2_glm_binomial_workspace(10000, D, 8))
        assert call(p, p, p, 1, p, 10000, D, 0, p, need - 1) == -5, D

    def pot(X, y, m, per_row, D, bias, z, Dz, w_off, b_off, s_w=1.0, s_b=1.0, U=p, g=p):
        r = N.b2_glm_regression(kind=N.GLM_BINOMIAL, X=X, y=y, N=10000, D=D, K=1, trials=m, trials_per_row=per_row,
                                has_bias=bias, w_off=w_off, b_off=b_off, s_w=s_w, s_b=s_b, s_off=-1)
        return L.b2_glm_potential(ctypes.byref(r), z, 8, Dz, U, g, None, 0, None)

    assert pot(None, p, p, 1, 10, 1, p, 11, 0, 10) == -4
    assert pot(p, p, None, 1, 10, 1, p, 11, 0, 10) == -4
    assert pot(p, p, p, 1, 10, 1, None, 11, 0, 10) == -4
    assert pot(p, p, p, 1, 10, 1, p, 12, 0, 10) == -2                # Dz != D + 1
    assert pot(p, p, p, 1, 10, 1, p, 11, 2, 0) == -2                 # weights out of the row
    assert pot(p, p, p, 1, 10, 1, p, 11, 0, 5) == -2                 # bias inside the weights
    assert pot(p, p, p, 1, 10, 1, p, 11, 0, 10, s_w=0.0) == -2
    assert pot(p, p, p, 3, 10, 1, p, 11, 0, 10) == -2
    assert pot(p, p, q, 1, 10, 1, p, 11, 0, 10) == -2
    assert pot(p, p, p, 1, 129, 0, p, 129, 0, 0) == -2
    assert pot(p, p, p, 1, 10, 1, p, 11, 0, 10) == -5                # valid: workspace next
    assert pot(p, p, p, 0, 10, 0, p, 10, 0, 0) == -5


# ---- CPU tier: the kernels' SASS ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    from test_glm_tc_sass import _tools
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp("glm_binomial_sass") / "glm_binomial_tc.o")
    src = os.path.join(_build.CSRC, "glm_binomial_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _g2(key):
    return "64x%dx8" % (32 * key[2] + 8)


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_no_serialisation_note_and_no_spills(compiled, key):
    from test_glm_tc_sass import _ptxas_properties
    log, _ = compiled
    assert "C7515" not in log and "C7520" not in log, log
    props, used = _ptxas_properties(log, KERNELS[key])
    assert "0 bytes spill stores, 0 bytes spill loads" in props, props + " / " + used


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_one_wait_per_contraction(compiled, key):
    """GEMM 1 is m64n64k8 over 4 DC k-steps (2 or 3 split products each), GEMM 2 m64n(32 DC + 8)k8 over 8
    k-steps; a WARPGROUP.DEPBAR or WARPGROUP.ARRIVE between two HGMMA of one shape breaks the chain."""
    import re

    from test_glm_tc_sass import _sass_function
    _, _, dc, split_x = key
    _, sass = compiled
    shapes, bad = [], []
    prev, between = None, []
    for line in _sass_function(sass, KERNELS[key]):
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            if m.group(1) == prev and between:
                bad.append("%s after %s" % (m.group(1), between))
            shapes.append(m.group(1))
            prev, between = m.group(1), []
        elif "WARPGROUP.DEPBAR" in line or "WARPGROUP.ARRIVE" in line:
            between.append(line.split(";")[0].split("*/")[-1].strip())
    assert shapes.count("64x64x8") == 4 * dc * (3 if split_x else 2), shapes
    assert shapes.count(_g2(key)) == 8, shapes
    assert not bad, bad


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_mufu_ops_per_logit_in_the_tile_loop(compiled, key):
    """ex2 and lg2 per logit (32 each per thread and tile); the log binomial coefficients are summed after the
    loop."""
    from test_glm_flat import _opcode, _tile_loop
    from test_glm_tc_sass import _sass_function
    _, sass = compiled
    loop = _tile_loop(_sass_function(sass, KERNELS[key]), _g2(key))
    ops = [_opcode(l) for l in loop]
    assert ops.count("MUFU.EX2") >= 32, ops.count("MUFU.EX2")
    # (the loop holds the epilogue twice: the masked last tile and the others)
    assert 32 <= ops.count("MUFU.LG2") <= 72, ops.count("MUFU.LG2")


# ---- CPU tier: recognition ------------------------------------------------------------------------------------
def binomial_model(X, y, trials):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        l = w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b
        pyro.sample("y", dist.Binomial(trials, logits=l), obs=y)


def binomial_model_nobias(X, y, trials):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 0.5).to_event(1))
    with pyro.plate("data", X.shape[0]):
        l = w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w
        pyro.sample("y", dist.Binomial(trials, logits=l), obs=y)


def _variant(change):
    def model(X, y, trials):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        with pyro.plate("data", X.shape[0]):
            l = w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b
            if change == "times2":
                l = 2 * l
            if change == "probs":
                d = dist.Binomial(trials, probs=torch.sigmoid(l))
            elif change == "moving_trials":
                d = dist.Binomial(trials + torch.floor(10 * w.detach().abs().sum()), logits=l)
            else:
                d = dist.Binomial(trials, logits=l)
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool))
            pyro.sample("y", d, obs=y)
    return model


def _data(n, D, dtype=torch.float32, dev="cpu", seed=0, trials="rows", level=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    X = torch.randn(n, D, generator=g, dtype=torch.float64)
    w = 0.5 * torch.randn(D, generator=g, dtype=torch.float64) / D ** 0.5
    m = (torch.randint(0, 201, (n,), generator=g).double() if trials == "rows"
         else torch.full((n,), float(trials), dtype=torch.float64))
    y = torch.binomial(m, torch.sigmoid(X @ w + level), generator=g)
    tr = m.to(dtype).to(dev) if trials == "rows" else float(trials)
    return X.to(dtype).to(dev), y.to(dtype).to(dev), tr


def _recognised(model, *args):
    import cpu_emulation

    from pyro_b200.infer.mcmc.compile import recognise
    with cpu_emulation.enabled():
        return recognise(model, args)


@pytest.mark.parametrize("trials", ["rows", 10])
@pytest.mark.parametrize("name", ["bias", "nobias"])
def test_recognises_binomial_regression(name, trials):
    X, y, m = _data(300, 10, trials=trials)
    model = binomial_model if name == "bias" else binomial_model_nobias
    pot = _recognised(model, X, y, m)
    assert isinstance(pot, GlmPotential) and pot.binomial
    assert pot.trials_per_row == (1 if trials == "rows" else 0)
    if trials == "rows":
        assert torch.equal(pot.trials, m)
    else:
        assert float(pot.trials) == 10.0
    tp = TracePotential(model, (X, y, m))
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, _, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
    assert pot.has_bias == (name == "bias")


@pytest.mark.parametrize("change", ["times2", "probs", "moving_trials", "mask", "fp64", "grad_trials"])
def test_near_misses_are_not_recognised(change):
    if change == "fp64":
        X, y, m = _data(300, 10, dtype=torch.float64)
        pot = _recognised(binomial_model, X, y, m)
    elif change == "grad_trials":
        X, y, m = _data(300, 10)
        pot = _recognised(binomial_model, X, y, m.clone().requires_grad_(True))
    else:
        X, y, m = _data(300, 10)
        pot = _recognised(_variant(change), X, y, m)
    assert not isinstance(pot, GlmPotential), change


# ---- GPU tier: the site kernel --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["logits", "probs"])
@pytest.mark.parametrize("n,large", [(300, False), (300, True), (50000, False)], ids=["small", "small_large", "big"])
def test_site_kernel_against_fp64(kind, n, large):
    """[N] trials against [P, N] parameters, scale and mask, the one-CTA and the multi-CTA kernels: the value and
    the parameter gradients against torch fp64."""
    if EMULATE:
        pytest.skip("kernel test")
    P = 5
    g = torch.Generator().manual_seed(n + (kind == "probs"))
    m = torch.randint(0, 60, (n,), generator=g).float()
    k = torch.floor(torch.rand(P, n, generator=g) * (m + 1)).clamp(max=m)
    l = 2 * torch.randn(P, n, generator=g)
    p = torch.sigmoid(l).clamp(1e-4, 1 - 1e-4)
    mask = torch.rand(P, n, generator=g) < 0.8
    m, k, l, p, mask = m.to(DEV), k.to(DEV), l.to(DEV), p.to(DEV), mask.to(DEV)
    par = (l if kind == "logits" else p).clone().requires_grad_(True)
    saved = N.FORCE_LARGE_SITE_KERNELS
    N.FORCE_LARGE_SITE_KERNELS = large
    try:
        d = dist.Binomial(m, **{kind: par})
        lp = d.log_prob(k)
        total = d._fused_sum(k, mask, 0.5, 1.0, 1.0)
        (gp,) = torch.autograd.grad(total, [par])
    finally:
        N.FORCE_LARGE_SITE_KERNELS = saved
    pd = par.detach().double().requires_grad_(True)
    ld = pd if kind == "logits" else torch.log(pd) - torch.log1p(-pd)
    ref = binomial_lp(k.double(), m.double(), ld)
    ref_total = 0.5 * torch.where(mask, ref, torch.zeros_like(ref)).sum()
    (gref,) = torch.autograd.grad(ref_total, [pd])
    assert float((lp.double() - ref).abs().max()) <= 2e-3 + 2e-5 * float(ref.abs().max())
    assert abs(float(total) - float(ref_total)) <= 2e-5 * abs(float(ref_total)) + 1e-2
    assert float((gp.double() - gref).abs().max()) <= 1e-4 * max(1.0, float(gref.abs().max()))


# ---- GPU tier: the GLM kernel against fp64 --------------------------------------------------------------------
def _launch(X, y, m, W, b, flags):
    n, D = X.shape
    P = W.shape[0]
    per_row = 1 if m.numel() == n and n > 1 else 0
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dW = torch.empty(P, D, device=DEV)
    db = torch.empty(P, device=DEV)
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_binomial_workspace(n, D, P)), tag="glm_binomial")
    N.check(N.lib().b2_glm_binomial_logits(X.data_ptr(), y.data_ptr(), m.data_ptr(), per_row, W.data_ptr(),
                                           b.data_ptr() if b is not None else None, n, D, P, 1.0, 1.0, 1.0, flags,
                                           sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(),
                                           ws.data_ptr(), ws.numel(), N.stream_ptr(torch.device(DEV))),
            "b2_glm_binomial_logits")
    torch.cuda.synchronize()
    return sum_p, total, dW, db


def _reference(X, y, m, W, b):
    """fp64 per-particle sums and their gradients by autograd (on the device)."""
    Wd = W.double().requires_grad_(True)
    bd = (b if b is not None else torch.zeros(W.shape[0], device=W.device)).double().requires_grad_(True)
    s = binomial_lp(y.double(), m.double().expand(y.shape), Wd @ X.double().t() + bd[:, None]).sum(1)
    gW, gb = torch.autograd.grad(s.sum(), [Wd, bd])
    return s.detach(), gW, gb


def _term_size(X, y, m, W, b):
    """Per particle, SUM_n |y l| + m softplus(l) + |log C(m, y)| in fp64: the size of the terms of sum_p."""
    l = W.double() @ X.double().t() + (b.double()[:, None] if b is not None else 0.0)
    yd, md = y.double(), m.double().expand(y.shape)
    lb = torch.lgamma(md + 1) - torch.lgamma(yd + 1) - torch.lgamma(md - yd + 1)
    return ((yd * l).abs() + md * torch.nn.functional.softplus(l) + lb.abs()).sum(1)


def _full_data(n, P, D, trials, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=g)
    wt = 0.5 * torch.randn(D, generator=g) / D ** 0.5
    m = torch.randint(0, 201, (n,), generator=g).float() if trials == "rows" else torch.full((1,), float(trials))
    y = torch.binomial(m.expand(n), torch.sigmoid(X @ wt), generator=g)
    W = 0.05 * torch.randn(P, D, generator=g) / D ** 0.5 + wt
    b = 0.1 * torch.randn(P, generator=g)
    return X.to(DEV), y.to(DEV), m.to(DEV), W.to(DEV), b.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("trials", [1, 10, 100, "rows"])
@pytest.mark.parametrize("D", [1, 10, 31, 32, 33, 64, 100, 128])
def test_kernel_full_size_against_fp64(D, trials):
    """N = 1e6, P = 64: sums within 2e-5 relative, dW and db within 2e-4 of the largest gradient, two launches
    bitwise equal.  Per-row counts are drawn from 0..200, zeros included."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, m, W, b = _full_data(1_000_000, 64, D, trials, 300 + D)
    s_ref, gW, gb = _reference(X, y, m, W, b)
    sum_p, total, dW, db = _launch(X, y, m, W, b, 0)
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    ew = float((dW.double() - gW).abs().max()) / float(gW.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    print("\nbinomial D=%d trials=%s: sum %.1e dW %.1e db %.1e" % (D, trials, es, ew, eb))
    assert es <= 2e-5 and ew <= 2e-4 and eb <= 2e-4, (es, ew, eb)
    assert abs(float(total) - float(s_ref.sum())) <= 2e-5 * abs(float(s_ref.sum()))
    sum2, total2, dW2, db2 = _launch(X, y, m, W, b, 0)
    assert torch.equal(sum_p, sum2) and torch.equal(total, total2)
    assert torch.equal(dW, dW2) and torch.equal(db, db2)


_RAGGED = [(1, 1, 1, True), (63, 7, 32, False), (64, 65, 10, True), (65, 1, 33, False), (8191, 7, 100, True),
           (70001, 65, 32, True), (70001, 1, 127, False), (65, 130, 32, True), (8191, 130, 3, False),
           (70001, 7, 10, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("trials", [10, "rows"])
@pytest.mark.parametrize("n,P,D,bias", _RAGGED, ids=["-".join(map(str, c)) for c in _RAGGED])
def test_kernel_ragged_shapes_against_fp64(n, P, D, bias, trials):
    """Partial last tiles, a CTA's only tile, one to three particle slabs: sums within 2e-5 of the size of their
    terms, dW and db within 5e-4 of the largest gradient (1e-3 below one full tile, as for the Poisson kernel).

    A few rows' sum can cancel far below its terms: one row with a hundred-odd trials scores y l - m softplus(l) -
    log C(m, y) as terms of about 100 each that can add up to a few units.  Each term carries the rounding of its fp32 value (an lgamma near
    500 has an ulp of 3e-5), as it does on the materialised fp32 path, so the bound is taken against
    SUM |y l| + m softplus(l) + |log C(m, y)|, not against the sum itself."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, m, W, b = _full_data(n, P, D, trials, 7 * n + 3 * P + D)
    b = b if bias else None
    if trials == "rows" and n == 1:
        m = m.clone()
    s_ref, gW, gb = _reference(X, y, m, W, b)
    sum_p, total, dW, db = _launch(X, y, m, W, b, 0)
    tol_g = 5e-4 if n >= 64 else 1e-3
    size = _term_size(X, y, m, W, b)
    assert bool(((sum_p.double() - s_ref).abs() <= 2e-5 * size.clamp(min=1.0)).all()), \
        float(((sum_p.double() - s_ref).abs() / size.clamp(min=1.0)).max())
    assert float((dW.double() - gW).abs().max()) <= tol_g * max(1e-6, float(gW.abs().max()))
    if bias:
        assert float((db.double() - gb).abs().max()) <= tol_g * max(1e-6, float(gb.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 32])
def test_one_trial_agrees_with_the_bernoulli_kernel(D):
    if EMULATE:
        pytest.skip("kernel test")
    X, y, m, W, b = _full_data(1_000_000, 64, D, 1, 500 + D)
    sum_p, total, dW, db = _launch(X, y, m, W, b, 0)
    n, P = X.shape[0], W.shape[0]
    s2, t2, dW2, db2 = (torch.empty(P, device=DEV), torch.empty((), device=DEV), torch.empty(P, D, device=DEV),
                        torch.empty(P, device=DEV))
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_workspace(n, D, P)), tag="glm_bern")
    N.check(N.lib().b2_glm_bernoulli_logits(X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr(), n, D, P, 1.0,
                                            1.0, 1.0, 0, s2.data_ptr(), t2.data_ptr(), dW2.data_ptr(),
                                            db2.data_ptr(), ws.data_ptr(), ws.numel(),
                                            N.stream_ptr(torch.device(DEV))), "b2_glm_bernoulli_logits")
    torch.cuda.synchronize()
    assert float(((sum_p - s2).abs() / s2.abs()).max()) <= 2e-5
    assert float((dW - dW2).abs().max()) <= 2e-4 * float(dW2.abs().max())
    assert float((db - db2).abs().max()) <= 2e-4 * float(db2.abs().max())


# ---- GPU tier: the unchanged model under SVI ------------------------------------------------------------------
def binomial_guide(X, y, trials):
    D = X.shape[-1]
    w_loc = pyro.param("w_loc", X.new_zeros(D))
    w_scale = pyro.param("w_scale", X.new_full((D,), 0.1), constraint=dist.constraints.positive)
    b_loc = pyro.param("b_loc", X.new_zeros(()))
    b_scale = pyro.param("b_scale", X.new_full((), 0.1), constraint=dist.constraints.positive)
    pyro.sample("w", dist.Normal(w_loc, w_scale).to_event(1))
    pyro.sample("b", dist.Normal(b_loc, b_scale))


def binomial_model_masked(X, y, trials, mask):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Binomial(trials, logits=w.squeeze(-2) @ X.T + b).mask(mask), obs=y)


def binomial_model_offset(X, y, trials):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Binomial(trials, logits=w.squeeze(-2) @ X.T + b + 0.25), obs=y)


def _run(model, X, y, m, eps_w, eps_b, lazy, elbo_cls=Trace_ELBO, extra=()):
    import models
    pyro.clear_param_store()
    bw, bb = torch.empty_like(eps_w[0]), torch.empty_like(eps_b[0])
    calls = []
    real = dist._GlmBinomialFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)

    def guide(*args):
        with models.InjectNoise({"w": bw, "b": bb}):
            binomial_guide(*args[:3])

    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    dist._GlmBinomialFn.apply = spy
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  elbo_cls(num_particles=eps_w.shape[1], vectorize_particles=True, max_plate_nesting=1))
        losses = []
        for i in range(eps_w.shape[0]):
            bw.copy_(eps_w[i])
            bb.copy_(eps_b[i])
            losses.append(svi.step(X, y, m, *extra))
    finally:
        elbo_mod.LAZY_LINEAR = saved
        dist._GlmBinomialFn.apply = real
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in ("w_loc", "w_scale", "b_loc", "b_scale")}, len(calls)


def _svi_data(n, D, P, steps, seed, trials="rows", dtype=torch.float32):
    X, y, m = _data(n, D, dtype=dtype, seed=seed, trials=trials, dev=DEV)
    g = torch.Generator().manual_seed(seed + 1)
    eps_w = torch.randn(steps, P, 1, D, generator=g, dtype=dtype).to(DEV)
    eps_b = torch.randn(steps, P, 1, generator=g, dtype=dtype).to(DEV)
    return X, y, m, eps_w, eps_b


class _materialisations:
    """Records every materialisation of lazy Binomial logits: ``_BinomialLinear._params`` (the eager expression or
    the dense predictor) and ``LinearPredictor.dense``."""

    def __enter__(self):
        self.calls = []
        self.real_params = dist._BinomialLinear.__dict__["_params"]
        self.real_dense = dist.LinearPredictor.dense
        calls, real_params, real_dense = self.calls, self.real_params, self.real_dense

        def params(obj):
            if obj._dense is None:
                calls.append("_params")
            return real_params.fget(obj)

        def dense(obj):
            calls.append("dense")
            return real_dense(obj)
        dist._BinomialLinear._params = property(params)
        dist.LinearPredictor.dense = dense
        return self.calls

    def __exit__(self, *exc):
        dist._BinomialLinear._params = self.real_params
        dist.LinearPredictor.dense = self.real_dense


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 12])
@pytest.mark.parametrize("D", [10, 32, 100])
def test_unchanged_model_under_svi_matches_materialised(D, trials):
    """N = 70 000, 16 vectorised particles: every step's site goes through the kernel, the [P, N] logits are never
    materialised, and three steps match LAZY_LINEAR = False (loss 2e-5 relative, parameters 2e-4)."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, m, ew, eb = _svi_data(70000, D, 16, 3, D, trials)
    with _materialisations() as dense_calls:
        l_f, p_f, calls = _run(binomial_model, X, y, m, ew, eb, True)
    assert calls == 3 and not dense_calls
    l_m, p_m, calls_m = _run(binomial_model, X, y, m, ew, eb, False)
    assert calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 12])
@pytest.mark.parametrize("D", [10, 32, 100])
def test_reference_pyro_model_under_bind_matches_materialised(D, trials):
    """The same model written against the unmodified reference, through bind.Trace_ELBO: the kernel scores the
    site (torch's broadcast_all and type_as keep the logits lazy), and three steps match the model whose logits
    are materialised by ``* 1.0`` (scored by the Binomial site kernel)."""
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference tree not built")
    import pyro as rpyro
    import pyro.distributions as rdist
    X, y, m, _, _ = _svi_data(70000, D, 16, 3, 77 + D, trials)

    def run(lazy):
        # the guide draws with torch's generator, reseeded so both runs see the same noise
        torch.manual_seed(0)

        def model(X, y, trials):
            D = X.shape[-1]
            w = rpyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
            b = rpyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
            with rpyro.plate("data", X.shape[0]):
                logits = w.squeeze(-2) @ X.T + b
                rpyro.sample("y", rdist.Binomial(trials, logits=logits if lazy else logits * 1.0), obs=y)

        rpyro.clear_param_store()

        def guide(X, y, trials):
            D = X.shape[-1]
            w_loc = rpyro.param("w_loc", X.new_zeros(D))
            w_scale = rpyro.param("w_scale", X.new_full((D,), 0.1), constraint=rdist.constraints.positive)
            b_loc = rpyro.param("b_loc", X.new_zeros(()))
            b_scale = rpyro.param("b_scale", X.new_full((), 0.1), constraint=rdist.constraints.positive)
            rpyro.sample("w", rdist.Normal(w_loc, w_scale).to_event(1))
            rpyro.sample("b", rdist.Normal(b_loc, b_scale))

        calls = []
        real = dist._GlmBinomialFn.apply
        dist._GlmBinomialFn.apply = lambda *a: calls.append(1) or real(*a)
        try:
            svi = bind.SVI(model, guide, bind.ClippedAdam({"lr": 0.01}),
                           bind.Trace_ELBO(num_particles=16, vectorize_particles=True, max_plate_nesting=1))
            with _materialisations() as dense_calls:
                losses = [svi.step(X, y, m) for _ in range(3)]
            if lazy:
                assert not dense_calls, dense_calls
        finally:
            dist._GlmBinomialFn.apply = real
        store = rpyro.get_param_store()
        return losses, {k: store[k].detach().clone() for k in ("w_loc", "w_scale", "b_loc", "b_scale")}, len(calls)

    l_f, p_f, calls = run(True)
    l_m, p_m, calls_m = run(False)
    assert calls == 3 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_captured_graph_step_equals_eager():
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, y, m, ew, eb = _svi_data(70000, 32, 16, 4, 5)
    l_e, p_e, n_e = _run(binomial_model, X, y, m, ew, eb, True)
    l_g, p_g, n_g = _run(binomial_model, X, y, m, ew, eb, True, JitTrace_ELBO)
    assert n_e == 4 and n_g >= 3
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["N8191", "masked", "fp64", "D129", "offset", "per_particle"])
def test_out_of_scope_sites_keep_the_materialised_path(case):
    if EMULATE:
        pytest.skip("kernel test")
    n, D, P = 9000, 10, 4
    dtype = torch.float64 if case == "fp64" else torch.float32
    D = 129 if case == "D129" else D
    n = 8191 if case == "N8191" else n
    X, y, m, ew, eb = _svi_data(n, D, P, 2, 31, dtype=dtype)
    model, extra = binomial_model, ()
    if case == "masked":
        model = binomial_model_masked
        extra = (torch.rand(n, device=DEV) < 0.7,)
    if case == "offset":
        model = binomial_model_offset
    if case == "per_particle":
        m = torch.full((P, 1), 50.0, device=DEV)
        y = y.clamp(max=50)
    l_f, p_f, calls = _run(model, X, y, m, ew, eb, True, extra=extra)
    assert calls == 0
    l_m, p_m, _ = _run(model, X, y, m, ew, eb, False, extra=extra)
    tol = 1e-12 if dtype == torch.float64 else 2e-6
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= tol * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=tol, rtol=tol), k


# ---- GPU tier: GlmPotential -----------------------------------------------------------------------------------
def _direct_potential(X, y, m, bias):
    D = X.shape[1]
    sites = {"w": (slice(0, D), "identity", (D,))}
    if bias:
        sites["b"] = (slice(D, D + 1), "identity", ())
    return GlmPotential(X, y, "Binomial", sites, "w", "b" if bias else None, s_w=1.0, s_b=10.0, trials=m)


def _oracle_value_and_grad(X, y, m, pot, z):
    Xd, yd = X.double(), y.double()
    md = (m.double() if isinstance(m, torch.Tensor) else torch.full_like(yd, float(m))).expand(yd.shape)
    step = max(1, (1 << 27) // X.shape[0])
    Us, Gs = [], []
    for i in range(0, z.shape[0], step):
        zc = z[i:i + step].double().detach().requires_grad_(True)
        zero = torch.zeros((), dtype=zc.dtype, device=zc.device)
        w = zc[..., pot.sites["w"][0]]
        lp = od.normal(w, zero, zero + pot.s_w).sum(-1)
        bv = 0.0
        if pot.bias is not None:
            bv = zc[..., pot.sites["b"][0]]
            lp = lp + od.normal(bv, zero, zero + pot.s_b).sum(-1)
        u = -(lp + binomial_lp(yd, md, w @ Xd.T + bv).sum(-1))
        (g,) = torch.autograd.grad(u.sum(), zc)
        Us.append(u.detach())
        Gs.append(g)
    return torch.cat(Us), torch.cat(Gs)


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 20])
@pytest.mark.parametrize("n", [300, 1_000_000])
@pytest.mark.parametrize("bias", [True, False], ids=["b", "nob"])
def test_potential_against_fp64(bias, n, trials):
    """U and dU/dz for C = 1, 8, 130 chains against fp64 (U 2e-6 relative, the gradient 5e-4 of max |grad|),
    bitwise repeatable, four native launches per evaluation."""
    if EMULATE:
        pytest.skip("kernel test")
    D = 10
    X, y, m = _data(n, D, dev=DEV, seed=n, trials=trials)
    pot = _direct_potential(X, y, m, bias)
    for C in (1, 8, 130):
        g = torch.Generator(device=DEV).manual_seed(C)
        z = 0.1 * torch.randn(C, pot.dim, generator=g, device=DEV)
        c0 = N.launch_count()
        U, G = pot.value_and_grad(z)
        assert N.launch_count() - c0 == 4
        U2, G2 = pot.value_and_grad(z)
        assert torch.equal(U, U2) and torch.equal(G, G2)
        Ur, Gr = _oracle_value_and_grad(X, y, m, pot, z)
        eu = float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max())
        eg = float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max()))
        print("\nbinomial potential n=%d C=%d trials=%s: U %.1e grad %.1e" % (n, C, trials, eu, eg))
        assert eu <= 2e-6 and eg <= 5e-4, (C, eu, eg)


# ---- GPU tier: NUTS / HMC on the unchanged model ----------------------------------------------------------------
def _oracle_potential(X, y, m, pot):
    """fp64 U(z) on the host: -(Normal prior log densities + the Binomial log likelihood with logits X @ w + b)."""
    Xd, yd = X.double().cpu(), y.double().cpu()
    md = (m.double().cpu() if isinstance(m, torch.Tensor) else torch.full_like(yd, float(m))).expand(yd.shape)

    def U(z):
        zero = torch.zeros((), dtype=z.dtype)
        w = z[..., pot.sites["w"][0]]
        lp = od.normal(w, zero, zero + pot.s_w).sum(-1)
        bv = 0.0
        if pot.bias is not None:
            bv = z[..., pot.sites["b"][0]]
            lp = lp + od.normal(bv, zero, zero + pot.s_b).sum(-1)
        return -(lp + binomial_lp(yd, md, w @ Xd.T + bv).sum(-1))
    return U


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 20])
def test_hmc_trajectory_matches_oracle_integrator(trials):
    """Twenty leapfrog steps of HMC's integrator on GlmPotential against oracle.mcmc.velocity_verlet in fp64."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.0005
    X, y, m = _data(n, 32, dev=DEV, seed=11, trials=trials)
    pot = _direct_potential(X, y, m, True)
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    g0 = torch.Generator(device=DEV).manual_seed(12)
    z0 = 0.05 * torch.randn(C, pot.dim, device=DEV, generator=g0)
    r0 = torch.randn(C, pot.dim, device=DEV, generator=g0)
    z, r = z0.clone(), r0.clone()
    _, g = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, g, U, _ = kernel._leapfrog(z, r, g, epsv, minv)
    Uo = _oracle_potential(X, y, m, pot)
    errs = []
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        errs.append((float((z[c].double().cpu() - zr).abs().max()),
                     float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max())),
                     abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))))
    print("\nhmc trajectory Binomial trials=%s: (z err, r err, U err) %s" % (trials, ["%.1e %.1e %.1e" % e
                                                                                   for e in errs]))
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 20])
def test_nuts_binomial_model_posterior_matches_trace_potential(trials):
    """NUTS(binomial_model) at N = 10^4, D = 8, 8 chains: recognised (GlmPotential), and its posterior moments
    agree with a run on TracePotential (compile_model = False) of the same model: means within 0.3 posterior
    standard deviations, standard deviations within 25 %."""
    if EMULATE:
        pytest.skip("kernel test")
    D = 8
    X, y, m = _data(10_000, D, dev=DEV, seed=21, trials=trials)
    out = {}
    for compile_model in (True, False):
        kernel = NUTS(binomial_model)
        kernel.compile_model = compile_model
        mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1 if compile_model else 2)
        mc.run(X, y, m)
        want = GlmPotential if compile_model else TracePotential
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        s = mc.get_samples()
        out[compile_model] = torch.cat([s["w"].reshape(-1, D), s["b"].reshape(-1, 1)], -1).double().cpu()
    got, ref = out[True], out[False]
    m_, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    print("\nnuts Binomial trials=%s: max |mean diff| / sd %.2f, max |sd diff| / sd %.2f"
          % (trials, float(((m_ - rm).abs() / rs).max()), float(((sd - rs).abs() / rs).max())))
    assert bool(((m_ - rm).abs() <= 0.3 * rs).all()), float(((m_ - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


@pytest.mark.gpu
def test_routes_taken_by_nuts_model():
    """NUTS(model) picks GlmPotential for Binomial regression with per-row or constant counts, with or without an
    intercept, samples on it, and keeps TracePotential for the near misses."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, m = _data(9000, 33, dev=DEV, seed=1)
    Xc, yc, mc = _data(9000, 33, dev=DEV, seed=1, trials=10)
    for model, args, want in ((binomial_model, (X, y, m), GlmPotential),
                              (binomial_model, (Xc, yc, mc), GlmPotential),
                              (binomial_model_nobias, (X, y, m), GlmPotential),
                              (_variant("times2"), (X, y, m), TracePotential),
                              (_variant("probs"), (X, y, m), TracePotential),
                              (binomial_model, (X.double(), y.double(), m.double()), TracePotential)):
        kernel = NUTS(model)
        kernel.setup(5, 4, *args)
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        if want is GlmPotential:
            assert kernel.potential.binomial
            n0 = N.launch_count()
            kernel.sample()
            assert N.launch_count() - n0 > 0 and kernel.leapfrog_count() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("trials", ["rows", 15])
def test_bind_nuts_recognises_reference_pyro_binomial_model(trials):
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as ref_pyro
    import pyro.distributions as rdist
    from pyro.infer import MCMC as RefMCMC

    def model(X, y, m):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Binomial(m, logits=X @ w + b), obs=y)

    X, y, m = _data(4000, 12, dev=DEV, seed=1, trials=trials)
    pot = bind.recognise(model, (X, y, m), {}, poutine=ref_pyro.poutine)
    assert isinstance(pot, GlmPotential) and pot.binomial and pot.trials_per_row == (1 if trials == "rows" else 0)
    kernel = bind.NUTS(model, num_chains=4, seed=0)
    mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
    mc.run(X, y, m)
    assert isinstance(kernel._kernel.potential, GlmPotential)
    for v in mc.get_samples().values():
        assert bool(torch.isfinite(v).all())
