"""Poisson regression (log link) on the fused GLM path: `Poisson(rate = exp(X @ w + b))` scored by one pass of
`b2_glm_poisson_log_rate` (glm_poisson_tc.cu) under SVI, and `GlmPotential` of kind B2_GLM_POISSON under NUTS / HMC.

CPU tier: the lazy exp predictor (shape, dtype and value of the eager expression, bit for bit; every other use
materialises), the SASS of all ten kernel instantiations, the entry point's argument checks and the recognition
of the model by `NUTS(model)`.
GPU tier: the kernel against fp64 at full size and at ragged shapes, overflowing rates, the unchanged model
under SVI against the materialised path, out-of-scope sites, and GlmPotential against fp64, TracePotential,
the oracle integrator and the oracle NUTS sampler."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
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
# (atoms of 32 columns, split X) -> mangled-name fragment; D = 32 runs the TMA tile pipeline
KERNELS = {("flat", dc, sx): "glm_poisson_flat_tc_kernelILi%dELb%dE" % (dc, int(sx)) for dc in (1, 2, 3, 4)
           for sx in (False, True)}
KERNELS.update({("d32", 1, sx): "glm_poisson_tc_kernelILb%dE" % int(sx) for sx in (False, True)})
IDS = ["%s-DC%d-%s" % (k, dc, "split_x" if sx else "default") for k, dc, sx in sorted(KERNELS)]


# ---- models ------------------------------------------------------------------------------------------------
def poisson_model(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        l = w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b
        pyro.sample("y", dist.Poisson(torch.exp(l)), obs=y)


def poisson_model_nobias(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 0.5).to_event(1))
    with pyro.plate("data", X.shape[0]):
        l = w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w
        pyro.sample("y", dist.Poisson(l.exp()), obs=y)


def _variant(change):
    """poisson_model with one change: the near misses that must not be recognised."""
    def model(X, y):
        D = X.shape[-1]
        loc = X.new_full((D,), 0.5) if change == "loc" else X.new_zeros(D)
        scale = torch.linspace(0.5, 1.5, D, dtype=X.dtype) if change == "scale" else X.new_ones(D)
        w = pyro.sample("w", dist.Normal(loc, scale).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
        if change == "extra":
            pyro.sample("s", dist.Normal(X.new_zeros(()), 1.0))
        with pyro.plate("data", X.shape[0]):
            rate = torch.exp(w.squeeze(-2) @ X.T + b if w.dim() > 1 else X @ w + b)
            if change == "times2":
                rate = rate * 2
            d = dist.Poisson(rate)
            if change == "mask":
                d = d.mask(torch.ones(X.shape[0], dtype=torch.bool))
            if change == "scale_site":
                with poutine.scale(scale=2.0):
                    pyro.sample("y", d, obs=y)
            else:
                pyro.sample("y", d, obs=y)
    return model


def _data(n, D, dtype=torch.float32, dev="cpu", seed=0, level=0.5):
    """X [n, D], counts y drawn from the model with log-rates around `level`."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    X = torch.randn(n, D, generator=g, dtype=torch.float64)
    w = 0.3 * torch.randn(D, generator=g, dtype=torch.float64) / D ** 0.5
    y = torch.poisson(torch.exp(X @ w + level), generator=g)
    return X.to(dtype).to(dev), y.to(dtype).to(dev)


# ---- CPU tier: lazy semantics ----------------------------------------------------------------------------
def _lazy_mk():
    torch.manual_seed(0)
    X = torch.randn(50, 12)
    w = torch.randn(8, 1, 12, requires_grad=True)
    b = torch.randn(8, 1, requires_grad=True)
    return X, w, b


def test_exp_patterns_stay_lazy_and_match_eager_bitwise():
    X, w, b = _lazy_mk()
    ws, bs = SiteValue.wrap(w * 1.0), SiteValue.wrap(b * 1.0)
    w1, b1 = SiteValue.wrap(torch.randn(12)), SiteValue.wrap(torch.randn(()))
    pw1, pb1 = w1.as_subclass(torch.Tensor), b1.as_subclass(torch.Tensor)
    cases = [
        (torch.exp(ws.squeeze(-2) @ X.T + bs), torch.exp(w.squeeze(-2) @ X.T + b)),
        ((ws.squeeze(-2) @ X.T + bs).exp(), (w.squeeze(-2) @ X.T + b).exp()),
        ((ws.squeeze(-2) @ X.T).exp(), (w.squeeze(-2) @ X.T).exp()),
        (torch.exp(X @ w1 + b1), torch.exp(X @ pw1 + pb1)),
        ((X @ w1).exp(), (X @ pw1).exp()),
        (F.linear(X, w1).add(b1).exp(), F.linear(X, pw1).add(pb1).exp()),
        (F.linear(X, w1).exp(), F.linear(X, pw1).exp()),
    ]
    for i, (lz, ref) in enumerate(cases):
        assert isinstance(lz, LinearPredictorTensor) and isinstance(lz.lazy, dist.ExpLinearPredictor), i
        assert tuple(lz.shape) == tuple(ref.shape) and lz.dtype == ref.dtype, i
        assert torch.equal(lz.dense(), ref), i


def test_other_uses_of_exp_materialise_exactly():
    X, w, b = _lazy_mk()
    ws, bs = SiteValue.wrap(w * 1.0), SiteValue.wrap(b * 1.0)
    ref = torch.exp(w.squeeze(-2) @ X.T + b)
    rate = torch.exp(ws.squeeze(-2) @ X.T + bs)
    off = torch.randn(50)
    for got, want in ((rate + off, ref + off), (rate * 2, ref * 2), (rate + 1.0, ref + 1.0),
                      (rate.log(), ref.log()), (rate.sum(), ref.sum())):
        assert type(got) is torch.Tensor and torch.equal(got, want)
    # comparisons and finiteness checks look at the value: exp may underflow to 0 or overflow to inf
    w0 = torch.zeros(1, 1, 12)
    w0[..., 0] = 100.0
    X0 = torch.tensor([[-2.0] + [0.0] * 11, [-0.63] + [0.0] * 11, [0.72] + [0.0] * 11, [1.0] + [0.0] * 11])
    big = torch.exp(SiteValue.wrap(w0).squeeze(-2) @ X0.T)
    want = torch.exp(w0.squeeze(-2) @ X0.T)
    assert bool((want == 0).any()) and bool(torch.isinf(want).any())
    for got, exact in ((big == 0, want == 0), (big != 0, want != 0), (torch.isinf(big), torch.isinf(want)),
                       (torch.isfinite(big), torch.isfinite(want)), (torch.isnan(big), torch.isnan(want)),
                       (big.eq(0), want.eq(0)), (big.ne(0), want.ne(0))):
        assert torch.equal(got, exact)
    # autograd through the materialised value
    (rate * 2).sum().backward()
    gw, gb = torch.autograd.grad((ref * 2).sum(), [w, b])
    assert torch.allclose(w.grad, gw) and torch.allclose(b.grad, gb)


def test_exp_of_other_lazy_tensors_materialises():
    torch.manual_seed(1)
    X = torch.randn(40, 6)
    W = SiteValue.wrap(torch.randn(3, 6))
    cls = (X @ W.mT).exp()                                      # class logits
    assert type(cls) is torch.Tensor and torch.equal(cls, (X @ W.as_subclass(torch.Tensor).mT).exp())
    import pyro_b200.lazy as lazy
    saved = lazy._FACTOR_DEVICE_TYPES
    lazy._FACTOR_DEVICE_TYPES = ("cpu",)
    try:
        z, v = SiteValue.wrap(torch.rand(40, 4)), SiteValue.wrap(torch.rand(4, 5))
        fp = torch.matmul(z, v)
        assert isinstance(fp, LinearPredictorTensor)
        e = fp.exp()                                            # factor product
        assert type(e) is torch.Tensor
        assert torch.equal(e, torch.matmul(z.as_subclass(torch.Tensor), v.as_subclass(torch.Tensor)).exp())
    finally:
        lazy._FACTOR_DEVICE_TYPES = saved


def test_poisson_of_lazy_rate_is_fused_and_validation_keeps_it_lazy():
    X, w, b = _lazy_mk()
    rate = torch.exp(SiteValue.wrap(w * 1.0).squeeze(-2) @ X.T + SiteValue.wrap(b * 1.0))
    d = dist.Poisson(rate)
    assert type(d).__name__ == "_PoissonLinear" and tuple(d.batch_shape) == (8, 50)
    assert d._dense is None
    # the rate check of torch / reference Pyro (constraints.nonnegative) is answered without the dense value
    td = torch.distributions.Poisson(rate, validate_args=True)
    assert isinstance(td.__dict__["rate"], LinearPredictorTensor) and rate._dense is None
    assert bool(torch.distributions.constraints.nonnegative.check(rate).all()) and rate._dense is None
    y = torch.poisson(torch.ones(50))
    ref = torch.distributions.Poisson(torch.exp(w.squeeze(-2) @ X.T + b)).log_prob(y)
    assert torch.allclose(td.log_prob(y), ref, atol=1e-5)


# ---- CPU tier: SASS ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    from test_glm_tc_sass import _tools
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp("glm_poisson_sass") / "glm_poisson_tc.o")
    src = os.path.join(_build.CSRC, "glm_poisson_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _g2(key):
    return "64x%dx8" % (32 * key[1] + 8)


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
    _, dc, split_x = key
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
def test_one_ex2_per_logit_and_no_lg2_in_the_tile_loop(compiled, key):
    """The epilogue is one MUFU.EX2 per logit (32 per thread and tile); SUM lgamma(y + 1) is evaluated after
    the tile loop, so the loop takes no MUFU.LG2 at all."""
    from test_glm_flat import _opcode, _tile_loop
    from test_glm_tc_sass import _sass_function
    _, sass = compiled
    loop = _tile_loop(_sass_function(sass, KERNELS[key]), _g2(key))
    ops = [_opcode(l) for l in loop]
    assert ops.count("MUFU.EX2") >= 32, ops.count("MUFU.EX2")
    assert ops.count("MUFU.LG2") == 0, ops.count("MUFU.LG2")


# ---- CPU tier: argument checks -----------------------------------------------------------------------------
def test_entry_point_validates_arguments_before_any_cuda_call():
    """The pointers are never dereferenced and no workspace is passed: the checks come first."""
    L = N.lib()
    assert L.b2_version() == 104
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)

    def call(X, y, W, n, D, flags, ws=None, nbytes=0):
        return L.b2_glm_poisson_log_rate(X, y, W, None, n, D, 8, 1.0, 1.0, 1.0, flags, None, None, None, None,
                                         ws, nbytes, None)

    assert call(None, p, p, 10000, 10, 0) == -4                  # B2_ERR_NULL
    assert call(p, None, p, 10000, 10, 0) == -4
    assert call(p, p, None, 10000, 10, 0) == -4
    assert call(p, p, p, 0, 10, 0) == -2                         # B2_ERR_BAD_SHAPE
    assert call(p, p, p, -5, 10, 0) == -2
    for D in (0, -1, 129):
        assert call(p, p, p, 10000, D, 0) == -2, D
    assert call(q, p, p, 10000, 10, 0) == -2                     # X not 16-byte aligned
    assert call(p, q, p, 10000, 10, 0) == -2                     # y not 16-byte aligned
    assert call(p, p, p, 10000, 32, N.B2_FLAG_GLM_FP32) == -2    # no fp32 SIMT kernel
    assert call(p, p, p, 1 << 31, 10, 0) == -8                   # B2_ERR_TOO_LARGE
    for D in (1, 10, 32, 33, 128):                               # valid: the workspace check is next
        assert call(p, p, p, 10000, D, 0) == -5, D
        need = int(L.b2_glm_poisson_workspace(10000, D, 8))
        assert call(p, p, p, 10000, D, 0, p, need - 1) == -5, D


# ---- CPU tier: recognition ---------------------------------------------------------------------------------
def _recognised(model, *args):
    import cpu_emulation

    from pyro_b200.infer.mcmc.compile import recognise
    with cpu_emulation.enabled():
        return recognise(model, args)


@pytest.mark.parametrize("name", ["bias", "nobias"])
def test_recognises_poisson_regression(name):
    X, y = _data(300, 10)
    model = poisson_model if name == "bias" else poisson_model_nobias
    pot = _recognised(model, X, y)
    assert isinstance(pot, GlmPotential) and pot.kind == N.GLM_POISSON
    tp = TracePotential(model, (X, y))
    assert list(pot.sites) == list(tp.sites) and pot.dim == tp.dim
    for site, (sl, _, shape) in pot.sites.items():
        assert sl == tp.sites[site][0] and tuple(shape) == tp.sites[site][2], site
    if name == "bias":
        assert (pot.has_bias, pot.s_w, pot.s_b, pot.K) == (True, 1.0, 10.0, 1)
    else:
        assert (pot.has_bias, pot.s_w, pot.K) == (False, 0.5, 1)


@pytest.mark.parametrize("change", ["loc", "scale", "extra", "times2", "mask", "scale_site", "fp64"])
def test_near_misses_are_not_recognised(change):
    if change == "fp64":
        X, y = _data(300, 10, dtype=torch.float64)
        pot = _recognised(poisson_model, X, y)
    else:
        X, y = _data(300, 10)
        pot = _recognised(_variant(change), X, y)
    assert not isinstance(pot, GlmPotential), change


# ---- GPU tier: the kernel against fp64 ---------------------------------------------------------------------
def _launch(X, y, W, b, flags):
    n, D = X.shape
    P = W.shape[0]
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dW = torch.empty(P, D, device=DEV)
    db = torch.empty(P, device=DEV)
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_poisson_workspace(n, D, P)), tag="glm_poisson")
    N.check(N.lib().b2_glm_poisson_log_rate(X.data_ptr(), y.data_ptr(), W.data_ptr(),
                                            b.data_ptr() if b is not None else None, n, D, P, 1.0, 1.0, 1.0,
                                            flags, sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(),
                                            db.data_ptr(), ws.data_ptr(), ws.numel(),
                                            N.stream_ptr(torch.device(DEV))), "b2_glm_poisson_log_rate")
    torch.cuda.synchronize()
    return sum_p, total, dW, db


def _reference(X, y, W, b):
    """fp64 per-particle sums and their gradients by autograd through oracle/dists.py (on the device)."""
    Wd = W.double().requires_grad_(True)
    bd = (b if b is not None else torch.zeros(W.shape[0], device=W.device)).double().requires_grad_(True)
    s = od.poisson(y.double(), torch.exp(Wd @ X.double().t() + bd[:, None])).sum(1)
    gW, gb = torch.autograd.grad(s.sum(), [Wd, bd])
    return s.detach(), gW, gb


_FULL = {}


@pytest.mark.gpu
@pytest.mark.parametrize("flag_name", ["default", "B2_FLAG_GLM_3XTF32"])
@pytest.mark.parametrize("D,level", [(1, 0.5), (10, 0.5), (32, 0.5), (32, 4.6), (33, 0.5), (64, 0.5),
                                     (100, 4.6), (128, 0.5)])
def test_kernel_full_size_against_oracle(D, level, flag_name):
    """N = 1e6, P = 64: sums within 2e-5 relative, dW and db within 2e-4 of the largest gradient, and two
    launches bitwise equal.  level 4.6 draws counts with a mean around 100, where each row's lp is about +360
    before the lgamma term and about -3 after it, so a bias of the log-rate shows in the sum: the bias is added in
    the epilogue, not by the tensor cores' truncating accumulator (see poisson_epilogue)."""
    if EMULATE:
        pytest.skip("kernel test")
    n, P = 1_000_000, 64
    key = (D, level)
    if key not in _FULL:
        _FULL.clear()
        g = torch.Generator().manual_seed(200 + D)
        X = torch.randn(n, D, generator=g)
        wt = 0.3 * torch.randn(D, generator=g) / D ** 0.5
        y = torch.poisson(torch.exp(X @ wt + level), generator=g)
        W = 0.05 * torch.randn(P, D, generator=g) / D ** 0.5 + wt
        b = level + 0.05 * torch.randn(P, generator=g)
        Xg, yg, Wg, bg = X.to(DEV), y.to(DEV), W.to(DEV), b.to(DEV)
        _FULL[key] = (Xg, yg, Wg, bg) + _reference(Xg, yg, Wg, bg)
    Xg, yg, Wg, bg, s_ref, gW, gb = _FULL[key]
    flags = 0 if flag_name == "default" else getattr(N, flag_name)
    sum_p, total, dW, db = _launch(Xg, yg, Wg, bg, flags)
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    ew = float((dW.double() - gW).abs().max()) / float(gW.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    print("\npoisson D=%d level=%.1f %s: sum %.1e dW %.1e db %.1e" % (D, level, flag_name, es, ew, eb))
    assert es <= 2e-5 and ew <= 2e-4 and eb <= 2e-4, (es, ew, eb)
    assert abs(float(total) - float(s_ref.sum())) <= 2e-5 * abs(float(s_ref.sum()))
    sum2, total2, dW2, db2 = _launch(Xg, yg, Wg, bg, flags)
    assert torch.equal(sum_p, sum2) and torch.equal(total, total2)
    assert torch.equal(dW, dW2) and torch.equal(db, db2)


_RAGGED = [(n, P, D, bias) for n, P, D, bias in
           [(1, 1, 1, True), (63, 7, 32, False), (64, 65, 10, True), (65, 1, 33, False), (8191, 7, 100, True),
            (70001, 65, 32, True), (70001, 1, 127, False), (65, 65, 32, True), (1, 7, 32, False),
            (8191, 65, 3, False), (63, 1, 64, True), (70001, 7, 10, False)]]


@pytest.mark.gpu
@pytest.mark.parametrize("n,P,D,bias", _RAGGED, ids=["-".join(map(str, c)) for c in _RAGGED])
def test_kernel_ragged_shapes_against_oracle(n, P, D, bias):
    """Partial last tiles, a CTA's only tile, one and two particle slabs: sums within 2e-5, dW and db within
    5e-4 of the largest gradient.  A single row (n = 1) has nothing to average its two TF32 roundings (g and x,
    2^-11 relative each) over: measured 5.2e-4 at D = 1 on an H100, so below one full tile the bound is 1e-3 of
    the largest gradient."""
    if EMULATE:
        pytest.skip("kernel test")
    g = torch.Generator().manual_seed(7 * n + 3 * P + D)
    X = torch.randn(n, D, generator=g)
    y = torch.poisson(torch.full((n,), 2.0), generator=g)
    W = 0.3 * torch.randn(P, D, generator=g) / D ** 0.5
    b = 0.5 * torch.randn(P, generator=g) if bias else None
    Xg, yg, Wg = X.to(DEV), y.to(DEV), W.to(DEV)
    bg = b.to(DEV) if bias else None
    s_ref, gW, gb = _reference(Xg, yg, Wg, bg)
    sum_p, total, dW, db = _launch(Xg, yg, Wg, bg, 0)
    tol_g = 5e-4 if n >= 64 else 1e-3
    assert float((sum_p.double() - s_ref).abs().max()) <= 2e-5 * max(1.0, float(s_ref.abs().max()))
    assert float((dW.double() - gW).abs().max()) <= tol_g * float(gW.abs().max())
    if bias:
        assert float((db.double() - gb).abs().max()) <= tol_g * float(gb.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 32])
def test_overflowing_rates(D):
    """A log-rate above 88.72 overflows exp to +inf.  The kernel then gives sum_p = -inf, db = -inf and a
    non-finite dW for that particle, without a fault, and leaves the other particles finite and correct.  The
    materialised path gives NaN for the sum (xlogy(y, inf) - inf at a positive count) and NaN gradients."""
    if EMULATE:
        pytest.skip("kernel test")
    n, P = 9000, 3
    g = torch.Generator().manual_seed(D)
    X = torch.randn(n, D, generator=g)
    y = torch.poisson(torch.full((n,), 3.0), generator=g)
    y[0] = 2.0
    W = 0.1 * torch.randn(P, D, generator=g)
    b = torch.tensor([1.0, 90.0, 1.0])                 # particle 1: every log-rate near 90
    Xg, yg, Wg, bg = X.to(DEV), y.to(DEV), W.to(DEV), b.to(DEV)
    sum_p, total, dW, db = _launch(Xg, yg, Wg, bg, 0)
    assert float(sum_p[1]) == float("-inf") and float(db[1]) == float("-inf")
    assert not bool(torch.isfinite(dW[1]).any())
    assert float(total) == float("-inf")
    s_ref, gW, gb = _reference(Xg, yg, Wg, bg)
    for p in (0, 2):
        assert abs(float(sum_p[p]) - float(s_ref[p])) <= 2e-5 * abs(float(s_ref[p]))
        assert float((dW[p].double() - gW[p]).abs().max()) <= 5e-4 * float(gW[p].abs().max())
    mat = torch.distributions.Poisson(torch.exp(Wg @ Xg.T + bg[:, None])).log_prob(yg).sum(1)
    assert bool(torch.isnan(mat[1]))


# ---- GPU tier: the unchanged model under SVI ---------------------------------------------------------------
def poisson_guide(X, y):
    D = X.shape[-1]
    w_loc = pyro.param("w_loc", X.new_zeros(D))
    w_scale = pyro.param("w_scale", X.new_full((D,), 0.1), constraint=dist.constraints.positive)
    b_loc = pyro.param("b_loc", X.new_zeros(()))
    b_scale = pyro.param("b_scale", X.new_full((), 0.1), constraint=dist.constraints.positive)
    pyro.sample("w", dist.Normal(w_loc, w_scale).to_event(1))
    pyro.sample("b", dist.Normal(b_loc, b_scale))


def poisson_model_masked(X, y, mask):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Poisson(torch.exp(w.squeeze(-2) @ X.T + b)).mask(mask), obs=y)


def poisson_model_offset(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Poisson(torch.exp(w.squeeze(-2) @ X.T + b) + 0.5), obs=y)


def poisson_model_simt(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Poisson(dist.ExpLinearPredictor(dist.LinearPredictor(X, w, b, tensor_cores=False))),
                    obs=y)


def poisson_model_simt_eager(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        rate = torch.exp(dist.LinearPredictor(X, w, b).dense())
        pyro.sample("y", dist.Poisson(rate), obs=y)


def _run(model, X, y, eps_w, eps_b, lazy, elbo_cls=Trace_ELBO, extra=()):
    """SVI steps with the guide's noise injected through fixed device buffers; returns the losses, the
    parameters and the number of kernel calls."""
    import models
    pyro.clear_param_store()
    bw, bb = torch.empty_like(eps_w[0]), torch.empty_like(eps_b[0])
    calls = []
    real = dist._GlmPoissonFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)

    def guide(*args):
        with models.InjectNoise({"w": bw, "b": bb}):
            poisson_guide(*args[:2])

    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    dist._GlmPoissonFn.apply = spy
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  elbo_cls(num_particles=eps_w.shape[1], vectorize_particles=True, max_plate_nesting=1))
        losses = []
        for i in range(eps_w.shape[0]):
            bw.copy_(eps_w[i])
            bb.copy_(eps_b[i])
            losses.append(svi.step(X, y, *extra))
    finally:
        elbo_mod.LAZY_LINEAR = saved
        dist._GlmPoissonFn.apply = real
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in ("w_loc", "w_scale", "b_loc", "b_scale")}, len(calls)


def _svi_data(n, D, P, steps, seed, dtype=torch.float32):
    X, y = _data(n, D, dtype=dtype, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    eps_w = torch.randn(steps, P, 1, D, generator=g, dtype=dtype)
    eps_b = torch.randn(steps, P, 1, generator=g, dtype=dtype)
    return X, y, eps_w, eps_b


@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 32, 100])
def test_unchanged_model_under_svi_matches_materialised(D):
    """The Poisson model at N = 70 000, 16 vectorised particles: every step's site goes through the kernel, and
    three steps match LAZY_LINEAR = False (loss 2e-5 relative, parameters 2e-4)."""
    if EMULATE:
        pytest.skip("kernel test")
    X, y, ew, eb = _svi_data(70000, D, 16, 3, D)
    X, y, ew, eb = X.to(DEV), y.to(DEV), ew.to(DEV), eb.to(DEV)
    dense_calls = []
    real_dense = dist.ExpLinearPredictor.dense

    def spy(self):
        dense_calls.append(1)
        return real_dense(self)
    dist.ExpLinearPredictor.dense = spy
    try:
        l_f, p_f, calls = _run(poisson_model, X, y, ew, eb, True)
    finally:
        dist.ExpLinearPredictor.dense = real_dense
    assert calls == 3 and not dense_calls       # every site on the kernel, the [P, N] rate never materialised
    l_m, p_m, calls_m = _run(poisson_model, X, y, ew, eb, False)
    assert calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_captured_graph_step_equals_eager():
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, y, ew, eb = _svi_data(70000, 32, 16, 4, 5)
    X, y, ew, eb = X.to(DEV), y.to(DEV), ew.to(DEV), eb.to(DEV)
    l_e, p_e, n_e = _run(poisson_model, X, y, ew, eb, True)
    l_g, p_g, n_g = _run(poisson_model, X, y, ew, eb, True, JitTrace_ELBO)
    assert n_e == 4 and n_g >= 3
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["N8191", "masked", "fp64", "y_offset1", "D129", "no_tensor_cores", "offset"])
def test_out_of_scope_sites_keep_the_materialised_path(case):
    if EMULATE:
        pytest.skip("kernel test")
    n, D, P = 9000, 10, 4
    dtype = torch.float64 if case == "fp64" else torch.float32
    if case == "D129":
        D = 129
    if case == "N8191":
        n = 8191
    X, y, ew, eb = _svi_data(n, D, P, 2, 31, dtype)
    X, y, ew, eb = X.to(DEV), y.to(DEV), ew.to(DEV), eb.to(DEV)
    model, model_m, extra = poisson_model, poisson_model, ()
    if case == "masked":
        model = model_m = poisson_model_masked
        extra = (torch.rand(n, device=DEV) < 0.7,)
    if case == "y_offset1":
        y = torch.cat([torch.zeros(1, device=DEV), y])[1:]
        assert y.data_ptr() % 16 != 0
    if case == "no_tensor_cores":
        model, model_m = poisson_model_simt, poisson_model_simt_eager
    if case == "offset":
        model = model_m = poisson_model_offset
    l_f, p_f, calls = _run(model, X, y, ew, eb, True, extra=extra)
    assert calls == 0
    l_m, p_m, _ = _run(model_m, X, y, ew, eb, False, extra=extra)
    tol = 1e-12 if dtype == torch.float64 else 2e-6
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= tol * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=tol, rtol=tol), k


# ---- GPU tier: GlmPotential --------------------------------------------------------------------------------
def _direct_potential(X, y, bias):
    D = X.shape[1]
    sites = {"w": (slice(0, D), "identity", (D,))}
    if bias:
        sites["b"] = (slice(D, D + 1), "identity", ())
    return GlmPotential(X, y, "Poisson", sites, "w", "b" if bias else None, s_w=1.0, s_b=10.0)


def _oracle_potential(X, y, pot):
    """fp64 U(z): -(Normal prior log densities + the Poisson log likelihood with log-rate X @ w + b)."""
    Xd, yd = X.double(), y.double()

    def U(z):
        zero = torch.zeros((), dtype=z.dtype, device=z.device)
        w = z[..., pot.sites[pot.weight][0]]
        lp = od.normal(w, zero, zero + pot.s_w).sum(-1)
        bv = 0.0
        if pot.bias is not None:
            bv = z[..., pot.sites[pot.bias][0]]
            lp = lp + od.normal(bv, zero, zero + pot.s_b).sum(-1)
        return -(lp + od.poisson(yd, torch.exp(w @ Xd.T + bv)).sum(-1))
    return U


def _trace_model(bias):
    def model(X, y):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0))) if bias else 0.0
        with pyro.plate("data", X.shape[0]):
            pyro.sample("y", dist.Poisson(torch.exp((w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w) + b)), obs=y)
    return model


def _oracle_value_and_grad(U, z, n):
    step = max(1, (1 << 27) // n)
    Us, Gs = [], []
    for i in range(0, z.shape[0], step):
        zc = z[i:i + step].double().detach().requires_grad_(True)
        u = U(zc)
        (g,) = torch.autograd.grad(u.sum(), zc)
        Us.append(u.detach())
        Gs.append(g)
    return torch.cat(Us), torch.cat(Gs)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [300, 8192, 70001, 1_000_000])
@pytest.mark.parametrize("bias", [True, False], ids=["b", "nob"])
def test_potential_against_fp64_and_trace(bias, n):
    """U and dU/dz for C = 1, 7, 64, 130 chains against fp64 (U 2e-6 relative, the gradient 2e-4 of max |grad|
    at N = 1e6 with up to 64 chains and 5e-4 otherwise), bitwise repeatable, and against TracePotential."""
    if EMULATE:
        pytest.skip("kernel test")
    D = 10
    X, y = _data(n, D, dev=DEV, seed=n)
    pot = _direct_potential(X, y, bias)
    U_ref_fn = _oracle_potential(X, y, pot)
    errs = []
    for C in (1, 7, 64, 130):
        g = torch.Generator(device=DEV).manual_seed(C)
        z = 0.1 * torch.randn(C, pot.dim, generator=g, device=DEV)
        U, G = pot.value_and_grad(z)
        U2, G2 = pot.value_and_grad(z)
        assert torch.equal(U, U2) and torch.equal(G, G2)
        Ur, Gr = _oracle_value_and_grad(U_ref_fn, z, n)
        eu = float(((U.double() - Ur).abs() / Ur.abs().clamp(min=1.0)).max())
        eg = float((G.double() - Gr).abs().max()) / max(1.0, float(Gr.abs().max()))
        et = gt = 0.0
        if C * n <= 64 * 70001 * 16:
            tp = TracePotential(_trace_model(bias), (X, y), num_chains=C)
            assert list(tp.sites) == list(pot.sites) and tp.dim == pot.dim
            Ut, Gt = tp.value_and_grad(z)
            et = float(((U - Ut).abs() / Ut.abs().clamp(min=1.0)).max())
            gt = float((G - Gt).abs().max()) / max(1.0, float(Gt.abs().max()))
        errs.append((C, eu, eg, et, gt))
    print("\nglm potential Poisson bias=%d n=%d: (C, U vs fp64, grad vs fp64, U vs trace, grad vs trace) %s"
          % (bias, n, ["%d %.1e %.1e %.1e %.1e" % e for e in errs]))
    for C, eu, eg, et, gt in errs:
        gtol = 2e-4 if n == 1_000_000 and C <= 64 else 5e-4
        assert eu <= 2e-6 and eg <= gtol, (C, eu, eg)
        assert et <= 2e-6 and gt <= 5e-4, (C, et, gt)


@pytest.mark.gpu
def test_captured_graph_replay_equals_eager():
    if EMULATE:
        pytest.skip("needs CUDA graphs")
    X, y = _data(70001, 33, dev=DEV, seed=3)
    pot = _direct_potential(X, y, True)
    z = 0.1 * torch.randn(64, pot.dim, device=DEV)
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
    """Twenty leapfrog steps of HMC's integrator on GlmPotential against oracle.mcmc.velocity_verlet."""
    if EMULATE:
        pytest.skip("kernel test")
    n, C, L, eps = 8192, 4, 20, 0.002
    X, y = _data(n, 32, dev=DEV, seed=11)
    pot = _direct_potential(X, y, True)
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = 0.05 * torch.randn(C, pot.dim, device=DEV)
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
    print("\nhmc trajectory Poisson: (z err, r err, U err) %s" % ["%.1e %.1e %.1e" % e for e in errs])
    for ez, er, eu in errs:
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


@pytest.mark.gpu
def test_nuts_poisson_model_posterior():
    """NUTS(poisson_model) at N = 10^4, D = 8, 8 chains, on GlmPotential, against the oracle sampler: means
    within 0.3 posterior standard deviations, standard deviations within 25 %."""
    if EMULATE:
        pytest.skip("kernel test")
    D = 8
    X, y = _data(10_000, D, dev=DEV, seed=21)
    kernel = NUTS(poisson_model)
    mc = MCMC(kernel, num_samples=250, warmup_steps=200, num_chains=8, seed=1)
    mc.run(X, y)
    assert isinstance(kernel.potential, GlmPotential) and kernel.potential.kind == N.GLM_POISSON
    s = mc.get_samples()
    got = torch.cat([s["w"].reshape(-1, D), s["b"].reshape(-1, 1)], -1).double().cpu()
    chain = omcmc.NUTSChain(_oracle_potential(X.cpu(), y.cpu(), kernel.potential), D + 1, seed=2)
    ref, _ = chain.run(torch.zeros(D + 1, dtype=torch.float64), 200, 800)
    m, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    assert bool(((m - rm).abs() <= 0.3 * rs).all()), float(((m - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


@pytest.mark.gpu
def test_routes_taken_by_nuts_model():
    if EMULATE:
        pytest.skip("kernel test")
    X, y = _data(9000, 33, dev=DEV, seed=1)
    for model, args, want in ((poisson_model, (X, y), GlmPotential),
                              (poisson_model_nobias, (X, y), GlmPotential),
                              (_variant("times2"), (X, y), TracePotential),
                              (poisson_model, (X.double(), y.double()), TracePotential)):
        kernel = NUTS(model)
        kernel.setup(5, 4, *args)
        assert type(kernel.potential) is want, (type(kernel.potential).__name__)
        if want is GlmPotential:
            n0 = N.launch_count()
            kernel.sample()
            assert N.launch_count() - n0 > 0 and kernel.leapfrog_count() > 0


@pytest.mark.gpu
def test_bind_nuts_recognises_reference_pyro_poisson_model():
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as ref_pyro
    import pyro.distributions as rdist
    from pyro.infer import MCMC as RefMCMC

    def model(X, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Poisson(torch.exp(X @ w + b)), obs=y)

    X, y = _data(4000, 12, dev=DEV, seed=1)
    assert isinstance(bind.recognise(model, (X, y), {}, poutine=ref_pyro.poutine), GlmPotential)
    kernel = bind.NUTS(model, num_chains=4, seed=0)
    mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
    mc.run(X, y)
    assert isinstance(kernel._kernel.potential, GlmPotential)
    for v in mc.get_samples().values():
        assert bool(torch.isfinite(v).all())
