"""Fused Poisson matrix factorisation: ``Poisson(rate = z @ w)`` with both factors latent, scored by the wgmma
kernel of poisson_product_tc.cu (``b2_poisson_product``).

CPU tier: the lazy factor-product patterns of pyro_b200/lazy.py (shape, dtype and values equal the eager
expression, and the near misses stay eager), what ptxas makes of the kernel, and argument validation.  GPU
tier: the kernel against fp64 at full size and at ragged shapes, the rate == 0 edge against the generic
Poisson kernel, determinism and graph replay, and the unchanged sparse gamma DEF reaching the kernel under
TraceMeanField_ELBO and Trace_ELBO, eager and graph-captured."""
import ctypes
import math
import os
import re
import subprocess

import pytest
import torch

import models
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from pyro_b200 import _build, lazy
from pyro_b200 import _native as N
from pyro_b200.infer import SVI, Trace_ELBO, TraceMeanField_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.lazy import LinearPredictorTensor, SiteValue
from pyro_b200.optim import AdagradRMSProp

S = SiteValue.wrap


def _factor(t):
    return isinstance(t, LinearPredictorTensor) and isinstance(t.lazy, dist.FactorProduct)


# ---- CPU tier: lazy semantics ------------------------------------------------------------------------------
@pytest.fixture
def cpu_factors(monkeypatch):
    """Let products of CPU site values stay lazy, so the patterns can be checked without a GPU."""
    monkeypatch.setattr(lazy, "_FACTOR_DEVICE_TYPES", ("cuda", "cpu"))


def _recognised_cases():
    torch.manual_seed(0)
    P, n, K, J = 3, 7, 5, 12
    z2, w2 = torch.rand(n, K), torch.rand(K, J)
    z3, w3 = torch.rand(P, n, K), torch.rand(P, K, J)
    wflat = torch.rand(P, K * J)
    z1, w1 = torch.rand(1, n, K), torch.rand(1, K, J)
    return [
        ("z@w", lambda: S(z2) @ S(w2), lambda: z2 @ w2),
        ("matmul(z,w)", lambda: torch.matmul(S(z2), S(w2)), lambda: torch.matmul(z2, w2)),
        ("z3@w3", lambda: S(z3) @ S(w3), lambda: z3 @ w3),
        ("matmul(z3,w3)", lambda: torch.matmul(S(z3), S(w3)), lambda: torch.matmul(z3, w3)),
        ("bmm(z3,w3)", lambda: torch.bmm(S(z3), S(w3)), lambda: torch.bmm(z3, w3)),
        ("z3@w.reshape", lambda: torch.matmul(S(z3), S(wflat).reshape(-1, K, J)),
         lambda: torch.matmul(z3, wflat.reshape(-1, K, J))),
        ("P=1", lambda: torch.matmul(S(z1), S(w1)), lambda: torch.matmul(z1, w1)),
        ("K=16", lambda: S(torch.rand(n, 16)) @ S(torch.rand(16, J)), None),
        ("K=1", lambda: S(torch.rand(P, n, 1)) @ S(torch.rand(P, 1, J)), None),
    ]


@pytest.mark.parametrize("case", _recognised_cases(), ids=lambda c: c[0])
def test_factor_product_patterns_stay_lazy(cpu_factors, case):
    _, lazy_fn, eager_fn = case
    out = lazy_fn()
    assert _factor(out), type(out)
    lz = out.lazy
    ref = eager_fn() if eager_fn is not None else torch.matmul(lz.A, lz.B)
    assert out.shape == ref.shape and out.dtype == ref.dtype
    assert torch.equal(out.dense(), ref)


def _excluded_cases():
    torch.manual_seed(1)
    P, n, K, J = 3, 7, 5, 12
    return [
        ("fp64", lambda: S(torch.rand(n, K, dtype=torch.float64)) @ S(torch.rand(K, J, dtype=torch.float64))),
        ("K=17", lambda: S(torch.rand(n, 17)) @ S(torch.rand(17, J))),
        ("data operand", lambda: S(torch.rand(n, K)) @ torch.rand(K, J)),
        ("data operand 3-d", lambda: torch.matmul(S(torch.rand(P, n, K)), torch.rand(P, K, J))),
        ("mismatched P", lambda: torch.matmul(S(torch.rand(1, n, K)), S(torch.rand(P, K, J)))),
        ("broadcast [N,K]@[P,K,J]", lambda: torch.matmul(S(torch.rand(n, K)), S(torch.rand(P, K, J)))),
        ("bmm of 2-d", lambda: S(torch.rand(P, n, K)) @ S(torch.rand(K, J))),
    ]


@pytest.mark.parametrize("case", _excluded_cases(), ids=lambda c: c[0])
def test_factor_product_near_misses_stay_eager(cpu_factors, case):
    out = case[1]()
    assert isinstance(out, torch.Tensor) and not isinstance(out, LinearPredictorTensor), type(out)


def test_cpu_factor_products_stay_eager():
    """Without the widening fixture a product of CPU site values is computed eagerly: the kernel is CUDA only."""
    z, w = torch.rand(4, 3), torch.rand(3, 8)
    out = S(z) @ S(w)
    assert not isinstance(out, LinearPredictorTensor)
    assert torch.equal(out.as_subclass(torch.Tensor), z @ w)


def test_other_uses_materialise(cpu_factors):
    torch.manual_seed(2)
    z, w, t = torch.rand(2, 6, 4), torch.rand(2, 4, 8), torch.rand(2, 6, 8) + 0.5
    lazy_rate = S(z) @ S(w)
    assert _factor(lazy_rate)
    assert lazy_rate._with_bias(t) is None
    for got, ref in ((lazy_rate + t, z @ w + t), (t + lazy_rate, t + z @ w), (lazy_rate / t, (z @ w) / t),
                     (t / lazy_rate, t / (z @ w)), (lazy_rate.sum(-1), (z @ w).sum(-1))):
        assert not isinstance(got, LinearPredictorTensor)
        assert torch.equal(got.as_subclass(torch.Tensor), ref)


@pytest.mark.parametrize("shapes", [((3, 6, 4), (4, 8)), ((6, 4), (3, 4, 8)), ((2, 6, 4), (3, 4, 8)),
                                    ((6, 4), (5, 8)), ((3, 6, 4), (3, 5, 8)), ((6, 4, 1, 1), (1, 1, 4, 8))],
                         ids=["shared B", "shared A", "P mismatch", "K mismatch", "K mismatch 3-d", "4-d"])
def test_factor_product_rejects_mismatched_factors(shapes):
    """A FactorProduct is [N, K] @ [K, J] or [P, N, K] @ [P, K, J]; anything else, which the kernel would read
    out of bounds, is refused when it is built."""
    with pytest.raises(ValueError, match="FactorProduct"):
        dist.FactorProduct(torch.rand(shapes[0]), torch.rand(shapes[1]))
    with pytest.raises(ValueError, match="FactorProduct"):
        dist.FactorProduct(torch.rand(6, 4), torch.rand(4, 8, dtype=torch.float64))


def test_poisson_of_factor_product_builds_fused_subclass(cpu_factors):
    z, w = torch.rand(2, 6, 4), torch.rand(2, 4, 8)
    d = dist.Poisson(S(z) @ S(w))
    assert type(d).__name__ == "_PoissonProduct" and d.batch_shape == (2, 6, 8)
    assert torch.equal(d.rate, z @ w)
    e = d.to_event(1).expand((2, 6))
    assert type(e.base_dist).__name__ == "_PoissonProduct" and e.event_shape == (8,)
    assert type(dist.Poisson(z @ w)) is dist.Poisson


# ---- CPU tier: compiled kernel and argument validation ------------------------------------------------------
KERNEL = "poisson_product_tc_kernel"


def test_kernel_compiles_without_spills_or_serialisation(tmp_path):
    from test_glm_tc_sass import _ptxas_properties, _sass_function, _tools
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path / "poisson_product_tc.o")
    src = os.path.join(_build.CSRC, "poisson_product_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert "C7515" not in log and "C7520" not in log, log
    props, used = _ptxas_properties(log, KERNEL)
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    body = _sass_function(sass, KERNEL)
    shapes = [m.group(1) for m in (re.search(r"HGMMA\.(\d+x\d+x\d+)", l) for l in body) if m]
    # GEMM 1: 2 k-steps x 3 split products; GEMM 2 and GEMM 3: 8 k-steps x 3 split products each
    assert shapes.count("64x64x8") == 6 and shapes.count("64x16x8") == 48, shapes
    # each contraction is one chain: no warpgroup wait or arrive between two HGMMA of one shape
    prev, between, bad = None, [], []
    for line in body:
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            if m.group(1) == prev and between:
                bad.append(between)
            prev, between = m.group(1), []
        elif "WARPGROUP" in line and prev is not None:
            between.append(line.split("*/", 1)[1].strip())
    assert not bad, bad


def test_entry_point_validates_before_launching():
    L = N.lib()
    assert L.b2_version() == 104
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)

    def call(A, B, x, n, K, J, P):
        return L.b2_poisson_product(A, B, x, n, K, J, P, 1.0, 1.0, 1.0, 0, None, None, None, None, None, 0, None)

    assert call(None, p, p, 320, 15, 4096, 4) == -4
    assert call(p, None, p, 320, 15, 4096, 4) == -4
    assert call(p, p, None, 320, 15, 4096, 4) == -4
    for n, K, J, P in ((320, 0, 4096, 4), (320, 17, 4096, 4), (0, 15, 4096, 4), (320, 15, 4094, 4),
                       (320, 15, 0, 4), (320, 15, 4096, 0), (-1, 15, 4096, 4), (320, 15, 4096, 70000)):
        assert call(p, p, p, n, K, J, P) == -2, (n, K, J, P)
    # a valid shape without a workspace is refused before any launch
    assert call(p, p, p, 320, 15, 4096, 4) == -5
    assert L.b2_poisson_product_workspace(320, 15, 4096, 256) > 256 + 256 * 320 * 15 * 4


# ---- GPU tier -------------------------------------------------------------------------------------------------
def _gamma(shape, conc, rate, gen):
    """Gamma(conc, rate) draws from ``gen`` (the inputs are fixed by the test's seed, whatever ran before)."""
    return torch._standard_gamma(torch.full(shape, float(conc)), generator=gen) / rate


def _counts(n, J, gen, dev):
    rate = _gamma((n, J), 0.5, 0.5, gen) * 2.0
    x = torch.poisson(rate, generator=gen)
    big = torch.rand(n, J, generator=gen) < 0.002
    x[big] = torch.randint(50, 400, (int(big.sum()),), generator=gen).float()
    return x.to(dev)


def _factors(P, n, K, J, gen, dev):
    A = _gamma((P, n, K), 0.3, 0.3, gen)
    B = _gamma((P, K, J), 0.3, 0.3, gen)
    A[..., 0, :] *= 1e-4           # tiny rates
    return A.to(dev), B.to(dev)


def _ref64(A, B, x):
    """fp64 sum_p, dA, dB of the formulas (torch autograd on xlogy(x, rate) - rate - lgamma(x + 1))."""
    A64 = A.double().requires_grad_()
    B64 = B.double().requires_grad_()
    rate = A64 @ B64
    x64 = x.double()
    lp = torch.xlogy(x64, rate) - rate - torch.lgamma(x64 + 1)
    sp = lp.sum((-1, -2))
    sp.sum().backward()
    return sp.detach(), A64.grad, B64.grad


def _run(A, B, x, scale=1.0, weight=1.0, coeff=1.0, flags=0, total=None):
    P, n, K = A.shape
    J = B.shape[-1]
    dev = A.device
    sum_p = torch.empty(P, device=dev)
    total = torch.zeros((), device=dev) if total is None else total
    dA, dB = torch.empty_like(A), torch.empty_like(B)
    ws = N.workspace(torch.device(dev), int(N.lib().b2_poisson_product_workspace(n, K, J, P)), tag="glm")
    N.check(N.lib().b2_poisson_product(A.data_ptr(), B.data_ptr(), x.data_ptr(), n, K, J, P, scale, weight, coeff,
                                       flags, sum_p.data_ptr(), total.data_ptr(), dA.data_ptr(), dB.data_ptr(),
                                       ws.data_ptr(), ws.numel(), N.stream_ptr(torch.device(dev))),
            "b2_poisson_product")
    return sum_p, total, dA, dB


# measured on the H100: sum_p within 8.4e-7 relative, dA within 1.5e-6 and dB within 5.5e-6 of the
# particle's largest gradient at P = 256, N = 320, K = 15, J = 4096; with one TF32-rounded operand in the
# gradient contractions dA and dB were off by 2-6e-4, which GRAD_TOL must catch
SUM_TOL, GRAD_TOL = 2e-6, 2e-5


def _check(A, B, x, got, scale=1.0, weight=1.0):
    sum_p, _, dA, dB = got
    rs, rA, rB = _ref64(A, B, x)
    rel = ((sum_p.double() - scale * rs).abs() / (scale * rs).abs().clamp_min(1e-30)).max().item()
    assert rel <= SUM_TOL, rel
    for g, r in ((dA, rA), (dB, rB)):
        r = weight * scale * r
        tol = GRAD_TOL * r.abs().flatten(1).amax(1).clamp_min(1e-30)
        err = (g.double() - r).abs().flatten(1).amax(1)
        assert (err <= tol).all(), (err / tol).max().item()


@pytest.mark.gpu
def test_kernel_matches_fp64_full_size():
    gen = torch.Generator().manual_seed(0)
    P, n, K, J = 256, 320, 15, 4096
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    got = _run(A, B, x)
    # the fp64 reference in slices of particles (a [256, 320, 4096] fp64 graph would take 10 GB)
    for s in range(0, P, 32):
        _check(A[s:s + 32], B[s:s + 32], x, tuple(t[s:s + 32] if t.dim() else t for t in got))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 65, 320])
@pytest.mark.parametrize("J", [4, 260, 4096])
@pytest.mark.parametrize("K", [1, 2, 8, 15, 16])
@pytest.mark.parametrize("P", [1, 3])
def test_kernel_matches_fp64_ragged(n, J, K, P):
    gen = torch.Generator().manual_seed(n * 7 + J + K * 13 + P)
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    _check(A, B, x, _run(A, B, x))


def _blocks_per_cta(J, P):
    """J blocks of 64 columns per CTA, as poisson_product_tc.cu chooses them (two waves of 3 CTAs per SM, <= 8)."""
    nb = (J + 63) // 64
    return nb, max(1, min(8, P * nb // (2 * 3 * 132)))


@pytest.mark.gpu
@pytest.mark.parametrize("P,n,K,J", [(64, 65, 15, 4228), (40, 65, 3, 4100), (64, 1, 16, 4228), (256, 130, 15, 1028)])
def test_kernel_matches_fp64_several_blocks_per_cta(P, n, K, J):
    """CTAs that walk several J blocks (the dA partial re-read and added) and whose last block lies past J."""
    nb, S = _blocks_per_cta(J, P)
    assert S > 1 and nb % S != 0, (nb, S)
    gen = torch.Generator().manual_seed(P + n + K + J)
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    got = _run(A, B, x)
    for s in range(0, P, 64):
        _check(A[s:s + 64], B[s:s + 64], x, tuple(t[s:s + 64] if t.dim() else t for t in got))


@pytest.mark.gpu
def test_scale_weight_coeff_and_accumulate():
    gen = torch.Generator().manual_seed(5)
    P, n, K, J = 3, 65, 15, 260
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    got = _run(A, B, x, scale=0.25, weight=-1.5, coeff=3.0)
    _check(A, B, x, got, scale=0.25, weight=-1.5)
    sum_p, total = got[0], got[1]
    assert torch.allclose(total.double(), 3.0 * sum_p.double().sum(), rtol=1e-6)
    acc = torch.full((), 10.0, device="cuda")
    _run(A, B, x, scale=0.25, coeff=3.0, flags=N.B2_FLAG_ACCUMULATE_SUM, total=acc)
    assert torch.allclose(acc.double(), 10.0 + 3.0 * sum_p.double().sum(), rtol=1e-6)


@pytest.mark.gpu
def test_deterministic_and_graph_replay():
    gen = torch.Generator().manual_seed(6)
    P, n, K, J = 32, 320, 15, 4096
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    first = _run(A, B, x)
    second = _run(A, B, x)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    out = [torch.empty_like(t) for t in first]
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            res = _run(A, B, x)
            for o, r in zip(out, res):
                o.copy_(r)
    torch.cuda.current_stream().wait_stream(s)
    for o in out:
        o.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(first, out):
        assert torch.equal(a, b)


def _site_sum(rate, x):
    """The observation site's fused sum and its factor gradients, through Poisson(rate).to_event(1)."""
    return dist.Poisson(rate).to_event(1)._fused_sum(x, None, 1.0, 1.0, 1.0, True)


def _both_paths(A, B, x):
    """(value, dA, dB) of the observation site on the fused path and on the generic Poisson kernel."""
    out = []
    for use_lazy in (True, False):
        a, b = A.clone().requires_grad_(), B.clone().requires_grad_()
        rate = SiteValue.wrap(a) @ SiteValue.wrap(b) if use_lazy else a @ b
        assert _factor(rate) == use_lazy
        tot = _site_sum(rate, x)
        tot.backward()
        out.append((tot.item(), a.grad, b.grad))
    return out


def _same_edges(fused, generic):
    """Non-finite in the same entries; NaN wherever the generic path has NaN (an entry it gives as +-inf may be
    NaN on the fused path: a split product multiplies inf by a factor's zero low part); finite entries close."""
    for f, g in zip(fused, generic):
        assert torch.equal(torch.isfinite(f), torch.isfinite(g))
        assert not (torch.isnan(g) & ~torch.isnan(f)).any()
        inf = torch.isinf(g)
        assert (torch.isnan(f[inf]) | (f[inf] == g[inf])).all()
        fin = torch.isfinite(g)
        if fin.any():
            assert torch.allclose(f[fin], g[fin], rtol=1e-3, atol=1e-3 * g[fin].abs().max().item())


@pytest.mark.gpu
def test_zero_rate_edge_equals_generic_poisson_kernel():
    """rate == 0 with x == 0 (lp 0, G NaN) and with x > 0 (lp -inf, G +inf): the value equals the generic
    Poisson site kernel's, and so does which factor gradients are non-finite."""
    gen = torch.Generator().manual_seed(7)
    P, n, K, J = 2, 65, 8, 260
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    A[0, 3] = 0.0                  # row 3 of particle 0: rate 0 everywhere
    x[3] = 0.0                     # ... with x == 0: finite value, NaN gradient
    A[1, 5] = 0.0
    x[5, 7] = 2.0                  # row 5 of particle 1 has one x > 0 at rate 0: -inf
    fused, generic = _both_paths(A, B, x)
    assert fused[0] == generic[0] == float("-inf")
    _same_edges(fused[1:], generic[1:])
    # particle 0 alone (x == 0 at rate 0): finite value, NaN gradient in both paths
    fused, generic = _both_paths(A[:1], B[:1], x)
    assert math.isfinite(fused[0]) and abs(fused[0] - generic[0]) <= SUM_TOL * abs(generic[0])
    assert torch.isnan(fused[1][0, 3]).all()


@pytest.mark.gpu
def test_zero_rate_column_with_positive_counts():
    """A zero column of B with x > 0 in every row of it: G = +inf down the column and nowhere x == 0, so dB of
    that column is +inf on the generic path (A > 0) and +inf or NaN on the fused path; all else agrees."""
    gen = torch.Generator().manual_seed(8)
    P, n, K, J = 2, 65, 8, 260
    x = _counts(n, J, gen, "cuda")
    A, B = _factors(P, n, K, J, gen, "cuda")
    B[1, :, 11] = 0.0
    x[:, 11] = x[:, 11].clamp_min(1.0)
    fused, generic = _both_paths(A, B, x)
    assert fused[0] == generic[0] == float("-inf")
    assert torch.isposinf(generic[2][1, :, 11]).all()
    _same_edges(fused[1:], generic[1:])
    assert torch.isfinite(fused[2][0]).all() and torch.isfinite(fused[2][1, :, :11]).all()


@pytest.mark.gpu
def test_out_of_scope_factor_product_takes_dense_path(count_fused):
    """K = 17 is outside the kernel's scope: a FactorProduct built by hand scores the materialised rate."""
    gen = torch.Generator().manual_seed(9)
    x = _counts(20, 64, gen, "cuda")
    A, B = _factors(2, 20, 17, 64, gen, "cuda")
    a, b = A.clone().requires_grad_(), B.clone().requires_grad_()
    tot = _site_sum(LinearPredictorTensor(dist.FactorProduct(a, b)), x)
    tot.backward()
    ref_a, ref_b = A.clone().requires_grad_(), B.clone().requires_grad_()
    ref = _site_sum(ref_a @ ref_b, x)
    ref.backward()
    assert not count_fused
    assert tot.item() == ref.item() and torch.equal(a.grad, ref_a.grad) and torch.equal(b.grad, ref_b.grad)


# ---- GPU tier: the unchanged sparse gamma DEF --------------------------------------------------------------
def _def_setup(P, n=40, J=256, dtype=torch.float32, seed=0):
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed)
    x = _counts(n, J, gen, "cuda").to(dtype)
    widths = (100, 40, 15)
    sizes = {"w_top": (widths[0] * widths[1],), "w_mid": (widths[1] * widths[2],), "w_bottom": (widths[2] * J,),
             "z_top": (n, widths[0]), "z_mid": (n, widths[1]), "z_bottom": (n, widths[2])}
    # per-particle latent values, a deterministic function of the guide parameters
    mult = {k: (0.5 + torch.rand(((P,) if P > 1 else ()) + v, generator=gen)).to("cuda", dtype)
            for k, v in sizes.items()}
    inj = {k: (lambda a, r, k=k: (a / r) * mult[k]) for k in sizes}
    return x, models.SparseGammaDEF(J, widths, device="cuda", dtype=dtype, inject=inj, particles=1)


def _loss_and_grads(elbo_cls, P, lazy_on, dtype=torch.float32, capture=False, steps=1):
    elbo_mod.LAZY_LINEAR = lazy_on
    try:
        pyro.clear_param_store()
        x, m = _def_setup(P, dtype=dtype)
        elbo = elbo_cls(num_particles=P, vectorize_particles=P > 1, max_plate_nesting=1)
        if capture:
            elbo.capture_graph = True
            svi = SVI(m.model, m.guide, AdagradRMSProp({"eta": 0.05, "t": 0.1}), elbo)
            losses = [svi.step(x) for _ in range(steps)]
            params = {k: v.detach().clone() for k, v in pyro.get_param_store().named_parameters()}
            return losses, params
        loss = elbo.loss_and_grads(m.model, m.guide, x)
        grads = {k: v.grad.detach().clone() for k, v in pyro.get_param_store().named_parameters()}
        return loss, grads
    finally:
        elbo_mod.LAZY_LINEAR = True


@pytest.fixture
def count_fused(monkeypatch):
    calls = []
    orig = dist._PoissonProductFn.apply

    def apply(*args):
        calls.append(1)
        return orig(*args)

    monkeypatch.setattr(dist._PoissonProductFn, "apply", apply)
    return calls


def _close(a, b):
    assert abs(a - b) <= 2e-6 * abs(b), (a, b)


def _grads_close(got, ref):
    assert set(got) == set(ref)
    for k in ref:
        tol = 2e-4 * ref[k].abs().max().item()
        err = (got[k] - ref[k]).abs().max().item()
        assert err <= tol, (k, err, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("elbo_cls", [TraceMeanField_ELBO, Trace_ELBO], ids=["meanfield", "trace"])
def test_def_model_takes_fused_path_and_matches(elbo_cls, count_fused):
    P = 8
    loss, grads = _loss_and_grads(elbo_cls, P, True)
    assert len(count_fused) == 1
    ref_loss, ref_grads = _loss_and_grads(elbo_cls, P, False)
    assert len(count_fused) == 1
    _close(loss, ref_loss)
    _grads_close(grads, ref_grads)


@pytest.mark.gpu
def test_def_model_single_particle(count_fused):
    loss, grads = _loss_and_grads(TraceMeanField_ELBO, 1, True)
    assert len(count_fused) == 1
    ref_loss, ref_grads = _loss_and_grads(TraceMeanField_ELBO, 1, False)
    _close(loss, ref_loss)
    _grads_close(grads, ref_grads)


@pytest.mark.gpu
def test_def_model_graph_captured(count_fused):
    P = 8
    losses, params = _loss_and_grads(TraceMeanField_ELBO, P, True, capture=True, steps=4)
    assert len(count_fused) >= 1
    ref_losses, ref_params = _loss_and_grads(TraceMeanField_ELBO, P, False, capture=True, steps=4)
    for a, b in zip(losses, ref_losses):
        _close(a, b)
    for k in ref_params:
        assert torch.allclose(params[k], ref_params[k], rtol=1e-4, atol=1e-5), k


@pytest.mark.gpu
def test_masked_and_fp64_sites_take_materialised_path(count_fused):
    P = 4
    # fp64: the factor product stays eager
    loss64, _ = _loss_and_grads(TraceMeanField_ELBO, P, True, dtype=torch.float64)
    ref64, _ = _loss_and_grads(TraceMeanField_ELBO, P, False, dtype=torch.float64)
    assert not count_fused
    assert abs(loss64 - ref64) <= 1e-9 * abs(ref64)
    # a masked observation site: lazy rate, materialised score
    gen = torch.Generator().manual_seed(3)
    x = _counts(20, 64, gen, "cuda")
    A, B = _factors(2, 20, 15, 64, gen, "cuda")
    mask = torch.rand(20, generator=gen).to("cuda") < 0.7
    out = []
    for use_lazy in (True, False):
        a, b = A.clone().requires_grad_(), B.clone().requires_grad_()
        rate = SiteValue.wrap(a) @ SiteValue.wrap(b) if use_lazy else a @ b
        assert _factor(rate) == use_lazy
        d = dist.Poisson(rate).to_event(1).mask(mask)
        tot = d._fused_sum(x, None, 1.0, 1.0, 1.0, True)
        tot.backward()
        out.append((tot.item(), a.grad, b.grad))
    assert not count_fused
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])
