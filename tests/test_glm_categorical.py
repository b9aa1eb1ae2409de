"""Fused softmax regression: ``Categorical(logits = X @ W.mT + b)`` scored by the wgmma kernel of
glm_categorical_tc.cu (``b2_glm_categorical_logits``).

CPU tier: the lazy class-axis patterns of pyro_b200/lazy.py (shape, dtype and values equal the eager
expression) and what ptxas makes of the kernel.  GPU tier: the kernel against fp64 at full size and at
ragged shapes, the unchanged softmax model reaching the kernel under Trace_ELBO and JitTrace_ELBO, and the
cases that take the materialised Categorical path."""
import os
import re
import subprocess

import pytest
import torch
import torch.nn.functional as F

import models
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from pyro_b200 import _build
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.lazy import LinearPredictorTensor, SiteValue
from pyro_b200.optim import ClippedAdam

DEV = device()


def softmax_model(X, y, K):
    D = X.shape[-1]
    W = pyro.sample("W", dist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
    b = pyro.sample("b", dist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1))
    with pyro.plate("data", X.shape[0]):
        Wm = W.squeeze(-3) if W.dim() > 2 else W
        pyro.sample("y", dist.Categorical(logits=X @ Wm.mT + b), obs=y)


def softmax_model_masked(X, y, K, mask):
    D = X.shape[-1]
    W = pyro.sample("W", dist.Normal(X.new_zeros(K, D), X.new_ones(K, D)).to_event(2))
    b = pyro.sample("b", dist.Normal(X.new_zeros(K), X.new_full((K,), 10.0)).to_event(1))
    with pyro.plate("data", X.shape[0]):
        Wm = W.squeeze(-3) if W.dim() > 2 else W
        pyro.sample("y", dist.Categorical(logits=X @ Wm.mT + b).mask(mask), obs=y)


def softmax_guide(X, y, K, *args):
    D = X.shape[-1]
    W_loc = pyro.param("W_loc", lambda: X.new_zeros(K, D))
    W_scale = pyro.param("W_scale", lambda: X.new_full((K, D), 0.1), constraint=torch.distributions.constraints.positive)
    b_loc = pyro.param("b_loc", lambda: X.new_zeros(K))
    b_scale = pyro.param("b_scale", lambda: X.new_full((K,), 0.1), constraint=torch.distributions.constraints.positive)
    pyro.sample("W", dist.Normal(W_loc, W_scale).to_event(2))
    pyro.sample("b", dist.Normal(b_loc, b_scale).to_event(1))


# ---- CPU tier: lazy semantics ------------------------------------------------------------------------------
def _class_lazy(t):
    return isinstance(t, LinearPredictorTensor) and isinstance(t.lazy, dist.ClassLinearPredictor)


def _lazy_cases():
    torch.manual_seed(0)
    N, D, K, P = 7, 5, 3, 4
    X = torch.randn(N, D)
    W2, W3, W4 = torch.randn(K, D), torch.randn(P, K, D), torch.randn(P, 1, K, D)
    bK, bP = torch.randn(K), torch.randn(P, 1, K)
    S = SiteValue.wrap
    return [
        ("X@W.mT", lambda: X @ S(W2).mT, lambda: X @ W2.mT),
        ("X@W.transpose", lambda: X @ S(W2).transpose(-1, -2), lambda: X @ W2.transpose(-1, -2)),
        ("matmul(X,W.mT)", lambda: torch.matmul(X, S(W2).mT), lambda: torch.matmul(X, W2.mT)),
        ("X@W3.mT", lambda: X @ S(W3).mT, lambda: X @ W3.mT),
        ("matmul(X,W3.mT)", lambda: torch.matmul(X, S(W3).mT), lambda: torch.matmul(X, W3.mT)),
        ("X@W4.squeeze.mT+b", lambda: X @ S(W4).squeeze(-3).mT + S(bP), lambda: X @ W4.squeeze(-3).mT + bP),
        ("X@W.mT+b", lambda: X @ S(W2).mT + S(bK), lambda: X @ W2.mT + bK),
        ("b+X@W.mT", lambda: S(bK) + X @ S(W2).mT, lambda: bK + X @ W2.mT),
        ("X@W3.mT+bK", lambda: X @ S(W3).mT + bK, lambda: X @ W3.mT + bK),
        ("linear(X,W)", lambda: F.linear(X, S(W2)), lambda: F.linear(X, W2)),
        ("linear(X,W,b)", lambda: F.linear(X, S(W2), S(bK)), lambda: F.linear(X, W2, bK)),
        ("linear(X,W)+b", lambda: F.linear(X, S(W2)) + bK, lambda: F.linear(X, W2) + bK),
    ]


@pytest.mark.parametrize("case", range(12))
def test_class_lazy_patterns_equal_eager(case):
    name, lazy_fn, eager_fn = _lazy_cases()[case]
    lazy, eager = lazy_fn(), eager_fn()
    assert _class_lazy(lazy), name
    assert tuple(lazy.shape) == tuple(eager.shape) and lazy.dtype == eager.dtype, name
    assert torch.equal(lazy.dense(), eager), name


def test_linear_with_matrix_weight_gives_rows_by_classes():
    X = torch.randn(5, 3)
    W = SiteValue.wrap(torch.randn(2, 3))
    assert tuple(F.linear(X, W).shape) == (5, 2)


def test_other_uses_of_class_logits_materialise_exactly():
    torch.manual_seed(1)
    X, W, b = torch.randn(6, 4), torch.randn(3, 4), torch.randn(3)
    S = SiteValue.wrap
    lazy = X @ S(W).mT + S(b)
    eager = X @ W.mT + b
    for f in (lambda t: t * 2.0, lambda t: t.softmax(-1), lambda t: t + torch.ones(6, 3), lambda t: t.sum(0)):
        out = f(lazy)
        assert not isinstance(out, LinearPredictorTensor)
        assert torch.equal(out, f(eager))
    # a bias that does not fit [K] / [P, 1, K] is added eagerly
    odd = torch.randn(6, 1)
    out = X @ S(W).mT + odd
    assert not isinstance(out, LinearPredictorTensor) and torch.equal(out, X @ W.mT + odd)


def test_categorical_of_class_logits_materialises_on_log_prob():
    torch.manual_seed(2)
    X, W, b = torch.randn(6, 4), torch.randn(2, 3, 4), torch.randn(2, 1, 3)
    S = SiteValue.wrap
    d = dist.Categorical(logits=X @ S(W).mT + S(b))
    assert isinstance(d, dist._CategoricalLinear) and tuple(d.batch_shape) == (2, 6)
    ref = X @ W.mT + b
    assert torch.equal(d._logits_raw, ref)
    assert torch.allclose(d.logits, torch.log_softmax(ref, -1), atol=1e-6)
    assert torch.allclose(d.probs, torch.softmax(ref, -1))


def test_bernoulli_patterns_unchanged():
    torch.manual_seed(3)
    N, D, P = 9, 4, 3
    X = torch.randn(N, D)
    S = SiteValue.wrap
    w1, wP, bP, b0 = torch.randn(D), torch.randn(P, 1, D), torch.randn(P, 1), torch.randn(())
    for lazy, shape in ((S(wP).squeeze(-2) @ X.T + S(bP), (P, N)), (X @ S(w1) + S(b0), (N,)),
                        (F.linear(X, S(w1), S(b0)), (N,))):
        assert type(lazy) is LinearPredictorTensor and isinstance(lazy.lazy, dist.LinearPredictor)
        assert tuple(lazy.shape) == shape
    assert isinstance(dist.Bernoulli(logits=X @ S(w1) + S(b0)), dist._BernoulliLinear)


# ---- CPU tier: SASS of the kernel ----------------------------------------------------------------------------
SASS_KERNELS = ["glm_categorical_tc_kernelILi%dELb%dE" % (kp, sx) for kp in (2, 4, 8, 16) for sx in (0, 1)]


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, cuobjdump = sass_test._tools()
    obj = str(tmp_path_factory.mktemp("glm_cat_sass") / "glm_categorical_tc.o")
    src = os.path.join(_build.CSRC, "glm_categorical_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


@pytest.mark.parametrize("mangled", SASS_KERNELS)
def test_categorical_kernel_sass(compiled, mangled):
    """No C7515/C7520 serialisation note, no spills, and no warpgroup wait or arrive between two HGMMA of
    one contraction, for every instantiation (class padding x split X)."""
    import test_glm_tc_sass as sass_test
    log, sass = compiled
    for line in log.splitlines():
        if mangled in line:
            assert "C7515" not in line and "C7520" not in line, line
    props, used = sass_test._ptxas_properties(log, mangled)
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used
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
    assert "64x64x8" in shapes and "64x40x8" in shapes, shapes
    assert not bad, bad


# ---- GPU tier: the kernel against fp64 -----------------------------------------------------------------------
def _reference(X, y, W, b):
    """fp64 per-particle sums, dW and db on the CPU, one particle at a time."""
    Xd = X.double()
    P, K, _ = W.shape
    s = torch.empty(P, dtype=torch.float64)
    gW = torch.empty(W.shape, dtype=torch.float64)
    gb = torch.empty(P, K, dtype=torch.float64)
    onehot = F.one_hot(y.clamp(0, K - 1), K).double()
    bad = (y < 0) | (y >= K)
    for p in range(P):
        lg = Xd @ W[p].double().t() + (b[p].double() if b is not None else 0.0)
        lse = lg.logsumexp(-1)
        lpn = lg.gather(1, y.clamp(0, K - 1)[:, None]).squeeze(1) - lse
        s[p] = lpn.sum() if not bool(bad.any()) else float("nan")
        g = onehot - torch.softmax(lg, -1)
        gW[p] = g.t() @ Xd
        gb[p] = g.sum(0)
    return s, gW, gb


def _launch(X, y, W, b, flags=0, out_total=None):
    from pyro_b200 import _native as N
    n, D = X.shape
    P, K, _ = W.shape
    sum_p = torch.empty(P, device=DEV)
    dW = torch.empty(P, K, D, device=DEV)
    db = torch.empty(P, K, device=DEV)
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_categorical_workspace(n, D, K, P)), tag="glm_cat_test")
    N.check(N.lib().b2_glm_categorical_logits(
        X.data_ptr(), y.data_ptr(), W.data_ptr(), b.data_ptr() if b is not None else None, n, D, K, P,
        1.0, 1.0, 1.0, flags, sum_p.data_ptr(), out_total.data_ptr() if out_total is not None else None,
        dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(torch.device(DEV))),
        "b2_glm_categorical_logits")
    torch.cuda.synchronize()
    return sum_p.cpu(), dW.cpu(), db.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 10, 16])
def test_categorical_kernel_full_size_against_fp64(K):
    """N = 1e6, D = 32, P = 64: sum_p within 2e-5 relative, dW / db within 2e-4 of max |grad|, and a second
    launch bitwise equal (fixed-order reductions, no float atomics)."""
    if EMULATE:
        pytest.skip("kernel test")
    torch.manual_seed(K)
    n, D, P = 1_000_000, 32, 64
    X = torch.randn(n, D)
    Wt = torch.randn(K, D) / D ** 0.5
    y = torch.distributions.Categorical(logits=X @ Wt.t()).sample()
    W = Wt + 0.3 * torch.randn(P, K, D)
    b = 0.2 * torch.randn(P, K)
    s_ref, gW, gb = _reference(X, y, W, b)
    Xg, yg, Wg, bg = X.to(DEV), y.to(DEV), W.to(DEV), b.to(DEV)
    total = torch.empty((), device=DEV)
    s, dW, db = _launch(Xg, yg, Wg, bg, out_total=total)
    assert float(((s.double() - s_ref).abs() / s_ref.abs()).max()) <= 2e-5
    assert abs(float(total) - float(s_ref.sum())) <= 2e-5 * abs(float(s_ref.sum()))
    assert float((dW.double() - gW).abs().max()) <= 2e-4 * float(gW.abs().max())
    assert float((db.double() - gb).abs().max()) <= 2e-4 * float(gb.abs().max())
    s2, dW2, db2 = _launch(Xg, yg, Wg, bg)
    assert torch.equal(s, s2) and torch.equal(dW, dW2) and torch.equal(db, db2)


# (n, P, K, bias, labels): "rand", "same" (every label the same class)
_RAGGED = [(1, 1, 2, True, "rand"), (63, 3, 3, False, "rand"), (64, 7, 5, True, "rand"),
           (65, 65, 9, True, "rand"), (8191, 7, 16, False, "rand"), (70001, 65, 16, True, "rand"),
           (70001, 3, 2, True, "rand"), (70001, 7, 5, False, "same"), (8191, 65, 3, True, "same"),
           (64, 1, 16, True, "same")]


@pytest.mark.gpu
@pytest.mark.parametrize("n,P,K,bias,labels", _RAGGED, ids=["-".join(map(str, c)) for c in _RAGGED])
def test_categorical_kernel_ragged_shapes_against_fp64(n, P, K, bias, labels):
    """Single rows, tile boundaries (63 / 64 / 65), ragged last tiles (70001 = 1093 * 64 + 49), ragged
    particle slabs (P = 65 with 4 .. 32 particles per slab), every class padding (K = 2, 3, 5, 9, 16), no
    bias, one class only.  Tolerances of the Bernoulli ragged-shape test on the tensor-core kernel."""
    if EMULATE:
        pytest.skip("kernel test")
    torch.manual_seed(n + P + K)
    D = 32
    X = torch.randn(n, D)
    y = torch.randint(0, K, (n,)) if labels == "rand" else torch.full((n,), K - 1, dtype=torch.int64)
    W = 0.3 * torch.randn(P, K, D)
    b = torch.randn(P, K) if bias else None
    s_ref, gW, gb = _reference(X, y, W, b)
    s, dW, db = _launch(X.to(DEV), y.to(DEV), W.to(DEV), b.to(DEV) if bias else None)
    assert float((s.double() - s_ref).abs().max()) <= 2e-5 * max(1.0, float(s_ref.abs().max()))
    assert float((dW.double() - gW).abs().max()) <= 5e-4 * max(1.0, float(gW.abs().max()))
    assert float((db.double() - gb).abs().max()) <= 5e-4 * max(1.0, float(gb.abs().max()))


@pytest.mark.gpu
def test_categorical_kernel_out_of_range_label_gives_nan():
    """A label outside [0, K) is compared, never used as an index: the sums it enters are NaN, nothing faults,
    and the next launch with valid labels is exact.  The labels are one vector shared by all P particles (every
    particle scores every row), so a bad label makes EVERY particle's sum NaN; "NaN for its particle only" can
    only mean the particle scoring that row, which here is all of them."""
    if EMULATE:
        pytest.skip("kernel test")
    torch.manual_seed(5)
    n, D, P, K = 9000, 32, 5, 5
    X = torch.randn(n, D)
    y = torch.randint(0, K, (n,))
    W = 0.3 * torch.randn(P, K, D)
    Xg, Wg = X.to(DEV), W.to(DEV)
    for bad in (K, -1, 1 << 40):
        yb = y.clone()
        yb[1234] = bad
        s, dW, db = _launch(Xg, yb.to(DEV), Wg, None)
        assert bool(torch.isnan(s).all()) and bool(torch.isfinite(dW).all()) and bool(torch.isfinite(db).all())
    s_ref, _, _ = _reference(X, y, W, None)
    s, _, _ = _launch(Xg, y.to(DEV), Wg, None)
    assert float((s.double() - s_ref).abs().max()) <= 2e-5 * float(s_ref.abs().max())


# ---- GPU tier: the unchanged softmax model ---------------------------------------------------------------
def _svi(model, elbo_cls, X, y, K, eps_W, eps_b, lazy, P, extra=()):
    """Steps of SVI with noise injected through fixed device buffers (refilled before every step), so an
    eager and a captured run consume identical draws."""
    pyro.clear_param_store()
    bW, bb = torch.empty_like(eps_W[0]), torch.empty_like(eps_b[0])

    def guide(*args):
        with models.InjectNoise({"W": bW, "b": bb}):
            softmax_guide(*args)

    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  elbo_cls(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
        losses = []
        for i in range(eps_W.shape[0]):
            bW.copy_(eps_W[i])
            bb.copy_(eps_b[i])
            losses.append(svi.step(X, y, K, *extra))
    finally:
        elbo_mod.LAZY_LINEAR = saved
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in ("W_loc", "W_scale", "b_loc", "b_scale")}


def _data(n, D, K, P, steps, seed):
    torch.manual_seed(seed)
    X = torch.randn(n, D)
    y = torch.distributions.Categorical(logits=X @ (torch.randn(K, D) / D ** 0.5).t()).sample()
    eps_W, eps_b = torch.randn(steps, P, 1, K, D), torch.randn(steps, P, 1, K)
    return X.to(DEV), y.to(DEV), eps_W.to(DEV), eps_b.to(DEV)


@pytest.mark.gpu
def test_unchanged_softmax_model_takes_the_kernel():
    """P = 16 vectorised particles, N = 70 000, K = 10: every step's likelihood site is scored by the
    kernel, and three Trace_ELBO + ClippedAdam steps match the materialised path (LAZY_LINEAR = False):
    loss within 2e-5 relative, parameters within 2e-4."""
    if EMULATE:
        pytest.skip("kernel test")
    P, K = 16, 10
    X, y, eps_W, eps_b = _data(70000, 32, K, P, 3, 11)
    calls = []
    real = dist._GlmCategoricalFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)
    dist._GlmCategoricalFn.apply = spy
    try:
        l_f, p_f = _svi(softmax_model, Trace_ELBO, X, y, K, eps_W, eps_b, True, P)
    finally:
        dist._GlmCategoricalFn.apply = real
    assert len(calls) == 3
    l_m, p_m = _svi(softmax_model, Trace_ELBO, X, y, K, eps_W, eps_b, False, P)
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_softmax_model_captured_graph_step_equals_eager():
    """JitTrace_ELBO (the step captured in a CUDA graph) with the fused site gives bit for bit the losses and
    parameters of the eager steps: the same kernels run on the same inputs, and every Python-level scoring of
    the site, the capturing one included, went through the kernel."""
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    P, K = 16, 10
    X, y, eps_W, eps_b = _data(70000, 32, K, P, 3, 12)
    sites, calls = [], []
    real_sum, real_apply = dist._CategoricalLinear._fused_sum, dist._GlmCategoricalFn.apply

    def spy_sum(self, *a, **k):
        sites.append(1)
        return real_sum(self, *a, **k)

    def spy_apply(*a):
        calls.append(1)
        return real_apply(*a)
    dist._CategoricalLinear._fused_sum = spy_sum
    dist._GlmCategoricalFn.apply = spy_apply
    try:
        l_e, p_e = _svi(softmax_model, Trace_ELBO, X, y, K, eps_W, eps_b, True, P)
        n_eager = len(calls)
        l_g, p_g = _svi(softmax_model, JitTrace_ELBO, X, y, K, eps_W, eps_b, True, P)
    finally:
        dist._CategoricalLinear._fused_sum = real_sum
        dist._GlmCategoricalFn.apply = real_apply
    assert n_eager == 3
    # JitTrace: one eager step, then the capturing call (one real update + the capture), then a replay
    assert len(calls) - n_eager >= 3 and len(calls) == len(sites)
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("n,D,K,masked", [(9000, 10, 4, False), (9000, 32, 20, False), (4000, 32, 10, False),
                                          (9000, 32, 10, True)], ids=["D10", "K20", "N4000", "masked"])
def test_softmax_model_fallback_matches_materialised(n, D, K, masked):
    """Outside the kernel's scope (D != 32, K > 16, N < 8192, a masked site) the site is scored from the
    materialised logits, with the same results as LAZY_LINEAR = False."""
    if EMULATE:
        pytest.skip("kernel test")
    P = 4
    X, y, eps_W, eps_b = _data(n, D, K, P, 2, 13)
    model, extra = softmax_model, ()
    if masked:
        model, extra = softmax_model_masked, (torch.rand(n, device=DEV) < 0.7,)
    calls = []
    real = dist._GlmCategoricalFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)
    dist._GlmCategoricalFn.apply = spy
    try:
        l_f, p_f = _svi(model, Trace_ELBO, X, y, K, eps_W, eps_b, True, P, extra)
    finally:
        dist._GlmCategoricalFn.apply = real
    assert not calls
    l_m, p_m = _svi(model, Trace_ELBO, X, y, K, eps_W, eps_b, False, P, extra)
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 1e-6 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=1e-6), k


# ---- other families keep their results when the model contracts data with a matrix latent ---------------------
def matrix_weight_model(X, Y, kind, seen):
    D, K = X.shape[1], Y.shape[1]
    W = pyro.sample("W", dist.Normal(X.new_zeros(D, K), X.new_ones(D, K)).to_event(2))
    with pyro.plate("data", X.shape[0]):
        Wm = W.squeeze(-3) if W.dim() > 2 else W
        if kind == "vector":                       # X @ w with a 1-d latent w: a Bernoulli-style lazy predictor
            mean = X @ Wm[..., 0]
            seen.append(mean)
            pyro.sample("y", dist.Normal(mean, 1.0), obs=Y[:, 0])
            return
        if kind == "linear":
            logits = F.linear(X, Wm.mT)
        elif kind == "mT":
            logits = X @ Wm.mT.mT
        else:
            logits = X @ Wm
        seen.append(logits)
        if kind == "bernoulli":
            pyro.sample("y", dist.Bernoulli(logits=logits).to_event(1), obs=(Y > 0).to(Y.dtype))
        else:
            pyro.sample("y", dist.Normal(logits, 1.0).to_event(1), obs=Y)


def matrix_weight_guide(X, Y, kind, seen):
    D, K = X.shape[1], Y.shape[1]
    W_loc = pyro.param("W_loc", lambda: X.new_zeros(D, K))
    pyro.sample("W", dist.Normal(W_loc, X.new_full((D, K), 0.1)).to_event(2))


def _matrix_weight_run(kind, lazy, particles, dev):
    torch.manual_seed(21)
    n, D, K = 3000, 6, 3
    X, Y = torch.randn(n, D).to(dev), torch.randn(n, K).to(dev)
    shape = (particles, 1, D, K) if particles > 1 else (D, K)
    eps = torch.randn((2,) + shape).to(dev)
    buf = torch.empty_like(eps[0])
    pyro.clear_param_store()
    seen = []

    def guide(*args):
        with models.InjectNoise({"W": buf}):
            matrix_weight_guide(*args)

    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    try:
        elbo = Trace_ELBO(num_particles=particles, vectorize_particles=particles > 1, max_plate_nesting=1)
        svi = SVI(matrix_weight_model, guide, ClippedAdam({"lr": 0.05}), elbo)
        losses = []
        for i in range(2):
            buf.copy_(eps[i])
            losses.append(svi.step(X, Y, kind, seen))
    finally:
        elbo_mod.LAZY_LINEAR = saved
    return losses, pyro.get_param_store()["W_loc"].detach().clone(), seen


_MATRIX_CASES = [("normal", 4), ("mT", 4), ("bernoulli", 4), ("linear", 1), ("vector", 1)]


def _check_matrix_weight(kind, particles, dev):
    l_lazy, w_lazy, seen = _matrix_weight_run(kind, True, particles, dev)
    l_eager, w_eager, seen_eager = _matrix_weight_run(kind, False, particles, dev)
    # the contraction was kept lazy, so the case exercises the hand-over of a lazy tensor to another family
    assert all(isinstance(t, LinearPredictorTensor) for t in seen) and seen
    assert not any(isinstance(t, LinearPredictorTensor) for t in seen_eager)
    assert l_lazy == l_eager, (l_lazy, l_eager)
    assert torch.equal(w_lazy, w_eager)
    assert float(w_lazy.abs().max()) > 0      # the likelihood gradient reached W


@pytest.mark.parametrize("kind,particles", _MATRIX_CASES, ids=[c[0] for c in _MATRIX_CASES])
def test_matrix_latent_in_other_families_emulated(kind, particles):
    """CPU tier (native seams emulated): ``Normal(X @ W, 1)``, ``Bernoulli(logits=X @ W)`` and friends with a
    matrix latent W give the same losses and updates as LAZY_LINEAR = False."""
    import cpu_emulation
    with cpu_emulation.enabled():
        _check_matrix_weight(kind, particles, "cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,particles", _MATRIX_CASES, ids=[c[0] for c in _MATRIX_CASES])
def test_matrix_latent_in_other_families(kind, particles):
    """On the device: a lazy contraction handed to Normal or Bernoulli is materialised before the native
    kernel, with its gradient to W, and gives bit for bit the losses and updates of LAZY_LINEAR = False."""
    _check_matrix_weight(kind, particles, DEV)


def test_class_linear_predictor_validates_bias():
    X, W = torch.randn(5, 4), torch.randn(2, 3, 4)
    assert tuple(dist.class_linear_predictor(X, W, torch.randn(3)).shape) == (2, 5, 3)
    assert tuple(dist.class_linear_predictor(X, W, torch.randn(2, 1, 3)).shape) == (2, 5, 3)
    for bad in (torch.randn(2, 3), torch.randn(3, dtype=torch.float64), torch.randn(4)):
        with pytest.raises(ValueError):
            dist.class_linear_predictor(X, W, bad)
    with pytest.raises(ValueError):
        dist.class_linear_predictor(X, torch.randn(3, 5))
