"""Multilevel regression under SVI past 128 columns: ``X @ w + b + alpha[g] + SUM_k beta_k[g] * X[:, c_k]`` with
D + G (1 + S) > 128 and the rows sorted by group, scored by ``b2_glm_group_gather_sum``: the gathered tile kernel of
the potential's wide route, glm_finish_kernel D wide, and a group finish that writes d/dalpha and d/dbeta_k in the
particle layout.

CPU tier: SVI steps of logistic, Poisson and linear regression with the kernel seam replaced by an fp64 torch
restatement match ``LAZY_LINEAR = False``, with one gathered call per step; the near misses make no gathered call and
match exactly; narrow models keep their call; the sortedness cache; the entry point's argument checks and workspace;
what ptxas makes of the new pack and finish kernels.
GPU tier: the call against fp64 (P = 1, 64, 65; D = 1 .. 128; ragged N; G = 38 .. 65536; one group, runs across many
ranges, runs ending on tile boundaries, empty groups), bitwise repeatable, and against ``b2_glm_group_slope_sum`` at
narrow widths; the NaN policy; SVI against the materialised path; a captured graph; the fallbacks; reference Pyro
through ``bind.Trace_ELBO``."""
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
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.lazy import LinearPredictorTensor
from pyro_b200.optim import ClippedAdam
from test_glm_group_svi import KIND_CODE, group_guide, group_model
from test_glm_slope_svi import _Noise, _data, _operands, _reference, slope_guide, slope_model

DEV = device()
WIDE_KINDS = ["Bernoulli", "Poisson", "Normal"]


def _sorted(X, g, y, m):
    """The rows ordered by group (stable): the posterior does not depend on the order of the rows."""
    order = torch.argsort(g, stable=True)
    return X[order].contiguous(), g[order].contiguous(), y[order].contiguous(), m[order].contiguous()


def _cols(D, S):
    return [0, D - 1, D // 2][:S]


def _wide(kind, n, D, G, S, seed, dev=DEV):
    return _sorted(*_data(kind, n, D, G, S=S, seed=seed, dev=dev, cols=_cols(D, S)))


def _model(kind, form, S, G):
    if S == 0:
        return group_model(kind, form), group_guide(kind, form)
    return slope_model(kind, form, S, cols=_cols(5, S)), slope_guide(kind, form, S)


# ---- the kernel seam restated in fp64 ------------------------------------------------------------------------------
def _fp64_gather(meta, X, y, W, b, sigma, *T):
    """What b2_glm_group_gather_sum returns through _GlmGatherFn.launch, restated in fp64 with torch.distributions and
    autograd."""
    scale, weight, coeff, _, kind, idx, s_stride, cols = meta
    ops = [t.detach().double().requires_grad_(t.requires_grad) if t is not None else None for t in (W, b, sigma) + T]
    Wd, bd, sd = ops[:3]
    G = T[0].shape[-1]
    gi = idx.long()
    with torch.enable_grad():
        eta = Wd @ X.double().T + ops[3].reshape(-1, G)[:, gi]
        for Bd, c in zip(ops[4:], cols):
            eta = eta + Bd.reshape(-1, G)[:, gi] * X.double()[:, c]
        if bd is not None:
            eta = eta + bd[:, None]
        yd = y.double()
        if kind == N.GLM_BERNOULLI:
            lp = torch.distributions.Bernoulli(logits=eta).log_prob(yd)
        elif kind == N.GLM_POISSON:
            lp = yd * eta - eta.exp() - torch.lgamma(yd + 1)
        else:
            lp = torch.distributions.Normal(eta, sd.reshape(-1, 1) if s_stride else sd.reshape(())).log_prob(yd)
        lps = scale * lp.sum()
        need = [o for o in ops if o is not None and o.requires_grad]
        grads = iter(torch.autograd.grad(lps, need))
    out = [weight * next(grads) if o is not None and o.requires_grad else None for o in ops]
    out = [o.float() if o is not None else None for o in out]
    return ((coeff * lps).detach().float(), None, None) + tuple(out)


def _svi(model, guide, args, steps, lazy, elbo_cls=Trace_ELBO, P=8, seed=0):
    """``steps`` SVI steps with guide noise from seed ``seed`` injected through fixed buffers; returns the losses, the
    parameters, the number of gathered calls and the metas of the one-hot group and slope calls."""
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
    calls, metas = [], []
    real_a, real_s, real_g = dist._GlmGatherFn.apply, dist._GlmSlopeFn.apply, dist._GlmGroupFn.apply
    dist._GlmGatherFn.apply = lambda *a: calls.append(1) or real_a(*a)
    dist._GlmSlopeFn.apply = lambda *a: metas.append(("slope", a[0])) or real_s(*a)
    dist._GlmGroupFn.apply = lambda *a: metas.append(("group", a[0])) or real_g(*a)
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
        dist._GlmGatherFn.apply, dist._GlmSlopeFn.apply, dist._GlmGroupFn.apply = real_a, real_s, real_g
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls), metas


@pytest.fixture
def fp64_seam():
    """The CPU stand-ins of the native seams, with the gathered sum restated in fp64 (and _BernoulliLinear's own
    _fused_sum, which the stand-ins replace by the dense path)."""
    import cpu_emulation
    fused = dist._BernoulliLinear._fused_sum
    with cpu_emulation.enabled():
        dist._BernoulliLinear._fused_sum = fused
        saved = dist._GlmGatherFn.launch
        dist._GlmGatherFn.launch = _fp64_gather
        try:
            yield
        finally:
            dist._GlmGatherFn.launch = saved


def _close(l_f, p_f, l_m, p_m, rel, atol):
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= rel * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=atol, rtol=atol), k


def _equal(l_f, p_f, l_m, p_m):
    assert l_f == l_m, (l_f, l_m)
    for k in p_m:
        assert torch.equal(p_f[k], p_m[k]), k


# ---- CPU tier: SVI on the gathered route ------------------------------------------------------------------------------
# (S, G): radon's 85 counties with slopes (5 + 85 (1 + S) columns), and 1 000 groups
_SHAPES = [(0, 1000), (1, 85), (2, 85), (3, 1000)]


@pytest.mark.parametrize("S,G", _SHAPES, ids=["S%d-G%d" % c for c in _SHAPES])
@pytest.mark.parametrize("form", ["centred", "noncentred"])
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_svi_on_the_gathered_route_matches_materialised_with_the_seam_restated(fp64_seam, kind, form, S, G):
    """Three steps, 8 particles (per-particle tables; Normal with a latent sigma): one gathered call per step and no
    one-hot call, losses and parameters within 1e-5 of LAZY_LINEAR = False."""
    X, g, y, m = _wide(kind, 8192, 5, G, S, seed=3 + S, dev="cpu")
    args = (X, g, y, m, None, G)
    model, guide = _model(kind, form, S, G)
    l_f, p_f, calls, metas = _svi(model, guide, args, 3, True)
    l_m, p_m, calls_m, metas_m = _svi(model, guide, args, 3, False)
    assert calls == 3 and calls_m == 0 and not metas and not metas_m
    _close(l_f, p_f, l_m, p_m, 1e-5, 1e-5)


@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_shared_tables_with_one_particle(fp64_seam, kind):
    """One particle: every table and sigma is one row shared by the particle axis (stride 0), its gradient summed."""
    X, g, y, m = _wide(kind, 8192, 5, 85, 2, seed=9, dev="cpu")
    model, guide = _model(kind, "noncentred", 2, 85)
    l_f, p_f, calls, metas = _svi(model, guide, (X, g, y, m, None, 85), 3, True, P=1)
    l_m, p_m, _, _ = _svi(model, guide, (X, g, y, m, None, 85), 3, False, P=1)
    assert calls == 3 and not metas
    _close(l_f, p_f, l_m, p_m, 1e-5, 1e-5)


def test_shared_table_gradient_is_summed_over_particles(fp64_seam):
    """_gather_sum with a [G] table and a [P, G] table: d/dtable takes each table's shape."""
    X, g, y, m = _wide("Poisson", 8192, 6, 200, 1, seed=10, dev="cpu")
    P = 4
    w = torch.randn(P, 6).mul_(0.1).requires_grad_(True)
    A = torch.randn(200).mul_(0.1).requires_grad_(True)
    B = torch.randn(P, 200).mul_(0.1).requires_grad_(True)
    lp = dist.LinearPredictor(X, w.reshape(P, 1, 6), None, group=dist.GroupGather(A, g),
                              slopes=(dist.SlopeGather(B, g, X[:, 0]).with_col(0),))
    meta = (1.0, 1.0, 1.0, True)
    total = dist._gather_sum(N.GLM_POISSON, lp, y, None, lp.shape, meta, (None, 0))
    total.backward()
    eta = (w @ X.T + A[g] + B[:, g] * X[:, 0]).double()
    ref = (y.double() * eta - eta.exp() - torch.lgamma(y.double() + 1)).sum()
    gw, gA, gB = torch.autograd.grad(ref, [w, A, B])
    assert A.grad.shape == A.shape and B.grad.shape == B.shape
    for got, want in ((w.grad, gw), (A.grad, gA), (B.grad, gB)):
        assert torch.allclose(got.double(), want.double(), rtol=1e-5, atol=1e-5)


# ---- CPU tier: near misses -----------------------------------------------------------------------------------------
_MISSES = ["descending_pair", "binomial_one_count", "binomial_row_counts", "G65537", "D129", "N8191", "masked",
           "fp64", "no_tensor_cores"]


@pytest.mark.parametrize("case", _MISSES)
def test_near_misses_make_no_gathered_call_and_match_materialised(fp64_seam, case):
    kind = "Binomial" if case.startswith("binomial") else "Poisson"
    n = 8191 if case == "N8191" else 8192
    D = 129 if case == "D129" else 5
    G = 65537 if case == "G65537" else 85
    X, g, y, m = _wide("BinomialRows" if case == "binomial_row_counts" else kind, n, D, G, 1, seed=12, dev="cpu")
    if case == "descending_pair":
        i = int(torch.nonzero(g[1:] > g[:-1])[0]) + 1     # the first step up becomes a step down
        g = g.clone()
        g[i - 1], g[i] = int(g[i]), int(g[i - 1])
    mask = (torch.rand(n, generator=torch.Generator().manual_seed(1)) < 0.7) if case == "masked" else None
    if case == "fp64":
        X, y, m = X.double(), y.double(), m.double()
    if case == "no_tensor_cores":
        def model(X, g, y, m=None, mask=None, G=6):
            w = pyro.sample("w", dist.Normal(X.new_zeros(X.shape[-1]), 1.0).to_event(1))
            b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
            A = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1)).squeeze(-2)
            B0 = pyro.sample("beta0", dist.Normal(X.new_zeros(G), 0.3).to_event(1)).squeeze(-2)
            with pyro.plate("data", X.shape[0]):
                lp = dist.LinearPredictor(X, w, b, tensor_cores=False)
                eta = LinearPredictorTensor(lp) + A[..., g] + B0[..., g] * X[:, 0]
                pyro.sample("y", dist.Poisson(torch.exp(eta)), obs=y)
    else:
        model = slope_model(kind, S=1, cols=[0])
    guide = slope_guide(kind, S=1)
    args = (X, g, y, m, mask, G)
    l_f, p_f, calls, metas = _svi(model, guide, args, 2, True, P=4)
    l_m, p_m, _, _ = _svi(model, guide, args, 2, False, P=4)
    assert calls == 0 and not metas
    _equal(l_f, p_f, l_m, p_m)


@pytest.mark.parametrize("S", [0, 2])
def test_narrow_sorted_models_keep_their_call_and_meta(fp64_seam, S):
    """A sorted index at D + G (1 + S) <= 128 columns keeps the one-hot call (b2_glm_group_sum or
    b2_glm_group_slope_sum) with the parent's meta."""
    import test_glm_group_svi as group_test
    import test_glm_slope_svi as slope_test
    X, g, y, m = _wide("Normal", 8192, 5, 7, S, seed=5, dev="cpu")
    model, guide = _model("Normal", "centred", S, 7)
    saved = dist._GlmGroupFn.launch, dist._GlmSlopeFn.launch
    dist._GlmGroupFn.launch, dist._GlmSlopeFn.launch = group_test._fp64_launch, slope_test._fp64_launch
    try:
        _, _, calls, metas = _svi(model, guide, (X, g, y, m, None, 7), 2, True)
    finally:
        dist._GlmGroupFn.launch, dist._GlmSlopeFn.launch = saved
    assert calls == 0 and len(metas) == 2
    for which, meta in metas:
        if S == 0:
            scale, weight, coeff, unit, kind, idx, trials, per_row, s_stride = meta
            assert which == "group"
        else:
            scale, weight, coeff, unit, kind, idx, trials, per_row, s_stride, cols = meta
            assert which == "slope" and cols == tuple(_cols(5, S))
        assert kind == N.GLM_NORMAL and idx.dtype == torch.int32 and trials is None and per_row == 0


# ---- CPU tier: the sortedness cache ---------------------------------------------------------------------------------
class _Syncs:
    """Counts the host reads of tensor values (tolist, item, bool) while active."""

    def __enter__(self):
        self.n = 0
        self.saved = (torch.Tensor.tolist, torch.Tensor.item, torch.Tensor.__bool__)
        tolist, item, tbool = self.saved

        def counted(f):
            def g(*a, **k):
                self.n += 1
                return f(*a, **k)
            return g
        torch.Tensor.tolist, torch.Tensor.item, torch.Tensor.__bool__ = counted(tolist), counted(item), counted(tbool)
        return self

    def __exit__(self, *exc):
        torch.Tensor.tolist, torch.Tensor.item, torch.Tensor.__bool__ = self.saved


def test_sortedness_is_found_with_the_range_check_and_cached():
    g = torch.sort(torch.randint(0, 50, (1000,), generator=torch.Generator().manual_seed(0))).values
    with _Syncs() as s:
        assert dist.group_index_sorted(g, 50) is True
    assert s.n == 1                                        # one host sync for the range and the order
    with _Syncs() as s:
        c = dist.group_index_int32(g, 50)
        assert dist.group_index_sorted(g, 50) is True and dist.group_index_int32(g, 50) is c
    assert s.n == 0
    g[10], g[11] = 40, 3                                   # an in-place write: a new version, checked again
    with _Syncs() as s:
        assert dist.group_index_sorted(g, 50) is False
    assert s.n == 1
    assert dist.group_index_int32(g, 50) is not c and int(dist.group_index_int32(g, 50)[11]) == 3
    assert dist.group_index_sorted(torch.zeros(1, dtype=torch.int64), 1) is True
    with pytest.raises(IndexError):
        dist.group_index_sorted(g, 40)


def test_glm_potential_sets_sorted_as_before():
    """On the wide potential fixtures and their unsorted and narrow twins, `sorted` is the non-decreasing test of
    the index."""
    from test_glm_many_groups_potential import _data as pot_data
    from test_glm_many_groups_potential import _recognised, _sorted as pot_sorted
    from test_glm_slope_potential import slope_model as pot_slope_model
    from pyro_b200.infer.mcmc import GlmPotential
    for G, cols, srt in ((70, (2,), True), (6, (), True), (6, (), False), (40, (2, 0), True), (40, (2, 0), False)):
        X, g, y = pot_data("Poisson", 400, 8, G, dev="cpu", seed=G, slopes=list(cols))
        if srt:
            X, g, y = pot_sorted(X, g, y)
        pot = _recognised(pot_slope_model("Poisson", tuple(("centred", "const", c) for c in cols), G=G), X, g, y)
        assert isinstance(pot, GlmPotential), (G, cols, srt)
        assert pot.group_effect.sorted == int(bool((g[1:] >= g[:-1]).all())) == int(srt), (G, cols, srt)


# ---- CPU tier: the entry point's argument checks ---------------------------------------------------------------------
def test_gather_sum_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p, q = ctypes.c_void_p(4096), ctypes.c_void_p(4100)
    D, G, P, n = 10, 200, 4, 10000

    def tables(S=2, cols=(3, 7, 0), beta=(4096, 4096, 4096), strides=(G, 0, G)):
        sl = N.b2_glm_slope_tables(S)
        for k in range(3):
            sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], beta[k], strides[k]
        return ctypes.byref(sl)

    def call(kind=N.GLM_POISSON, X=p, y=p, sigma=p, s_stride=0, groups=p, nG=G, W=p, w_stride=D, A=p, a_stride=G,
             sl="default", nD=D, flags=0, dT=p, ws=None, nbytes=0, rows=n):
        sl = tables() if sl == "default" else sl
        return L.b2_glm_group_gather_sum(kind, X, y, sigma, s_stride, groups, nG, W, w_stride, A, a_stride, sl, None,
                                         rows, nD, P, 1.0, 1.0, 1.0, flags, None, None, None, None, None, dT, ws,
                                         nbytes, None)

    assert call() == -5                                                    # valid: the workspace check is next
    for k in ("X", "y", "groups", "W", "A", "dT"):
        assert call(**{k: None}) == -4, k
    assert call(kind=N.GLM_NORMAL, sigma=None) == -4 and call(sigma=None) == -5
    assert call(kind=N.GLM_BINOMIAL) == -2 and call(kind=N.GLM_CATEGORICAL) == -2 and call(kind=7) == -2
    for kind in (N.GLM_BERNOULLI, N.GLM_NORMAL):
        assert call(kind=kind) == -5
    assert call(nG=0, a_stride=0) == -2 and call(nD=0, w_stride=0) == -2 and call(rows=0) == -2
    assert call(nD=129, w_stride=129) == -2 and call(nD=128, w_stride=128) == -5
    assert call(nG=65537) == -2 and call(nG=65536, a_stride=0, sl=tables(strides=(0, 0, 0))) == -5
    assert call(w_stride=0) == -5 and call(a_stride=0) == -5 and call(w_stride=D - 1) == -2
    assert call(a_stride=G - 1) == -2
    assert call(X=q) == -2 and call(y=q) == -2 and call(groups=q) == -2
    assert call(kind=N.GLM_NORMAL, s_stride=2) == -2 and call(kind=N.GLM_NORMAL, s_stride=1) == -5
    assert call(flags=N.B2_FLAG_GLM_FP32) == -2 and call(flags=N.B2_FLAG_GLM_3XTF32) == -5
    assert call(rows=1 << 31) == -8
    # the slopes: NULL or S = 0 is none; S, columns, tables, strides
    assert call(sl=None) == -5 and call(sl=tables(S=0)) == -5
    assert call(sl=tables(S=-1)) == -2 and call(sl=tables(S=4)) == -2
    assert call(sl=tables(S=1, beta=(0, 4096, 4096))) == -4 and call(sl=tables(S=3, beta=(4096, 4096, 0))) == -4
    for cols in ((3, -1, 0), (3, D, 0), (3, 7, 3), (3, 3, 0)):
        assert call(sl=tables(S=3, cols=cols)) == -2, cols
    assert call(sl=tables(S=2, cols=(3, 7, 3))) == -5                 # only the first S columns are read
    assert call(sl=tables(S=2, strides=(G - 1, 0, 0))) == -2 and call(sl=tables(S=2, strides=(0, 3, 0))) == -2
    # narrow widths are taken too
    assert call(nG=5, a_stride=5, sl=tables(S=1, strides=(0, 0, 0))) == -5
    need = int(L.b2_glm_group_gather_sum_workspace(N.GLM_POISSON, n, D, G, 2, P))
    assert call(ws=p, nbytes=need - 1) == -5
    for kind in (N.GLM_BINOMIAL, N.GLM_CATEGORICAL):
        assert L.b2_glm_group_gather_sum_workspace(kind, n, D, G, 2, P) == 256
    for bad in ((n, D, G, 4, P), (n, D, 65537, 0, P), (n, 129, G, 0, P), (0, D, G, 0, P), (n, D, G, -1, P)):
        assert L.b2_glm_group_gather_sum_workspace(N.GLM_POISSON, *bad) == 256, bad


def test_workspace_grows_with_groups_slopes_and_particles_not_rows():
    L = N.lib()

    def ws(n=1_000_000, D=16, G=1000, S=1, P=64):
        return int(L.b2_glm_group_gather_sum_workspace(N.GLM_BERNOULLI, n, D, G, S, P))
    base = ws()
    assert ws(G=10000) > base and ws(S=3) > base and ws(P=65) > base
    # past the point where every SM has its CTA, more rows add nothing (the CTA partials stop growing)
    assert ws(n=1_000_000) == ws(n=100_000_000 // 64 * 64) == ws(n=(1 << 31) - 1)
    # the tables: (1 + S) G cp floats twice; the slots and status: per range, not per row
    assert ws(G=10000) - base >= 2 * 2 * 9000 * 64 * 4
    assert L.b2_glm_group_gather_sum_workspace(N.GLM_BERNOULLI, 1 << 31, 16, 1000, 1, 64) == 256


# ---- CPU tier: what ptxas makes of the new kernels -------------------------------------------------------------------
@pytest.fixture(scope="module")
def group_log(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, _ = sass_test._tools()
    obj = str(tmp_path_factory.mktemp("glm_group_gather_sum") / "glm_group.o")
    src = os.path.join(_build.CSRC, "glm_group.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", ["glm_group_gather_sum_pack_kernel", "glm_group_gather_sum_finish_kernel"])
def test_new_kernels_have_no_stack_frame_or_spills(group_log, kernel):
    import test_glm_tc_sass as sass_test
    props, used = sass_test._ptxas_properties(group_log, kernel)
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used


# ---- GPU tier: the call against fp64 ----------------------------------------------------------------------------------
def _layout(n, G, layout, seed):
    """A sorted [N] index: random groups, all rows in group 0, three groups spanning many ranges with the rest empty,
    one group per 64-row tile (runs ending on tile boundaries, the groups past the last tile empty)."""
    gen = torch.Generator().manual_seed(seed)
    if layout == "random":
        g = torch.randint(0, G, (n,), generator=gen)
    elif layout == "one":
        g = torch.zeros(n, dtype=torch.int64)
    elif layout == "span":
        g = torch.arange(n) * 3 // n * (G // 3)
    else:
        g = (torch.arange(n) // 64).clamp(max=G - 1)
    return torch.sort(g).values


def _gather_launch(kind, X, y, g32, W, A, Bs, cols, b, sigma, shared=(), flags=0):
    n, D = X.shape
    G, S = A.shape[-1], len(Bs)
    P = b.shape[0]
    dev = torch.device(DEV)
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dW = torch.empty(P, D, device=DEV)
    db = torch.empty(P, device=DEV)
    dsig = torch.empty(P, device=DEV)
    dT = torch.empty(1 + S, P, G, device=DEV)
    code = KIND_CODE[kind]
    sl = N.b2_glm_slope_tables(S)
    for k in range(S):
        sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], Bs[k].data_ptr(), 0 if "beta" in shared else G
    ws = N.workspace(dev, int(N.lib().b2_glm_group_gather_sum_workspace(code, n, D, G, S, P)), tag="glm_gather_test")
    N.check(N.lib().b2_glm_group_gather_sum(
        code, X.data_ptr(), y.data_ptr(), sigma.data_ptr(), 1, g32.data_ptr(), G, W.data_ptr(),
        0 if "w" in shared else D, A.data_ptr(), 0 if "alpha" in shared else G, ctypes.byref(sl), b.data_ptr(), n, D,
        P, 1.0, 1.0, 1.0, flags, sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(), db.data_ptr(), dsig.data_ptr(),
        dT.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)), "b2_glm_group_gather_sum")
    torch.cuda.synchronize()
    return sum_p, total, dW, db, dsig, dT


# (kind, n, D, G, S, P, layout, shared): P = 1, 64, 65; D = 1, 31, 33, 128; ragged N, so a partial last tile falls
# anywhere in its range; G from 38 to 65536
_CASES = [("Bernoulli", 8192, 1, 38, 1, 1, "random", ""),
          ("Poisson", 33793, 31, 1000, 3, 64, "random", "beta"),
          ("Normal", 250001, 33, 10000, 1, 65, "random", ""),
          ("Bernoulli", 250001, 128, 65536, 0, 64, "tile", ""),
          ("Normal", 33793, 16, 39, 2, 65, "span", "w,alpha"),
          ("Poisson", 250001, 16, 38, 0, 1, "one", ""),
          ("Bernoulli", 33793, 33, 85, 2, 65, "tile", ""),
          ("Poisson", 8192, 128, 2000, 1, 64, "span", ""),
          ("Normal", 250001, 31, 65536, 3, 64, "random", "alpha,beta")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _CASES, ids=["%s-%d-D%d-G%d-S%d-P%d-%s-%s" % c for c in _CASES])
def test_gather_sum_against_fp64(case):
    """sum_p and total within 2e-6 relative; dW, db and dsigma within 2e-4 of their largest entry, each block of
    out_dT within 5e-4 (2^-11, one TF32 rounding: a group of a few rows sums a few TF32-rounded residuals, which
    do not average out); empty groups exactly 0; two calls bitwise equal."""
    if EMULATE:
        pytest.skip("kernel test")
    kind, n, D, G, S, P, layout, shared = case
    shared = shared.split(",")
    cols = _cols(D, S)
    X, _, y, m = _data(kind, n, D, 7, S=S, seed=n + D, cols=cols)
    g = _layout(n, G, layout, n + G).to(DEV)
    # the labels of a model with this index, drawn from tables of their own (not the operands, whose gradients would
    # then be pure noise)
    W, A, Bs, b, sigma = _operands(n, D, G, S, P, shared, P + D + S)
    gen = torch.Generator(device=DEV).manual_seed(1)
    eta = X @ (0.3 * torch.randn(D, device=DEV, generator=gen) / D ** 0.5) + 0.3
    eta = eta + 0.5 * torch.randn(G, device=DEV, generator=gen)[g]
    for c in cols:
        eta = eta + 0.3 * torch.randn(G, device=DEV, generator=gen)[g] * X[:, c]
    if kind == "Bernoulli":
        y = torch.bernoulli(torch.sigmoid(eta), generator=gen)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta.clamp(max=8.0)), generator=gen)
    else:
        y = eta + 0.6 * torch.randn(n, device=DEV, generator=gen)
    g32 = g.to(torch.int32)
    out = _gather_launch(kind, X, y, g32, W, A, Bs, cols, b, sigma, shared)
    sum_p, total, dW, db, dsig, dT = out
    s_ref, (gW, gA, gb, gs, *gB) = _reference(kind, X, y, m, g, W, A, Bs, cols, b, sigma, P)

    def rel(got, want):
        return float((got.double() - want).abs().max()) / max(float(want.abs().max()), 1e-30)
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    et = abs(float(total) - float(s_ref.sum())) / abs(float(s_ref.sum()))
    errs = {"dW": rel(dW, gW), "db": rel(db, gb), "dalpha": rel(dT[0], gA)}
    for k in range(S):
        errs["dbeta%d" % k] = rel(dT[k + 1], gB[k])
    if kind == "Normal":
        errs["dsigma"] = rel(dsig, gs)
    print("\n%s: sum %.1e total %.1e %s" % (case, es, et, " ".join("%s %.1e" % kv for kv in errs.items())))
    tol = {k: 5e-4 if k.startswith(("dalpha", "dbeta")) else 2e-4 for k in errs}
    assert es <= 2e-6 and et <= 2e-6 and all(e <= tol[k] for k, e in errs.items()), (es, et, errs)
    # the empty groups get exactly 0
    empty = torch.bincount(g, minlength=G) == 0
    if bool(empty.any()):
        assert bool((dT[:, :, empty] == 0).all())
    again = _gather_launch(kind, X, y, g32, W, A, Bs, cols, b, sigma, shared)
    for i, (u, v) in enumerate(zip(out, again)):
        assert i == 4 and kind != "Normal" or torch.equal(u, v), i     # dsigma is written for Normal only


@pytest.mark.gpu
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_narrow_widths_agree_with_the_one_hot_call(kind):
    """At D + G (1 + S) <= 128 the gathered call and b2_glm_group_slope_sum with B2_FLAG_GLM_3XTF32 agree to fp32
    rounding: both take the same TF32-rounded residuals, but the gathered walk sums each group's run of about 3 000
    rows in row order in fp32 and the one-hot contraction in its own order, so the table gradients are compared to
    1e-4 of their largest entry."""
    if EMULATE:
        pytest.skip("kernel test")
    from test_glm_slope_svi import _launch as slope_launch
    n, D, G, S, P = 70001, 16, 24, 2, 64
    cols = _cols(D, S)
    X, g, y, m = _wide(kind, n, D, G, S, seed=31)
    W, A, Bs, b, sigma = _operands(n, D, G, S, P, [], 32)
    g32 = g.to(torch.int32)
    sum_p, total, dW, db, dsig, dT = _gather_launch(kind, X, y, g32, W, A, Bs, cols, b, sigma)
    s_p, s_total, dWAB, s_db, s_dsig = slope_launch(kind, X, y, m, g32, W, A, Bs, cols, b, sigma,
                                                    N.B2_FLAG_GLM_3XTF32)

    def close(u, v, tol=2e-5):
        assert float((u - v).abs().max()) <= tol * float(v.abs().max()), (float((u - v).abs().max()),
                                                                          float(v.abs().max()))
    close(sum_p, s_p, 2e-6)
    close(db, s_db)
    close(dW, dWAB[:, :D])
    for k in range(1 + S):
        close(dT[k], dWAB[:, D + k * G:D + (k + 1) * G], 1e-4)
    if kind == "Normal":
        close(dsig, s_dsig)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["out_of_range", "descending_pair"])
def test_bad_index_gives_nan_total_and_table_gradients(bad):
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G, S, P = 70001, 16, 300, 1, 8
    cols = _cols(D, S)
    X, g, y, _ = _wide("Bernoulli", n, D, G, S, seed=41)
    W, A, Bs, b, sigma = _operands(n, D, G, S, P, [], 42)
    for where in (4321, n - 1):
        g32 = g.to(torch.int32)
        if bad == "out_of_range":
            g32[where] = G
        else:
            steps = torch.nonzero(g32[1:] > g32[:-1]).reshape(-1)      # the step up nearest `where` goes down
            i = int(steps[(steps - where).abs().argmin()])
            g32[i], g32[i + 1] = int(g32[i + 1]), int(g32[i])
        sum_p, total, _, _, _, dT = _gather_launch("Bernoulli", X, y, g32, W, A, Bs, cols, b, sigma)
        assert bool(torch.isnan(total)) and bool(torch.isnan(sum_p).all()) and bool(torch.isnan(dT).all()), where
    # a good call on the same workspace afterwards is finite again (status is rewritten every call)
    sum_p, total, _, _, _, dT = _gather_launch("Bernoulli", X, y, g.to(torch.int32), W, A, Bs, cols, b, sigma)
    assert bool(torch.isfinite(total)) and bool(torch.isfinite(dT).all())


# ---- GPU tier: SVI --------------------------------------------------------------------------------------------------
def _elbo_grads(model, guide, args, lazy, P):
    """One Trace_ELBO.loss_and_grads at the initial parameters with injected guide noise: the loss and the gradient
    of each unconstrained parameter."""
    pyro.clear_param_store()
    X, G = args[0], args[5]
    shapes = {"w": (X.shape[1],), "b": (), "sigma": (), "alpha": (G,), "beta0": (G,), "s_b0": (), "eb0": (G,)}
    gen = torch.Generator().manual_seed(7)
    bufs = {k: torch.randn((P, 1) + sh, generator=gen).to(X.device) for k, sh in shapes.items()}

    def noisy_guide(*a):
        with _Noise(bufs):
            guide(*a)
    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    try:
        loss = Trace_ELBO(num_particles=P, vectorize_particles=True, max_plate_nesting=1).loss_and_grads(
            model, noisy_guide, *args)
    finally:
        elbo_mod.LAZY_LINEAR = saved
    return float(loss), {k: p.grad.detach().clone() for k, p in pyro.get_param_store().named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_svi_matches_materialised(kind):
    """N = 1e5, D = 16, G = 2 000, S = 1, 16 particles: four Trace_ELBO + ClippedAdam steps make one gathered call
    each, with losses within 2e-5 relative of LAZY_LINEAR = False; and the ELBO's gradient of every parameter is
    within 2e-4 of its largest entry.  (Parameters after Adam steps are not compared: Adam's first steps are about lr
    times the sign of each gradient entry, and with 50 rows per group some entries lie within TF32 rounding of 0.)"""
    if EMULATE:
        pytest.skip("kernel test")
    X, g, y, m = _wide(kind, 100_000, 16, 2000, 1, seed=11)
    model, guide = slope_model(kind, "noncentred", 1, cols=[0]), slope_guide(kind, "noncentred", 1)
    args = (X, g, y, m, None, 2000)
    l_f, _, calls, metas = _svi(model, guide, args, 4, True, P=16)
    l_m, _, calls_m, _ = _svi(model, guide, args, 4, False, P=16)
    assert calls == 4 and calls_m == 0 and not metas
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    lf, gf = _elbo_grads(model, guide, args, True, 16)
    lm, gm = _elbo_grads(model, guide, args, False, 16)
    assert abs(lf - lm) <= 2e-5 * abs(lm), (lf, lm)
    for k in gm:
        err = float((gf[k] - gm[k]).abs().max()) / float(gm[k].abs().max())
        assert err <= 2e-4, (k, err)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Bernoulli", "Normal"])
def test_captured_graph_step_equals_eager(kind):
    """A JitTrace_ELBO (graph-captured) run equals the eager one bit for bit; every gathered site is four launches."""
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, g, y, m = _wide(kind, 70000, 16, 500, 2, seed=14)
    model, guide = slope_model(kind, S=2, cols=_cols(16, 2)), slope_guide(kind, S=2)
    per_call = []
    real = dist._GlmGatherFn.launch

    def counted(*a):
        n0 = N.launch_count()
        out = real(*a)
        per_call.append(N.launch_count() - n0)
        return out
    dist._GlmGatherFn.launch = counted
    try:
        l_e, p_e, n_e, _ = _svi(model, guide, (X, g, y, m, None, 500), 4, True, P=16)
        l_g, p_g, n_g, _ = _svi(model, guide, (X, g, y, m, None, 500), 4, True, JitTrace_ELBO, P=16)
    finally:
        dist._GlmGatherFn.launch = real
    assert n_e == 4 and n_g >= 1 and per_call and set(per_call) == {4}, per_call
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["unsorted", "index_on_cpu", "binomial"])
def test_fallbacks_match_materialised(case):
    """Wide sites outside the gathered scope make no fused call and match LAZY_LINEAR = False to 1e-6."""
    if EMULATE:
        pytest.skip("kernel test")
    kind = "Binomial" if case == "binomial" else "Poisson"
    X, g, y, m = _data(kind, 9000, 16, 120, S=1, seed=15, cols=[0])
    if case != "unsorted":
        X, g, y, m = _sorted(X, g, y, m)
    if case == "index_on_cpu":
        g = g.cpu()
    model, guide = slope_model(kind, S=1, cols=[0]), slope_guide(kind, S=1)
    l_f, p_f, calls, metas = _svi(model, guide, (X, g, y, m, None, 120), 2, True, P=4)
    l_m, p_m, _, _ = _svi(model, guide, (X, g, y, m, None, 120), 2, False, P=4)
    assert calls == 0 and not metas
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 1e-6 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=1e-6, rtol=1e-6), k


@pytest.mark.gpu
def test_reference_pyro_model_under_bind_matches_materialised():
    """Radon-shaped multilevel logistic regression (85 groups, one slope, 171 columns, rows sorted by group) written
    against the unmodified reference, through bind.Trace_ELBO: the gathered call scores the site, and three steps
    match the model whose logits are materialised by ``* 1.0``."""
    if EMULATE:
        pytest.skip("kernel test")
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as rpyro
    import pyro.distributions as rdist
    X, g, y, _ = _wide("Bernoulli", 70000, 16, 85, 1, seed=16)

    def run(lazy):
        torch.manual_seed(0)

        def model(X, g, y):
            D = X.shape[-1]
            w = rpyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
            b = rpyro.sample("b", rdist.Normal(X.new_zeros(()), 5.0))
            a = rpyro.sample("alpha", rdist.Normal(X.new_zeros(85), 0.5).to_event(1))
            be = rpyro.sample("beta", rdist.Normal(X.new_zeros(85), 0.3).to_event(1))
            with rpyro.plate("data", X.shape[0]):
                logits = w.squeeze(-2) @ X.T + b + a.squeeze(-2)[..., g] + be.squeeze(-2)[..., g] * X[:, 0]
                rpyro.sample("y", rdist.Bernoulli(logits=logits if lazy else logits * 1.0), obs=y)

        def guide(X, g, y):
            D = X.shape[-1]
            for name, shape in (("w", (D,)), ("b", ()), ("alpha", (85,)), ("beta", (85,))):
                loc = rpyro.param(name + "_loc", X.new_zeros(shape))
                scale = rpyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=rdist.constraints.positive)
                d = rdist.Normal(loc, scale)
                rpyro.sample(name, d.to_event(1) if shape else d)

        rpyro.clear_param_store()
        calls = []
        real = dist._GlmGatherFn.apply
        dist._GlmGatherFn.apply = lambda *a: calls.append(1) or real(*a)
        try:
            svi = bind.SVI(model, guide, bind.ClippedAdam({"lr": 0.01}),
                           bind.Trace_ELBO(num_particles=16, vectorize_particles=True, max_plate_nesting=1))
            losses = [svi.step(X, g, y) for _ in range(3)]
        finally:
            dist._GlmGatherFn.apply = real
        store = rpyro.get_param_store()
        return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls)

    l_f, p_f, calls = run(True)
    l_m, p_m, calls_m = run(False)
    assert calls == 3 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k
