"""Multilevel regression under SVI: ``X @ w + b + alpha[g]`` kept lazy by pyro_b200/lazy.py and scored by
``b2_glm_group_sum``, one pass of the family's fused kernel over ``[X | onehot(g)]`` with d/dalpha from the same
contraction, for logistic, Poisson, linear and Binomial regression.

CPU tier: every spelling of the gather stays lazy and its ``dense()`` equals the model's eager expression bit for bit;
every other use, and every near miss, materialises exactly; SVI steps of all four families with the kernel seam
replaced by an fp64 torch restatement match ``LAZY_LINEAR = False``; an out-of-range index raises IndexError before
anything reads it; the entry point's argument checks; what ptxas makes of the group kernels with X rounded to TF32.
GPU tier: the kernel against fp64 (every kind and count form, shared and per-particle w and alpha, both precisions,
P = 1, 64, 65, ragged N, D + G on each side of 32, 64 and 96), determinism, the IndexError of an out-of-range index,
SVI steps against the materialised path, a captured-graph step against the eager one, the fallbacks, and
``bind.Trace_ELBO`` with reference Pyro."""
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
from pyro_b200 import poutine
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO, TraceMeanField_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.lazy import LinearPredictorTensor, SiteValue
from pyro_b200.optim import ClippedAdam

DEV = device()
KINDS = ["Bernoulli", "Poisson", "Normal", "Binomial"]
KIND_CODE = {"Bernoulli": N.GLM_BERNOULLI, "Poisson": N.GLM_POISSON, "Normal": N.GLM_NORMAL,
             "Binomial": N.GLM_BINOMIAL, "BinomialRows": N.GLM_BINOMIAL}
TRIALS = 10.0


# ---- models ------------------------------------------------------------------------------------------------------
def _likelihood(kind, eta, sigma, m):
    if kind == "Bernoulli":
        return dist.Bernoulli(logits=eta)
    if kind == "Poisson":
        return dist.Poisson(torch.exp(eta))
    if kind == "Binomial":
        return dist.Binomial(m, logits=eta)
    return dist.Normal(eta, sigma)


def group_model(kind, form="centred", spelling="ellipsis", order="w_first", change=None):
    """Regression of ``kind`` with a varying intercept ``alpha ~ Normal(0, 0.5)[G]`` (centred) or ``s_a * eta`` with a
    latent scale (non-centred), gathered by the int64 group index ``g``.  ``order``: where the gather is added (after
    the bias, before it, or in front of ``X @ w``); ``change`` makes a fallback or a near miss."""
    def model(X, g, y, m=None, mask=None, G=6):
        D = X.shape[-1]
        w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
        sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.0))) if kind == "Normal" else None
        if form == "centred":
            A = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
            A = A.squeeze(-2) if A.dim() > 1 else A
            ag = {"ellipsis": lambda: A[..., g], "index_select": lambda: A.index_select(-1, g),
                  "torch_index_select": lambda: torch.index_select(A, -1, g)}[spelling]()
        else:
            s = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
            e = pyro.sample("eta", dist.Normal(X.new_zeros(G), 1.0).to_event(1))
            e = e.squeeze(-2) if e.dim() > 1 else e
            ag = s * e[..., g]
        if change == "offset":
            ag = ag + 0.25
        lin = w.squeeze(-2) @ X.T if w.dim() > 1 else X @ w
        with pyro.plate("data", X.shape[0]):
            if order == "w_first":
                eta = lin + b + ag
            elif order == "group_before_bias":
                eta = (lin + ag) + b
            else:
                eta = ag + (lin + b)
            d = _likelihood(kind, eta, sigma, m)
            if mask is not None:
                d = d.mask(mask)
            pyro.sample("y", d, obs=y)
    return model


def group_guide(kind, form="centred"):
    def guide(X, g, y, m=None, mask=None, G=6):
        D = X.shape[-1]
        sites = [("w", (D,)), ("b", ())]
        if kind == "Normal":
            sites.append(("sigma_u", ()))
        sites += [("alpha", (G,))] if form == "centred" else [("s_u", ()), ("eta", (G,))]
        for name, shape in sites:
            loc = pyro.param(name + "_loc", X.new_zeros(shape))
            scale = pyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=dist.constraints.positive)
            d = dist.Normal(loc, scale)
            d = d.to_event(1) if shape else d
            if name == "sigma_u":
                pyro.sample("sigma", dist.LogNormal(loc, scale))
            elif name == "s_u":
                pyro.sample("s_a", dist.LogNormal(loc, scale))
            else:
                pyro.sample(name, d)
    return guide


def _data(kind, n, D, G, seed=0, dev=DEV):
    gen = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=gen)
    g = torch.randint(0, G, (n,), generator=gen)
    a = 0.5 * torch.randn(G, generator=gen)
    eta = X @ (0.3 * torch.randn(D, generator=gen) / D ** 0.5) + 0.3 + a[g]
    m = torch.randint(1, 20, (n,), generator=gen).float() if kind == "BinomialRows" else torch.full((n,), TRIALS)
    if kind == "Bernoulli":
        y = torch.bernoulli(torch.sigmoid(eta), generator=gen)
    elif kind == "Poisson":
        y = torch.poisson(torch.exp(eta), generator=gen)
    elif kind == "Normal":
        y = eta + 0.6 * torch.randn(n, generator=gen)
    else:
        y = torch.binomial(m, torch.sigmoid(eta), generator=gen)
    return X.to(dev), g.to(dev), y.to(dev), m.to(dev)


# ---- CPU tier: lazy semantics -------------------------------------------------------------------------------------
def _mk(P=4, n=50, D=6, G=5):
    torch.manual_seed(0)
    X = torch.randn(n, D)
    g = torch.randint(0, G, (n,))
    w, b = torch.randn(P, 1, D), torch.randn(P, 1)
    A, A1 = torch.randn(P, 1, G), torch.randn(G)
    s = torch.rand(P, 1) + 0.5
    return X, g, w, b, A, A1, s


def _sv(t):
    return SiteValue.wrap(t.clone())


def test_every_spelling_stays_lazy_and_dense_equals_the_eager_expression_bitwise():
    X, g, w, b, A, A1, s = _mk()
    ws, bs, As, A1s, ss = _sv(w), _sv(b), _sv(A), _sv(A1), _sv(s)
    lin, lin_e = ws.squeeze(-2) @ X.T, w.squeeze(-2) @ X.T
    Ap, A2 = As.squeeze(-2), A.squeeze(-2)
    A2s = _sv(A2)
    gathers = [  # (lazy gather, eager gather)
        (Ap[..., g], A2[..., g]), (A2s[..., g], A2[..., g]), (Ap.index_select(-1, g), A2.index_select(-1, g)),
        (torch.index_select(Ap, -1, g), torch.index_select(A2, -1, g)), (A1s[g], A1[g]), (A1s[..., g], A1[..., g]),
        (ss * Ap[..., g], s * A2[..., g]), (Ap[..., g] * ss, A2[..., g] * s), (0.7 * Ap[..., g], 0.7 * A2[..., g]),
        (ss * A1s[..., g], s * A1[..., g]), (_sv(torch.tensor([1.3])) * Ap[..., g], torch.tensor([1.3]) * A2[..., g]),
    ]
    n_cases = 0
    for i, (lz, ref) in enumerate(gathers):
        assert isinstance(lz, LinearPredictorTensor) and isinstance(lz.lazy, dist.GroupGather), i
        assert torch.equal(lz.dense(), ref), i
        for j, (got, want) in enumerate([(lin + bs + lz, lin_e + b + ref), ((lin + lz) + bs, (lin_e + ref) + b),
                                         (lz + (lin + bs), ref + (lin_e + b)), (lz + lin, ref + lin_e),
                                         (bs + (lin + lz), b + (lin_e + ref))]):
            assert isinstance(got, LinearPredictorTensor) and isinstance(got.lazy, dist.LinearPredictor), (i, j)
            assert got.lazy.group is not None and got.shape == want.shape, (i, j)
            assert torch.equal(got.dense(), want), (i, j)
            assert torch.equal(torch.exp(got).dense(), torch.exp(want)), (i, j)           # the Poisson rate
            nd = dist.Normal(got, 0.6)
            assert type(nd).__name__ == "_NormalLinear" and torch.equal(nd.loc, want), (i, j)   # the Normal loc
            bd = dist.Binomial(torch.tensor(TRIALS), logits=got)
            assert type(bd).__name__ == "_BinomialLinear" and torch.equal(bd.logits, want), (i, j)
            assert type(dist.Bernoulli(logits=got)).__name__ == "_BernoulliLinear", (i, j)
            n_cases += 1
    # a shared weight vector: X @ w [N] plus a [G] table
    w1, b1 = torch.randn(6), torch.randn(())
    got = X @ _sv(w1) + _sv(b1) + A1s[g]
    assert got.lazy.group is not None and torch.equal(got.dense(), X @ w1 + b1 + A1[g])
    assert n_cases == 5 * len(gathers)


def test_other_uses_materialise_exactly():
    X, g, w, b, A, A1, s = _mk()
    Ap, A2 = _sv(A).squeeze(-2), A.squeeze(-2)
    lin, lin_e = _sv(w).squeeze(-2) @ X.T, w.squeeze(-2) @ X.T
    off = torch.randn(50)
    cases = [(Ap[..., g] + off, A2[..., g] + off), (Ap[..., g] + 1.0, A2[..., g] + 1.0),
             (Ap[..., g] * torch.randn(50), None), (Ap[..., g].sum(), A2[..., g].sum()),
             (Ap[..., g].exp(), A2[..., g].exp()), (Ap[..., g].isfinite(), A2[..., g].isfinite()),
             (torch.broadcast_tensors(Ap[..., g], off)[0], torch.broadcast_tensors(A2[..., g], off)[0]),
             (Ap[..., g].detach(), A2[..., g].detach()), (Ap[..., g][..., g], A2[..., g][..., g]),
             (Ap[g[:4] % 4], A2[g[:4] % 4]),                                       # a dim-0 gather of a 2-d value
             ((_sv(A)[..., g] + lin), A[..., g] + lin_e)]                          # [P, 1, N]: broadcasts to [P, P, N]
    for i, (got, want) in enumerate(cases):
        # a plain tensor (a dim-0 gather is a view of the site value, which stays a SiteValue as before)
        assert type(got) in (torch.Tensor, SiteValue), (i, type(got))
        if want is not None:
            assert torch.equal(got.as_subclass(torch.Tensor), want), i
    # a second group effect materialises the sum (the first stays as written)
    two = lin + Ap[..., g] + Ap[..., g]
    assert type(two) is torch.Tensor and torch.equal(two, lin_e + A2[..., g] + A2[..., g])
    # near misses of the index: float (torch refuses it the same way), requires grad, 2-d
    with pytest.raises(IndexError):
        Ap[..., g.float()]
    with pytest.raises(IndexError):
        A2[..., g.float()]
    for idx in (g.reshape(5, 10), g.to(torch.int32)):
        got = Ap[..., idx]
        assert type(got) is not LinearPredictorTensor and torch.equal(got.as_subclass(torch.Tensor), A2[..., idx])


# ---- CPU tier: SVI with the kernel seam replaced by an fp64 torch restatement ----------------------------------------
def _fp64_launch(meta, X, y, W, b, A, sigma):
    """What b2_glm_group_sum returns, restated in fp64 with torch.distributions and autograd."""
    scale, weight, coeff, _, kind, idx, trials, per_row, s_stride = meta
    ops = [t.detach().double().requires_grad_(t.requires_grad) if t is not None else None for t in (W, b, A, sigma)]
    Wd, bd, Ad, sd = ops
    G = A.shape[-1]
    with torch.enable_grad():
        eta = Wd @ X.double().T + Ad.reshape(-1, G)[:, idx.long()]
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


class _Noise(poutine.Messenger):
    """The guide's draws as loc + eps * scale (exp of that for LogNormal) with recorded eps, so two runs see the same
    noise (the technique of models.InjectNoise)."""

    def __init__(self, eps):
        self.eps = eps

    def _pyro_sample(self, msg):
        if msg["name"] in self.eps and not msg["is_observed"]:
            base = msg["fn"]
            while hasattr(base, "base_dist"):
                base = base.base_dist
            v = base.loc + self.eps[msg["name"]] * base.scale
            msg["value"] = v.exp() if isinstance(base, dist.LogNormal) else v
            msg["done"] = True


def _svi(kind, model, guide, args, steps, lazy, elbo_cls=Trace_ELBO, P=8, seed=0):
    """``steps`` SVI steps with guide noise from seed ``seed`` injected through fixed buffers; returns the losses, the
    parameters and the fused calls."""
    pyro.clear_param_store()
    X, G = args[0], args[5]
    shapes = {"w": (X.shape[1],), "b": (), "sigma": (), "alpha": (G,), "s_a": (), "eta": (G,)}
    gen = torch.Generator().manual_seed(seed)
    eps = {k: torch.randn((steps, P, 1) + sh, generator=gen, dtype=X.dtype).to(X.device) for k, sh in shapes.items()}
    bufs = {k: torch.empty_like(v[0]) for k, v in eps.items()}

    def noisy_guide(*a):
        with _Noise(bufs):
            guide(*a)
    calls = []
    real = dist._GlmGroupFn.apply
    dist._GlmGroupFn.apply = lambda *a: calls.append(1) or real(*a)
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
        dist._GlmGroupFn.apply = real
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls)


@pytest.fixture
def fp64_seam():
    """The CPU stand-ins of the native seams, with the group sum restated in fp64 (and _BernoulliLinear's own
    _fused_sum, which the stand-ins replace by the dense path)."""
    import cpu_emulation
    fused = dist._BernoulliLinear._fused_sum
    with cpu_emulation.enabled():
        dist._BernoulliLinear._fused_sum = fused
        saved = dist._GlmGroupFn.launch
        dist._GlmGroupFn.launch = _fp64_launch
        try:
            yield
        finally:
            dist._GlmGroupFn.launch = saved


@pytest.mark.parametrize("kind", KINDS + ["BinomialRows"])
@pytest.mark.parametrize("form", ["centred", "noncentred"])
def test_svi_on_the_lazy_route_matches_materialised_with_the_seam_restated(fp64_seam, kind, form):
    fam = "Binomial" if kind == "BinomialRows" else kind
    X, g, y, m = _data(kind, 8192, 5, 7, seed=3, dev="cpu")
    args = (X, g, y, m, None, 7)
    model, guide = group_model(fam, form), group_guide(fam, form)
    l_f, p_f, calls = _svi(fam, model, guide, args, 3, True)
    l_m, p_m, calls_m = _svi(fam, model, guide, args, 3, False)
    assert calls == 3 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 1e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=1e-5), k


def test_out_of_range_index_raises_before_anything_reads_it(fp64_seam):
    X, g, y, m = _data("Bernoulli", 8192, 5, 7, seed=4, dev="cpu")
    launched = []
    dist._GlmGroupFn.launch = lambda *a: launched.append(1)

    def refuse(self):
        raise AssertionError("materialised")
    saved = (dist.GroupGather.dense, dist.LinearPredictor.dense)
    dist.GroupGather.dense = dist.LinearPredictor.dense = refuse
    try:
        for bad in (-1, 7):
            g2 = g.clone()
            g2[100] = bad
            with pytest.raises(IndexError):
                _svi("Bernoulli", group_model("Bernoulli"), group_guide("Bernoulli"), (X, g2, y, m, None, 7), 1, True)
    finally:
        dist.GroupGather.dense, dist.LinearPredictor.dense = saved
    assert not launched


def test_index_copy_is_built_once_per_index_and_version():
    g = torch.randint(0, 5, (100,))
    c1 = dist.group_index_int32(g, 5)
    assert c1.dtype == torch.int32 and torch.equal(c1, g.to(torch.int32)) and c1.data_ptr() != g.data_ptr()
    assert dist.group_index_int32(g, 5) is c1
    g[3] = 4
    c2 = dist.group_index_int32(g, 5)
    assert c2 is not c1 and int(c2[3]) == 4
    with pytest.raises(IndexError):
        dist.group_index_int32(g, 4)


# ---- CPU tier: the entry point's argument checks -------------------------------------------------------------------
def test_group_sum_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p, q = ctypes.c_void_p(4096), ctypes.c_void_p(4100)
    D, G, P, n = 10, 20, 4, 10000

    def call(kind=N.GLM_POISSON, X=p, y=p, trials=p, per_row=0, sigma=p, s_stride=0, groups=p, nG=G, W=p, w_stride=D,
             A=p, a_stride=G, nD=D, flags=0, ws=None, nbytes=0, rows=n):
        return L.b2_glm_group_sum(kind, X, y, trials, per_row, sigma, s_stride, groups, nG, W, w_stride, A, a_stride,
                                  None, rows, nD, P, 1.0, 1.0, 1.0, flags, None, None, None, None, None, ws, nbytes,
                                  None)

    assert call() == -5                                                    # valid: the workspace check is next
    for k in ("X", "y", "groups", "W", "A"):
        assert call(**{k: None}) == -4, k
    assert call(kind=N.GLM_BINOMIAL, trials=None) == -4 and call(kind=N.GLM_NORMAL, sigma=None) == -4
    assert call(kind=N.GLM_CATEGORICAL) == -2 and call(kind=7) == -2
    for kind in (N.GLM_BERNOULLI, N.GLM_NORMAL, N.GLM_BINOMIAL):
        assert call(kind=kind) == -5
    assert call(nD=109, w_stride=109) == -2 and call(nD=108, w_stride=108) == -5     # D + G <= 128
    assert call(nG=0, a_stride=0) == -2 and call(nD=0, w_stride=0) == -2 and call(rows=0) == -2
    assert call(w_stride=0) == -5 and call(a_stride=0) == -5 and call(w_stride=D - 1) == -2 and call(a_stride=3) == -2
    assert call(X=q) == -2 and call(y=q) == -2 and call(groups=q) == -2
    assert call(kind=N.GLM_BINOMIAL, trials=q, per_row=1) == -2 and call(kind=N.GLM_BINOMIAL, trials=q) == -5
    assert call(kind=N.GLM_BINOMIAL, per_row=2) == -2
    assert call(kind=N.GLM_NORMAL, s_stride=2) == -2 and call(kind=N.GLM_NORMAL, s_stride=1) == -5
    assert call(flags=N.B2_FLAG_GLM_FP32) == -2 and call(rows=1 << 31) == -8
    need = int(L.b2_glm_group_sum_workspace(N.GLM_POISSON, n, D, G, P))
    assert need > 256 and call(ws=p, nbytes=need - 1) == -5
    assert L.b2_glm_group_sum_workspace(N.GLM_CATEGORICAL, n, D, G, P) == 256
    assert L.b2_glm_group_sum_workspace(N.GLM_POISSON, n, 100, 29, P) == 256


# ---- CPU tier: what ptxas makes of the group kernels with X rounded to TF32 -----------------------------------------
RN_KERNELS = ["glm_group_rn_tc_kernelINS_2tc9BernoulliELi%dE" % dc for dc in (1, 2, 3, 4)] + \
             ["glm_group_rn_tc_kernelINS_2tc7PoissonELi%dE" % dc for dc in (1, 2, 3, 4)] + \
             ["glm_group_rn_tc_kernelINS_2tc8BinomialILb%dEEELi%dE" % (r, dc) for r in (0, 1) for dc in (2, 3, 4)]


@pytest.fixture(scope="module")
def rn_sass(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, cuobjdump = sass_test._tools()
    obj = str(tmp_path_factory.mktemp("glm_group_rn") / "glm_group.o")
    src = os.path.join(_build.CSRC, "glm_group.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


@pytest.mark.parametrize("mangled", RN_KERNELS)
def test_rn_group_kernel_sass(rn_sass, mangled):
    """No C7515/C7520 serialisation note, no spills and no stack frame, and no warpgroup wait or arrive between two
    HGMMA of one contraction (GEMM 1 m64n64k8, GEMM 2 m64n(32 DC + 8)k8)."""
    import test_glm_tc_sass as sass_test
    log, sass = rn_sass
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


# ---- GPU tier: the kernel against fp64 ------------------------------------------------------------------------------
def _launch(kind, X, y, m, g32, W, A, b, sigma, flags, shared_w=False, shared_a=False):
    n, D = X.shape
    G = A.shape[-1]
    P = max(W.shape[0] if not shared_w else 1, A.shape[0] if not shared_a else 1, b.shape[0])
    dev = torch.device(DEV)
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dWA = torch.empty(P, D + G, device=DEV)
    db = torch.empty(P, device=DEV)
    dsig = torch.empty(P, device=DEV)
    code = KIND_CODE[kind]
    ws = N.workspace(dev, int(N.lib().b2_glm_group_sum_workspace(code, n, D, G, P)), tag="glm_group_test")
    N.check(N.lib().b2_glm_group_sum(
        code, X.data_ptr(), y.data_ptr(), m.data_ptr() if kind == "BinomialRows" else m[:1].clone().data_ptr(),
        int(kind == "BinomialRows"), sigma.data_ptr(), 1, g32.data_ptr(), G, W.data_ptr(), 0 if shared_w else D,
        A.data_ptr(), 0 if shared_a else G, b.data_ptr(), n, D, P, 1.0, 1.0, 1.0, flags, sum_p.data_ptr(),
        total.data_ptr(), dWA.data_ptr(), db.data_ptr(), dsig.data_ptr(), ws.data_ptr(), ws.numel(),
        N.stream_ptr(dev)), "b2_glm_group_sum")
    torch.cuda.synchronize()
    return sum_p, total, dWA, db, dsig


def _reference(kind, X, y, m, g, W, A, b, sigma, P):
    D, G = X.shape[1], A.shape[-1]
    Wd = W.double().expand(P, D).clone().requires_grad_(True)
    Ad = A.double().expand(P, G).clone().requires_grad_(True)
    bd = b.double().clone().requires_grad_(True)
    sd = sigma.double().clone().requires_grad_(True)
    eta = Wd @ X.double().T + bd[:, None] + Ad[:, g]
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
    gW, gA, gb, gs = torch.autograd.grad(s.sum(), [Wd, Ad, bd, sd], allow_unused=True)
    return s.detach(), gW, gA, gb, gs


# (n, D, G, P, shared, flags): ragged N from 8192 to 1e6, D + G = 31, 33, 63, 65, 95, 97, 128
_CASES = [(8192, 10, 21, 1, "none", "split"), (8193, 10, 23, 64, "w", "split"), (70001, 16, 47, 65, "alpha", "default"),
          (99999, 16, 49, 64, "none", "default"), (250003, 30, 65, 1, "w", "default"),
          (1_000_000, 30, 67, 65, "none", "split"), (1_000_000, 16, 48, 64, "alpha", "default"),
          (65537, 100, 28, 64, "none", "default")]
_KERNEL_KINDS = ["Bernoulli", "Poisson", "Normal", "Binomial", "BinomialRows"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _CASES, ids=["%d-D%d-G%d-P%d-%s-%s" % c for c in _CASES])
@pytest.mark.parametrize("kind", _KERNEL_KINDS)
def test_kernel_against_fp64(kind, case):
    """sum_p within 2e-6 relative, dW, d/dalpha and db within 2e-4 of the largest gradient; two launches bitwise
    equal."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G, P, shared, prec = case
    X, g, y, m = _data(kind, n, D, G, seed=n + D + G)
    gen = torch.Generator().manual_seed(P + D)
    W = (0.3 * torch.randn(1 if shared == "w" else P, D, generator=gen) / D ** 0.5).to(DEV)
    A = (0.5 * torch.randn(1 if shared == "alpha" else P, G, generator=gen)).to(DEV)
    b = (0.3 + 0.05 * torch.randn(P, generator=gen)).to(DEV)
    sigma = (0.6 + 0.1 * torch.rand(P, generator=gen)).to(DEV)
    flags = N.B2_FLAG_GLM_3XTF32 if prec == "split" else 0
    g32 = g.to(torch.int32)
    sum_p, total, dWA, db, dsig = _launch(kind, X, y, m, g32, W, A, b, sigma, flags, shared == "w", shared == "alpha")
    s_ref, gW, gA, gb, gs = _reference(kind, X, y, m, g, W, A, b, sigma, P)
    es = float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max())
    ew = float((dWA[:, :D].double() - gW).abs().max()) / float(gW.abs().max())
    ea = float((dWA[:, D:].double() - gA).abs().max()) / float(gA.abs().max())
    eb = float((db.double() - gb).abs().max()) / float(gb.abs().max())
    print("\n%s %s: sum %.1e dW %.1e dalpha %.1e db %.1e" % (kind, case, es, ew, ea, eb))
    assert es <= 2e-6 and ew <= 2e-4 and ea <= 2e-4 and eb <= 2e-4, (es, ew, ea, eb)
    if kind == "Normal":
        assert float((dsig.double() - gs).abs().max()) <= 2e-4 * float(gs.abs().max())
    again = _launch(kind, X, y, m, g32, W, A, b, sigma, flags, shared == "w", shared == "alpha")
    for u, v in zip((sum_p, total, dWA, db), again):
        assert torch.equal(u, v)


# ---- GPU tier: SVI -------------------------------------------------------------------------------------------------
_SVI_TOL = {"Bernoulli": 2e-5, "Poisson": 2e-5, "Normal": 2e-5, "Binomial": 2e-5}


@pytest.mark.gpu
@pytest.mark.parametrize("case", [("Bernoulli", "centred", "ellipsis", "w_first"),
                                  ("Bernoulli", "noncentred", "ellipsis", "group_before_bias"),
                                  ("Poisson", "centred", "index_select", "w_first"),
                                  ("Poisson", "noncentred", "ellipsis", "group_first"),
                                  ("Normal", "centred", "torch_index_select", "group_before_bias"),
                                  ("Normal", "noncentred", "ellipsis", "w_first"),
                                  ("Binomial", "centred", "ellipsis", "group_first"),
                                  ("Binomial", "noncentred", "index_select", "w_first"),
                                  ("BinomialRows", "centred", "ellipsis", "w_first")], ids=lambda c: "-".join(c))
def test_svi_matches_materialised(case):
    """Four Trace_ELBO + ClippedAdam steps at N = 70 000, D = 16, G = 48, 16 particles: one fused call per step,
    losses within 2e-5 relative and parameters within 2e-4 of LAZY_LINEAR = False."""
    if EMULATE:
        pytest.skip("kernel test")
    kind, form, spelling, order = case
    fam = "Binomial" if kind == "BinomialRows" else kind
    X, g, y, m = _data(kind, 70000, 16, 48, seed=11)
    model, guide = group_model(fam, form, spelling, order), group_guide(fam, form)
    l_f, p_f, calls = _svi(fam, model, guide, (X, g, y, m, None, 48), 4, True, P=16)
    l_m, p_m, calls_m = _svi(fam, model, guide, (X, g, y, m, None, 48), 4, False, P=16)
    assert calls == 4 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= _SVI_TOL[fam] * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_mean_field_elbo_matches_materialised():
    if EMULATE:
        pytest.skip("kernel test")
    X, g, y, m = _data("Poisson", 70000, 16, 48, seed=12)
    model, guide = group_model("Poisson"), group_guide("Poisson")
    l_f, p_f, calls = _svi("Poisson", model, guide, (X, g, y, m, None, 48), 3, True, TraceMeanField_ELBO, P=16)
    l_m, p_m, _ = _svi("Poisson", model, guide, (X, g, y, m, None, 48), 3, False, TraceMeanField_ELBO, P=16)
    assert calls == 3
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_out_of_range_index_raises_on_the_fused_path():
    """Nothing gathers with the bad index: both dense paths are replaced by a refusal, so only the fused path's range
    check (a comparison, not a gather) reads the index."""
    if EMULATE:
        pytest.skip("kernel test")
    X, g, y, m = _data("Bernoulli", 70000, 16, 48, seed=13)
    launched = []
    real = dist._GlmGroupFn.launch

    def refuse(self):
        raise AssertionError("materialised")
    saved = (dist.GroupGather.dense, dist.LinearPredictor.dense)
    dist.GroupGather.dense = dist.LinearPredictor.dense = refuse
    dist._GlmGroupFn.launch = lambda *a: launched.append(1)
    try:
        for bad in (-1, 48):
            g2 = g.clone()
            g2[1234] = bad
            with pytest.raises(IndexError):
                _svi("Bernoulli", group_model("Bernoulli"), group_guide("Bernoulli"), (X, g2, y, m, None, 48), 1,
                     True, P=16)
    finally:
        dist.GroupGather.dense, dist.LinearPredictor.dense = saved
        dist._GlmGroupFn.launch = real
    assert not launched


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Bernoulli", "Normal"])
def test_captured_graph_step_equals_eager(kind):
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, g, y, m = _data(kind, 70000, 16, 48, seed=14)
    model, guide = group_model(kind), group_guide(kind)
    l_e, p_e, n_e = _svi(kind, model, guide, (X, g, y, m, None, 48), 4, True, P=16)
    l_g, p_g, n_g = _svi(kind, model, guide, (X, g, y, m, None, 48), 4, True, JitTrace_ELBO, P=16)
    assert n_e == 4 and n_g >= 1
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["N8191", "masked", "fp64", "DG129", "no_tensor_cores", "index_on_cpu"])
def test_fallbacks_match_materialised(case):
    """Sites outside the fused scope make no fused call and match LAZY_LINEAR = False to 1e-6."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, G = (8191 if case == "N8191" else 9000), 16, (114 if case == "DG129" else 12)
    X, g, y, m = _data("Poisson", n, D, G, seed=15)
    mask = (torch.rand(n, device=DEV) < 0.7) if case == "masked" else None
    if case == "fp64":
        X, y = X.double(), y.double()
    if case == "index_on_cpu":
        g = g.cpu()
    model = group_model("Poisson")
    if case == "no_tensor_cores":
        def model(X, g, y, m=None, mask=None, G=6):
            D = X.shape[-1]
            w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
            b = pyro.sample("b", dist.Normal(X.new_zeros(()), 5.0))
            A = pyro.sample("alpha", dist.Normal(X.new_zeros(G), 0.5).to_event(1))
            with pyro.plate("data", X.shape[0]):
                lp = dist.LinearPredictor(X, w, b, tensor_cores=False)
                eta = LinearPredictorTensor(lp) + A.squeeze(-2)[..., g]
                pyro.sample("y", dist.Poisson(torch.exp(eta)), obs=y)
    guide = group_guide("Poisson")
    l_f, p_f, calls = _svi("Poisson", model, guide, (X, g, y, m, mask, G), 2, True, P=4)
    l_m, p_m, _ = _svi("Poisson", model, guide, (X, g, y, m, mask, G), 2, False, P=4)
    assert calls == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 1e-6 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=1e-6, rtol=1e-6), k


@pytest.mark.gpu
def test_reference_pyro_model_under_bind_matches_materialised():
    """The multilevel logistic model written against the unmodified reference, through bind.Trace_ELBO: the kernel
    scores the site, and three steps match the model whose logits are materialised by ``* 1.0``."""
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
            with rpyro.plate("data", X.shape[0]):
                logits = w.squeeze(-2) @ X.T + b + a.squeeze(-2)[..., g]
                rpyro.sample("y", rdist.Bernoulli(logits=logits if lazy else logits * 1.0), obs=y)

        def guide(X, g, y):
            D = X.shape[-1]
            for name, shape in (("w", (D,)), ("b", ()), ("alpha", (48,))):
                loc = rpyro.param(name + "_loc", X.new_zeros(shape))
                scale = rpyro.param(name + "_scale", X.new_full(shape, 0.1), constraint=rdist.constraints.positive)
                d = rdist.Normal(loc, scale)
                rpyro.sample(name, d.to_event(1) if shape else d)

        rpyro.clear_param_store()
        calls = []
        real = dist._GlmGroupFn.apply
        dist._GlmGroupFn.apply = lambda *a: calls.append(1) or real(*a)
        try:
            svi = bind.SVI(model, guide, bind.ClippedAdam({"lr": 0.01}),
                           bind.Trace_ELBO(num_particles=16, vectorize_particles=True, max_plate_nesting=1))
            losses = [svi.step(X, g, y) for _ in range(3)]
        finally:
            dist._GlmGroupFn.apply = real
        store = rpyro.get_param_store()
        return losses, {k: store[k].detach().clone() for k in store.keys()}, len(calls)

    l_f, p_f, calls = run(True)
    l_m, p_m, calls_m = run(False)
    assert calls == 3 and calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k
