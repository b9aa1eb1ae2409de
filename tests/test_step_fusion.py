"""The fixed cost of a Bayesian-logistic-regression SVI step: deferred Normal draws launched together at their first
read (one b2_latent_normal_draw for all sites, bitwise equal to separate launches), and the loss assembled in the
finish kernel of the fused GLM call (b2_glm_bernoulli_logits_elbo, bitwise equal to the separate
b2_latent_normal_prior_combine launch)."""
import ctypes

import pytest
import torch

import models
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from torch.distributions import constraints
from conftest import device, EMULATE
from pyro_b200 import _native as N
from pyro_b200.distributions import _ops
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO
from pyro_b200.optim import ClippedAdam

DEV = device()


def _data(n, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=g)
    y = (torch.rand(n, generator=g) < torch.sigmoid(X[:, 0] - 0.5 * X[:, 1])).float()
    return X.to(DEV), y.to(DEV)


def _run(elbo_cls, X, y, steps, assemble=True, batch_draws=True, P=64, model=models.logistic_model,
         guide=models.logistic_guide):
    pyro.clear_param_store()
    pyro.set_rng_seed(7)
    svi = SVI(model, guide, ClippedAdam({"lr": 0.02}),
              elbo_cls(num_particles=P, vectorize_particles=True, max_plate_nesting=1))
    take, draw = _ops.take_elbo_assembly, _ops.defer_latent_draw
    if not assemble:
        _ops.take_elbo_assembly = lambda device: (take(device), None)[1]
    if not batch_draws:
        # every draw launched on its own, at once (the behaviour the batched flush must reproduce)
        def draw_now(*a):
            out = draw(*a)
            _ops.flush_draws()
            return out
        _ops.defer_latent_draw = draw_now
    try:
        losses = [svi.step(X, y) for _ in range(steps)]
    finally:
        _ops.take_elbo_assembly, _ops.defer_latent_draw = take, draw
    store = pyro.get_param_store()
    params = {}
    for k in store.keys():
        v = store[k]
        params[k] = (v.dense() if hasattr(v, "dense") else v).detach().cpu().clone()
    return losses, params


def _assert_same(a, b):
    la, pa = a
    lb, pb = b
    assert la == lb
    assert pa.keys() == pb.keys()
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k


# ---- CPU: when the assembly is handed out ---------------------------------------------------------------
def test_assembly_taken_once_and_only_when_it_fits():
    z = torch.zeros(4, 1, 3)
    prior = (torch.zeros(3), torch.ones(3))
    term = torch.zeros(())
    assert _ops.take_elbo_assembly(z.device) is None                       # none open
    with _ops.elbo_assembly([(z, *prior)], [1.0], [term], [1.0], -1.0) as asm:
        got = _ops.take_elbo_assembly(z.device)
        assert got is not None and got[0] is asm and got[2] == 1 and got[6] == 2   # own total = last term
        assert _ops.take_elbo_assembly(z.device) is None                   # a later call does not see it
    assert asm.loss is None
    too_many = [(z, *prior)] * (N.LATENT_MAX_JOBS + 1)
    zd = z.double()
    for items, terms in ((too_many, [term]), ([(zd, prior[0].double(), prior[1].double())], [term.double()]),
                         ([(z, *prior)], [term] * N.LATENT_MAX_TERMS), ([], [term])):
        with _ops.elbo_assembly(items, [1.0] * len(items), terms, [1.0] * len(terms), -1.0):
            assert _ops.take_elbo_assembly(z.device) is None
    assert _ops._ELBO_ASSEMBLY is None


def test_deferred_value_is_flushed_before_any_read(monkeypatch):
    """A pending draw is launched before any torch operation reads a deferred value, a site value handed to the
    model, or a plain alias of one, and before any native launch; metadata queries leave it pending."""
    from pyro_b200.lazy import SiteValue
    calls = []
    monkeypatch.setattr(_ops, "_PENDING_DRAWS", [])

    def fake_flush():
        if _ops._PENDING_DRAWS:
            calls.append(1)
            _ops._PENDING_DRAWS.clear()
    monkeypatch.setattr(_ops, "flush_draws", fake_flush)
    monkeypatch.setattr(N, "before_launch", fake_flush)
    z = torch.zeros(4, 3).as_subclass(_ops.DeferredDraw)
    sv = z.as_subclass(SiteValue)
    reads = [lambda: z + 1, lambda: z.sum(), lambda: float(z[0, 0]), lambda: z.data_ptr(), lambda: repr(z),
             lambda: torch.stack([z, z]), lambda: sv.squeeze(-1), lambda: sv @ torch.ones(3),
             lambda: _ops.plain_value(sv), lambda: N.stream_ptr() if torch.cuda.is_available() else fake_flush()]
    for k, read in enumerate(reads):
        _ops._PENDING_DRAWS.append(("job", (), None))
        z.shape, z.dim(), z.numel(), z.dtype, z.device, z.is_contiguous(), sv.shape, sv.size(-1)
        assert len(_ops._PENDING_DRAWS) == 1 and len(calls) == k, k
        read()
        assert not _ops._PENDING_DRAWS and len(calls) == k + 1, k


def test_glm_elbo_entry_validates_arguments():
    L = N.lib()
    one = (N.b2_latent_job * 1)()
    j = one[0]
    j.dtype, j.ndim = N._DTYPES[torch.float32], 1
    j.shape[0] = 8
    d = ctypes.c_void_p(4096)                          # never dereferenced: validation fails first
    jc = (ctypes.c_double * 1)(1.0)
    tc = (ctypes.c_double * 1)(1.0)
    terms = (ctypes.c_void_p * 1)(None)
    ws = int(L.b2_glm_elbo_workspace())
    assert ws >= N.LATENT_MAX_JOBS * 32 * 8

    def call(out_total=d, jobs=one, n_jobs=1, n_terms=1, loss=d, warp_sums=d, warp_bytes=ws):
        return L.b2_glm_bernoulli_logits_elbo(d, d, d, None, 100000, 32, 64, 1.0, 1.0, 1.0, 0, None, out_total, d, d,
                                              d, 1 << 30, jobs, n_jobs, jc, terms, tc, n_terms, loss, warp_sums,
                                              warp_bytes, None)
    assert call(out_total=None) == -4                                   # no own total
    assert call(loss=None) == -4                                        # no loss output
    assert call(n_terms=N.LATENT_MAX_TERMS + 1) == -8
    assert call(warp_sums=None) == -5 and call(warp_bytes=ws - 8) == -5
    assert call(n_jobs=0) == -2 and call(n_jobs=N.LATENT_MAX_JOBS + 1) == -2
    assert call() == -4                                                 # job without z / prior
    j.dtype = N._DTYPES[torch.float64]
    assert call() == -1                                                 # fp64 jobs


# ---- GPU ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [70000, 1 << 20])
def test_finish_loss_equals_prior_combine(n):
    """The GLM call with the assembly open writes the loss latent_prior_combine computes from the same priors,
    terms and the call's own total, bit for bit; its own outputs are unchanged."""
    if EMULATE:
        pytest.skip("fused GLM kernel needs a GPU")
    from pyro_b200.distributions import _GlmBernoulliFn
    D, P = 32, 64
    X, y = _data(n, D)
    g = torch.Generator().manual_seed(3)
    zw = (0.3 * torch.randn(P, 1, D, generator=g)).to(DEV)
    zb = torch.randn(P, 1, generator=g).to(DEV)
    priors = [(zw, torch.zeros(D, device=DEV), torch.ones(D, device=DEV)),
              (zb, torch.zeros((), device=DEV), torch.full((), 10.0, device=DEV))]
    guide_terms = [torch.randn((), generator=g).to(DEV) * 100 for _ in range(2)]
    jc, tc, own = [-1.0 / P, -1.0 / P], [1.0 / P, 1.0 / P], -1.0 / P
    meta = (1.0, -1.0 / P, 1.0, True, 0)
    W, b = zw.reshape(P, D), zb.reshape(P)

    plain = _GlmBernoulliFn.apply(meta, X, y, W, b)
    ref = _ops.latent_prior_combine(priors, jc, guide_terms + [plain], tc + [own])
    with _ops.elbo_assembly(priors, jc, guide_terms, tc, own) as asm:
        fused = _GlmBernoulliFn.apply(meta, X, y, W, b)
    assert asm.loss is not None
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)
    assert torch.equal(asm.loss, ref), (float(asm.loss), float(ref))


@pytest.mark.gpu
@pytest.mark.parametrize("elbo_cls", [Trace_ELBO, JitTrace_ELBO])
def test_step_trajectory_unchanged_by_finish_assembly(elbo_cls):
    """Losses and parameters of config-2-shaped SVI steps (eager and graph-replayed) with the loss assembled in
    the GLM finish equal those with the separate prior-combine launch, bit for bit."""
    if EMULATE:
        pytest.skip("fused GLM kernel needs a GPU")
    X, y = _data(1 << 17, 32)
    _assert_same(_run(elbo_cls, X, y, 6, assemble=True), _run(elbo_cls, X, y, 6, assemble=False))


@pytest.mark.gpu
def test_graph_replay_equals_eager_steps():
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, y = _data(1 << 17, 32)
    _assert_same(_run(Trace_ELBO, X, y, 6), _run(JitTrace_ELBO, X, y, 6))


@pytest.mark.gpu
@pytest.mark.parametrize("n_sites", [2, 11])
def test_batched_draw_equals_separate_launches(n_sites):
    """n_sites deferred draws flushed together (one launch per 8) equal the same draws launched one by one: values,
    noise, scores and the Philox counter afterwards, bit for bit."""
    if EMULATE:
        pytest.skip("Philox draw kernel needs a GPU")
    g = torch.Generator().manual_seed(5)
    shapes = [(64, 1, 32), (64, 1), (7,), (3, 5)] * 3
    sites = [(torch.randn(shapes[k], generator=g).to(DEV), (0.1 + torch.rand(shapes[k], generator=g)).to(DEV))
             for k in range(n_sites)]

    def draws(together):
        pyro.set_rng_seed(11)
        out = []
        for loc, scale in sites:
            out.append(_ops.defer_latent_draw(loc, scale, False, loc.shape))
            if not together:
                _ops.flush_draws()
        assert len(_ops._PENDING_DRAWS) == (n_sites if together else 0)
        n0 = N.launch_count()
        _ops.flush_draws()
        launches = N.launch_count() - n0
        torch.cuda.synchronize()
        state = _ops.rng_state(sites[0][0].device).cpu().clone()
        return [[t.as_subclass(torch.Tensor).cpu() for t in o] for o in out], state, launches

    a, sa, la = draws(True)
    b, sb, _ = draws(False)
    assert la == (n_sites + 7) // 8
    assert torch.equal(sa, sb) and int(sa[1]) == n_sites and int(sa[2]) == 0
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)


def _hier_guide(X, y):
    """Out of the lazy scope: the second site's loc is the first site's value (read before it is flushed)."""
    D = X.shape[-1]
    m_loc = pyro.param("m_loc", lambda: X.new_zeros(()))
    w_scale = pyro.param("w_scale", lambda: X.new_full((D,), 0.1), constraint=constraints.positive)
    b_loc = pyro.param("b_loc", lambda: X.new_zeros(()))
    m = pyro.sample("m", dist.Normal(m_loc, 1.0))
    pyro.sample("w", dist.Normal(m.unsqueeze(-1).expand(m.shape + (D,)), w_scale).to_event(1))
    pyro.sample("b", dist.Normal(b_loc, 0.1))


def _hier_model(X, y):
    D = X.shape[-1]
    m = pyro.sample("m", dist.Normal(X.new_zeros(()), 1.0))
    w = pyro.sample("w", dist.Normal(m.unsqueeze(-1).expand(m.shape + (D,)), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=w.squeeze(-2) @ X.T + b), obs=y)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["lazy", "materialised", "out_of_scope"])
def test_deferred_draws_keep_trajectory(case):
    """Batched deferred draws give the trajectory of draws launched one by one, for the lazy model, the same model
    with its logits materialised, and a guide whose draw depends on an earlier draw."""
    if EMULATE:
        pytest.skip("Philox draw kernel needs a GPU")
    from pyro_b200.infer import elbo as elbo_mod
    X, y = _data(1 << 16, 32)
    kw = dict(model=_hier_model, guide=_hier_guide, P=8) if case == "out_of_scope" else {}
    prev = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = case != "materialised"
    try:
        _assert_same(_run(Trace_ELBO, X, y, 4, **kw), _run(Trace_ELBO, X, y, 4, batch_draws=False, **kw))
    finally:
        elbo_mod.LAZY_LINEAR = prev


@pytest.mark.gpu
def test_config2_step_native_launches():
    """one draw for both guide sites, GLM kernel, GLM finish (loss included), draws' backward, ClippedAdam."""
    if EMULATE:
        pytest.skip("fused GLM kernel needs a GPU")
    X, y = _data(1 << 17, 32)
    pyro.clear_param_store()
    svi = SVI(models.logistic_model, models.logistic_guide, ClippedAdam({"lr": 0.02}),
              Trace_ELBO(num_particles=64, vectorize_particles=True, max_plate_nesting=1))
    svi.step(X, y)
    n0 = N.launch_count()
    svi.step(X, y)
    assert N.launch_count() - n0 == 5
