"""Model-class recognition: let ``NUTS(model)`` / ``HMC(model)`` run on a native potential.

The reference evaluates ``U(z)`` by re-running the Python model under ``condition`` + ``trace`` for
every leapfrog step (pyro/infer/mcmc/util.py:275-286; 36 % of a leapfrog is the re-trace, SURVEY.md
3.5).  For the model classes of the BASELINE configs a fused potential+gradient kernel exists behind
the C ABI (``b2_potential_grad``, ``b2_nuts_small``, ``b2_nuts_leaf_hier``).  ``recognise`` decides,
WITHOUT touching the user's code, whether a model belongs to such a class:

* structure: the prototype trace (one ordinary execution, as pyro/infer/mcmc/util.py:370-482
  ``initialize_model`` takes) must have exactly the sites of the class, with the right families,
  shapes and constant prior parameters;
* function: the observed site's parameters are PROBED -- the model is re-run under
  ``poutine.condition`` on random latent values and the likelihood's location (or logits) must equal
  the class's closed form (``mu + tau * eta``; ``X @ beta``) at every probe, and its scale must not
  move.  A model that merely looks similar fails the probe and falls back to the traced potential.

The returned potential uses the model's own site names, so ``MCMC.get_samples()`` is unchanged.
"""
import torch


def _base(fn):
    """(innermost distribution, its class name) under Independent / Expanded / Masked wrappers."""
    seen = 0
    # only the pure wrappers are looked through: torch's HalfCauchy / LogNormal are
    # TransformedDistributions that own a ``base_dist`` too
    while type(fn).__name__ in ("Independent", "ExpandedDistribution", "MaskedDistribution") and seen < 8:
        fn = fn.base_dist
        seen += 1
    return fn, type(fn).__name__.lstrip("_")


def _is_masked(fn):
    seen = 0
    while seen < 8:
        if type(fn).__name__ == "MaskedDistribution":
            return True
        if not hasattr(fn, "base_dist"):
            return False
        fn = fn.base_dist
        seen += 1
    return False


def _const(t):
    """python float if ``t`` is (a tensor of) one repeated gradient-free value, else None."""
    if isinstance(t, (int, float)):
        return float(t)
    if not isinstance(t, torch.Tensor) or t.requires_grad or t.numel() == 0:
        return None
    flat = t.detach().reshape(-1)
    v = flat[0]
    if not bool((flat == v).all()):
        return None
    return float(v)


def _sites(trace):
    latent, observed = {}, {}
    for name, site in trace.nodes.items():
        if site["type"] != "sample":
            continue
        # plates record a subsample site: flagged in pyro_b200, a ``_Subsample`` distribution in Pyro
        if site.get("infer", {}).get("_subsample") or type(site["fn"]).__name__ == "_Subsample":
            continue
        (observed if site["is_observed"] else latent)[name] = site
    return latent, observed


def _plain_site(site):
    scale = site.get("scale", 1.0)
    if isinstance(scale, torch.Tensor) or scale != 1.0:
        return False
    if site.get("mask") is not None or _is_masked(site["fn"]):
        return False
    return not (site.get("args") or site.get("kwargs"))


def _probe(poutine, model, args, kwargs, data, obs_name):
    tr = poutine.trace(poutine.condition(model, data=data)).get_trace(*args, **kwargs)
    return _base(tr.nodes[obs_name]["fn"])[0]


def _close(a, b, dtype):
    tol = 1e-10 if dtype == torch.float64 else 2e-5
    a, b = torch.broadcast_tensors(a.detach(), b.detach())
    return bool(((a - b).abs() <= tol * (1.0 + b.abs())).all())


def _try_hier_normal(poutine, model, args, kwargs, latent, observed):
    from .potential import HierNormalPotential
    if len(latent) != 3 or len(observed) != 1:
        return None
    (obs_name, obs), = observed.items()
    ofn, oname = _base(obs["fn"])
    if oname != "Normal" or not _plain_site(obs):
        return None
    y = obs["value"]
    if not (isinstance(y, torch.Tensor) and y.is_floating_point() and y.dim() == 1 and y.numel() >= 1):
        return None
    J = y.numel()
    mu = tau = eta = None
    s_mu = s_tau = None
    for name, site in latent.items():
        fn, cls = _base(site["fn"])
        v = site["value"]
        if not _plain_site(site) or not isinstance(v, torch.Tensor):
            return None
        if cls == "HalfCauchy" and v.numel() == 1 and tau is None:
            s_tau = _const(fn.scale)
            tau = name
        elif cls == "Normal" and v.numel() == 1 and J != 1 and mu is None and _const(fn.loc) == 0.0:
            s_mu = _const(fn.scale)
            mu = name
        elif cls == "Normal" and tuple(v.shape) == (J,) and eta is None \
                and _const(fn.loc) == 0.0 and _const(fn.scale) == 1.0:
            eta = name
        else:
            return None
    if None in (mu, tau, eta, s_mu, s_tau):
        return None
    sigma0 = ofn.scale
    if not isinstance(sigma0, torch.Tensor) or sigma0.requires_grad:
        return None
    sigma0 = sigma0.detach().expand(J) if sigma0.numel() in (1, J) else None
    if sigma0 is None:
        return None
    # ---- functional probe: loc == mu + tau * eta, scale constant -------------------------------------
    gen = torch.Generator(device="cpu").manual_seed(20240229)
    for _ in range(3):
        m = torch.randn((), generator=gen).to(y)
        t = (0.2 + torch.rand((), generator=gen) * 3).to(y)
        e = torch.randn(J, generator=gen).to(y)
        data = {mu: m.reshape(latent[mu]["value"].shape), tau: t.reshape(latent[tau]["value"].shape),
                eta: e}
        pfn = _probe(poutine, model, args, kwargs, data, obs_name)
        if not _close(pfn.loc, m + t * e, y.dtype) or not _close(pfn.scale, sigma0, y.dtype):
            return None
    pot = HierNormalPotential(y.detach(), sigma0.contiguous(), s_mu=s_mu, s_tau=s_tau,
                              names=(mu, tau, eta),
                              shapes=(tuple(latent[mu]["value"].shape), tuple(latent[tau]["value"].shape)))
    return pot


def _try_logistic(poutine, model, args, kwargs, latent, observed):
    from .potential import LogisticPotential
    if len(latent) != 1 or len(observed) != 1:
        return None
    (bname, bsite), = latent.items()
    (obs_name, obs), = observed.items()
    bfn, bcls = _base(bsite["fn"])
    ofn, ocls = _base(obs["fn"])
    if bcls != "Normal" or ocls != "Bernoulli" or not _plain_site(bsite) or not _plain_site(obs):
        return None
    beta = bsite["value"]
    if beta.dim() != 1 or _const(bfn.loc) != 0.0:
        return None
    s = _const(bfn.scale)
    if s is None:
        return None
    D = beta.numel()
    y = obs["value"]
    if not isinstance(y, torch.Tensor) or y.dim() != 1:
        return None
    X = None
    for a in list(args) + list(kwargs.values()):
        if isinstance(a, torch.Tensor) and a.dim() == 2 and tuple(a.shape) == (y.numel(), D) \
                and a.is_floating_point() and not a.requires_grad:
            X = a
    if X is None or "logits" not in getattr(ofn, "__dict__", {"logits": 1}) and not hasattr(ofn, "logits"):
        return None
    gen = torch.Generator(device="cpu").manual_seed(20240301)
    for _ in range(3):
        bv = torch.randn(D, generator=gen).to(X)
        pfn = _probe(poutine, model, args, kwargs, {bname: bv}, obs_name)
        logits = pfn.logits
        if hasattr(logits, "dense"):
            logits = logits.dense()
        if not _close(logits, X @ bv, X.dtype):
            return None
    return LogisticPotential(X, y.to(X.dtype), prior_scale=s, site_name=bname)


def _try_glm(poutine, model, args, kwargs, latent, observed):
    """Logistic regression with an intercept, or softmax or Poisson (log link) regression with or without one,
    in fp32, within the GLM kernels' scope: Bernoulli D in {4, 8, 16, 32}; Categorical D == 32, 2 <= K <= 16;
    Poisson 1 <= D <= 128."""
    from .potential import GlmPotential
    if len(observed) != 1 or len(latent) not in (1, 2):
        return None
    (obs_name, obs), = observed.items()
    _, kind = _base(obs["fn"])
    # lazy linear-predictor logits build _BernoulliLinear / _CategoricalLinear (pyro_b200/distributions)
    # (and _PoissonLinear for a lazy exp of one)
    kind = {"BernoulliLinear": "Bernoulli", "CategoricalLinear": "Categorical",
            "PoissonLinear": "Poisson"}.get(kind, kind)
    if kind not in ("Bernoulli", "Categorical", "Poisson") or not _plain_site(obs):
        return None
    y = obs["value"]
    if not isinstance(y, torch.Tensor) or y.dim() != 1:
        return None
    n = y.numel()
    X = None
    for a in list(args) + list(kwargs.values()):
        if isinstance(a, torch.Tensor) and a.dim() == 2 and a.shape[0] == n and a.dtype == torch.float32 \
                and not a.requires_grad:
            X = a
    if X is None or not X.is_contiguous() or X.data_ptr() % 16 != 0:
        return None
    D = X.shape[1]
    scales, shapes = {}, {}
    for name, site in latent.items():
        fn, cls = _base(site["fn"])
        v = site["value"]
        if cls != "Normal" or not _plain_site(site) or not isinstance(v, torch.Tensor) \
                or v.dtype != torch.float32 or _const(fn.loc) != 0.0:
            return None
        s = _const(fn.scale)
        if s is None or not s > 0.0:
            return None
        scales[name], shapes[name] = s, tuple(v.shape)
    if kind == "Bernoulli":
        K = 1
        wshapes, bshapes = [(D,)], [(), (1,)]
        if D not in (4, 8, 16, 32) or y.dtype != torch.float32:
            return None
    elif kind == "Poisson":
        K = 1
        wshapes, bshapes = [(D,)], [(), (1,)]
        if not 1 <= D <= 128 or y.dtype != torch.float32:
            return None
    else:
        wmat = [s for s in shapes.values() if len(s) == 2]
        K = wmat[0][0] if len(wmat) == 1 else 0
        wshapes, bshapes = [(K, D)], [(K,)]
        if D != 32 or not 2 <= K <= 16 or y.dtype != torch.int64:
            return None
    weight = [name for name, s in shapes.items() if s in wshapes]
    bias = [name for name, s in shapes.items() if s in bshapes]
    if len(weight) != 1 or len(bias) + 1 != len(latent):
        return None
    weight, bias = weight[0], (bias[0] if bias else None)
    if kind == "Bernoulli" and bias is None:
        return None   # intercept-free logistic regression keeps LogisticPotential's route
    # ---- functional probe: logits == X @ w + b  /  log_softmax(logits) == log_softmax(X @ W.mT + b)  /
    # log(rate) == X @ w + b ----------------------------------------------------------------------------------
    gen = torch.Generator(device="cpu").manual_seed(20240302)
    for _ in range(3):
        wv = torch.randn(shapes[weight], generator=gen).to(X)
        if kind == "Poisson":
            wv = wv / D ** 0.5            # log-rates of a few units: exp neither overflows nor underflows
        bv = torch.randn(shapes[bias], generator=gen).to(X) if bias is not None else None
        data = {weight: wv} if bias is None else {weight: wv, bias: bv}
        pfn = _probe(poutine, model, args, kwargs, data, obs_name)
        logits = torch.log(pfn.rate) if kind == "Poisson" else pfn.logits
        if hasattr(logits, "dense"):
            logits = logits.dense()
        if kind == "Poisson":
            want = X @ wv + (bv.reshape(()) if bv is not None else 0.0)
        elif kind == "Bernoulli":
            want = X @ wv + bv.reshape(())
        else:
            want = X @ wv.mT + (bv if bv is not None else 0.0)
            logits, want = torch.log_softmax(logits, -1), torch.log_softmax(want, -1)
        if tuple(logits.shape) != tuple(want.shape) or not _close(logits, want, X.dtype):
            return None
    off, sites = 0, {}
    for name in latent:
        width = 1
        for d in shapes[name]:
            width *= d
        sites[name] = (slice(off, off + width), "identity", shapes[name])
        off += width
    return GlmPotential(X, y.detach(), kind, sites, weight, bias, s_w=scales[weight],
                        s_b=scales[bias] if bias is not None else 1.0)


def recognise(model, args=(), kwargs=None, poutine=None):
    """A native potential for ``model`` if it belongs to a compiled class, else None (never raises:
    any surprise means "not recognised")."""
    kwargs = kwargs or {}
    if poutine is None:
        from ... import poutine as _own
        poutine = _own
    try:
        with torch.no_grad():
            proto = poutine.trace(model).get_trace(*args, **kwargs)
            latent, observed = _sites(proto)
            for attempt in (_try_hier_normal, _try_logistic, _try_glm):
                pot = attempt(poutine, model, args, kwargs, latent, observed)
                if pot is not None:
                    return pot
    except Exception:  # noqa: BLE001 -- recognition is an optimisation, never an error source
        return None
    return None
