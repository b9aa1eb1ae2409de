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
import math

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


_POSITIVE = ("HalfNormal", "HalfCauchy", "Exponential", "LogNormal")


def _positive_prior(fn, cls):
    """``(cls, p0, p1)`` of a HalfNormal(p0), HalfCauchy(p0), Exponential(p0) or LogNormal(p0, p1) prior whose
    parameters are each one repeated gradient-free value, else None."""
    if cls == "LogNormal":
        p0, p1 = _const(fn.loc), _const(fn.scale)
    else:
        p0, p1 = _const(fn.rate if cls == "Exponential" else fn.scale), 1.0
    if p0 is None or p1 is None or not p1 > 0.0 or not math.isfinite(p0) or (cls != "LogNormal" and not p0 > 0.0):
        return None
    return cls, p0, p1


def _try_glm(poutine, model, args, kwargs, latent, observed):
    """Logistic regression with an intercept, or softmax, Poisson (log link), Binomial (logit link) or linear
    regression with or without one, in fp32, within the GLM kernels' scope: Bernoulli D in {4, 8, 16, 32};
    Categorical D == 32, 2 <= K <= 16; Poisson, Binomial and Normal 1 <= D <= 128.  Binomial's total_count is a
    constant or gradient-free fp32 [N] counts, the same at every probe.

    The weight prior is ``Normal(0, S)`` and the bias prior ``Normal(0, s_b)`` with a constant ``s_b``.  ``S`` is a
    constant, or latent: ``tau`` (one positive scalar site), ``lam`` (a positive site of the weight's shape) or
    ``tau * lam``.  Linear regression's noise scale is a constant or one latent positive scalar site.  Every
    latent positive site has a HalfNormal, HalfCauchy, Exponential or LogNormal prior with constant parameters
    (for ``lam`` one value for every coefficient), and exactly one role -- noise scale, ``tau``, ``lam`` or the group
    scale ``s_a`` -- which the probes establish: the observation's scale equals the drawn noise scale and the weight
    site's scale equals the drawn ``tau``, ``lam`` or ``tau * lam`` at every probe.  Intercept-free logistic
    regression with a constant weight scale keeps LogisticPotential's route.

    A varying intercept by group (every kind but softmax, with a constant weight scale, any D with D + G <= 128, or
    past that with the rows sorted by group, D <= 128 and G <= 65536, but for Binomial regression):
    the group index is the one gradient-free int64 ``[N]`` tensor among the arguments, and the group effect a
    latent ``Normal`` site of shape ``(G,)``, tried after the model without one fails.  The probes decide the form:
    the observation's logits (log-rate, loc) equal ``X @ w + b + alpha[g]`` with ``alpha ~ Normal(0, s_a)``
    (centred), or ``X @ w + b + s_a * eta[g]`` with ``eta ~ Normal(0, 1)`` (non-centred), ``s_a`` a constant or a
    drawn positive scalar site, at every probe.  So how the model writes the gather does not matter.

    Varying slopes (up to three, with a varying intercept, D + G (1 + S) <= 128 or a sorted index): further latent
    ``Normal`` sites of shape ``(G,)``, tried after the intercept-only model fails.  Slope k adds
    ``beta_k[g] * X[:, c_k]`` to the linear predictor, ``beta_k`` centred or non-centred with its own constant or
    latent scale, as the intercept.  A probe with only table k non-zero finds ``c_k``: the residual after
    ``X @ w + b + alpha[g]`` must be ``beta_k[g]`` times a column of X (the lowest such column when columns repeat);
    then the three probes with every table drawn confirm the whole sum.  So the covariate must be a column of X,
    whatever the model writes to take it."""
    if len(observed) != 1 or not 1 <= len(latent) <= 11:
        return None
    (obs_name, obs), = observed.items()
    _, kind = _base(obs["fn"])
    # lazy linear-predictor logits build _BernoulliLinear / _CategoricalLinear (pyro_b200/distributions)
    # (and _PoissonLinear for a lazy exp of one, _NormalLinear for a lazy loc)
    kind = {"BernoulliLinear": "Bernoulli", "CategoricalLinear": "Categorical",
            "PoissonLinear": "Poisson", "NormalLinear": "Normal", "BinomialLinear": "Binomial"}.get(kind, kind)
    if kind not in ("Bernoulli", "Categorical", "Poisson", "Normal", "Binomial") or not _plain_site(obs):
        return None
    order = list(latent)                   # TracePotential's site order
    # positive-support sites (z holds their logs): the noise scale and the weight scales, roles decided by probing
    positive, priors = {}, {}
    for name, site in latent.items():
        fn, cls = _base(site["fn"])
        if cls not in _POSITIVE:
            continue
        v = site["value"]
        if not _plain_site(site) or not isinstance(v, torch.Tensor) or v.dtype != torch.float32:
            return None
        priors[name] = _positive_prior(fn, cls)
        if priors[name] is None:
            return None
        positive[name] = tuple(v.shape)
    latent = {k: v for k, v in latent.items() if k not in positive}
    if not 1 <= len(latent) <= 6:
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
        scales[name], shapes[name] = _const(fn.scale), tuple(v.shape)
    attempts = [(None, ())]                # (the group-effect site, its slope sites): none, then each candidate
    ints = [a for a in list(args) + list(kwargs.values())
            if isinstance(a, torch.Tensor) and a is not y and a.dtype == torch.int64 and a.dim() == 1
            and a.numel() == n and not a.requires_grad]
    if kind != "Categorical" and len(ints) == 1 and len(latent) >= 2 and ints[0].numel() > 0:
        # only sites with a group for every index: the probes gather with it
        lo, hi = int(ints[0].min()), int(ints[0].max())
        groups = [name for name, s in shapes.items() if len(s) == 1 and lo >= 0 and hi < s[0]]
        # the one-hot columns fit the contraction, or the rows are sorted by group (the gathered route)
        ordered = bool((ints[0][1:] >= ints[0][:-1]).all())

        def fits(G, S):
            return D + G * (1 + S) <= 128 or (ordered and kind != "Binomial" and D <= 128 and G <= 65536)
        attempts += [(a, ()) for a in groups if fits(shapes[a][0], 0)]
        # then with slopes: the other sites of the intercept's shape (when D == G, bar one that may be the weight)
        for a in groups:
            G = shapes[a][0]
            rest = [name for name in groups if name != a and shapes[name] == (G,)]
            sets = [rest] + ([[b for b in rest if b != w] for w in rest] if D == G else [])
            attempts += [(a, tuple(b)) for b in sets if 1 <= len(b) <= 3 and fits(G, len(b))]
    for group_site, slope_sites in attempts:
        pot = _glm_roles(poutine, model, args, kwargs, kind, obs_name, obs, order, positive, priors, latent, X, y,
                         scales, shapes, group_site, ints[0] if group_site is not None else None, slope_sites)
        if pot is not None:
            return pot
    return None


def _glm_roles(poutine, model, args, kwargs, kind, obs_name, obs, order, positive, priors, latent, X, y, scales,
               shapes, group_site, gidx, slope_sites=()):
    """``_try_glm`` with the Normal site ``group_site`` (None: no group effect) as the group effect, and the Normal
    sites ``slope_sites`` as its varying slopes."""
    from .potential import GlmPotential
    n, D = y.numel(), X.shape[1]
    latent = {k: v for k, v in latent.items() if k != group_site and k not in slope_sites}
    if len(latent) not in (1, 2):
        return None
    if kind == "Bernoulli":
        K = 1
        wshapes, bshapes = [(D,)], [(), (1,)]
        if (group_site is None and D not in (4, 8, 16, 32)) or y.dtype != torch.float32:
            return None
    elif kind in ("Poisson", "Normal", "Binomial"):
        K = 1
        wshapes, bshapes = [(D,)], [(), (1,)]
        if not 1 <= D <= 128 or y.dtype != torch.float32:
            return None
    else:
        wmat = [shapes[name] for name in latent if len(shapes[name]) == 2]
        K = wmat[0][0] if len(wmat) == 1 else 0
        wshapes, bshapes = [(K, D)], [(K,)]
        if D != 32 or not 2 <= K <= 16 or y.dtype != torch.int64:
            return None
    weight = [name for name in latent if shapes[name] in wshapes]
    bias = [name for name in latent if shapes[name] in bshapes]
    if len(weight) != 1 or len(bias) + 1 != len(latent):
        return None
    weight, bias = weight[0], (bias[0] if bias else None)
    if bias is not None and not (scales[bias] is not None and scales[bias] > 0.0):
        return None
    # candidates by shape: tau (and the noise scale) one value, lam the weight's shape
    scalars = [name for name, s in positive.items() if s in ((), (1,))]
    lams = [name for name, s in positive.items() if s == shapes[weight]]
    # ---- functional probe: logits == X @ w + b  /  log_softmax(logits) == log_softmax(X @ W.mT + b)  /
    # log(rate) == X @ w + b, and the scales' roles ------------------------------------------------------------------
    gen = torch.Generator(device="cpu").manual_seed(20240302)
    sigma_site, sigma_const = None, None
    wform = None                           # (tau site or None, lam site or None); (None, None): the constant s_w
    trials = None                          # Binomial: the constant count, or the [N] counts of the prototype
    group = None                           # the group effect's form, once the first probe has found it
    slopes = {k: None for k in slope_sites}   # each slope's column and form, once its own probe has found them
    # with slopes, a probe of the intercept alone and one of each slope alone (the other tables zero) come first
    probes = [()] + [(k,) for k in slope_sites] if slope_sites else []
    probes += [tuple(slope_sites)] * 3
    if kind == "Binomial":
        trials = _binomial_trials(_base(obs["fn"])[0], n)
        if trials is None:
            return None

    def as_t(v):
        return torch.as_tensor(v, dtype=X.dtype, device=X.device)

    for i, drawn in enumerate(probes):
        wv = torch.randn(shapes[weight], generator=gen).to(X)
        if kind == "Poisson":
            wv = wv / D ** 0.5            # log-rates of a few units: exp neither overflows nor underflows
        bv = torch.randn(shapes[bias], generator=gen).to(X) if bias is not None else None
        data = {weight: wv} if bias is None else {weight: wv, bias: bv}
        for name, shape in positive.items():
            data[name] = torch.exp(0.5 * torch.randn(shape, generator=gen)).to(X)
        if group_site is not None:
            data[group_site] = torch.randn(shapes[group_site], generator=gen).to(X)
        for k in slope_sites:
            data[k] = torch.randn(shapes[k], generator=gen).to(X) if k in drawn else X.new_zeros(shapes[k])
        tr = poutine.trace(poutine.condition(model, data=data)).get_trace(*args, **kwargs)
        pfn = _base(tr.nodes[obs_name]["fn"])[0]
        # the priors: constant parameters that do not move with any latent
        for name in positive:
            fn, cls = _base(tr.nodes[name]["fn"])
            if cls != priors[name][0] or _positive_prior(fn, cls) != priors[name]:
                return None
        if bias is not None:
            bfn = _base(tr.nodes[bias]["fn"])[0]
            if _const(bfn.loc) != 0.0 or _const(bfn.scale) != scales[bias]:
                return None
        wfn = _base(tr.nodes[weight]["fn"])[0]
        if _const(wfn.loc) != 0.0:
            return None
        if kind == "Normal":
            # scale: a latent noise scale as drawn, or one constant that does not move with the latents
            sc = as_t(pfn.scale)
            if i == 0:
                hits = [name for name in scalars if _close(sc, data[name].reshape(()), X.dtype)]
                if len(hits) > 1:
                    return None
                sigma_site = hits[0] if hits else None
            if sigma_site is not None:
                if not _close(sc, data[sigma_site].reshape(()), X.dtype):
                    return None
            else:
                c = _const(sc)
                if c is None or not c > 0.0 or (sigma_const is not None and c != sigma_const):
                    return None
                sigma_const = c
        free_s = [name for name in scalars if name != sigma_site]
        # the weight scale: the constant of the prototype, or the drawn tau, lam or tau * lam
        def want_scale(form):
            t, lam = form
            if t is None and lam is None:
                return as_t(scales[weight]) if scales[weight] is not None and scales[weight] > 0.0 else None
            v = data[t].reshape(()) if t is not None else 1.0
            return v * data[lam] if lam is not None else v
        ws = as_t(wfn.scale)
        if i == 0:
            forms = [(None, None)]
            if group_site is None:
                forms += [(t, None) for t in free_s] + [(None, lam) for lam in lams] + \
                    [(t, lam) for t in free_s for lam in lams if t != lam]
            hits = [f for f in forms if want_scale(f) is not None and _close(ws, want_scale(f), X.dtype)]
            if len(hits) != 1:
                return None
            wform = hits[0]
        want = want_scale(wform)
        if tuple(torch.broadcast_shapes(ws.shape, want.shape, shapes[weight])) != shapes[weight] \
                or not _close(ws, want, X.dtype):
            return None
        if kind == "Binomial":
            # logits as the model gave them (not probs), and the same trial counts at every probe
            t = _binomial_trials(pfn, n)
            if t is None or type(t) is not type(trials) or (
                    isinstance(t, float) and t != trials) or (
                    isinstance(t, torch.Tensor) and not torch.equal(t, trials)):
                return None
            logits = pfn.logits
        elif kind == "Normal":
            logits = pfn.loc
        else:
            logits = torch.log(pfn.rate) if kind == "Poisson" else pfn.logits
        if hasattr(logits, "dense"):
            logits = logits.dense()
        if kind != "Categorical":
            want = X @ wv + (bv.reshape(()) if bv is not None else 0.0)
        else:
            want = X @ wv.mT + (bv if bv is not None else 0.0)
            logits, want = torch.log_softmax(logits, -1), torch.log_softmax(want, -1)
        if group_site is not None:
            group = _group_form(tr, group_site, data, gidx, logits, want, free_s, group, X.dtype)
            if group is None:
                return None
            sa = data[group["s_site"]].reshape(()) if group["s_site"] is not None else as_t(group["s_const"])
            e = data[group_site][gidx]
            want = want + (sa * e if group["noncentred"] else e)
        for k in drawn:
            claimed = [sigma_site, group["s_site"]] + [v["form"]["s_site"] for j, v in slopes.items()
                                                        if j != k and v is not None]
            free_k = [s for s in free_s if s not in claimed]
            if slopes[k] is None:
                # its own probe: the only table drawn, so the residual is its term alone.  The first column whose
                # form is found wins, one with a drawn scale before a constant one: over very few rows several
                # columns can fit, and only the drawn scale tells them apart.
                found = [(c, _group_form(tr, k, data, gidx, logits, want, free_k, None, X.dtype, cov=X[:, c]))
                         for c in _slope_columns(logits - want, data[k][gidx], X)]
                found = [f for f in found if f[1] is not None]
                found = [f for f in found if f[1]["s_site"] is not None] or found
                if not found:
                    return None
                slopes[k] = {"col": found[0][0], "form": found[0][1]}
            cov = X[:, slopes[k]["col"]]
            form = _group_form(tr, k, data, gidx, logits, want, free_k, slopes[k]["form"], X.dtype, cov=cov)
            if form is None:
                return None
            sk = data[form["s_site"]].reshape(()) if form["s_site"] is not None else as_t(form["s_const"])
            e = data[k][gidx] * cov
            want = want + (sk * e if form["noncentred"] else e)
        if tuple(logits.shape) != tuple(want.shape) or not _close(logits, want, X.dtype):
            return None
    tau_site, lam_site = wform
    # every positive site has exactly one role
    roles = [r for r in (sigma_site,) + wform + ((group["s_site"],) if group else ())
             + tuple(v["form"]["s_site"] for v in slopes.values()) if r is not None]
    if sorted(roles) != sorted(positive):
        return None
    if kind == "Bernoulli" and bias is None and tau_site is None and lam_site is None and group is None:
        return None   # intercept-free logistic regression with a constant weight scale keeps LogisticPotential
    off, sites = 0, {}
    for name in order:
        shape = positive.get(name, shapes.get(name))
        width = 1
        for d in shape:
            width *= d
        sites[name] = (slice(off, off + width), "exp" if name in positive else "identity", shape)
        off += width
    if group is not None:
        group = dict(group, site=group_site, index=gidx, s_prior=priors.get(group["s_site"]),
                     slopes=[dict(v["form"], site=k, col=v["col"], s_prior=priors.get(v["form"]["s_site"]))
                             for k, v in slopes.items()])
    return GlmPotential(X, y.detach(), kind, sites, weight, bias,
                        s_w=scales[weight] if wform == (None, None) else 1.0,
                        s_b=scales[bias] if bias is not None else 1.0,
                        sigma=sigma_const if sigma_const is not None else 1.0, sigma_site=sigma_site,
                        sigma_prior=priors.get(sigma_site), trials=trials,
                        tau_site=tau_site, tau_prior=priors.get(tau_site),
                        lam_site=lam_site, lam_prior=priors.get(lam_site), group=group)


def _slope_columns(r, e, X):
    """The columns c of X, lowest first, with ``r == s * e * X[:, c]`` for one number s."""
    cols = []
    for c in range(X.shape[1]):
        q = e * X[:, c]
        s = (r * q).sum() / (q * q).sum().clamp(min=1e-30)
        if _close(r, s * q, X.dtype):
            cols.append(c)
    return cols


def _group_form(tr, group_site, data, gidx, logits, want, free_s, group, dtype, cov=None):
    """The group effect's form at one probe: ``{"noncentred", "s_site", "s_const"}`` when the residual
    ``logits - want`` is ``alpha[g]`` with ``alpha ~ Normal(0, s_a)`` or ``s_a * eta[g]`` with ``eta ~ Normal(0, 1)``,
    ``s_a`` the drawn site of ``free_s`` or one constant; ``group`` is the first probe's answer, which later probes
    must repeat.  A varying slope's residual is that times its covariate ``cov``.  None otherwise."""
    afn = _base(tr.nodes[group_site]["fn"])[0]
    if _const(afn.loc) != 0.0:
        return None
    G = data[group_site].numel()
    scale = torch.as_tensor(afn.scale, dtype=dtype, device=logits.device).detach()
    if tuple(torch.broadcast_shapes(scale.shape, (G,))) != (G,):
        return None
    e = data[group_site][gidx]
    if cov is not None:
        e = e * cov
    r = logits - want
    if group is None:
        if _close(r, e, dtype):
            s, noncentred = scale, False
        elif _const(scale) == 1.0:
            # the least-squares s_a of r = s_a e; the comparison below confirms it
            s, noncentred = (r * e).sum() / (e * e).sum().clamp(min=1e-30), True
        else:
            return None
        hits = [name for name in free_s if _close(s, data[name].reshape(()), dtype)]
        if len(hits) > 1:
            return None
        c = _const(s) if not hits else None
        if not hits and not (c is not None and c > 0.0 and math.isfinite(c)):
            return None
        group = {"noncentred": noncentred, "s_site": hits[0] if hits else None, "s_const": c}
    sa = data[group["s_site"]].reshape(()) if group["s_site"] is not None else group["s_const"]
    if group["noncentred"]:
        return group if _const(scale) == 1.0 else None
    return group if _close(scale, torch.as_tensor(sa, dtype=dtype, device=scale.device), dtype) else None


def _binomial_trials(fn, n):
    """The trial counts of a logits-parameterised Binomial with ``n`` rows: a python float when they are one
    gradient-free value, else the fp32 ``[n]`` counts (no gradient); None for a Binomial given ``probs`` or any other
    total_count."""
    if getattr(fn, "family", None) is not None:
        from ... import _native as N
        if fn.family != N.BINOMIAL_LOGITS:
            return None
    elif "logits" not in fn.__dict__:
        return None
    tc = fn.total_count
    if not isinstance(tc, torch.Tensor) or tc.requires_grad or tc.dtype != torch.float32:
        return None
    c = _const(tc)
    if c is not None:
        return c
    if tc.numel() != n:
        return None
    return tc.detach().reshape(n)


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
