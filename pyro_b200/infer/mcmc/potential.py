"""Potential energies ``U(z) = -[sum_sites log_prob(T^-1(z)) + log|det dT^-1/dz|]`` for MANY chains.

Two providers share one interface, ``value_and_grad(z[C, D]) -> (U[C], dU/dz[C, D])``:

``NativePotential``  a "compiled model class": the whole potential and its gradient are one fused
                     kernel pair behind the C ABI (``b2_potential_grad``), and, for small latent
                     dimension, entire NUTS transitions run on the device (``b2_nuts_small``).
``TracePotential``   any model written with ``pyro_b200.sample``: the model is run once per
                     evaluation with a leading chain plate, sites are scored by the fused
                     log_prob kernels and differentiated by their fused backward -- the same
                     construction as pyro/infer/mcmc/util.py:275-286 (``_PEMaker._potential_fn``)
                     and pyro/ops/integrator.py:68-94 (``potential_grad``), but for all chains in
                     one pass.
"""
import ctypes

import torch
from torch.distributions import biject_to

from ... import _native as N
from ... import poutine
from ...distributions import group_index_int32, group_index_sorted, scale_and_mask
from ...primitives import plate


class NativePotential:
    """Base for native model classes.  ``sites`` maps site name -> (slice into z, transform name,
    event shape); ``transform`` is "identity" or "exp" (positive support: z = log value,
    torch/distributions/constraint_registry.py:184-188)."""

    def __init__(self, model_id, dtype, device, J, D, data0, data1, hyper, sites):
        self.model_id = model_id
        self.dtype = dtype
        self.device = device
        self.J, self.D = int(J), int(D)
        self._keep = (data0, data1)  # keep the data alive
        m = N.b2_model()
        m.model = model_id
        m.dtype = N._DTYPES[dtype]
        m.J = self.J
        m.D = self.D
        m.data0 = data0.data_ptr()
        m.data1 = data1.data_ptr()
        for i, h in enumerate(hyper):
            m.hyper[i] = float(h)
        self._model = m
        self.sites = sites

    @property
    def dim(self):
        return self.D

    def value_and_grad(self, z, active=None, out_grad=None):
        N.require_cuda(z, "NativePotential")
        C = z.shape[0]
        z = z.contiguous()
        U = torch.empty(C, dtype=self.dtype, device=z.device)
        g = out_grad if out_grad is not None else torch.empty_like(z)
        need = int(N.lib().b2_mcmc_workspace(C))
        ws = N.workspace(z.device, need, tag="mcmc")
        N.check(N.lib().b2_potential_grad(
            ctypes.byref(self._model), z.data_ptr(), U.data_ptr(), g.data_ptr(), C,
            active.data_ptr() if active is not None else None, ws.data_ptr(), ws.numel(),
            N.stream_ptr(z.device)), "b2_potential_grad")
        return U, g

    def unpack(self, z):
        """``[..., D]`` unconstrained -> dict of constrained site values ``[..., *event_shape]``."""
        return {name: self.unpack_site(name, z[..., sl]) for name, (sl, _, _) in self.sites.items()}

    def unpack_site(self, name, u):
        """Constrained value of ONE site from its unconstrained columns ``[..., n_site]``."""
        _, transform, shape = self.sites[name]
        v = u.exp() if transform == "exp" else u
        return v.reshape(u.shape[:-1] + tuple(shape))

    def init_uniform(self, num_chains, radius=2.0, generator=None):
        return (torch.rand(num_chains, self.D, dtype=self.dtype, device=self.device,
                           generator=generator) * 2 - 1) * radius


class HierNormalPotential(NativePotential):
    """eight_schools family (examples/eight_schools/mcmc.py:27-34):
    ``mu ~ Normal(0, s_mu)``, ``tau ~ HalfCauchy(s_tau)``, ``eta ~ Normal(0,1)[J]``,
    ``obs ~ Normal(mu + tau*eta, sigma)``;  z = [mu, log tau, eta]."""

    def __init__(self, y, sigma, s_mu=10.0, s_tau=25.0, names=("mu", "tau", "eta"), shapes=((1,), (1,))):
        N.require_cuda(y, "HierNormalPotential")
        y = y.contiguous()
        sigma = sigma.to(y.dtype).contiguous()
        J = y.numel()
        # ``names`` / ``shapes``: the site names and the (mu, tau) value shapes of the user's model when
        # the class was recognised from a model (infer/mcmc/compile.py)
        sites = {names[0]: (slice(0, 1), "identity", tuple(shapes[0])),
                 names[1]: (slice(1, 2), "exp", tuple(shapes[1])),
                 names[2]: (slice(2, 2 + J), "identity", (J,))}
        super().__init__(N.MODEL_HIER_NORMAL, y.dtype, y.device, J, J + 2, y, sigma, (s_mu, s_tau), sites)


class LogisticPotential(NativePotential):
    """Bayesian logistic regression (tests/infer/mcmc/test_hmc.py:189-198):
    ``beta ~ Normal(0, s)[D]``, ``y ~ Bernoulli(logits = X beta)``;  z = beta."""

    def __init__(self, X, y, prior_scale=1.0, site_name="beta"):
        N.require_cuda(X, "LogisticPotential")
        X = X.contiguous()
        y = y.to(X.dtype).contiguous()
        n, d = X.shape
        sites = {site_name: (slice(0, d), "identity", (d,))}
        super().__init__(N.MODEL_LOGISTIC, X.dtype, X.device, n, d, X, y, (prior_scale,), sites)


class GlmPotential:
    """Bayesian logistic, softmax or Poisson regression with constant-scale Normal priors:
    ``w ~ Normal(0, s_w)[D]``, ``b ~ Normal(0, s_b)``, ``y ~ Bernoulli(logits = X @ w + b)``, or
    ``W ~ Normal(0, s_w)[K, D]``, ``b ~ Normal(0, s_b)[K]`` (optional),
    ``y ~ Categorical(logits = X @ W.mT + b)``, or
    ``w ~ Normal(0, s_w)[D]``, ``b ~ Normal(0, s_b)`` (optional), ``y ~ Poisson(rate = exp(X @ w + b))``, or
    ``y ~ Binomial(trials, logits = X @ w + b)`` with ``trials`` one count or ``[N]`` counts, or
    ``w ~ Normal(0, s_w)[D]``, ``b ~ Normal(0, s_b)`` (optional), ``y ~ Normal(X @ w + b, sigma)`` with a constant
    ``sigma`` or a latent one (``sigma_site``) whose prior ``sigma_prior = (kind, p0, p1)`` is HalfNormal(p0),
    HalfCauchy(p0), Exponential(p0) or LogNormal(p0, p1); z then holds ``log sigma`` (transform ``"exp"``) and U
    carries the Jacobian ``-log sigma``, as ``TracePotential`` gives it.

    The weight scale may instead be latent (``weight_scale``): ``w ~ Normal(0, S)`` with ``S`` the
    positive scalar site ``tau_site``, the positive site ``lam_site`` of the weight's shape, or their product (the
    hierarchical, ARD and horseshoe priors).  ``tau_prior`` / ``lam_prior`` are ``(kind, p0, p1)`` as
    ``sigma_prior``, one value for every coefficient; z holds their logs (transform ``"exp"``), and U carries
    their Jacobians.

    A varying intercept by group (``group_effect``, every kind but softmax, constant weight scale): the
    linear predictor gains ``alpha[g]``, ``g`` the int64 ``[N]`` group index and ``alpha`` the ``G`` values of the
    site ``group["site"]``, drawn as ``Normal(0, s_a)`` (centred) or as ``eta ~ Normal(0, 1)`` with
    ``alpha = s_a * eta`` (``group["noncentred"]``).  ``s_a`` is the constant ``group["s_const"]`` or the positive
    scalar site ``group["s_site"]`` with prior ``group["s_prior"]`` (as ``sigma_prior``).  ``group["index"]`` must
    lie in ``[0, G)``; a private int32 copy is made once.  ``group["slopes"]`` lists up to three varying slopes,
    each a dict with the keys of the intercept (``site``, ``noncentred``, ``s_site``, ``s_const``, ``s_prior``) and
    ``col``: slope k adds ``beta_k[g] * X[:, col]``.  Up to ``D + G (1 + S) <= 128`` columns the group effect is
    more columns of the one contraction over ``[X | onehot(g) | X[:, col] onehot(g) ..]``.  Past that (up to
    ``G <= 65536``) it is gathered per row and its gradient summed over each group's rows, which needs the rows
    sorted by group: an index that is not non-decreasing raises ``ValueError`` there.  Sorting the rows of X, y
    and the index by group once changes nothing in the posterior.

    ``value_and_grad`` is one ``b2_glm_potential`` call on the ``b2_glm_regression`` built once here
    (``regression``): the likelihood of all chains comes from one pass of the fused GLM kernel over X, the chains
    being its particles.  ``sites`` maps each site name to
    ``(slice into z, transform, value shape)`` in the order and layout ``TracePotential`` gives the same
    model, so samples, ``initial_params`` and ``full_mass`` behave the same on either.  Every chain is
    evaluated; the sampler masks inactive chains, as it does for ``TracePotential``."""

    _SIGMA_PRIORS = {"HalfNormal": N.SIGMA_HALFNORMAL, "HalfCauchy": N.SIGMA_HALFCAUCHY,
                     "Exponential": N.SIGMA_EXPONENTIAL, "LogNormal": N.SIGMA_LOGNORMAL}

    def __init__(self, X, y, kind, sites, weight, bias=None, s_w=1.0, s_b=1.0, sigma=1.0, sigma_site=None,
                 sigma_prior=None, trials=None, tau_site=None, tau_prior=None, lam_site=None, lam_prior=None,
                 group=None):
        N.require_cuda(X, "GlmPotential")
        if X.dtype != torch.float32 or X.dim() != 2:
            raise ValueError("GlmPotential needs fp32 X of shape [N, D]")
        self.X = X.contiguous()
        self.normal = kind == "Normal"
        self.sigma, self.sigma_site = float(sigma), sigma_site
        if sigma_site is not None:
            pk, p0, p1 = sigma_prior
            self.sigma_prior = (self._SIGMA_PRIORS[pk], float(p0), float(p1))
        else:
            self.sigma_prior = (N.SIGMA_CONST, 0.0, 0.0)
        # a latent weight scale: b2_glm_weight_scale with the z columns of log tau / log lam (-1 when absent)
        self.tau_site, self.lam_site = tau_site, lam_site
        self.weight_scale = None
        if tau_site is not None or lam_site is not None:
            sc = N.b2_glm_weight_scale()
            sc.tau_off = sites[tau_site][0].start if tau_site is not None else -1
            sc.lam_off = sites[lam_site][0].start if lam_site is not None else -1
            for part, site, prior in (("tau", tau_site, tau_prior), ("lam", lam_site, lam_prior)):
                if site is None:
                    continue
                pk, p0, p1 = prior
                setattr(sc, part + "_prior", self._SIGMA_PRIORS[pk])
                setattr(sc, part + "_p0", float(p0))
                setattr(sc, part + "_p1", float(p1))
            self.weight_scale = sc
        self.kind = {"Bernoulli": N.GLM_BERNOULLI, "Categorical": N.GLM_CATEGORICAL, "Poisson": N.GLM_POISSON,
                     "Normal": N.GLM_NORMAL, "Binomial": N.GLM_BINOMIAL}[kind]
        self.binomial = kind == "Binomial"
        if self.binomial:
            # one count (on the device, read by the kernel) or the [N] counts, private and 16-byte aligned
            if isinstance(trials, torch.Tensor):
                self.trials, self.trials_per_row = trials.detach().to(X.device, torch.float32).reshape(-1).clone(), 1
            else:
                self.trials = torch.full((1,), float(trials), dtype=torch.float32, device=X.device)
                self.trials_per_row = 0
        # private contiguous copies: the kernels load y with TMA (16-byte aligned)
        self.y = (y.to(torch.int64) if self.kind == N.GLM_CATEGORICAL else y.to(torch.float32)).clone()
        self.sites = dict(sites)
        self.weight, self.bias = weight, bias
        self.n, self.Dx = self.X.shape
        wshape = self.sites[weight][2]
        self.K = int(wshape[0]) if self.kind == N.GLM_CATEGORICAL else 1
        self.w_off = self.sites[weight][0].start
        self.b_off = self.sites[bias][0].start if bias is not None else 0
        self.has_bias = bias is not None
        self.s_w, self.s_b = float(s_w), float(s_b)
        self.D = sum(sl.stop - sl.start for sl, _, _ in self.sites.values())
        self.dtype = torch.float32
        self.device = self.X.device
        self.group, self.group_effect = group, None
        if group is not None:
            self.group_effect = self._group_effect(group)
        self.regression = self._regression()

    def _regression(self):
        """b2_glm_regression of this potential: it points at the private X, y, trials and group-index copies and at
        the ``weight_scale`` / ``group_effect`` structs (a NULL pointer for a constant scale / no group effect)."""
        m = N.b2_glm_regression()
        m.kind, m.X, m.y = self.kind, self.X.data_ptr(), self.y.data_ptr()
        m.N, m.D, m.K = self.n, self.Dx, self.K
        if self.binomial:
            m.trials, m.trials_per_row = self.trials.data_ptr(), self.trials_per_row
        m.has_bias, m.w_off, m.b_off, m.s_w, m.s_b = int(self.has_bias), self.w_off, self.b_off, self.s_w, self.s_b
        m.s_off = self.sites[self.sigma_site][0].start if self.sigma_site is not None else -1
        (m.s_prior, m.sp0, m.sp1), m.sigma = self.sigma_prior, self.sigma
        if self.weight_scale is not None:
            m.scale = ctypes.pointer(self.weight_scale)
        if self.group_effect is not None:
            m.group = ctypes.pointer(self.group_effect)
        return m

    def _group_effect(self, group):
        """b2_glm_group_effect of ``group``, with the private int32 copy of the index it points to."""
        sl, _, shape = self.sites[group["site"]]
        G = int(shape[0])
        g = group["index"].detach().to(self.device).reshape(-1)
        if g.numel() != self.n or g.is_floating_point():
            raise ValueError("the group index must be an integer tensor of shape [N]")
        if G > 65536:
            raise ValueError("at most 65536 groups")
        try:
            self.groups = group_index_int32(g, G)
        except IndexError as e:
            raise ValueError(str(e)) from None
        ge = N.b2_glm_group_effect()
        # the gathered route past 128 columns needs the rows sorted by group (found by the same check)
        ge.sorted = int(bool(group_index_sorted(g, G)))
        ge.groups = self.groups.data_ptr()
        ge.a_off, ge.G, ge.noncentred = sl.start, G, int(bool(group["noncentred"]))
        s_site = group.get("s_site")
        if s_site is not None:
            pk, p0, p1 = group["s_prior"]
            ge.s_off, ge.s_prior, ge.sp0, ge.sp1 = self.sites[s_site][0].start, self._SIGMA_PRIORS[pk], p0, p1
        else:
            ge.s_off, ge.s_const = -1, float(group["s_const"])
        slopes = group.get("slopes", [])
        if len(slopes) > 3:
            raise ValueError("at most three varying slopes")
        ge.S = len(slopes)
        for k, sl in enumerate(slopes):
            e = ge.slope[k]
            bsl, _, bshape = self.sites[sl["site"]]
            if tuple(bshape) != (G,) or not 0 <= int(sl["col"]) < self.Dx:
                raise ValueError("a varying slope needs G values and a column of X")
            e.b_off, e.col, e.noncentred = bsl.start, int(sl["col"]), int(bool(sl["noncentred"]))
            if sl.get("s_site") is not None:
                pk, p0, p1 = sl["s_prior"]
                e.s_off, e.s_prior, e.sp0, e.sp1 = self.sites[sl["s_site"]][0].start, self._SIGMA_PRIORS[pk], p0, p1
            else:
                e.s_off, e.s_const = -1, float(sl["s_const"])
        if self.Dx + G * (1 + ge.S) > 128 and self.binomial:
            raise ValueError("Binomial regression takes at most 128 columns (D + G (1 + S)) with a group effect")
        if self.Dx + G * (1 + ge.S) > 128 and not ge.sorted:
            raise ValueError("past 128 columns (D + G (1 + S) = %d) the rows must be sorted by group"
                             % (self.Dx + G * (1 + ge.S)))
        return ge

    @property
    def dim(self):
        return self.D

    def value_and_grad(self, z, active=None):
        N.require_cuda(z, "GlmPotential")
        z = z.detach().to(torch.float32).contiguous()
        C = z.shape[0]
        U = torch.empty(C, dtype=torch.float32, device=z.device)
        g = torch.empty_like(z)
        lib = N.lib()
        need = int(lib.b2_glm_potential_workspace(ctypes.byref(self.regression), C))
        ws = N.workspace(z.device, need, tag="glm_potential")
        N.check(lib.b2_glm_potential(ctypes.byref(self.regression), z.data_ptr(), C, self.D, U.data_ptr(),
                                     g.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(z.device)),
                "b2_glm_potential")
        return U, g

    def unpack(self, z):
        return {name: self.unpack_site(name, z[..., sl]) for name, (sl, _, _) in self.sites.items()}

    def unpack_site(self, name, u):
        _, transform, shape = self.sites[name]
        v = u.exp() if transform == "exp" else u
        return v.reshape(u.shape[:-1] + tuple(shape))

    def init_uniform(self, num_chains, radius=2.0, generator=None):
        return (torch.rand(num_chains, self.D, dtype=self.dtype, device=self.device,
                           generator=generator) * 2 - 1) * radius


class TracePotential:
    """Potential of an arbitrary model, evaluated for ``C`` chains per call.

    The model is wrapped in an outermost ``plate("_num_chains", C, dim=-(max_plate_nesting+1))`` --
    the trick ``ELBO._vectorized_num_particles`` uses for particles (pyro/infer/elbo.py:186-203) --
    so the model must broadcast over a leading batch dim exactly as ``vectorize_particles`` requires.
    """

    def __init__(self, model, model_args=(), model_kwargs=None, num_chains=1, max_plate_nesting=None):
        self.model = model
        self.args = model_args
        self.kwargs = model_kwargs or {}
        self.C = num_chains
        # prototype trace (single execution, no chain plate) -> latent sites, transforms, layout
        proto = poutine.trace(model).get_trace(*self.args, **self.kwargs)
        proto = poutine.prune_subsample_sites(proto)
        if max_plate_nesting is None:
            # batch dims may be used without a plate (eight_schools does): reserve every batch dim
            # any site uses, so the chain dim sits to the left of all of them
            dims = [f.dim for s in proto.nodes.values() if s["type"] == "sample"
                    for f in s["cond_indep_stack"] if f.vectorized]
            nest = -min(dims) if dims else 0
            for s in proto.nodes.values():
                if s["type"] == "sample":
                    nest = max(nest, len(getattr(s["fn"], "batch_shape", ())))
            max_plate_nesting = nest
        self.max_plate_nesting = max_plate_nesting
        self.chain_dim = -(max_plate_nesting + 1)
        self.sites = {}
        self.transforms = {}
        off = 0
        ref = None
        for name, site in proto.nodes.items():
            if site["type"] != "sample" or site["is_observed"]:
                continue
            fn = site["fn"]
            if not site["value"].is_floating_point():
                raise ValueError("discrete latent site '{}' is not supported by HMC/NUTS here".format(name))
            t = biject_to(fn.support).inv  # constrained -> unconstrained (mcmc/util.py:452-453)
            u = t(site["value"].detach())
            n = u.numel()
            self.transforms[name] = t
            self.sites[name] = (slice(off, off + n), tuple(u.shape), tuple(site["value"].shape),
                                len(fn.batch_shape))
            off += n
            ref = site["value"]
        self.D = off
        self.dtype = ref.dtype if ref is not None else torch.get_default_dtype()
        self.device = ref.device if ref is not None else torch.device("cpu")
        self._proto = proto

    @property
    def dim(self):
        return self.D

    def _chain_shape(self, batch_ndim, ushape):
        """shape of a per-chain value carrying the chain dim at ``chain_dim`` of the batch shape"""
        event_ndim = len(ushape) - batch_ndim
        pad = self.max_plate_nesting - batch_ndim
        return (self.C,) + (1,) * pad + tuple(ushape)

    def constrain(self, z):
        """z [C, D] -> dict name -> constrained value with the chain dim in plate position,
        plus the summed log|det J| per chain."""
        C = z.shape[0]
        values = {}
        logdet = torch.zeros(C, dtype=z.dtype, device=z.device)
        for name, (sl, ushape, vshape, batch_ndim) in self.sites.items():
            t = self.transforms[name]
            u = z[:, sl].reshape((C,) + ushape)
            v = t.inv(u)
            ld = t.log_abs_det_jacobian(v, u)  # log|d u / d v|
            # U = -log_joint(v) + sum log|du/dv|  (mcmc/util.py:282-285)
            logdet = logdet + ld.reshape(C, -1).sum(-1) if ld.dim() > 0 else logdet + ld
            pad = self.max_plate_nesting - batch_ndim
            values[name] = v.reshape((C,) + (1,) * pad + tuple(v.shape[1:]))
        return values, logdet

    def value_and_grad(self, z, active=None):
        z = z.detach().requires_grad_(True)
        C = z.shape[0]
        with torch.enable_grad():
            values, logdet = self.constrain(z)
            chained = plate("_num_chains", C, dim=self.chain_dim)(self.model)
            trace = poutine.trace(poutine.condition(chained, data=values)).get_trace(*self.args, **self.kwargs)
            trace = poutine.prune_subsample_sites(trace)
            log_joint = torch.zeros(C, dtype=z.dtype, device=z.device)
            for name, site in trace.nodes.items():
                if site["type"] != "sample":
                    continue
                lp = site["fn"].log_prob(site["value"])
                lp = scale_and_mask(lp, site["scale"], site["mask"])
                # every site sits inside the chain plate, so the chain dim is batch dim
                # `chain_dim` (counted from the right); sum everything else
                lead = lp.dim() + self.chain_dim
                if lead < 0:
                    raise ValueError("site '{}' does not broadcast over the chain plate".format(name))
                other = [d for d in range(lp.dim()) if d != lead]
                if other:
                    lp = lp.sum(dim=other)
                log_joint = log_joint + lp
            U = -log_joint + logdet
            (g,) = torch.autograd.grad(U.sum(), z)
        return U.detach(), g

    def unpack(self, z):
        return {name: self.unpack_site(name, z[..., info[0]]) for name, info in self.sites.items()}

    def unpack_site(self, name, u):
        """Constrained value of ONE site from its unconstrained columns ``[..., n_site]``."""
        _, ushape, vshape, batch_ndim = self.sites[name]
        return self.transforms[name].inv(u.reshape(u.shape[:-1] + ushape))

    def init_uniform(self, num_chains, radius=2.0, generator=None):
        return (torch.rand(num_chains, self.D, dtype=self.dtype, device=self.device,
                           generator=generator) * 2 - 1) * radius


class WhitenedPotential:
    """``U'(z') = U(A z')`` for a per-chain lower-triangular factor ``A`` [C, D, D].

    Hamiltonian dynamics with mass matrix ``M = (A A^T)^-1`` on ``z`` are unit-mass dynamics on
    ``z' = A^-1 z`` (momenta map as ``r' = A^T r``; kinetic energy, the leapfrog map, the energy error and
    the U-turn products ``rho . M^-1 r`` are all invariant), so a DENSE adapted mass matrix
    (pyro/infer/mcmc/adaptation.py:238-392, ``full_mass=True``) costs two batched mat-vecs per potential
    evaluation here and every integrator / tree kernel stays on its identity-mass path.
    ``A`` is the Cholesky factor of the regularised sample covariance of a warm-up window
    (pyro/ops/welford.py:27-51 with ``diagonal=False``), i.e. the reference's inverse mass matrix."""

    def __init__(self, base):
        self.base = base
        self.A = None   # identity until the first mass-adaptation window closes
        self.sites = base.sites

    @property
    def dim(self):
        return self.base.dim

    @property
    def dtype(self):
        return self.base.dtype

    @property
    def device(self):
        return self.base.device

    def set_factor(self, A):
        self.A = A.contiguous()

    def to_original(self, zp):
        if self.A is None:
            return zp
        if zp.dim() == 2:
            return torch.bmm(self.A, zp.unsqueeze(-1)).squeeze(-1)
        # [C, T, D] sample arrays
        return torch.einsum("cij,ctj->cti", self.A, zp)

    def from_original(self, z):
        if self.A is None:
            return z
        return torch.linalg.solve_triangular(self.A, z.unsqueeze(-1), upper=False).squeeze(-1)

    def value_and_grad(self, zp, active=None, out_grad=None):
        z = self.to_original(zp).contiguous()
        U, g = self.base.value_and_grad(z, active)
        if self.A is not None:
            g = torch.bmm(self.A.transpose(-1, -2), g.unsqueeze(-1)).squeeze(-1)
        return U, g

    def unpack(self, z):
        return self.base.unpack(z)

    def unpack_site(self, name, u):
        return self.base.unpack_site(name, u)

    def init_uniform(self, num_chains, radius=2.0, generator=None):
        return self.base.init_uniform(num_chains, radius=radius, generator=generator)
