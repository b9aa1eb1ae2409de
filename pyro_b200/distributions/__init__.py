"""Distribution classes of the CUDA backend.

Host-side mirror of the reference's distribution protocol (pyro/distributions/distribution.py:29-222,
pyro/distributions/torch_distribution.py:19-232): ``sample/rsample/log_prob/score_parts/expand/
mask/to_event/has_rsample/batch_shape/event_shape/support``.  What differs is WHERE the arithmetic
runs: ``log_prob`` and ``score_parts`` dispatch to the fused sm_90a kernels through the C ABI
(``pyro_b200._native``); there is no ATen fallback -- scoring a CPU tensor raises.

Parameters are kept at their STORED shape; ``expand`` only records the new batch shape, and the
kernels read the operands through broadcast strides (what ExpandedDistribution does with views,
pyro/distributions/torch_distribution.py:399-488), so gradients are reduced to the stored shape
inside the backend instead of by autograd's ``sum_to_size``.

Sampling (``rsample``/``sample``) uses torch's generators; fusing it with scoring is the next
row of the scope table (SURVEY.md 8f rank 1).
"""
import ctypes
import math
import weakref
from collections import namedtuple
from numbers import Number

import torch
from torch.distributions import constraints

from .. import _native as N
from .._lazyparam import LazyExpParam, densify
from . import _ops


# ---------------------------------------------------------------------------------------------
# scale_and_mask / ScoreParts   (pyro/distributions/util.py:311-328, score_parts.py:11-38)
# ---------------------------------------------------------------------------------------------
def is_identically_zero(x):
    if isinstance(x, Number):
        return x == 0
    return False


def is_identically_one(x):
    if isinstance(x, Number):
        return x == 1
    return False


def scale_and_mask(tensor, scale=1.0, mask=None):
    if is_identically_zero(tensor) or (mask is None and is_identically_one(scale)):
        return tensor
    if mask is None or mask is True:
        return tensor * scale
    if mask is False:
        return torch.zeros_like(tensor)
    return torch.where(mask, tensor * scale, tensor.new_zeros(()))


class ScoreParts(namedtuple("ScoreParts", ["log_prob", "score_function", "entropy_term"])):
    def scale_and_mask(self, scale=1.0, mask=None):
        log_prob = scale_and_mask(self.log_prob, scale, mask)
        score_function = self.score_function  # not scaled
        entropy_term = scale_and_mask(self.entropy_term, scale, mask)
        return ScoreParts(log_prob, score_function, entropy_term)


def _as_tensor(x, like=None):
    if isinstance(x, torch.Tensor):
        return x
    if like is not None:
        return torch.as_tensor(x, dtype=like.dtype, device=like.device)
    return torch.as_tensor(x, dtype=torch.get_default_dtype())


_CONSTS = {}


def _const(value, dtype, device):
    """Cached 0-d constant: python-number parameters (``Normal(0., 1.)``) cost no fill kernel per
    step and stay valid under CUDA-graph capture (a fresh H2D copy of a scalar would not)."""
    key = (float(value), dtype, str(device))
    t = _CONSTS.get(key)
    if t is None:
        t = _CONSTS[key] = torch.full((), float(value), dtype=dtype, device=device)
    return t


def constant(value, like):
    """Cached 0-d tensor holding ``value`` on ``like``'s device/dtype (no kernel launch after the
    first call; safe to use inside a CUDA-graph captured step)."""
    return _const(value, like.dtype if like.is_floating_point() else torch.get_default_dtype(), like.device)


def _broadcast_params(*xs):
    """Tensor-ify python numbers next to the first tensor argument (dtype/device follow it; with no
    tensor argument they follow torch's default dtype and default device)."""
    ref = None
    for x in xs:
        if isinstance(x, torch.Tensor):
            ref = x
            break
    if ref is not None:
        dtype, device = (ref.dtype if ref.is_floating_point() else torch.get_default_dtype()), ref.device
    else:
        dtype, device = torch.get_default_dtype(), torch.get_default_device()
    out = []
    for x in xs:
        if isinstance(x, Number):
            t = _const(x, dtype, device)
        else:
            t = _as_tensor(x, ref)
            if ref is not None and t.dtype != ref.dtype and t.is_floating_point():
                t = t.to(ref.dtype)
        out.append(t)
    return out


# ---------------------------------------------------------------------------------------------
# base class
# ---------------------------------------------------------------------------------------------
class Distribution:
    has_rsample = False
    has_enumerate_support = False
    arg_constraints = {}
    support = constraints.real
    _event_ndim = 0

    def __init__(self, batch_shape=torch.Size(), event_shape=torch.Size()):
        self._batch_shape = torch.Size(batch_shape)
        self._event_shape = torch.Size(event_shape)

    # -- shapes ---------------------------------------------------------------------------------
    @property
    def batch_shape(self):
        return self._batch_shape

    @property
    def event_shape(self):
        return self._event_shape

    @property
    def event_dim(self):
        return len(self._event_shape)

    def shape(self, sample_shape=torch.Size()):
        return torch.Size(sample_shape) + self.batch_shape + self.event_shape

    # -- sampling -------------------------------------------------------------------------------
    def __call__(self, sample_shape=torch.Size()):
        # pyro/distributions/torch_distribution.py:31-52
        return self.rsample(sample_shape) if self.has_rsample else self.sample(sample_shape)

    def sample(self, sample_shape=torch.Size()):
        with torch.no_grad():
            return self.rsample(sample_shape)

    def rsample(self, sample_shape=torch.Size()):
        raise NotImplementedError

    def has_rsample_(self, value):
        if not (value is True or value is False):
            raise ValueError("Expected value in [False,True], actual {}".format(value))
        self.has_rsample = value
        return self

    # -- scoring --------------------------------------------------------------------------------
    def log_prob(self, value):
        raise NotImplementedError

    def score_parts(self, value):
        # pyro/distributions/distribution.py:98-125
        log_prob = self.log_prob(value)
        if self.has_rsample:
            return ScoreParts(log_prob=log_prob, score_function=0, entropy_term=log_prob)
        return ScoreParts(log_prob=log_prob, score_function=log_prob, entropy_term=0)

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        """0-d ``sum_coeff*sum(scale*mask*log_prob(value))`` with fused final gradients, or None
        if this distribution has no fused path (the caller then uses ``log_prob``)."""
        return None

    # -- structure ------------------------------------------------------------------------------
    def expand(self, batch_shape, _instance=None):
        raise NotImplementedError

    def expand_by(self, sample_shape):
        return self.expand(torch.Size(sample_shape) + self.batch_shape)

    def to_event(self, reinterpreted_batch_ndims=None):
        if reinterpreted_batch_ndims is None:
            reinterpreted_batch_ndims = len(self.batch_shape)
        if reinterpreted_batch_ndims == 0:
            return self
        return Independent(self, reinterpreted_batch_ndims)

    def independent(self, reinterpreted_batch_ndims=None):
        return self.to_event(reinterpreted_batch_ndims)

    def mask(self, mask):
        return MaskedDistribution(self, mask)


# ---------------------------------------------------------------------------------------------
# elementwise families on the fused kernel
# ---------------------------------------------------------------------------------------------
class _Elementwise(Distribution):
    family = None
    param_names = ()
    _torch_cls = None

    def __init__(self, *params, batch_shape=None):
        params = _broadcast_params(*params)
        self._params = params
        for n, p in zip(self.param_names, params):
            setattr(self, n, p)
        if batch_shape is None:
            batch_shape = torch.broadcast_shapes(*[p.shape for p in params])
        super().__init__(batch_shape)

    def _kernel_params(self):
        return self._params

    def expand(self, batch_shape, _instance=None):
        batch_shape = torch.Size(batch_shape)
        torch.broadcast_shapes(self.batch_shape, batch_shape)  # validates
        new = self.__class__.__new__(self.__class__)
        new.__dict__.update(self.__dict__)
        new._batch_shape = batch_shape
        return new

    def _torch(self):
        kw = {n: p.expand(self.batch_shape) if tuple(p.shape) != tuple(self.batch_shape) else p
              for n, p in zip(self.param_names, self._params)}
        return self._torch_cls(**kw, validate_args=False)

    def rsample(self, sample_shape=torch.Size()):
        return self._torch().rsample(sample_shape)

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)

    def _value(self, value):
        ref = self._params[0]
        if not isinstance(value, torch.Tensor):
            value = torch.as_tensor(value, dtype=ref.dtype, device=ref.device)
        if value.dtype != ref.dtype:
            value = value.to(ref.dtype)
        return value

    def log_prob(self, value):
        return _ops.log_prob_op(self.family, self._value(value), self._kernel_params(),
                                self.batch_shape)

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        return _ops.fused_site_sum(self.family, self._value(value), self._kernel_params(),
                                   self.batch_shape, mask=mask, scale=scale, weight=weight,
                                   sum_coeff=sum_coeff, assume_unit_upstream=unit)

    @property
    def mean(self):
        return self._torch().mean

    @property
    def variance(self):
        return self._torch().variance

    def entropy(self):
        return self._torch().entropy()

    def __repr__(self):
        args = ", ".join("{}: {}".format(n, tuple(p.shape)) for n, p in zip(self.param_names, self._params))
        return "{}({}; batch_shape={})".format(type(self).__name__, args, tuple(self.batch_shape))


class Normal(_Elementwise):
    family = N.NORMAL
    param_names = ("loc", "scale")
    arg_constraints = {"loc": constraints.real, "scale": constraints.positive}
    support = constraints.real
    has_rsample = True
    _torch_cls = torch.distributions.Normal

    def __init__(self, loc, scale, validate_args=None):
        super().__init__(loc, scale)
        # a positive parameter handed out as deferred exp(u) (pyro_b200/_lazyparam.py): the draw kernel takes
        # u = log(scale) as stored and returns d/du; every other use materialises exp(u)
        sc = self._params[1]
        self._log_scale = sc.log_value if isinstance(sc, LazyExpParam) and sc.dtype == self._params[0].dtype \
            else None

    def rsample(self, sample_shape=torch.Size()):
        """``loc + eps*scale`` (torch/distributions/normal.py:82-85).  On the GPU the draw and its
        own log density come out of ONE kernel (SURVEY.md 8(f) row 1): the returned tensor carries
        the 0-d ``sum log q(z)`` as ``z._b2_rsample`` so that an ELBO scoring this very site can
        claim it instead of launching a scoring kernel, and the backward of the pair is one kernel
        that hands (d/dloc, d/dscale) back in their stored shapes."""
        shape = self.shape(sample_shape)
        n = 1
        for d in shape:
            n *= int(d)
        loc = densify(self.loc)
        if (N.FUSED_DRAW and N.PHILOX_DRAW and loc.is_cuda and 0 < n <= N.RSAMPLE_MAX_N and len(shape) <= 6
                and loc.dtype == self.scale.dtype):
            # noise generated inside the draw kernel (Philox): no randn launch, graph-replay safe
            coeff = _Coeff()
            if self._log_scale is not None and N.LATENT_BLOCK:
                z, lq = _NormalRsampleFn.apply(coeff, loc, self._log_scale, None, torch.Size(shape), True)
            else:
                z, lq = _NormalRsampleFn.apply(coeff, loc, densify(self.scale), None, torch.Size(shape), False)
            if N.LATENT_BLOCK:
                # a deferred draw (_ops.defer_latent_draw): reading z or lq launches it first
                z, lq = z.as_subclass(_ops.DeferredDraw), lq.as_subclass(_ops.DeferredDraw)
            z._b2_rsample = _RsampleTag(self.loc, self.scale, lq, coeff)
            return z
        eps = torch.randn(shape, dtype=loc.dtype, device=loc.device)
        return self.rsample_with_noise(eps)

    def rsample_with_noise(self, eps):
        """The draw for given standard-normal noise ``eps`` (shape = sample_shape + batch_shape)."""
        loc = densify(self.loc)
        if not N.FUSED_DRAW or (not eps.is_cuda and not N.EMULATE_RSAMPLE):
            return torch.addcmul(loc, eps, densify(self.scale))   # plain draw; scored later by b2_site_score
        coeff = _Coeff()
        if self._log_scale is not None and N.LATENT_BLOCK:
            z, lq = _NormalRsampleFn.apply(coeff, loc, self._log_scale, eps, None, True)
        else:
            z, lq = _NormalRsampleFn.apply(coeff, loc, densify(self.scale), eps, None, False)
        z._b2_rsample = _RsampleTag(self.loc, self.scale, lq, coeff)
        return z


class _Coeff:
    """Coefficient with which a fused draw's ``sum log q`` entered the loss (set by whoever claims
    it).  Kept apart from the tag: the autograd node holds THIS object only -- holding the tag (which
    holds the node's own output) would be a reference cycle through the C++ graph that Python's GC
    cannot break, keeping every step's graph alive."""
    __slots__ = ("value", "prior", "__weakref__")

    def __init__(self):
        self.value = 0.0
        self.prior = None     # (prior_loc, prior_scale, weight of sum log p(z) in the loss): see claim_rsample_prior


class _RsampleTag:
    """Travels on a fused draw: the parameters it was drawn with, its summed log density, and the
    coefficient holder shared with the draw's autograd node."""
    __slots__ = ("loc", "scale", "lq", "coeff")

    def __init__(self, loc, scale, lq, coeff):
        self.loc, self.scale, self.lq, self.coeff = loc, scale, lq, coeff


class _NormalRsampleFn(torch.autograd.Function):
    """``(z, sum log q(z))`` of a Normal site.  ``scale`` is the scale, or with ``log_scale`` the unconstrained
    storage u = log(scale) of a positive parameter (the gradient then comes back w.r.t. u)."""

    @staticmethod
    def forward(ctx, coeff, loc, scale, eps, shape, log_scale=False):
        if eps is None:
            if N.LATENT_BLOCK:
                z, lq, eps = _ops.defer_latent_draw(loc, scale, log_scale, shape)
            else:
                z, lq, eps = _ops.normal_rsample_philox(loc, scale.exp() if log_scale else scale, shape)
        else:
            z, lq = _ops.normal_rsample_score(loc, scale.exp() if log_scale else scale, eps)
        ctx.coeff = coeff
        ctx.log_scale = log_scale
        ctx.save_for_backward(eps, loc, scale, z)
        ctx.set_materialize_grads(False)
        return z, lq

    @staticmethod
    @_ops.once_differentiable
    def backward(ctx, gz, glq):
        eps, loc, scale, z = ctx.saved_tensors
        # the sum log q output is only reachable through the tag; its consumer folds its
        # coefficient into tag.coeff and sends a unit upstream gradient (Trace_ELBO's contract).  A claimed
        # prior (claim_rsample_prior) rides on the same contract.
        c = ctx.coeff.value if glq is not None else 0.0
        prior = ctx.coeff.prior if glq is not None else None
        if N.LATENT_BLOCK:
            gloc, gscale = _ops.latent_backward(gz, eps, z, loc, scale, ctx.log_scale, c, prior,
                                                ctx.needs_input_grad[1], ctx.needs_input_grad[2],
                                                accumulate=N.LATENT_ACCUMULATE)
        else:
            if gz is None:
                gz = _const(0.0, eps.dtype, eps.device)
            s = scale.exp() if ctx.log_scale else scale
            gloc, gscale = _ops.normal_rsample_backward(gz, eps, loc, s, c, ctx.needs_input_grad[1],
                                                        ctx.needs_input_grad[2])
            if ctx.log_scale and gscale is not None:
                gscale = gscale * s
        return None, gloc, gscale, None, None, None


def claim_rsample_prior(fn, value, weight):
    """A model site ``value ~ fn`` whose value is a fused draw with a claimed score: if ``fn`` is a Normal with
    gradient-free parameters, register ``weight`` (the coefficient of ``sum log_prob(value)`` in the loss being
    differentiated) with the draw, whose backward kernel then adds ``weight * d log p/dz`` to the gradient
    reaching z -- no separate gradient kernel for the prior, no accumulation launch at z.  Returns
    ``(z, prior_loc, prior_scale)`` for the value-only scoring (``_ops.latent_prior``), or None."""
    if not N.LATENT_BLOCK:
        return None
    tag = getattr(value, "_b2_rsample", None)
    if tag is None or tag.coeff.value == 0.0 or tag.coeff.prior is not None:
        return None
    base = fn
    while isinstance(base, Independent):
        base = base.base_dist
    if type(base) is not Normal:
        return None
    ploc, pscale = base._params
    if isinstance(ploc, LazyExpParam) or isinstance(pscale, LazyExpParam):
        return None
    if ploc.requires_grad or pscale.requires_grad or not value.is_cuda and not N.EMULATE_RSAMPLE:
        return None
    if ploc.dtype != value.dtype or pscale.dtype != value.dtype or ploc.device != value.device:
        return None
    if value.numel() == 0 or value.numel() > N.RSAMPLE_MAX_N or value.dim() > 6:
        return None
    if torch.broadcast_shapes(value.shape, base.batch_shape) != value.shape:
        return None
    tag.coeff.prior = (ploc, pscale, float(weight))
    return value, ploc, pscale


def claim_rsample_score(fn, value, coeff):
    """If ``value`` is a fused draw from (the Normal underneath) ``fn``, register ``coeff`` -- the
    coefficient of ``sum log_prob(value)`` in the loss being differentiated -- and return the
    precomputed 0-d sum; else None."""
    tag = getattr(value, "_b2_rsample", None)
    if tag is None:
        return None
    base = fn
    while isinstance(base, Independent):
        base = base.base_dist
    if type(base) is not Normal or base.loc is not tag.loc or base.scale is not tag.scale:
        return None
    if torch.broadcast_shapes(value.shape, base.batch_shape) != value.shape:
        return None
    tag.coeff.value += float(coeff)
    return tag.lq


class Cauchy(_Elementwise):
    family = N.CAUCHY
    param_names = ("loc", "scale")
    arg_constraints = {"loc": constraints.real, "scale": constraints.positive}
    has_rsample = True
    _torch_cls = torch.distributions.Cauchy

    def __init__(self, loc, scale, validate_args=None):
        super().__init__(loc, scale)


class HalfCauchy(_Elementwise):
    family = N.HALFCAUCHY
    param_names = ("scale",)
    arg_constraints = {"scale": constraints.positive}
    support = constraints.nonnegative
    has_rsample = True
    _torch_cls = torch.distributions.HalfCauchy

    def __init__(self, scale, validate_args=None):
        super().__init__(scale)


class HalfNormal(_Elementwise):
    family = N.HALFNORMAL
    param_names = ("scale",)
    arg_constraints = {"scale": constraints.positive}
    support = constraints.nonnegative
    has_rsample = True
    _torch_cls = torch.distributions.HalfNormal

    def __init__(self, scale, validate_args=None):
        super().__init__(scale)


class LogNormal(_Elementwise):
    family = N.LOGNORMAL
    param_names = ("loc", "scale")
    arg_constraints = {"loc": constraints.real, "scale": constraints.positive}
    support = constraints.positive
    has_rsample = True
    _torch_cls = torch.distributions.LogNormal

    def __init__(self, loc, scale, validate_args=None):
        super().__init__(loc, scale)


class Exponential(_Elementwise):
    family = N.EXPONENTIAL
    param_names = ("rate",)
    arg_constraints = {"rate": constraints.positive}
    support = constraints.nonnegative
    has_rsample = True
    _torch_cls = torch.distributions.Exponential

    def __init__(self, rate, validate_args=None):
        super().__init__(rate)


class Uniform(_Elementwise):
    family = N.UNIFORM
    param_names = ("low", "high")
    arg_constraints = {"low": constraints.dependent, "high": constraints.dependent}
    has_rsample = True
    _torch_cls = torch.distributions.Uniform

    def __init__(self, low, high, validate_args=None):
        super().__init__(low, high)

    @property
    def support(self):
        return constraints.interval(self.low, self.high)


class Gamma(_Elementwise):
    family = N.GAMMA
    param_names = ("concentration", "rate")
    arg_constraints = {"concentration": constraints.positive, "rate": constraints.positive}
    support = constraints.nonnegative
    has_rsample = True
    _torch_cls = torch.distributions.Gamma

    def __init__(self, concentration, rate, validate_args=None):
        super().__init__(concentration, rate)

    def rsample(self, sample_shape=torch.Size()):
        """``_standard_gamma(concentration) / rate`` clamped away from 0 (torch/distributions/gamma.py:79-87).  On
        the GPU one kernel draws (Marsaglia-Tsang on the in-kernel Philox stream) and evaluates the
        implicit-reparameterisation derivative d z / d concentration that the backward pass needs
        (``b2_gamma_rsample``; SURVEY.md 8(f) row 1)."""
        shape = self.shape(sample_shape)
        conc, rate = densify(self.concentration), densify(self.rate)
        if (N.GAMMA_RSAMPLE and conc.is_cuda and conc.dtype == rate.dtype and len(shape) <= 6
                and conc.dtype in (torch.float32, torch.float64) and all(int(d) > 0 for d in shape)):
            return _GammaRsampleFn.apply(conc, rate, torch.Size(shape))
        return self._torch().rsample(sample_shape)


class _GammaRsampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, conc, rate, shape):
        need = ctx.needs_input_grad[0]
        z, dz = _ops.gamma_rsample(conc, rate, shape, want_grad=need)
        ctx.save_for_backward(z, dz, rate)
        ctx.shapes = (conc.shape, rate.shape)
        return z

    @staticmethod
    @_ops.once_differentiable
    def backward(ctx, gz):
        z, dz, rate = ctx.saved_tensors
        cshape, rshape = ctx.shapes
        gconc = (gz * dz).sum_to_size(cshape) if ctx.needs_input_grad[0] else None
        grate = (-(gz * z) / rate).sum_to_size(rshape) if ctx.needs_input_grad[1] else None
        return gconc, grate, None


class Beta(_Elementwise):
    family = N.BETA
    param_names = ("concentration1", "concentration0")
    arg_constraints = {"concentration1": constraints.positive, "concentration0": constraints.positive}
    support = constraints.unit_interval
    has_rsample = True
    _torch_cls = torch.distributions.Beta

    def __init__(self, concentration1, concentration0, validate_args=None):
        super().__init__(concentration1, concentration0)


class Poisson(_Elementwise):
    family = N.POISSON
    param_names = ("rate",)
    arg_constraints = {"rate": constraints.nonnegative}
    support = constraints.nonnegative_integer
    has_rsample = False
    _torch_cls = torch.distributions.Poisson

    def __init__(self, rate, validate_args=None, is_sparse=False):
        # is_sparse (pyro/distributions/torch.py:280-294) changes only which elements are
        # evaluated; the fused kernel evaluates the dense form in one pass either way.
        super().__init__(rate)

    def rsample(self, sample_shape=torch.Size()):
        raise NotImplementedError("Poisson has no rsample")

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)


class Bernoulli(_Elementwise):
    arg_constraints = {"probs": constraints.unit_interval, "logits": constraints.real}
    support = constraints.boolean
    has_rsample = False

    def __init__(self, probs=None, logits=None, validate_args=None):
        if (probs is None) == (logits is None):
            raise ValueError("Either `probs` or `logits` must be specified, but not both.")
        if logits is not None:
            self.family = N.BERNOULLI_LOGITS
            self.param_names = ("logits",)
            super().__init__(logits)
        else:
            self.family = N.BERNOULLI_PROBS
            self.param_names = ("probs",)
            super().__init__(probs)

    def _torch(self):
        p = self._params[0]
        p = p.expand(self.batch_shape) if tuple(p.shape) != tuple(self.batch_shape) else p
        if self.family == N.BERNOULLI_LOGITS:
            return torch.distributions.Bernoulli(logits=p, validate_args=False)
        return torch.distributions.Bernoulli(probs=p, validate_args=False)

    def rsample(self, sample_shape=torch.Size()):
        raise NotImplementedError("Bernoulli has no rsample")

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)


class Binomial(_Elementwise):
    """Binomial(total_count, probs | logits) of pyro/distributions/torch.py:83-101 with ``approx_log_prob_tol = 0``
    (the exact log binomial coefficient).  Gradients are those autograd gives for the reference expression, whose
    ``log_binomial`` is gradient-free: d/dlogits = k - n sigmoid(logits), d/dtotal_count = -softplus(logits)."""
    arg_constraints = {"total_count": constraints.nonnegative_integer, "probs": constraints.unit_interval,
                       "logits": constraints.real}
    has_rsample = False

    def __init__(self, total_count=1, probs=None, logits=None, validate_args=None):
        if (probs is None) == (logits is None):
            raise ValueError("Either `probs` or `logits` must be specified, but not both.")
        param = logits if logits is not None else probs
        param, total_count = _broadcast_params(param, total_count)
        if not total_count.is_floating_point() or total_count.dtype != param.dtype:
            total_count = total_count.to(param.dtype)
        if logits is not None:
            self.family = N.BINOMIAL_LOGITS
            self.param_names = ("total_count", "logits")
        else:
            self.family = N.BINOMIAL_PROBS
            self.param_names = ("total_count", "probs")
        super().__init__(total_count, param)

    @constraints.dependent_property(is_discrete=True, event_dim=0)
    def support(self):
        return constraints.integer_interval(0, self.total_count)

    def _torch(self):
        n, p = (t.expand(self.batch_shape) if tuple(t.shape) != tuple(self.batch_shape) else t
                for t in self._params)
        if self.family == N.BINOMIAL_LOGITS:
            return torch.distributions.Binomial(n, logits=p, validate_args=False)
        return torch.distributions.Binomial(n, probs=p, validate_args=False)

    def rsample(self, sample_shape=torch.Size()):
        raise NotImplementedError("Binomial has no rsample")

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)


# ---------------------------------------------------------------------------------------------
# event families
# ---------------------------------------------------------------------------------------------
def _event_contiguous(t, event_ndim):
    """The event kernels index the trailing event dims as one dense row-major block."""
    if t is None or event_ndim == 0:
        return t
    expect = 1
    for d in range(1, event_ndim + 1):
        if t.shape[-d] != 1 and t.stride(-d) != expect:
            return t.contiguous()
        expect *= t.shape[-d]
    return t


class _EventFamily(Distribution):
    family = None

    def expand(self, batch_shape, _instance=None):
        batch_shape = torch.Size(batch_shape)
        torch.broadcast_shapes(self.batch_shape, batch_shape)
        new = self.__class__.__new__(self.__class__)
        new.__dict__.update(self.__dict__)
        new._batch_shape = batch_shape
        return new

    def rsample(self, sample_shape=torch.Size()):
        return self._torch().rsample(sample_shape)

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)


class Dirichlet(_EventFamily):
    family = N.DIRICHLET
    arg_constraints = {"concentration": constraints.independent(constraints.positive, 1)}
    support = constraints.simplex
    has_rsample = True

    def __init__(self, concentration, validate_args=None):
        concentration = _event_contiguous(concentration, 1)
        self.concentration = concentration
        super().__init__(concentration.shape[:-1], concentration.shape[-1:])

    def _torch(self):
        c = self.concentration.expand(self.batch_shape + self.event_shape)
        return torch.distributions.Dirichlet(c, validate_args=False)

    def log_prob(self, value):
        value = _event_contiguous(value, 1)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape[:-1])
        return _ops.log_prob_op(self.family, value, [self.concentration], bshape,
                                event_size=self.event_shape[0])

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        value = _event_contiguous(value, 1)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape[:-1])
        return _ops.fused_site_sum(self.family, value, [self.concentration], bshape, mask=mask,
                                   scale=scale, weight=weight, sum_coeff=sum_coeff,
                                   event_size=self.event_shape[0], assume_unit_upstream=unit)


class Categorical(_EventFamily):
    family = N.CATEGORICAL
    arg_constraints = {"probs": constraints.simplex, "logits": constraints.real_vector}
    has_rsample = False
    has_enumerate_support = True

    def __init__(self, probs=None, logits=None, validate_args=None):
        if (probs is None) == (logits is None):
            raise ValueError("Either `probs` or `logits` must be specified, but not both.")
        if probs is not None:
            # torch/distributions/categorical.py:70-72 + utils.probs_to_logits: log of the
            # normalised, clamped probabilities.  The kernel normalises logits itself.
            eps = torch.finfo(probs.dtype).eps
            logits = torch.log((probs / probs.sum(-1, keepdim=True)).clamp(min=eps, max=1 - eps))
        logits = _event_contiguous(logits, 1)
        self._logits_raw = logits
        self._num_events = logits.shape[-1]
        super().__init__(logits.shape[:-1])

    @property
    def logits(self):
        return self._logits_raw - self._logits_raw.logsumexp(dim=-1, keepdim=True)

    @property
    def probs(self):
        return torch.softmax(self._logits_raw, dim=-1)

    @property
    def support(self):
        return constraints.integer_interval(0, self._num_events - 1)

    def _torch(self):
        lg = self._logits_raw.expand(self.batch_shape + (self._num_events,))
        return torch.distributions.Categorical(logits=lg, validate_args=False)

    def rsample(self, sample_shape=torch.Size()):
        raise NotImplementedError("Categorical has no rsample")

    def sample(self, sample_shape=torch.Size()):
        return self._torch().sample(sample_shape)

    def _value(self, value):
        if value.dtype != torch.int64:
            value = value.long()
        return value

    def log_prob(self, value):
        value = self._value(value)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape)
        return _ops.log_prob_op(self.family, value, [self._logits_raw], bshape,
                                event_size=self._num_events)

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        value = self._value(value)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape)
        return _ops.fused_site_sum(self.family, value, [self._logits_raw], bshape, mask=mask,
                                   scale=scale, weight=weight, sum_coeff=sum_coeff,
                                   event_size=self._num_events, assume_unit_upstream=unit)

    def enumerate_support(self, expand=True):
        return self._torch().enumerate_support(expand)


class MultivariateNormal(_EventFamily):
    family = N.MVN_TRIL
    arg_constraints = {"loc": constraints.real_vector, "scale_tril": constraints.lower_cholesky}
    support = constraints.real_vector
    has_rsample = True

    def __init__(self, loc, covariance_matrix=None, precision_matrix=None, scale_tril=None,
                 validate_args=None):
        if (covariance_matrix is not None) + (scale_tril is not None) + (precision_matrix is not None) != 1:
            raise ValueError("Exactly one of covariance_matrix or precision_matrix or scale_tril "
                             "may be specified.")
        if covariance_matrix is not None:
            scale_tril = torch.linalg.cholesky(covariance_matrix)
        elif precision_matrix is not None:
            # torch/distributions/multivariate_normal.py:_precision_to_scale_tril
            Lf = torch.linalg.cholesky(torch.flip(precision_matrix, (-2, -1)))
            L_inv = torch.transpose(torch.flip(Lf, (-2, -1)), -2, -1)
            Id = torch.eye(precision_matrix.shape[-1], dtype=precision_matrix.dtype,
                           device=precision_matrix.device)
            scale_tril = torch.linalg.solve_triangular(L_inv, Id, upper=False)
        self.loc = _event_contiguous(loc, 1)
        self.scale_tril = _event_contiguous(scale_tril, 2)
        batch = torch.broadcast_shapes(loc.shape[:-1], scale_tril.shape[:-2])
        super().__init__(batch, loc.shape[-1:])

    def _torch(self):
        return torch.distributions.MultivariateNormal(
            self.loc.expand(self.batch_shape + self.event_shape),
            scale_tril=self.scale_tril.expand(self.batch_shape + self.event_shape * 2),
            validate_args=False)

    def log_prob(self, value):
        value = _event_contiguous(value, 1)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape[:-1])
        return _ops.log_prob_op(self.family, value, [self.loc, self.scale_tril], bshape,
                                event_size=self.event_shape[0])

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        value = _event_contiguous(value, 1)
        bshape = torch.broadcast_shapes(self.batch_shape, value.shape[:-1])
        return _ops.fused_site_sum(self.family, value, [self.loc, self.scale_tril], bshape,
                                   mask=mask, scale=scale, weight=weight, sum_coeff=sum_coeff,
                                   event_size=self.event_shape[0], assume_unit_upstream=unit)


class Delta(Distribution):
    """Degenerate point mass (pyro/distributions/delta.py); pure bookkeeping, no kernel needed:
    log_prob is ``log_density`` where value == v (always true for replayed sites)."""
    has_rsample = True
    arg_constraints = {"v": constraints.dependent, "log_density": constraints.real}

    def __init__(self, v, log_density=0.0, event_dim=0, validate_args=None):
        self.v = v
        self.log_density = _as_tensor(log_density, v) if not isinstance(log_density, torch.Tensor) else log_density
        batch_dim = v.dim() - event_dim
        super().__init__(v.shape[:batch_dim], v.shape[batch_dim:])

    @property
    def support(self):
        return constraints.independent(constraints.real, len(self.event_shape))

    def expand(self, batch_shape, _instance=None):
        batch_shape = torch.Size(batch_shape)
        new = Delta.__new__(Delta)
        new.v = self.v.expand(batch_shape + self.event_shape)
        new.log_density = self.log_density.expand(batch_shape) if self.log_density.dim() else self.log_density
        Distribution.__init__(new, batch_shape, self.event_shape)
        return new

    def rsample(self, sample_shape=torch.Size()):
        return self.v.expand(self.shape(sample_shape))

    def log_prob(self, x):
        v = self.v.expand(self.shape())
        lp = (x == v).type(x.dtype).log()
        for _ in range(len(self.event_shape)):
            lp = lp.sum(-1)
        return lp + self.log_density


# ---------------------------------------------------------------------------------------------
# wrappers
# ---------------------------------------------------------------------------------------------
class Independent(Distribution):
    """Reinterprets batch dims as event dims (torch.distributions.Independent semantics,
    reached in the reference through TorchDistributionMixin.to_event,
    pyro/distributions/torch_distribution.py:163-213)."""

    def __init__(self, base_dist, reinterpreted_batch_ndims, validate_args=None):
        if reinterpreted_batch_ndims > len(base_dist.batch_shape):
            raise ValueError("Expected reinterpreted_batch_ndims <= len(base_distribution.batch_shape), "
                             "actual {} vs {}".format(reinterpreted_batch_ndims, len(base_dist.batch_shape)))
        self.base_dist = base_dist
        self.reinterpreted_batch_ndims = reinterpreted_batch_ndims
        shape = base_dist.batch_shape + base_dist.event_shape
        ev = reinterpreted_batch_ndims + len(base_dist.event_shape)
        super().__init__(shape[: len(shape) - ev], shape[len(shape) - ev:])

    @property
    def has_rsample(self):
        return self.base_dist.has_rsample

    @has_rsample.setter
    def has_rsample(self, value):
        self.base_dist.has_rsample = value

    @property
    def support(self):
        return constraints.independent(self.base_dist.support, self.reinterpreted_batch_ndims)

    def rsample(self, sample_shape=torch.Size()):
        return self.base_dist.rsample(sample_shape)

    def sample(self, sample_shape=torch.Size()):
        return self.base_dist.sample(sample_shape)

    def log_prob(self, value):
        lp = self.base_dist.log_prob(value)
        n = self.reinterpreted_batch_ndims
        return lp.sum(dim=tuple(range(-n, 0))) if n else lp

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        # the total over batch AND event dims is what the ELBO needs; a site mask has batch
        # shape, so align it with the base distribution's batch dims
        if mask is not None and isinstance(mask, torch.Tensor):
            mask = mask.reshape(mask.shape + (1,) * self.reinterpreted_batch_ndims)
        return self.base_dist._fused_sum(value, mask, scale, weight, sum_coeff, unit)

    def expand(self, batch_shape, _instance=None):
        batch_shape = torch.Size(batch_shape)
        n = self.reinterpreted_batch_ndims
        base_event = self.event_shape[:n]
        return Independent(self.base_dist.expand(batch_shape + base_event), n)

    def to_event(self, reinterpreted_batch_ndims=None):
        if reinterpreted_batch_ndims is None:
            reinterpreted_batch_ndims = len(self.batch_shape)
        if reinterpreted_batch_ndims == 0:
            return self
        return Independent(self.base_dist, self.reinterpreted_batch_ndims + reinterpreted_batch_ndims)

    def entropy(self):
        e = self.base_dist.entropy()
        n = self.reinterpreted_batch_ndims
        return e.sum(dim=tuple(range(-n, 0))) if n else e


class MaskedDistribution(Distribution):
    """pyro/distributions/torch_distribution.py:302-374."""

    def __init__(self, base_dist, mask):
        if isinstance(mask, bool):
            self._mask = mask
        else:
            batch_shape = torch.broadcast_shapes(mask.shape, base_dist.batch_shape)
            if mask.shape != batch_shape:
                mask = mask.expand(batch_shape)
            if base_dist.batch_shape != batch_shape:
                base_dist = base_dist.expand(batch_shape)
            self._mask = mask.bool()
        self.base_dist = base_dist
        super().__init__(base_dist.batch_shape, base_dist.event_shape)

    @property
    def has_rsample(self):
        return self.base_dist.has_rsample

    @has_rsample.setter
    def has_rsample(self, value):
        self.base_dist.has_rsample = value

    @property
    def support(self):
        return self.base_dist.support

    def expand(self, batch_shape, _instance=None):
        batch_shape = torch.Size(batch_shape)
        mask = self._mask
        if isinstance(mask, torch.Tensor):
            mask = mask.expand(batch_shape)
        return MaskedDistribution(self.base_dist.expand(batch_shape), mask)

    def rsample(self, sample_shape=torch.Size()):
        return self.base_dist.rsample(sample_shape)

    def sample(self, sample_shape=torch.Size()):
        return self.base_dist.sample(sample_shape)

    def log_prob(self, value):
        if self._mask is False:
            shape = torch.broadcast_shapes(self.base_dist.batch_shape,
                                           value.shape[: value.dim() - self.event_dim])
            return torch.zeros((), device=value.device).expand(shape)
        if self._mask is True:
            return self.base_dist.log_prob(value)
        return scale_and_mask(self.base_dist.log_prob(value), mask=self._mask)

    def score_parts(self, value):
        if isinstance(self._mask, bool):
            return super().score_parts(value)
        return self.base_dist.score_parts(value).scale_and_mask(mask=self._mask)

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        if self._mask is False:
            return None
        m = self._mask if isinstance(self._mask, torch.Tensor) else None
        if m is not None and mask is not None and isinstance(mask, torch.Tensor):
            m = m & mask
        elif m is None:
            m = mask
        return self.base_dist._fused_sum(value, m, scale, weight, sum_coeff, unit)


# ---------------------------------------------------------------------------------------------
# KL divergences on the fused kernel (torch/distributions/kl.py:301-306,468-471), used by
# TraceMeanField_ELBO (pyro/infer/trace_mean_field_elbo.py:117-132)
# ---------------------------------------------------------------------------------------------
def kl_divergence(p, q):
    if isinstance(p, Independent) and isinstance(q, Independent):
        if p.reinterpreted_batch_ndims != q.reinterpreted_batch_ndims:
            raise NotImplementedError
        kl = kl_divergence(p.base_dist, q.base_dist)
        n = p.reinterpreted_batch_ndims
        return kl.sum(dim=tuple(range(-n, 0))) if n else kl
    if type(p) is Normal and type(q) is Normal:
        fam = N.KL_NORMAL_NORMAL
    elif type(p) is Gamma and type(q) is Gamma:
        fam = N.KL_GAMMA_GAMMA
    else:
        raise NotImplementedError("kl_divergence({}, {})".format(type(p).__name__, type(q).__name__))
    shape = torch.broadcast_shapes(p.batch_shape, q.batch_shape)
    return _ops.log_prob_op(fam, None, list(p._params) + list(q._params), shape)


def fused_kl_sum(p, q, mask, scale, weight, sum_coeff, unit=True):
    """0-d ``sum_coeff*sum(scale*mask*KL(p||q))`` with fused final gradients, or None."""
    while isinstance(p, Independent) and isinstance(q, Independent) and \
            p.reinterpreted_batch_ndims == q.reinterpreted_batch_ndims:
        if mask is not None and isinstance(mask, torch.Tensor):
            mask = mask.reshape(mask.shape + (1,) * p.reinterpreted_batch_ndims)
        p, q = p.base_dist, q.base_dist
    if type(p) is Normal and type(q) is Normal:
        fam = N.KL_NORMAL_NORMAL
    elif type(p) is Gamma and type(q) is Gamma:
        fam = N.KL_GAMMA_GAMMA
    else:
        return None
    shape = torch.broadcast_shapes(p.batch_shape, q.batch_shape)
    return _ops.fused_site_sum(fam, None, list(p._params) + list(q._params), shape, mask=mask,
                               scale=scale, weight=weight, sum_coeff=sum_coeff, assume_unit_upstream=unit)


__all__ = ["Distribution", "Normal", "Bernoulli", "Binomial", "Gamma", "Beta", "Poisson", "Cauchy", "HalfCauchy",
           "HalfNormal", "LogNormal", "Exponential", "Uniform", "Dirichlet", "Categorical",
           "MultivariateNormal", "Delta", "Independent", "MaskedDistribution", "ScoreParts",
           "kl_divergence", "scale_and_mask", "is_identically_zero", "is_identically_one"]


# ---------------------------------------------------------------------------------------------
# fused generalised-linear likelihood (BASELINE config 2): Bernoulli(logits = X w + b)
# ---------------------------------------------------------------------------------------------
class LinearPredictor:
    """Lazy ``X @ w^T + b`` for P weight vectors: behaves like a ``[P, N]`` (or ``[N]``) logits
    tensor when handed to ``Bernoulli(logits=...)``, but lets the site be scored by ONE kernel
    that reads X and y once and emits sum, dW and db (``b2_glm_bernoulli_logits``) instead of
    materialising the [P, N] logits, log_prob and gradient tensors.

    ``w``: [D], [P, D] or [P, 1, D] (vectorised particles);  ``b``: None, [], [P] or [P, 1].

    ``group`` (a :class:`GroupGather`, or None): a varying intercept by group, ``+ table[..., index]``, which the
    unchanged model added (pyro_b200/lazy.py); its table has one row, or one per particle.  ``slopes`` (a tuple of up
    to three :class:`SlopeGather`, each with its ``col``): varying slopes by group on columns of X,
    ``+ table[..., index] * X[:, col]``, with the group's index and G.  ``eager`` then computes the predictor the way
    the model wrote it, so that :meth:`dense` is that value bit for bit.  A consumer that does not score the group
    and the slopes (``_weights``) must not see such a predictor: it is scored by ``b2_glm_group_sum`` (an intercept)
    or ``b2_glm_group_slope_sum`` (an intercept and slopes), past 128 columns with a sorted index by
    ``b2_glm_group_gather_sum``, or materialised (slopes without an intercept)."""

    def __init__(self, X, w, b=None, tensor_cores=True, group=None, eager=None, slopes=()):
        # latent values may arrive as lazy-aware SiteValue tensors (pyro_b200/lazy.py): score plain ones
        if type(w).__name__ == "SiteValue":
            w = _ops.plain_value(w)
        if type(b).__name__ == "SiteValue":
            b = _ops.plain_value(b)
        self.X, self.w, self.b = X, w, b
        self.group, self.eager, self.slopes = group, eager, tuple(slopes)
        self.tensor_cores = tensor_cores  # False: fp32 SIMT contractions (B2_FLAG_GLM_FP32)
        D = X.shape[-1]
        self.vectorised = w.dim() > 1
        self.P = w.numel() // D
        self.shape = torch.Size((self.P, X.shape[0])) if self.vectorised else torch.Size((X.shape[0],))
        self.dtype, self.device = X.dtype, X.device

    def dense(self):
        if self.eager is not None:
            return self.eager()
        W = self.w.reshape(self.P, -1)
        out = W @ self.X.t()
        if self.b is not None:
            out = out + self.b.reshape(self.P, 1)
        out = out if self.vectorised else out.squeeze(0)
        out = out if self.group is None else out + self.group.dense()
        for sg in self.slopes:
            out = out + sg.dense()
        return out


class GroupGather:
    """Lazy ``table[..., index]``: a latent table of G values per row (``[G]``, ``[P, G]``, ``[P, 1, G]``) gathered
    along its last dim by a gradient-free int64 ``[N]`` group index.  It stands for the ``[..., N]`` tensor only until
    it is added to a lazy ``X @ w + b`` (:class:`LinearPredictor` ``group``); every other use materialises it."""

    def __init__(self, table, index):
        if type(table).__name__ == "SiteValue":
            table = _ops.plain_value(table)
        self.table, self.index = table, index
        self.G = table.shape[-1]
        self.shape = table.shape[:-1] + index.shape
        self.dtype, self.device = table.dtype, table.device

    def dense(self):
        return self.table[..., self.index]


class SlopeGather:
    """Lazy ``table[..., index] * covariate``: a :class:`GroupGather` times a gradient-free fp32 ``[N]`` covariate on the
    table's device (either side of ``*``).  Added to a lazy ``X @ w + b`` whose X has the covariate as column ``col``
    (``X[:, col]``, ``X[..., col]``, ``X.select(-1, col)``), it becomes one of the predictor's varying slopes
    (:class:`LinearPredictor` ``slopes``, which sets ``col``); every other use materialises it."""

    def __init__(self, table, index, covariate):
        if type(table).__name__ == "SiteValue":
            table = _ops.plain_value(table)
        self.table, self.index, self.covariate = table, index, covariate
        self.col = None
        self.G = table.shape[-1]
        self.shape = torch.broadcast_shapes(table.shape[:-1] + index.shape, covariate.shape)
        self.dtype, self.device = table.dtype, table.device

    def with_col(self, col):
        out = SlopeGather(self.table, self.index, self.covariate)
        out.col = col
        return out

    def dense(self):
        # a product of two floats is commutative bit for bit: the model's order of the factors does not matter
        return self.table[..., self.index] * self.covariate


# int32 copies of group indices for b2_glm_group_sum and GlmPotential: id(index) -> (weakref, _version, device, G,
# copy, sorted).  A copy is built (one conversion, one host sync for its range check and for whether the index is
# non-decreasing) the first time an index is scored, e.g. in SVI's eager warm-up step, so a graph-captured step reuses
# it without a sync; a fresh index tensor every step (subsampling) pays the conversion and the check every step.
_INDEX32 = {}


def _index_entry(index, G):
    key = id(index)
    hit = _INDEX32.get(key)
    if hit is not None and hit[0]() is index and hit[1:4] == (index._version, index.device, G):
        return hit
    if N.capturing():
        return None
    g = index.detach().reshape(-1)
    # one host sync for both reductions
    bad, descends = torch.stack([((g < 0) | (g >= G)).any(), (g[1:] < g[:-1]).any()]).tolist()
    if bad:
        raise IndexError("group index outside [0, %d)" % G)
    copy = g.to(torch.int32, copy=True)
    hit = (weakref.ref(index, lambda _, k=key: _INDEX32.pop(k, None)), index._version, index.device, G, copy,
           not descends)
    _INDEX32[key] = hit
    return hit


def group_index_int32(index, G):
    """The int32 copy of the int64 group index ``index`` ([N], any device), checked once against ``[0, G)``: an index
    outside raises IndexError before anything reads it.  None while a CUDA graph is captured and no copy exists yet
    (the check needs a host sync), so the caller can materialise instead."""
    hit = _index_entry(index, G)
    return None if hit is None else hit[4]


def group_index_sorted(index, G):
    """Whether the group index ``index`` is non-decreasing (the rows sorted by group), found in the same check and
    cached with :func:`group_index_int32`'s copy; None while a CUDA graph is captured and nothing is cached yet."""
    hit = _index_entry(index, G)
    return None if hit is None else hit[5]


def linear_predictor(X, w, b=None, tensor_cores=True):
    return LinearPredictor(X, w, b, tensor_cores)


class ExpLinearPredictor:
    """Lazy ``exp(X @ w^T + b)`` of a :class:`LinearPredictor` ``lp``: behaves like the ``[P, N]`` (or ``[N]``)
    rate tensor when handed to ``Poisson(rate)``, which then scores the site with ONE kernel that reads X and the
    counts once and emits sum, dW and db (``b2_glm_poisson_log_rate``).  ``eager`` (optional) computes the
    log-rate the way the model wrote it, so that :meth:`dense` is ``torch.exp`` of the eager value bit for bit."""

    def __init__(self, lp, eager=None):
        self.lp, self._eager = lp, eager
        self.shape, self.dtype, self.device = lp.shape, lp.dtype, lp.device

    def dense(self):
        return torch.exp(self._eager() if self._eager is not None else self.lp.dense())


class _FusedSumFn(torch.autograd.Function):
    """The site sum of a fused likelihood kernel as one autograd node.  ``meta`` is ``(scale, weight, sum_coeff,
    unit, ...)`` with the family's own arguments after ``unit``; ``launch(meta, *operands)`` makes the native call
    and returns the total and one gradient per operand (None for a data operand).  ``backward`` returns those
    gradients, times ``gout`` unless ``unit`` (the kernel already applied the caller's coefficient)."""

    @staticmethod
    def forward(ctx, launch, meta, *operands):
        total, *grads = launch(meta, *operands)
        ctx.grads, ctx.unit = grads, meta[3]
        return total

    @staticmethod
    def backward(ctx, gout):
        grads = ctx.grads if ctx.unit else [g * gout if g is not None else None for g in ctx.grads]
        return (None, None, *grads)


class _FusedSum:
    """One family's fused site sum: ``apply(meta, *operands)`` is :class:`_FusedSumFn` with the family's launch.
    Every fused call of the family goes through ``apply`` of this one object, so a test or profile can count or
    intercept a family's calls by replacing it."""

    def __init__(self, launch):
        self.launch = launch

    def apply(self, meta, *operands):
        return _FusedSumFn.apply(self.launch, meta, *operands)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _glm_outputs(X, W, need):
    """The total, dW (W's shape) and db (W's shape without D) of a GLM likelihood call on X's device, and its
    ``"glm"`` workspace of ``need`` bytes."""
    dev = X.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    dW = torch.empty(W.shape, dtype=torch.float32, device=dev)
    db = torch.empty(W.shape[:-1], dtype=torch.float32, device=dev)
    return total, dW, db, N.workspace(dev, need, tag="glm")


def _glm_bernoulli(meta, X, y, W, b):
    scale, weight, coeff, _, flags = meta
    N.require_cuda(X, "fused GLM likelihood")
    P, D = W.shape
    n = X.shape[0]
    dev = X.device
    total, dW, db, ws = _glm_outputs(X, W, int(N.lib().b2_glm_workspace(n, D, P)))
    Wc, bc = W.contiguous(), b.contiguous() if b is not None else None
    args = (X.data_ptr(), y.data_ptr(), Wc.data_ptr(), _ptr(bc), n, D, P, float(scale), float(weight),
            float(coeff), int(flags), None, total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel())
    asm = _ops.take_elbo_assembly(dev)
    if asm is None:
        N.check(N.lib().b2_glm_bernoulli_logits(*args, N.stream_ptr(dev)), "b2_glm_bernoulli_logits")
    else:
        # the step's loss comes out of this call's finish kernel (the priors' sums and the other ELBO terms)
        asm, jobs, n_jobs, jc, ptrs, tc, n_terms, _keep = asm
        loss = torch.empty((), dtype=torch.float32, device=dev)
        sc = N.workspace(dev, int(N.lib().b2_glm_elbo_workspace()), tag="glm_elbo")
        N.check(N.lib().b2_glm_bernoulli_logits_elbo(*args, jobs, n_jobs, jc, ptrs, tc, n_terms, loss.data_ptr(),
                                                     sc.data_ptr(), sc.numel(), N.stream_ptr(dev)),
                "b2_glm_bernoulli_logits_elbo")
        asm.loss, asm.total = loss, total
    return total, None, None, dW, db if b is not None else None


_GlmBernoulliFn = _FusedSum(_glm_bernoulli)


def _lazy_as(x, cls):
    """The lazy object of type ``cls`` that ``x`` is or stands for (a LinearPredictorTensor wrapping it), or None."""
    if isinstance(x, cls):
        return x
    lz = getattr(x, "_lazy", None) if isinstance(x, torch.Tensor) else None
    return lz if isinstance(lz, cls) else None


def _weights(lp):
    """``(W [P, D], b [P] or None)`` of a LinearPredictor without a group effect or slopes."""
    if lp.group is not None or lp.slopes:
        raise RuntimeError("pyro_b200: a linear predictor with a group effect reached a kernel that does not score it")
    return lp.w.reshape(lp.P, lp.X.shape[-1]), lp.b.reshape(lp.P) if lp.b is not None else None


def _row_scope(lp, value, mask, batch_shape, D):
    """``(X, y)`` for the tensor-core kernels of the per-row GLM families (Bernoulli, Poisson, Normal, Binomial) at
    D contraction columns (1..128), or None outside their scope.  They take tensor cores asked for, fp32, contiguous
    16-byte aligned X and y, no mask, one value per row and the predictor's batch shape, from 8192 rows: below that
    the single-pass TF32 gradient has not averaged its rounding down to fp32 accuracy yet, and these kernels have no
    fp32 counterpart."""
    X = lp.X
    ok = (mask is None and X.dtype == torch.float32 and X.is_contiguous() and X.data_ptr() % 16 == 0
          and 1 <= D <= 128 and getattr(lp, "tensor_cores", True) and X.shape[0] >= 8192
          and isinstance(value, torch.Tensor) and value.numel() == X.shape[0]
          and tuple(batch_shape) == tuple(lp.shape))
    y = value.reshape(-1).to(torch.float32).contiguous() if ok else None
    if not ok or y.data_ptr() % 16 != 0:
        return None
    return X, y


def _per_row_scope(lp, value, mask, batch_shape):
    """``(X, y, W, b)`` of :func:`_row_scope` for a predictor without a group effect or slopes, or None."""
    rs = _row_scope(lp, value, mask, batch_shape, lp.X.shape[-1]) if lp.group is None and not lp.slopes else None
    return None if rs is None else rs + _weights(lp)


def _glm_group(meta, X, y, W, b, A, sigma):
    scale, weight, coeff, _, kind, idx, trials, per_row, s_stride = meta
    N.require_cuda(X, "fused multilevel-regression likelihood")
    P, D = W.shape
    G = A.shape[-1]
    n = X.shape[0]
    dev = X.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    dWA = torch.empty((P, D + G), dtype=torch.float32, device=dev)       # [d/dw | d/dalpha] per particle
    db = torch.empty(P, dtype=torch.float32, device=dev)
    dsig = torch.empty(P, dtype=torch.float32, device=dev) if sigma is not None and sigma.requires_grad else None
    ws = N.workspace(dev, int(N.lib().b2_glm_group_sum_workspace(kind, n, D, G, P)), tag="glm")
    Wc, Ac = W.contiguous(), A.contiguous()
    bc = b.contiguous() if b is not None else None
    sc = sigma.contiguous() if sigma is not None else None
    a_stride = 0 if Ac.numel() == G else G        # one table row shared by every particle, or one per particle
    N.check(N.lib().b2_glm_group_sum(
        kind, X.data_ptr(), y.data_ptr(), _ptr(trials), per_row, _ptr(sc), s_stride, idx.data_ptr(), G,
        Wc.data_ptr(), D, Ac.data_ptr(), a_stride, _ptr(bc), n, D, P, float(scale), float(weight), float(coeff), 0,
        None, total.data_ptr(), dWA.data_ptr(), db.data_ptr(), _ptr(dsig), ws.data_ptr(), ws.numel(),
        N.stream_ptr(dev)), "b2_glm_group_sum")
    dA = dWA[:, D:]
    dA = (dA.sum(0) if a_stride == 0 else dA).reshape(A.shape)
    if dsig is not None and s_stride == 0:
        dsig = dsig.sum().reshape(sigma.shape)      # one sigma shared by every particle
    return total, None, None, dWA[:, :D], db if b is not None else None, dA, dsig


_GlmGroupFn = _FusedSum(_glm_group)


def _glm_slope(meta, X, y, W, b, A, sigma, *B):
    scale, weight, coeff, _, kind, idx, trials, per_row, s_stride, cols = meta
    N.require_cuda(X, "fused multilevel-regression likelihood")
    P, D = W.shape
    G, S = A.shape[-1], len(B)
    Da = D + G * (1 + S)
    n = X.shape[0]
    dev = X.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    dWAB = torch.empty((P, Da), dtype=torch.float32, device=dev)     # [d/dw | d/dalpha | d/dbeta_1 ..] per particle
    db = torch.empty(P, dtype=torch.float32, device=dev)
    dsig = torch.empty(P, dtype=torch.float32, device=dev) if sigma is not None and sigma.requires_grad else None
    ws = N.workspace(dev, int(N.lib().b2_glm_group_slope_sum_workspace(kind, n, D, G, S, P)), tag="glm")
    Wc, Ac = W.contiguous(), A.contiguous()
    Bc = [t.contiguous() for t in B]
    bc = b.contiguous() if b is not None else None
    sc = sigma.contiguous() if sigma is not None else None
    a_stride = 0 if Ac.numel() == G else G        # one table row shared by every particle, or one per particle
    b_strides = [0 if t.numel() == G else G for t in Bc]
    sl = N.b2_glm_slope_tables(S)
    for k in range(S):
        sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], Bc[k].data_ptr(), b_strides[k]
    N.check(N.lib().b2_glm_group_slope_sum(
        kind, X.data_ptr(), y.data_ptr(), _ptr(trials), per_row, _ptr(sc), s_stride, idx.data_ptr(), G,
        Wc.data_ptr(), D, Ac.data_ptr(), a_stride, ctypes.byref(sl), _ptr(bc), n, D, P, float(scale), float(weight),
        float(coeff), 0, None, total.data_ptr(), dWAB.data_ptr(), db.data_ptr(), _ptr(dsig), ws.data_ptr(),
        ws.numel(), N.stream_ptr(dev)), "b2_glm_group_slope_sum")

    def table_grad(k, t, stride):          # block k of the group columns: alpha (0) or beta_k
        g = dWAB[:, D + k * G:D + (k + 1) * G]
        return (g.sum(0) if stride == 0 else g).reshape(t.shape)
    dA = table_grad(0, A, a_stride)
    dB = [table_grad(k + 1, t, st) for k, (t, st) in enumerate(zip(B, b_strides))]
    if dsig is not None and s_stride == 0:
        dsig = dsig.sum().reshape(sigma.shape)      # one sigma shared by every particle
    return (total, None, None, dWAB[:, :D], db if b is not None else None, dA, dsig) + tuple(dB)


_GlmSlopeFn = _FusedSum(_glm_slope)


def _glm_gather(meta, X, y, W, b, sigma, *T):
    scale, weight, coeff, _, kind, idx, s_stride, cols = meta
    N.require_cuda(X, "fused multilevel-regression likelihood")
    P, D = W.shape
    G, S = T[0].shape[-1], len(T) - 1
    n = X.shape[0]
    dev = X.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    dW = torch.empty((P, D), dtype=torch.float32, device=dev)
    db = torch.empty(P, dtype=torch.float32, device=dev)
    dT = torch.empty((1 + S, P, G), dtype=torch.float32, device=dev)   # d/dalpha, d/dbeta_1 .. per particle
    dsig = torch.empty(P, dtype=torch.float32, device=dev) if sigma is not None and sigma.requires_grad else None
    ws = N.workspace(dev, int(N.lib().b2_glm_group_gather_sum_workspace(kind, n, D, G, S, P)), tag="glm")
    Wc, bc = W.contiguous(), b.contiguous() if b is not None else None
    sc = sigma.contiguous() if sigma is not None else None
    Tc = [t.contiguous() for t in T]
    strides = [0 if t.numel() == G else G for t in Tc]   # one table row shared by every particle, or one per particle
    sl = N.b2_glm_slope_tables(S)
    for k in range(S):
        sl.col[k], sl.beta[k], sl.beta_stride[k] = cols[k], Tc[k + 1].data_ptr(), strides[k + 1]
    N.check(N.lib().b2_glm_group_gather_sum(
        kind, X.data_ptr(), y.data_ptr(), _ptr(sc), s_stride, idx.data_ptr(), G, Wc.data_ptr(), D, Tc[0].data_ptr(),
        strides[0], ctypes.byref(sl), _ptr(bc), n, D, P, float(scale), float(weight), float(coeff), 0, None,
        total.data_ptr(), dW.data_ptr(), db.data_ptr(), _ptr(dsig), dT.data_ptr(), ws.data_ptr(), ws.numel(),
        N.stream_ptr(dev)), "b2_glm_group_gather_sum")
    dTs = tuple((dT[k].sum(0) if st == 0 else dT[k]).reshape(t.shape) for k, (t, st) in enumerate(zip(T, strides)))
    if dsig is not None and s_stride == 0:
        dsig = dsig.sum().reshape(sigma.shape)      # one sigma shared by every particle
    return (total, None, None, dW, db if b is not None else None, dsig) + dTs


_GlmGatherFn = _FusedSum(_glm_gather)


def _gather_sum(kind, lp, value, mask, batch_shape, coeffs, sigma):
    """The site sum of a predictor with a group effect (and up to three slopes) past 128 columns through
    ``b2_glm_group_gather_sum``, or None outside its scope: :func:`_row_scope` at X's D columns, logistic, Poisson or
    linear regression, G <= 65536, tables of X's dtype and device, and a cached index that is sorted (a subsample, or
    any other unsorted index, materialises)."""
    grp, slopes = lp.group, lp.slopes
    D = lp.X.shape[-1]
    rs = _row_scope(lp, value, mask, batch_shape, D)
    tables = (grp.table,) + tuple(sg.table for sg in slopes)
    if (rs is None or kind not in (N.GLM_BERNOULLI, N.GLM_POISSON, N.GLM_NORMAL) or grp.G > 65536
            or any(t.dtype != torch.float32 or t.device != lp.X.device for t in tables)):
        return None
    idx = group_index_int32(grp.index, grp.G)
    if idx is None or not group_index_sorted(grp.index, grp.G):
        return None
    W, b = lp.w.reshape(lp.P, D), lp.b.reshape(lp.P) if lp.b is not None else None
    meta = coeffs + (kind, idx, sigma[1], tuple(sg.col for sg in slopes))
    return _GlmGatherFn.apply(meta, *rs, W, b, sigma[0], *tables)


def _slope_sum(kind, lp, value, mask, batch_shape, coeffs, trials=(None, 0), sigma=(None, 0)):
    """The site sum of a predictor with a group effect and varying slopes through ``b2_glm_group_slope_sum``, or None
    outside its scope: an intercept, :func:`_row_scope` at D + G (1 + S) columns, and tables of X's dtype and device.
    Past 128 columns, :func:`_gather_sum`.  An index outside ``[0, G)`` raises IndexError before any launch."""
    grp, slopes = lp.group, lp.slopes
    if grp is None:
        return None                 # slopes without an intercept: the kernel always scores alpha, so materialise
    D = lp.X.shape[-1]
    if D + grp.G * (1 + len(slopes)) > 128:
        return _gather_sum(kind, lp, value, mask, batch_shape, coeffs, sigma)
    rs = _row_scope(lp, value, mask, batch_shape, D + grp.G * (1 + len(slopes)))
    tables = (grp.table,) + tuple(sg.table for sg in slopes)
    if rs is None or any(t.dtype != torch.float32 or t.device != lp.X.device for t in tables):
        return None
    idx = group_index_int32(grp.index, grp.G)
    if idx is None:
        return None
    W, b = lp.w.reshape(lp.P, D), lp.b.reshape(lp.P) if lp.b is not None else None
    meta = coeffs + (kind, idx) + tuple(trials) + (sigma[1], tuple(sg.col for sg in slopes))
    return _GlmSlopeFn.apply(meta, *rs, W, b, grp.table, sigma[0], *(sg.table for sg in slopes))


def _group_sum(kind, lp, value, mask, batch_shape, coeffs, trials=(None, 0), sigma=(None, 0)):
    """The site sum of a predictor with a group effect through ``b2_glm_group_sum``, or None outside its scope:
    :func:`_row_scope` at D + G columns, and a table of X's dtype and device.  An index outside ``[0, G)`` raises
    IndexError before any launch.  A predictor with slopes goes to :func:`_slope_sum`, and past 128 columns to
    :func:`_gather_sum`."""
    if lp.slopes:
        return _slope_sum(kind, lp, value, mask, batch_shape, coeffs, trials, sigma)
    grp = lp.group
    D = lp.X.shape[-1]
    if D + grp.G > 128:
        return _gather_sum(kind, lp, value, mask, batch_shape, coeffs, sigma)
    rs = _row_scope(lp, value, mask, batch_shape, D + grp.G)
    if rs is None or grp.table.dtype != torch.float32 or grp.table.device != lp.X.device:
        return None
    idx = group_index_int32(grp.index, grp.G)
    if idx is None:
        return None
    W, b = lp.w.reshape(lp.P, D), lp.b.reshape(lp.P) if lp.b is not None else None
    return _GlmGroupFn.apply(coeffs + (kind, idx) + tuple(trials) + (sigma[1],), *rs, W, b, grp.table, sigma[0])


class _BernoulliLinear(Bernoulli):
    """Bernoulli whose logits are a LinearPredictor (built by ``Bernoulli(logits=lazy)``, or by an
    unchanged model whose ``w @ X.T + b`` was kept lazy by pyro_b200/lazy.py)."""

    def __init__(self, probs=None, logits=None, validate_args=None):
        lazy = _lazy_as(logits, LinearPredictor)
        self._lazy = lazy
        self.family = N.BERNOULLI_LOGITS
        self.param_names = ("logits",)
        self._dense = None
        Distribution.__init__(self, lazy.shape)

    @property
    def _params(self):
        if self._dense is None:
            self._dense = self._lazy.dense()
        return [self._dense]

    @property
    def logits(self):
        return self._params[0]

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        lz = self._lazy
        if lz.group is not None or lz.slopes:
            out = _group_sum(N.GLM_BERNOULLI, lz, value, mask, self.batch_shape, (scale, weight, sum_coeff, unit))
            return out if out is not None else super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        X = lz.X
        tc = getattr(lz, "tensor_cores", True)
        if X.shape[-1] in (4, 8, 16, 32):
            # these D also have the fp32 SIMT kernel of glm.cu: any N, with or without tensor cores, any y
            ok = (mask is None and X.dtype == torch.float32 and X.is_contiguous()
                  and isinstance(value, torch.Tensor) and value.numel() == X.shape[0]
                  and tuple(self.batch_shape) == tuple(lz.shape) and X.data_ptr() % 16 == 0)
            args = (X, value.reshape(-1).to(torch.float32).contiguous()) + _weights(lz) if ok else None
        else:
            args = _per_row_scope(lz, value, mask, self.batch_shape)
        if args is None:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        return _GlmBernoulliFn.apply((scale, weight, sum_coeff, unit, 0 if tc else N.B2_FLAG_GLM_FP32), *args)


def _bernoulli_new(cls, probs=None, logits=None, validate_args=None):
    # ``Bernoulli(logits=LinearPredictor)`` builds the fused-GLM subclass
    if cls is Bernoulli and _lazy_as(logits, LinearPredictor) is not None:
        return object.__new__(_BernoulliLinear)
    return object.__new__(cls)


Bernoulli.__new__ = staticmethod(_bernoulli_new)


# ---------------------------------------------------------------------------------------------
# fused softmax regression: Categorical(logits = X @ W.mT + b)
# ---------------------------------------------------------------------------------------------
class ClassLinearPredictor:
    """Lazy class-axis logits ``X @ W.mT + b`` for K classes: behaves like an ``[N, K]`` logits tensor
    (``W``: [K, D]) or a ``[P, N, K]`` one (``W``: [P, K, D], vectorised particles) when handed to
    ``Categorical(logits=...)``, which then scores the site with ONE kernel that reads X and the labels
    once and emits sum, dW and db (``b2_glm_categorical_logits``).  A separate type from
    :class:`LinearPredictor`, whose ``[P, D]`` weights are particles, not classes.

    ``Wt`` is the right-hand operand exactly as the model wrote it (``[.., D, K]``, usually the ``W.mT``
    view); ``b``: None, [K] or [P, 1, K].  ``linear`` records an ``F.linear(X, W[, b])`` call, so that
    :meth:`dense` repeats the eager computation bit for bit."""

    def __init__(self, X, Wt, b=None, linear=False, linear_bias=False):
        if type(Wt).__name__ == "SiteValue":
            Wt = _ops.plain_value(Wt)
        if type(b).__name__ == "SiteValue":
            b = _ops.plain_value(b)
        self.X, self.Wt, self.b = X, Wt, b
        self.linear, self.linear_bias = linear, linear_bias
        self.vectorised = Wt.dim() == 3
        self.P = Wt.shape[0] if self.vectorised else 1
        self.K = Wt.shape[-1]
        n = X.shape[0]
        self.shape = torch.Size((self.P, n, self.K)) if self.vectorised else torch.Size((n, self.K))
        self.dtype, self.device = X.dtype, X.device

    @property
    def W(self):
        return self.Wt.mT

    def with_bias(self, b):
        """The predictor plus ``b`` ([K], or [P, 1, K] with vectorised particles), or None."""
        if self.b is not None or not isinstance(b, torch.Tensor):
            return None
        shapes = [(self.K,)] + ([(self.P, 1, self.K)] if self.vectorised else [])
        if tuple(b.shape) not in shapes or b.dtype != self.dtype or b.device != self.device:
            return None
        return ClassLinearPredictor(self.X, self.Wt, b, self.linear)

    def bias_pk(self):
        """The bias as [P, K] (a view), or None."""
        return None if self.b is None else self.b.reshape(-1, self.K).expand(self.P, self.K)

    def dense(self):
        import torch.nn.functional as F
        if self.linear_bias:
            return F.linear(self.X, self.W, self.b)
        out = F.linear(self.X, self.W) if self.linear else self.X @ self.Wt
        return out if self.b is None else out + self.b


def class_linear_predictor(X, W, b=None):
    """Lazy ``X @ W.mT + b`` with ``W``: [K, D] (logits [N, K]) or [P, K, D] (logits [P, N, K]) and ``b``:
    None, [K] or [P, 1, K]; other shapes, dtypes or devices raise ValueError."""
    if not (isinstance(X, torch.Tensor) and X.dim() == 2 and isinstance(W, torch.Tensor) and W.dim() in (2, 3)
            and W.shape[-1] == X.shape[1] and W.dtype == X.dtype and W.device == X.device):
        raise ValueError("class_linear_predictor: expected X [N, D] and W [K, D] or [P, K, D] of X's dtype and "
                         "device, got X %s and W %s" % (tuple(getattr(X, "shape", ())), tuple(getattr(W, "shape", ()))))
    lp = ClassLinearPredictor(X, W.mT)
    if b is None:
        return lp
    out = lp.with_bias(_ops.plain_value(b) if type(b).__name__ == "SiteValue" else b)
    if out is None:
        raise ValueError("class_linear_predictor: the bias must be [K]%s of X's dtype and device, got %s"
                         % (" or [P, 1, K]" if lp.vectorised else "", tuple(getattr(b, "shape", ()))))
    return out


def _glm_categorical(meta, X, y, W, b):
    scale, weight, coeff, _ = meta
    N.require_cuda(X, "fused softmax-regression likelihood")
    P, K, D = W.shape
    n = X.shape[0]
    total, dW, db, ws = _glm_outputs(X, W, int(N.lib().b2_glm_categorical_workspace(n, D, K, P)))
    Wc, bc = W.contiguous(), b.contiguous() if b is not None else None
    N.check(N.lib().b2_glm_categorical_logits(
        X.data_ptr(), y.data_ptr(), Wc.data_ptr(), _ptr(bc), n, D, K, P, float(scale), float(weight),
        float(coeff), 0, None, total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(),
        N.stream_ptr(X.device)), "b2_glm_categorical_logits")
    return total, None, None, dW, db if b is not None else None


_GlmCategoricalFn = _FusedSum(_glm_categorical)


class _CategoricalLinear(Categorical):
    """Categorical whose logits are a ClassLinearPredictor (built by ``Categorical(logits=lazy)``, or by an
    unchanged model whose ``X @ W.mT + b`` was kept lazy by pyro_b200/lazy.py).  ``log_prob``, ``logits``
    and ``probs`` materialise the logits; the ELBO's site sum takes the fused kernel."""

    def __init__(self, probs=None, logits=None, validate_args=None):
        lazy = _lazy_as(logits, ClassLinearPredictor)
        self._lazy = lazy
        self._dense = None
        self._num_events = lazy.K
        Distribution.__init__(self, lazy.shape[:-1])

    @property
    def _logits_raw(self):
        if self._dense is None:
            self._dense = self._lazy.dense()
        return self._dense

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        lz = self._lazy
        X = lz.X
        n, D = X.shape
        # D == 32 and N >= 8192: the tensor-core kernel's scope and precision policy (as for Bernoulli)
        ok = (mask is None and X.dtype == torch.float32 and lz.Wt.dtype == torch.float32
              and X.is_contiguous() and X.data_ptr() % 16 == 0 and D == 32 and 2 <= lz.K <= 16 and n >= 8192
              and isinstance(value, torch.Tensor) and value.numel() == n
              and tuple(self.batch_shape) == tuple(lz.shape[:-1]))
        if not ok:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        y = self._value(value).reshape(-1).contiguous()
        if y.data_ptr() % 16 != 0:
            y = y.clone()
        W = lz.W.reshape(lz.P, lz.K, D)
        return _GlmCategoricalFn.apply((scale, weight, sum_coeff, unit), X, y, W, lz.bias_pk())


def _categorical_new(cls, probs=None, logits=None, validate_args=None):
    # ``Categorical(logits=ClassLinearPredictor)`` builds the fused softmax-regression subclass
    if cls is Categorical and probs is None and _lazy_as(logits, ClassLinearPredictor) is not None:
        return object.__new__(_CategoricalLinear)
    return object.__new__(cls)


Categorical.__new__ = staticmethod(_categorical_new)


# ---------------------------------------------------------------------------------------------
# fused Poisson matrix factorisation: Poisson(rate = A @ B) with both factors latent
# ---------------------------------------------------------------------------------------------
class FactorProduct:
    """Lazy product ``A @ B`` of two latent factors, either ``A`` [N, K] and ``B`` [K, J] or ``A`` [P, N, K] and
    ``B`` [P, K, J] with the same P (no broadcasting): behaves like an ``[N, J]`` / ``[P, N, J]`` rate tensor when
    handed to ``Poisson(rate)``, which then scores the site with ONE kernel that emits the sum and the gradients
    of both factors (``b2_poisson_product``, 1 <= K <= 16) without writing the ``[P, N, J]`` rate.  Other shapes
    raise ValueError.  ``bmm`` records a ``torch.bmm`` call, so that :meth:`dense` repeats the eager
    computation bit for bit."""

    def __init__(self, A, B, bmm=False):
        if type(A).__name__ == "SiteValue":
            A = _ops.plain_value(A)
        if type(B).__name__ == "SiteValue":
            B = _ops.plain_value(B)
        if not (isinstance(A, torch.Tensor) and isinstance(B, torch.Tensor) and A.dim() == B.dim()
                and A.dim() in (2, 3) and B.shape[-2] == A.shape[-1] and A.shape[:-2] == B.shape[:-2]
                and A.dtype == B.dtype and A.device == B.device):
            raise ValueError("FactorProduct: expected A [N, K] and B [K, J], or A [P, N, K] and B [P, K, J], of one "
                             "dtype and device, got A %s and B %s" % (tuple(getattr(A, "shape", ())),
                                                                      tuple(getattr(B, "shape", ()))))
        self.A, self.B, self.bmm = A, B, bmm
        self.vectorised = A.dim() == 3
        self.P = A.shape[0] if self.vectorised else 1
        self.K = A.shape[-1]
        self.shape = A.shape[:-1] + B.shape[-1:]
        self.dtype, self.device = A.dtype, A.device

    def dense(self):
        return torch.bmm(self.A, self.B) if self.bmm else torch.matmul(self.A, self.B)


def _poisson_product(meta, A, B, x):
    scale, weight, coeff, _ = meta
    N.require_cuda(A, "fused Poisson factorisation likelihood")
    Ac, Bc = A.contiguous(), B.contiguous()
    n, K = A.shape[-2:]
    J = B.shape[-1]
    P = A.shape[0] if A.dim() == 3 else 1
    dev = A.device
    total = torch.empty((), dtype=torch.float32, device=dev)
    dA = torch.empty(Ac.shape, dtype=torch.float32, device=dev)
    dB = torch.empty(Bc.shape, dtype=torch.float32, device=dev)
    need = int(N.lib().b2_poisson_product_workspace(n, K, J, P))
    ws = N.workspace(dev, need, tag="glm")
    N.check(N.lib().b2_poisson_product(
        Ac.data_ptr(), Bc.data_ptr(), x.data_ptr(), n, K, J, P, float(scale), float(weight), float(coeff), 0,
        None, total.data_ptr(), dA.data_ptr(), dB.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
        "b2_poisson_product")
    return total, dA, dB, None


_PoissonProductFn = _FusedSum(_poisson_product)


class _PoissonProduct(Poisson):
    """Poisson whose rate is a FactorProduct (built by ``Poisson(lazy)`` when an unchanged model's
    ``torch.matmul(z, w)`` of two latent values was kept lazy by pyro_b200/lazy.py).  ``rate``, ``log_prob``,
    ``mean`` and every other use materialise the rate; the ELBO's site sum takes the fused kernel."""

    def __init__(self, rate, validate_args=None, is_sparse=False):
        lazy = _lazy_as(rate, FactorProduct)
        self._lazy = lazy
        self._dense = None
        Distribution.__init__(self, lazy.shape)

    @property
    def _params(self):
        if self._dense is None:
            self._dense = self._lazy.dense()
        return [self._dense]

    @property
    def rate(self):
        return self._params[0]

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        lz = self._lazy
        n, J = lz.shape[-2:]
        # one [N, J] count matrix broadcast over the particles, fp32 on the factors' device
        ok = (mask is None and isinstance(value, torch.Tensor) and value.dtype == torch.float32
              and lz.A.dtype == torch.float32 and lz.B.dtype == torch.float32 and tuple(value.shape) == (n, J)
              and value.device == lz.device and lz.device.type == "cuda" and J % 4 == 0 and 1 <= lz.K <= 16
              and tuple(self.batch_shape) == tuple(lz.shape))
        if not ok:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        x = value.contiguous()
        if x.data_ptr() % 16 != 0:
            x = x.clone()
        return _PoissonProductFn.apply((scale, weight, sum_coeff, unit), lz.A, lz.B, x)


# ---------------------------------------------------------------------------------------------
# fused Poisson regression: Poisson(rate = exp(X @ w + b))
# ---------------------------------------------------------------------------------------------
def _glm_poisson(meta, X, y, W, b):
    scale, weight, coeff, _ = meta
    N.require_cuda(X, "fused Poisson-regression likelihood")
    P, D = W.shape
    n = X.shape[0]
    total, dW, db, ws = _glm_outputs(X, W, int(N.lib().b2_glm_poisson_workspace(n, D, P)))
    Wc, bc = W.contiguous(), b.contiguous() if b is not None else None
    N.check(N.lib().b2_glm_poisson_log_rate(
        X.data_ptr(), y.data_ptr(), Wc.data_ptr(), _ptr(bc), n, D, P, float(scale), float(weight),
        float(coeff), 0, None, total.data_ptr(), dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(),
        N.stream_ptr(X.device)), "b2_glm_poisson_log_rate")
    return total, None, None, dW, db if b is not None else None


_GlmPoissonFn = _FusedSum(_glm_poisson)


class _PoissonLinear(Poisson):
    """Poisson whose rate is an ExpLinearPredictor (built by ``Poisson(lazy)`` when an unchanged model's
    ``torch.exp(X @ w + b)`` was kept lazy by pyro_b200/lazy.py).  ``rate``, ``log_prob`` and every other use
    materialise the rate; the ELBO's site sum takes the fused kernel."""

    def __init__(self, rate, validate_args=None, is_sparse=False):
        lazy = _lazy_as(rate, ExpLinearPredictor)
        self._lazy = lazy
        self._dense = None
        Distribution.__init__(self, lazy.shape)

    @property
    def _params(self):
        if self._dense is None:
            self._dense = self._lazy.dense()
        return [self._dense]

    @property
    def rate(self):
        return self._params[0]

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        lp = self._lazy.lp
        if lp.group is not None or lp.slopes:
            out = _group_sum(N.GLM_POISSON, lp, value, mask, self.batch_shape, (scale, weight, sum_coeff, unit))
            return out if out is not None else super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        args = _per_row_scope(lp, value, mask, self.batch_shape)
        if args is None:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        return _GlmPoissonFn.apply((scale, weight, sum_coeff, unit), *args)


def _poisson_new(cls, rate=None, validate_args=None, is_sparse=False):
    # ``Poisson(FactorProduct)`` builds the fused factorisation subclass, ``Poisson(ExpLinearPredictor)`` the
    # fused Poisson-regression one
    if cls is Poisson and _lazy_as(rate, FactorProduct) is not None:
        return object.__new__(_PoissonProduct)
    if cls is Poisson and _lazy_as(rate, ExpLinearPredictor) is not None:
        return object.__new__(_PoissonLinear)
    return object.__new__(cls)


Poisson.__new__ = staticmethod(_poisson_new)


# ---------------------------------------------------------------------------------------------
# fused linear regression: Normal(loc = X @ w + b, scale = sigma)
# ---------------------------------------------------------------------------------------------
def _glm_normal(meta, X, y, W, b, sigma):
    scale, weight, coeff, _, stride = meta
    N.require_cuda(X, "fused linear-regression likelihood")
    P, D = W.shape
    n = X.shape[0]
    total, dW, db, ws = _glm_outputs(X, W, int(N.lib().b2_glm_normal_workspace(n, D, P)))
    dsig = torch.empty(P, dtype=torch.float32, device=X.device) if sigma.requires_grad else None
    Wc, bc, sc = W.contiguous(), b.contiguous() if b is not None else None, sigma.contiguous()
    N.check(N.lib().b2_glm_normal_loc(
        X.data_ptr(), y.data_ptr(), Wc.data_ptr(), _ptr(bc), sc.data_ptr(), stride, n, D,
        P, float(scale), float(weight), float(coeff), 0, None, total.data_ptr(), dW.data_ptr(), db.data_ptr(),
        _ptr(dsig), ws.data_ptr(), ws.numel(), N.stream_ptr(X.device)), "b2_glm_normal_loc")
    if dsig is not None and stride == 0:
        dsig = dsig.sum().reshape(sigma.shape)      # one sigma shared by every particle
    return total, None, None, dW, db if b is not None else None, dsig


_GlmNormalFn = _FusedSum(_glm_normal)


def _linear_loc_of(loc):
    """The LinearPredictorTensor behind a Normal loc (a lazy ``X @ w + b``), or None."""
    return loc if isinstance(loc, torch.Tensor) and _lazy_as(loc, LinearPredictor) is not None else None


def _per_particle_sigma(scale, lp):
    """``(sigma, stride)``: the stored tensor of a Normal scale that is one value per particle -- a number,
    ``[]``, ``[1]``, ``[P, 1]`` or a stride-0 expansion of one of these along N (as ``broadcast_all`` leaves it) --
    flattened to 1 (stride 0) or P (stride 1) values; None for any other scale.  An expansion is replaced by its
    base, never sliced: the backward of a slice would write a ``[P, N]`` zero tensor."""
    s = densify(scale)
    if type(s).__name__ == "SiteValue":
        s = _ops.plain_value(s)
    if not isinstance(s, torch.Tensor) or s.dtype != torch.float32 or s.device != lp.X.device:
        return None
    if s.dim() >= 1 and s.shape[-1] > 1 and s.stride(-1) == 0:
        # only an expansion along N is looked through (a [P, 1] scale expanded along P is taken as it is)
        s = _unexpanded(s)
        if s is None:
            return None
    if s.numel() == 1 and s.dim() <= len(lp.shape):
        return s.reshape(1), 0
    if lp.vectorised and tuple(s.shape) == (lp.P, 1) and lp.P > 1:
        return s.reshape(lp.P), 1
    return None


class _NormalLinear(Normal):
    """Normal whose loc is a lazy ``X @ w + b`` (built by ``Normal(lazy, scale)`` when an unchanged model's linear
    predictor was kept lazy by pyro_b200/lazy.py).  ``loc``, ``log_prob``, ``rsample`` and every other use
    materialise the loc as the model wrote it, bit for bit; the ELBO's site sum takes the fused kernel
    (``b2_glm_normal_loc``) when the scale is one value per particle."""

    def __init__(self, loc, scale, validate_args=None):
        _, sc = _broadcast_params(loc, scale)
        self._loc_lazy = loc
        self._scale = sc
        self._dense = None
        self._log_scale = sc.log_value if isinstance(sc, LazyExpParam) and sc.dtype == loc.dtype else None
        Distribution.__init__(self, torch.broadcast_shapes(loc.shape, sc.shape))

    @property
    def _params(self):
        if self._dense is None:
            self._dense = self._loc_lazy.eager()
        return [self._dense, self._scale]

    @property
    def loc(self):
        return self._params[0]

    @property
    def scale(self):
        return self._scale

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        lp = self._loc_lazy.lazy
        if lp.group is not None or lp.slopes:
            sig = _per_particle_sigma(self._scale, lp)
            out = None if sig is None else _group_sum(N.GLM_NORMAL, lp, value, mask, self.batch_shape,
                                                      (scale, weight, sum_coeff, unit), sigma=sig)
            return out if out is not None else super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        args = _per_row_scope(lp, value, mask, self.batch_shape)
        sig = _per_particle_sigma(self._scale, lp) if args is not None else None     # one noise scale per particle
        if sig is None:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        return _GlmNormalFn.apply((scale, weight, sum_coeff, unit, sig[1]), *args, sig[0])


def _normal_new(cls, loc=None, scale=None, validate_args=None):
    # ``Normal(lazy X @ w + b, scale)`` builds the fused linear-regression subclass
    if cls is Normal and _linear_loc_of(loc) is not None:
        return object.__new__(_NormalLinear)
    return object.__new__(cls)


Normal.__new__ = staticmethod(_normal_new)


# ---------------------------------------------------------------------------------------------
# fused Binomial regression: Binomial(total_count, logits = X @ w + b)
# ---------------------------------------------------------------------------------------------
def _glm_binomial(meta, X, y, W, b):
    scale, weight, coeff, _, trials, per_row = meta
    N.require_cuda(X, "fused Binomial-regression likelihood")
    P, D = W.shape
    n = X.shape[0]
    total, dW, db, ws = _glm_outputs(X, W, int(N.lib().b2_glm_binomial_workspace(n, D, P)))
    Wc, bc = W.contiguous(), b.contiguous() if b is not None else None
    N.check(N.lib().b2_glm_binomial_logits(
        X.data_ptr(), y.data_ptr(), trials.data_ptr(), per_row, Wc.data_ptr(), _ptr(bc), n, D, P,
        float(scale), float(weight), float(coeff), 0, None, total.data_ptr(), dW.data_ptr(), db.data_ptr(),
        ws.data_ptr(), ws.numel(), N.stream_ptr(X.device)), "b2_glm_binomial_logits")
    return total, None, None, dW, db if b is not None else None


_GlmBinomialFn = _FusedSum(_glm_binomial)


def _unexpanded(t):
    """The stored tensor behind a stride-0 expansion (``broadcast_all`` of pyro_b200/lazy.py remembers it; an expand
    of a tensor that is not itself a view has it as its autograd base), ``t`` itself when it is not an expansion,
    None for anything else, such as an expansion of a slice."""
    if all(s == 1 or st != 0 for s, st in zip(t.shape, t.stride())):
        return t
    base = getattr(t, "_b2_unexpanded", None)
    base = t._base if base is None else base
    if base is None or base.dim() > t.dim() or base.data_ptr() != t.data_ptr():
        return None
    try:
        if torch.broadcast_shapes(base.shape, t.shape) != t.shape:
            return None
    except RuntimeError:
        return None
    return base if base.expand(t.shape).stride() == t.stride() else None


def _binomial_trials(total_count, lp):
    """``(trials, per_row)`` for the fused kernel: ONE count (a number, ``[]``, ``[1]``) as a 1-element device tensor
    (per_row 0), or the counts of the N rows (``[N]``, contiguous, 16-byte aligned) as stored (per_row 1); None for
    any other total_count, one that requires grad, or a slice of one."""
    t = densify(total_count)
    if type(t).__name__ == "SiteValue":
        t = _ops.plain_value(t)
    if not isinstance(t, torch.Tensor) or t.requires_grad or t.dtype != torch.float32 or t.device != lp.X.device:
        return None
    t = _unexpanded(t)
    if t is None:
        return None
    n = lp.X.shape[0]
    if t.numel() == 1 and t.dim() <= len(lp.shape):
        return t.reshape(1), 0
    if t.dim() >= 1 and t.shape[-1] == n and t.numel() == n and t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t.reshape(n), 1
    return None


class _BinomialLinear(Binomial):
    """Binomial whose logits are a lazy ``X @ w + b`` (built by ``Binomial(total_count, logits=lazy)``, also when an
    unchanged model's linear predictor was kept lazy by pyro_b200/lazy.py).  ``logits``, ``log_prob``, ``sample`` and
    every other use materialise the logits as the model wrote them, bit for bit; the ELBO's site sum takes the fused
    kernel (``b2_glm_binomial_logits``) when total_count is one count or one count per row."""

    def __init__(self, total_count=1, probs=None, logits=None, validate_args=None):
        lz = _lazy_as(logits, LinearPredictor)
        self._lazy, self._logits_src = lz, logits
        self.family = N.BINOMIAL_LOGITS
        self.param_names = ("total_count", "logits")
        tc = total_count
        if isinstance(tc, Number):
            tc = _const(tc, lz.dtype, lz.device)
        elif not tc.is_floating_point() or tc.dtype != lz.dtype:
            tc = tc.to(lz.dtype)
        self._total_count = tc
        self._dense = None
        Distribution.__init__(self, torch.broadcast_shapes(tc.shape, lz.shape))

    @property
    def _params(self):
        if self._dense is None:
            src = self._logits_src
            self._dense = src.eager() if hasattr(src, "eager") else self._lazy.dense()
        return [self._total_count, self._dense]

    @property
    def total_count(self):
        return self._total_count

    @property
    def logits(self):
        return self._params[1]

    def _fused_sum(self, value, mask, scale, weight, sum_coeff, unit=True):
        if self._lazy.group is not None or self._lazy.slopes:
            trials = _binomial_trials(self._total_count, self._lazy)
            out = None if trials is None else _group_sum(N.GLM_BINOMIAL, self._lazy, value, mask, self.batch_shape,
                                                         (scale, weight, sum_coeff, unit), trials=trials)
            return out if out is not None else super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        args = _per_row_scope(self._lazy, value, mask, self.batch_shape)
        # the counts as the kernel reads them, passed in meta: they are data, never differentiated
        trials = _binomial_trials(self._total_count, self._lazy) if args is not None else None
        if trials is None:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        return _GlmBinomialFn.apply((scale, weight, sum_coeff, unit) + trials, *args)


def _binomial_new(cls, total_count=1, probs=None, logits=None, validate_args=None):
    # ``Binomial(total_count, logits=lazy X @ w + b)`` builds the fused Binomial-regression subclass
    if cls is Binomial and probs is None and _lazy_as(logits, LinearPredictor) is not None:
        return object.__new__(_BinomialLinear)
    return object.__new__(cls)


Binomial.__new__ = staticmethod(_binomial_new)
__all__ += ["LinearPredictor", "linear_predictor", "ExpLinearPredictor", "GroupGather", "SlopeGather",
            "ClassLinearPredictor", "class_linear_predictor", "FactorProduct", "constant"]

from .hmm import GaussianHMM  # noqa: E402,F401
__all__ += ["GaussianHMM"]
