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
import math
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
                z, lq, eps = _ops.latent_draw(loc, scale, log_scale, shape)
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


__all__ = ["Distribution", "Normal", "Bernoulli", "Gamma", "Beta", "Poisson", "Cauchy", "HalfCauchy",
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

    ``w``: [D], [P, D] or [P, 1, D] (vectorised particles);  ``b``: None, [], [P] or [P, 1]."""

    def __init__(self, X, w, b=None, tensor_cores=True):
        # latent values may arrive as lazy-aware SiteValue tensors (pyro_b200/lazy.py): score plain ones
        if type(w).__name__ == "SiteValue":
            w = w.as_subclass(torch.Tensor)
        if type(b).__name__ == "SiteValue":
            b = b.as_subclass(torch.Tensor)
        self.X, self.w, self.b = X, w, b
        self.tensor_cores = tensor_cores  # False: fp32 SIMT contractions (B2_FLAG_GLM_FP32)
        D = X.shape[-1]
        self.vectorised = w.dim() > 1
        self.P = w.numel() // D
        self.shape = torch.Size((self.P, X.shape[0])) if self.vectorised else torch.Size((X.shape[0],))
        self.dtype, self.device = X.dtype, X.device

    def dense(self):
        W = self.w.reshape(self.P, -1)
        out = W @ self.X.t()
        if self.b is not None:
            out = out + self.b.reshape(self.P, 1)
        return out if self.vectorised else out.squeeze(0)


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


class _GlmBernoulliFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, X, y, W, b):
        import ctypes
        scale, weight, coeff, unit, flags = meta
        N.require_cuda(X, "fused GLM likelihood")
        P, D = W.shape
        n = X.shape[0]
        dev = X.device
        Wc = W.contiguous()
        bc = b.contiguous() if b is not None else None
        total = torch.empty((), dtype=torch.float32, device=dev)
        dW = torch.empty(P, D, dtype=torch.float32, device=dev)
        db = torch.empty(P, dtype=torch.float32, device=dev)
        need = int(N.lib().b2_glm_workspace(n, D, P))
        ws = N.workspace(dev, need, tag="glm")
        N.check(N.lib().b2_glm_bernoulli_logits(
            X.data_ptr(), y.data_ptr(), Wc.data_ptr(), bc.data_ptr() if bc is not None else None,
            n, D, P, float(scale), float(weight), float(coeff), int(flags), None, total.data_ptr(),
            dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
            "b2_glm_bernoulli_logits")
        ctx.grads = (dW, db if b is not None else None)
        ctx.unit = unit
        return total

    @staticmethod
    def backward(ctx, gout):
        dW, db = ctx.grads
        if not ctx.unit:
            dW = dW * gout
            db = db * gout if db is not None else None
        return None, None, None, dW, db


def _lazy_of(logits):
    if isinstance(logits, LinearPredictor):
        return logits
    lz = getattr(logits, "_lazy", None) if type(logits).__name__ == "LinearPredictorTensor" else None
    return lz if isinstance(lz, LinearPredictor) else None


class _BernoulliLinear(Bernoulli):
    """Bernoulli whose logits are a LinearPredictor (built by ``Bernoulli(logits=lazy)``, or by an
    unchanged model whose ``w @ X.T + b`` was kept lazy by pyro_b200/lazy.py)."""

    def __init__(self, probs=None, logits=None, validate_args=None):
        lazy = _lazy_of(logits)
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
        X = lz.X
        D = X.shape[-1]
        tc = getattr(lz, "tensor_cores", True)
        # D in {4, 8, 16, 32} have their own kernels; every other D up to 128 takes the wgmma kernel of
        # glm_flat_tc.cu, from 8192 rows (below that its TF32 gradient has not averaged its rounding down to
        # fp32 accuracy yet, and there is no fp32 kernel for these D)
        flat = D not in (4, 8, 16, 32)
        ok = (mask is None and X.dtype == torch.float32 and X.is_contiguous()
              and (not flat or (1 <= D <= 128 and tc and X.shape[0] >= 8192))
              and isinstance(value, torch.Tensor) and value.numel() == X.shape[0]
              and tuple(self.batch_shape) == tuple(lz.shape) and X.data_ptr() % 16 == 0)
        y = value.reshape(-1).to(torch.float32).contiguous() if ok else None
        if not ok or (flat and y.data_ptr() % 16 != 0):
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        W = lz.w.reshape(lz.P, D)
        b = lz.b.reshape(lz.P) if lz.b is not None else None
        flags = 0 if tc else N.B2_FLAG_GLM_FP32
        return _GlmBernoulliFn.apply((scale, weight, sum_coeff, unit, flags), X, y, W, b)


def _bernoulli_new(cls, probs=None, logits=None, validate_args=None):
    # ``Bernoulli(logits=LinearPredictor)`` builds the fused-GLM subclass
    if cls is Bernoulli and _lazy_of(logits) is not None:
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
            Wt = Wt.as_subclass(torch.Tensor)
        if type(b).__name__ == "SiteValue":
            b = b.as_subclass(torch.Tensor)
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
    out = lp.with_bias(b.as_subclass(torch.Tensor) if type(b).__name__ == "SiteValue" else b)
    if out is None:
        raise ValueError("class_linear_predictor: the bias must be [K]%s of X's dtype and device, got %s"
                         % (" or [P, 1, K]" if lp.vectorised else "", tuple(getattr(b, "shape", ()))))
    return out


class _GlmCategoricalFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, X, y, W, b):
        scale, weight, coeff, unit, flags = meta
        N.require_cuda(X, "fused softmax-regression likelihood")
        P, K, D = W.shape
        n = X.shape[0]
        dev = X.device
        Wc = W.contiguous()
        bc = b.contiguous() if b is not None else None
        total = torch.empty((), dtype=torch.float32, device=dev)
        dW = torch.empty(P, K, D, dtype=torch.float32, device=dev)
        db = torch.empty(P, K, dtype=torch.float32, device=dev)
        need = int(N.lib().b2_glm_categorical_workspace(n, D, K, P))
        ws = N.workspace(dev, need, tag="glm")
        N.check(N.lib().b2_glm_categorical_logits(
            X.data_ptr(), y.data_ptr(), Wc.data_ptr(), bc.data_ptr() if bc is not None else None,
            n, D, K, P, float(scale), float(weight), float(coeff), int(flags), None, total.data_ptr(),
            dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
            "b2_glm_categorical_logits")
        ctx.grads = (dW, db if b is not None else None)
        ctx.unit = unit
        return total

    @staticmethod
    def backward(ctx, gout):
        dW, db = ctx.grads
        if not ctx.unit:
            dW = dW * gout
            db = db * gout if db is not None else None
        return None, None, None, dW, db


def _class_lazy_of(logits):
    if isinstance(logits, ClassLinearPredictor):
        return logits
    lz = getattr(logits, "_lazy", None) if isinstance(logits, torch.Tensor) else None
    return lz if isinstance(lz, ClassLinearPredictor) else None


class _CategoricalLinear(Categorical):
    """Categorical whose logits are a ClassLinearPredictor (built by ``Categorical(logits=lazy)``, or by an
    unchanged model whose ``X @ W.mT + b`` was kept lazy by pyro_b200/lazy.py).  ``log_prob``, ``logits``
    and ``probs`` materialise the logits; the ELBO's site sum takes the fused kernel."""

    def __init__(self, probs=None, logits=None, validate_args=None):
        lazy = _class_lazy_of(logits)
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
        return _GlmCategoricalFn.apply((scale, weight, sum_coeff, unit, 0), X, y, W, lz.bias_pk())


def _categorical_new(cls, probs=None, logits=None, validate_args=None):
    # ``Categorical(logits=ClassLinearPredictor)`` builds the fused softmax-regression subclass
    if cls is Categorical and probs is None and _class_lazy_of(logits) is not None:
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
            A = A.as_subclass(torch.Tensor)
        if type(B).__name__ == "SiteValue":
            B = B.as_subclass(torch.Tensor)
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


class _PoissonProductFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, A, B, x):
        scale, weight, coeff, unit = meta
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
        ctx.grads = (dA, dB)
        ctx.unit = unit
        return total

    @staticmethod
    def backward(ctx, gout):
        dA, dB = ctx.grads
        if not ctx.unit:
            dA, dB = dA * gout, dB * gout
        return None, dA, dB, None


def _factor_lazy_of(rate):
    if isinstance(rate, FactorProduct):
        return rate
    lz = getattr(rate, "_lazy", None) if isinstance(rate, torch.Tensor) else None
    return lz if isinstance(lz, FactorProduct) else None


class _PoissonProduct(Poisson):
    """Poisson whose rate is a FactorProduct (built by ``Poisson(lazy)`` when an unchanged model's
    ``torch.matmul(z, w)`` of two latent values was kept lazy by pyro_b200/lazy.py).  ``rate``, ``log_prob``,
    ``mean`` and every other use materialise the rate; the ELBO's site sum takes the fused kernel."""

    def __init__(self, rate, validate_args=None, is_sparse=False):
        lazy = _factor_lazy_of(rate)
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
class _GlmPoissonFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meta, X, y, W, b):
        scale, weight, coeff, unit = meta
        N.require_cuda(X, "fused Poisson-regression likelihood")
        P, D = W.shape
        n = X.shape[0]
        dev = X.device
        Wc = W.contiguous()
        bc = b.contiguous() if b is not None else None
        total = torch.empty((), dtype=torch.float32, device=dev)
        dW = torch.empty(P, D, dtype=torch.float32, device=dev)
        db = torch.empty(P, dtype=torch.float32, device=dev)
        need = int(N.lib().b2_glm_poisson_workspace(n, D, P))
        ws = N.workspace(dev, need, tag="glm")
        N.check(N.lib().b2_glm_poisson_log_rate(
            X.data_ptr(), y.data_ptr(), Wc.data_ptr(), bc.data_ptr() if bc is not None else None,
            n, D, P, float(scale), float(weight), float(coeff), 0, None, total.data_ptr(),
            dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr(dev)),
            "b2_glm_poisson_log_rate")
        ctx.grads = (dW, db if b is not None else None)
        ctx.unit = unit
        return total

    @staticmethod
    def backward(ctx, gout):
        dW, db = ctx.grads
        if not ctx.unit:
            dW = dW * gout
            db = db * gout if db is not None else None
        return None, None, None, dW, db


def _exp_lazy_of(rate):
    if isinstance(rate, ExpLinearPredictor):
        return rate
    lz = getattr(rate, "_lazy", None) if isinstance(rate, torch.Tensor) else None
    return lz if isinstance(lz, ExpLinearPredictor) else None


class _PoissonLinear(Poisson):
    """Poisson whose rate is an ExpLinearPredictor (built by ``Poisson(lazy)`` when an unchanged model's
    ``torch.exp(X @ w + b)`` was kept lazy by pyro_b200/lazy.py).  ``rate``, ``log_prob`` and every other use
    materialise the rate; the ELBO's site sum takes the fused kernel."""

    def __init__(self, rate, validate_args=None, is_sparse=False):
        lazy = _exp_lazy_of(rate)
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
        X = lp.X
        D = X.shape[-1]
        # the scope of the any-D logistic-regression kernel: tensor cores asked for, 1 <= D <= 128, from 8192
        # rows (below that the TF32 gradient has not averaged its rounding down to fp32 accuracy yet), fp32,
        # contiguous 16-byte aligned X and y, no mask
        ok = (mask is None and X.dtype == torch.float32 and X.is_contiguous() and X.data_ptr() % 16 == 0
              and 1 <= D <= 128 and getattr(lp, "tensor_cores", True) and X.shape[0] >= 8192
              and isinstance(value, torch.Tensor) and value.numel() == X.shape[0]
              and tuple(self.batch_shape) == tuple(lp.shape))
        y = value.reshape(-1).to(torch.float32).contiguous() if ok else None
        if not ok or y.data_ptr() % 16 != 0:
            return super()._fused_sum(value, mask, scale, weight, sum_coeff, unit)
        W = lp.w.reshape(lp.P, D)
        b = lp.b.reshape(lp.P) if lp.b is not None else None
        return _GlmPoissonFn.apply((scale, weight, sum_coeff, unit), X, y, W, b)


def _poisson_new(cls, rate=None, validate_args=None, is_sparse=False):
    # ``Poisson(FactorProduct)`` builds the fused factorisation subclass, ``Poisson(ExpLinearPredictor)`` the
    # fused Poisson-regression one
    if cls is Poisson and _factor_lazy_of(rate) is not None:
        return object.__new__(_PoissonProduct)
    if cls is Poisson and _exp_lazy_of(rate) is not None:
        return object.__new__(_PoissonLinear)
    return object.__new__(cls)


Poisson.__new__ = staticmethod(_poisson_new)
__all__ += ["LinearPredictor", "linear_predictor", "ExpLinearPredictor", "ClassLinearPredictor",
            "class_linear_predictor", "FactorProduct", "constant"]

from .hmm import GaussianHMM  # noqa: E402,F401
__all__ += ["GaussianHMM"]
