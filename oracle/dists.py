"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (torch fp64/fp32 CPU tensors, elementary ops only) of the log-densities reference
Pyro evaluates on the two hot paths.  The arithmetic of these families is NOT in the reference
repo: ``pyro.distributions.Normal`` etc. are thin subclasses of ``torch.distributions``
(pyro/distributions/torch.py:23-257, third-party dependency ``torch>=2.0`` pinned by setup.py:109;
torch 2.11.0 in this image).  Each function cites the torch source it restates; ``torch`` in the
citations means site-packages/torch.

Pinned by tests/test_oracle_golden.py against
  * the reference's own fixtures (tests/distributions/conftest.py, scipy log-pdfs, atol 1e-5) and
  * ``torch.distributions`` outputs on seeded random batches,
both captured by tests/golden/make_golden.py with the UNMODIFIED reference imported from
/root/reference.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this package.
Written with autograd-friendly ops so ``torch.autograd.grad`` of these functions is the
reference gradient.
"""
import math

import torch

LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))


def normal(x, loc, scale):
    """torch/distributions/normal.py:87-102"""
    var = scale ** 2
    return -((x - loc) ** 2) / (2 * var) - scale.log() - LOG_SQRT_2PI


def bernoulli_logits(x, logits):
    """torch/distributions/bernoulli.py:121-125: -binary_cross_entropy_with_logits(logits, x)
    = x*l - softplus(l), with softplus(l) = log(1 + e^l) evaluated stably as that loss does (torch's
    nn.functional.softplus returns l itself above its threshold of 20)"""
    return x * logits - torch.logaddexp(logits, torch.zeros_like(logits))


def bernoulli_probs(x, probs):
    """torch/distributions/bernoulli.py (probs -> logits via utils.probs_to_logits with clamp)"""
    eps = torch.finfo(probs.dtype).eps
    p = probs.clamp(min=eps, max=1 - eps)
    logits = torch.log(p) - torch.log1p(-p)
    return bernoulli_logits(x, logits)


def gamma(x, concentration, rate):
    """torch/distributions/gamma.py:89-98"""
    return (torch.xlogy(concentration, rate) + torch.xlogy(concentration - 1, x) - rate * x
            - torch.lgamma(concentration))


def dirichlet(x, concentration):
    """torch/distributions/dirichlet.py:90-97"""
    return (torch.xlogy(concentration - 1.0, x).sum(-1) + torch.lgamma(concentration.sum(-1))
            - torch.lgamma(concentration).sum(-1))


def beta(x, concentration1, concentration0):
    """torch/distributions/beta.py:87-91 -> Dirichlet([c1, c0]).log_prob([x, 1-x])"""
    c1, c0 = torch.broadcast_tensors(concentration1, concentration0)
    x = x.expand(torch.broadcast_shapes(x.shape, c1.shape))
    c1, c0 = c1.expand(x.shape), c0.expand(x.shape)
    return dirichlet(torch.stack([x, 1.0 - x], -1), torch.stack([c1, c0], -1))


def poisson(x, rate):
    """torch/distributions/poisson.py:75-79"""
    return torch.xlogy(x, rate) - rate - torch.lgamma(x + 1)


def binomial_logits(x, total_count, logits):
    """pyro/distributions/torch.py:83-101 with log_binomial at tol = 0 (pyro/ops/special.py:93-108):
    k*l - n*(max(l, 0) + log1p(exp(-|l|))) + lgamma(n + 1) - lgamma(k + 1) - lgamma(n - k + 1).
    log_binomial runs under torch.no_grad, so the lgamma terms carry no gradient.
    max(l, 0) + log1p(exp(-|l|)) is log(1 + e^l), evaluated here by logaddexp in the same way.  Its gradient is
    sigmoid(l), 0.5 at l = 0 as with the reference's _clamp_by_zero (pyro/distributions/torch.py:18-20), whose
    backward instead adds and cancels +-n/2 and so rounds n*sigmoid(l) at the scale of ulp(n/2)."""
    with torch.no_grad():
        n1 = total_count + 1
        log_binom = n1.lgamma() - (x + 1).lgamma() - (n1 - x).lgamma()
    norm = total_count * torch.logaddexp(logits, torch.zeros_like(logits))
    return x * logits - norm + log_binom


def binomial_probs(x, total_count, probs):
    """Binomial(total_count, probs): logits from torch's probs_to_logits with the clamp, as bernoulli_probs"""
    eps = torch.finfo(probs.dtype).eps
    p = probs.clamp(min=eps, max=1 - eps)
    return binomial_logits(x, total_count, torch.log(p) - torch.log1p(-p))


def cauchy(x, loc, scale):
    """torch/distributions/cauchy.py:81-88"""
    return -math.log(math.pi) - scale.log() - (((x - loc) / scale) ** 2).log1p()


def half_cauchy(x, scale):
    """torch/distributions/half_cauchy.py:73-81"""
    lp = cauchy(x, torch.zeros_like(scale), scale) + math.log(2)
    return torch.where(x >= 0, lp, torch.full_like(lp, -math.inf))


def half_normal(x, scale):
    """torch/distributions/half_normal.py (Normal(0, scale).log_prob + log 2, -inf below 0)"""
    lp = normal(x, torch.zeros_like(scale), scale) + math.log(2)
    return torch.where(x >= 0, lp, torch.full_like(lp, -math.inf))


def log_normal(x, loc, scale):
    """torch/distributions/log_normal.py via transformed_distribution.py log_prob:
    Normal.log_prob(log x) - log x"""
    return normal(x.log(), loc, scale) - x.log()


def exponential(x, rate):
    """torch/distributions/exponential.py log_prob: rate.log() - rate * x"""
    return rate.log() - rate * x


def uniform(x, low, high):
    """torch/distributions/uniform.py log_prob"""
    inside = (low <= x) & (x < high)
    lp = -torch.log(high - low)
    return torch.where(inside, lp.expand(inside.shape), torch.full(inside.shape, -math.inf, dtype=lp.dtype))


def categorical(value, logits):
    """torch/distributions/categorical.py:78 (normalise) and :151-157 (gather)"""
    logits = logits - logits.logsumexp(dim=-1, keepdim=True)
    value = value.long().unsqueeze(-1)
    value, log_pmf = torch.broadcast_tensors(value, logits)
    value = value[..., :1]
    return log_pmf.gather(-1, value).squeeze(-1)


def mvn_tril(x, loc, scale_tril):
    """torch/distributions/multivariate_normal.py:256-264 with _batch_mahalanobis :29-80"""
    diff = x - loc
    n = diff.shape[-1]
    L = scale_tril.expand(diff.shape[:-1] + (n, n))
    zsol = torch.linalg.solve_triangular(L, diff.unsqueeze(-1), upper=False).squeeze(-1)
    M = (zsol ** 2).sum(-1)
    half_log_det = scale_tril.diagonal(dim1=-2, dim2=-1).log().sum(-1)
    return -0.5 * (n * math.log(2 * math.pi) + M) - half_log_det


def kl_normal_normal(loc_p, scale_p, loc_q, scale_q):
    """torch/distributions/kl.py:468-471"""
    var_ratio = (scale_p / scale_q) ** 2
    t1 = ((loc_p - loc_q) / scale_q) ** 2
    return 0.5 * (var_ratio + t1 - 1 - var_ratio.log())


def kl_gamma_gamma(conc_p, rate_p, conc_q, rate_q):
    """torch/distributions/kl.py:301-306"""
    t1 = conc_q * (rate_p / rate_q).log()
    t2 = torch.lgamma(conc_q) - torch.lgamma(conc_p)
    t3 = (conc_p - conc_q) * torch.digamma(conc_p)
    t4 = (rate_q - rate_p) * (conc_p / rate_p)
    return t1 + t2 + t3 + t4


def scale_and_mask(lp, scale=1.0, mask=None):
    """pyro/distributions/util.py:311-328"""
    if mask is None:
        return lp if scale == 1.0 else lp * scale
    return torch.where(mask, lp * scale, torch.zeros((), dtype=lp.dtype))


# family id -> (fn(value, *params), number of params); ids as include/pyro_b200.h
ELEMENTWISE = {
    0: (normal, 2), 1: (bernoulli_logits, 1), 2: (gamma, 2), 3: (beta, 2), 4: (poisson, 1),
    5: (cauchy, 2), 6: (half_cauchy, 1), 7: (exponential, 1), 8: (log_normal, 2),
    9: (half_normal, 1), 10: (bernoulli_probs, 1), 11: (uniform, 2),
    12: (lambda x, a, b, c, d: kl_normal_normal(a, b, c, d), 4),
    13: (lambda x, a, b, c, d: kl_gamma_gamma(a, b, c, d), 4),
    16: (binomial_logits, 2), 17: (binomial_probs, 2),
}
EVENT = {32: dirichlet, 33: categorical, 34: mvn_tril}
