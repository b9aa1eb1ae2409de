"""Trace_ELBO on the fused kernels.

Semantics restate pyro/infer/trace_elbo.py:20-29 (``_compute_log_r``), :82-112
(``_differentiable_loss_particle``) and :130-159 (``loss_and_grads``).

Fast path (every guide site reparameterised, which is the case for all BASELINE configs): each
sample site costs ONE fused kernel that returns its ``sum(scale*mask*log_prob)`` and, in the same
pass, the FINAL gradient contributions ``-/+ (1/P) d lp / d operand`` -- the reference's
``.backward()`` through ~10 ATen kernels per site collapses into handing those tensors to
autograd.  The loss value is accumulated on the device and read back once per step (the
reference syncs once per site, trace_elbo.py:90,97).

General path (non-reparameterised guide sites): materialised ``log_prob`` tensors, the
Rao-Blackwellised ``log_r`` of :20-29 and the score-function surrogate of :104-110.
"""
import torch

from ..distributions import is_identically_zero
from ..poutine.trace_struct import ScaledTerm, _fused
from ..util import torch_item, warn_if_nan
from .elbo import ELBO, get_importance_trace
from .util import MultiFrameTensor, get_plate_stacks


def _compute_log_r(model_trace, guide_trace):
    log_r = MultiFrameTensor()
    stacks = get_plate_stacks(model_trace)
    for name, model_site in model_trace.nodes.items():
        if model_site["type"] == "sample":
            log_r_term = model_site["log_prob"]
            if not model_site["is_observed"]:
                log_r_term = log_r_term - guide_trace.nodes[name]["log_prob"]
            log_r.add((stacks[name], log_r_term.detach()))
    return log_r


_ONES = {}


def _one_like(t):
    key = (t.device, t.dtype)
    one = _ONES.get(key)
    if one is None:
        one = _ONES[key] = torch.ones((), device=t.device, dtype=t.dtype)
    return one


def _all_reparam(guide_trace):
    for site in guide_trace.nodes.values():
        if site["type"] == "sample" and not getattr(site["fn"], "has_rsample", False):
            return False
    return True


class Trace_ELBO(ELBO):
    """Drop-in for ``pyro.infer.Trace_ELBO`` (same constructor, ``loss``, ``differentiable_loss``,
    ``loss_and_grads``)."""

    def _get_trace(self, model, guide, args, kwargs):
        # traces come back UNSCORED; scoring happens per site below
        return get_importance_trace("flat", self.max_plate_nesting, model, guide, args, kwargs,
                                    score=False)

    # ---- value only -------------------------------------------------------------------------
    def loss(self, model, guide, *args, **kwargs):
        elbo = 0.0
        with torch.no_grad():
            for model_trace, guide_trace in self._get_traces(model, guide, args, kwargs):
                elbo_particle = model_trace.log_prob_sum() - guide_trace.log_prob_sum()
                elbo = elbo + elbo_particle / self.num_particles
        loss = -torch_item(elbo)
        warn_if_nan(loss, "loss")
        return loss

    # ---- general path: reference algorithm on materialised log_probs ---------------------------
    def _differentiable_loss_particle(self, model_trace, guide_trace):
        model_trace.compute_log_prob()
        guide_trace.compute_score_parts()
        elbo_particle = 0
        surrogate_elbo_particle = 0
        log_r = None
        for name, site in model_trace.nodes.items():
            if site["type"] == "sample":
                elbo_particle = elbo_particle + site["log_prob_sum"].detach()
                surrogate_elbo_particle = surrogate_elbo_particle + site["log_prob_sum"]
        for name, site in guide_trace.nodes.items():
            if site["type"] == "sample":
                log_prob, score_function_term, entropy_term = site["score_parts"]
                elbo_particle = elbo_particle - site["log_prob_sum"].detach()
                if not is_identically_zero(entropy_term):
                    surrogate_elbo_particle = surrogate_elbo_particle - entropy_term.sum()
                if not is_identically_zero(score_function_term):
                    if log_r is None:
                        log_r = _compute_log_r(model_trace, guide_trace)
                    site_log_r = log_r.sum_to(site["cond_indep_stack"])
                    surrogate_elbo_particle = surrogate_elbo_particle + (site_log_r * score_function_term).sum()
        return -elbo_particle, -surrogate_elbo_particle

    def differentiable_loss(self, model, guide, *args, **kwargs):
        loss = 0.0
        surrogate_loss = 0.0
        for model_trace, guide_trace in self._get_traces(model, guide, args, kwargs):
            loss_particle, surrogate_loss_particle = self._differentiable_loss_particle(model_trace, guide_trace)
            surrogate_loss = surrogate_loss + surrogate_loss_particle / self.num_particles
            loss = loss + loss_particle / self.num_particles
        return loss + (surrogate_loss - surrogate_loss.detach())

    # ---- fused path ------------------------------------------------------------------------------
    def _fused_particle(self, model_trace, guide_trace):
        """Returns (loss contribution ``-elbo/P`` as a 0-d device tensor, [0-d terms whose backward
        with unit upstream yields the surrogate-loss gradients])."""
        from ..distributions import scale_and_mask
        P = self.num_particles
        terms, parts, coeffs = [], [], []

        def add_site(site, coeff):
            # surrogate_loss = -(1/P) * sum_sites coeff * lp_sum ; elbo = sum coeff * lp_sum
            w = -coeff / P
            t = _fused(site, weight=w, sum_coeff=coeff, unit=True, claim=True)
            if isinstance(t, ScaledTerm):
                # drawn and scored by one kernel at sampling time (fused Normal rsample)
                parts.append(t.tensor.detach())
                coeffs.append(t.coeff)
                if t.tensor.requires_grad:
                    terms.append(t.tensor)
                return
            if t is not None:
                parts.append(t.detach())
                coeffs.append(1.0)
                if t.requires_grad:
                    terms.append(t)
                return
            # no fused kernel for this site: materialised log_prob + autograd
            lp = site["fn"].log_prob(site["value"], *site["args"], **site["kwargs"])
            lp = scale_and_mask(lp, site["scale"], site["mask"]).sum()
            parts.append(lp.detach())
            coeffs.append(coeff)
            if lp.requires_grad:
                terms.append(w * lp)

        # guide sites first: a fused draw whose score has been claimed can also carry its model site's prior
        for name, site in guide_trace.nodes.items():
            if site["type"] == "sample":
                add_site(site, -1.0)
        from ..distributions import _ops
        priors, prior_coeffs = [], []
        model_sites = [site for site in model_trace.nodes.values() if site["type"] == "sample"]
        for i, site in enumerate(model_sites):
            job = None
            if (not site["is_observed"] and (site["mask"] is None or site["mask"] is True)
                    and not site["args"] and not site["kwargs"]
                    and not isinstance(site["scale"], torch.Tensor)):
                # Normal prior on a fused draw: value-only scoring now (batched below), its d/dz inside
                # the draw's backward kernel
                from ..distributions import claim_rsample_prior
                sc = float(site["scale"])
                job = claim_rsample_prior(site["fn"], site["value"], -sc / P)
                if job is not None:
                    priors.append(job)
                    prior_coeffs.append(sc)
            if job is None:
                if priors and i == len(model_sites) - 1:
                    # the last site to score: a fused likelihood call can assemble the loss in its own
                    # finish kernel (the priors' sums, the parts so far, then its own term)
                    with _ops.elbo_assembly(priors, [-c / P for c in prior_coeffs], list(parts),
                                            [-c / P for c in coeffs], -1.0 / P) as asm:
                        add_site(site, 1.0)
                    # the assembly's last term is the GLM call's own total with coefficient -1/P: valid only when
                    # that total is the part this site added, with coefficient 1, which is checked here
                    if (asm.loss is not None and coeffs and coeffs[-1] == 1.0
                            and parts[-1].data_ptr() == asm.total.data_ptr()):
                        return asm.loss, terms
                else:
                    add_site(site, 1.0)
        if priors:
            # the priors' value-only sums and the assembly of the loss in one launch when the sites are small
            loss = _ops.latent_prior_combine(priors, [-c / P for c in prior_coeffs], parts, [-c / P for c in coeffs])
            if loss is not None:
                return loss, terms
            parts.extend(_ops.latent_prior(priors))
            coeffs.extend(prior_coeffs)
        if not parts:
            return torch.zeros(()), terms
        # loss = sum_i (-coeff_i / P) * part_i, assembled on the device in one launch
        parts = [e.to(parts[0].dtype) if e.dtype != parts[0].dtype else e for e in parts]
        loss = _ops.elbo_combine(parts, [-c / P for c in coeffs])
        return loss, terms

    def _score_and_backward(self, model_trace, guide_trace, allow_general=False):
        """Score one (model, guide) trace pair with the fused kernels and run the backward of the
        surrogate loss; returns this pair's loss contribution (0-d device tensor), or None when a guide
        site has no reparameterised sampler and ``allow_general`` is false (pyro_b200/bind.py then hands
        the pair to the reference algorithm)."""
        trainable = any(site["type"] == "param" for trace in (model_trace, guide_trace)
                        for site in trace.nodes.values())
        if _all_reparam(guide_trace):
            loss_particle, terms = self._fused_particle(model_trace, guide_trace)
            from ..distributions import _ops as _o
            _o.flush_draws()    # a draw nothing has read yet still runs inside this step
            if trainable and terms:
                # every term's upstream gradient is exactly 1 (contract of the fused nodes);
                # pass one cached ones-scalar instead of letting autograd fill a new one per term
                ones = [_one_like(t) for t in terms]
                with _o.deferred_latent_backward():
                    torch.autograd.backward(terms, ones, retain_graph=self.retain_graph)
            return loss_particle
        if not allow_general:
            return None
        loss_particle, surrogate = self._differentiable_loss_particle(model_trace, guide_trace)
        loss_particle = loss_particle / self.num_particles
        if trainable and getattr(surrogate, "requires_grad", False):
            (surrogate / self.num_particles).backward(retain_graph=self.retain_graph)
        return loss_particle

    def loss_and_grads_tensor(self, model, guide, *args, **kwargs):
        """Like ``loss_and_grads`` but returns the loss as a 0-d DEVICE tensor without
        synchronising (used by the graph-captured step)."""
        loss = None
        for model_trace, guide_trace in self._get_traces(model, guide, args, kwargs):
            loss_particle = self._score_and_backward(model_trace, guide_trace, allow_general=True)
            loss = loss_particle if loss is None else loss + loss_particle
        return loss if loss is not None else 0.0

    def loss_and_grads(self, model, guide, *args, **kwargs):
        loss = torch_item(self.loss_and_grads_tensor(model, guide, *args, **kwargs))
        warn_if_nan(loss, "loss")
        return loss


class JitTrace_ELBO(Trace_ELBO):
    """Analogue of pyro/infer/trace_elbo.py:162-257: instead of ``torch.jit.trace`` the whole
    SVI step (guide sampling, model, fused scoring, backward, fused optimiser) is captured once
    into a CUDA graph and replayed, which removes the Python/poutine overhead from every
    subsequent ``svi.step``.  Same restrictions as the reference's JIT variant: static model
    structure and tensor-only ``*args``."""
    capture_graph = True
