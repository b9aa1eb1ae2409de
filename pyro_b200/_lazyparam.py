"""A positive-constrained parameter whose constraint transform has not run yet.

``pyro.param(name, init, constraint=constraints.positive)`` returns ``exp(u)`` of the unconstrained storage
``u`` (pyro/params/param_store.py:125-156 with ``transform_to(positive) = exp``): one launch per parameter per
step, and one more in the backward pass.  The usual consumer is ``Normal(loc, scale)`` of a mean-field guide,
whose draw kernel can take ``u`` itself (``b2_latent_normal_draw`` with ``B2_LATENT_LOG_SCALE``) and hand back
``d/du`` directly.  :class:`LazyExpParam` is that deferred ``exp(u)``: a storage-less tensor with the right
metadata; ``Normal`` recognises it, and ANY other use (a torch function, a native kernel argument) computes
``u.exp()`` on the spot -- once, autograd-connected -- so arbitrary guide code keeps its meaning.
"""
import weakref

import torch
from torch.utils._pytree import tree_map

_META = {"size", "dim", "ndimension", "numel", "nelement", "__len__", "is_floating_point", "is_complex",
         "element_size", "get_device", "__repr__", "__str__", "__format__"}
# attributes (property getters arrive as ``__get__`` of their descriptor) answered from the metadata alone
_META_ATTRS = {"shape", "dtype", "device", "ndim", "layout", "is_cuda", "is_cpu", "is_sparse", "is_quantized",
               "is_meta", "is_leaf", "requires_grad", "grad_fn", "names", "is_mkldnn", "is_xpu", "is_nested",
               "itemsize", "nbytes", "output_nr", "_version"}


class LazyExpParam(torch.Tensor):
    @staticmethod
    def __new__(cls, u):
        t = torch.Tensor._make_wrapper_subclass(cls, tuple(u.shape), dtype=u.dtype, device=u.device,
                                                requires_grad=False)
        t._u = u
        t._dense = None
        return t

    def __init__(self, u):
        pass

    @property
    def log_value(self):
        """The unconstrained storage ``u`` (a leaf that requires grad)."""
        return self._u

    def dense(self):
        if self._dense is None:
            d = self._u.exp()
            d.unconstrained = weakref.ref(self._u)
            d._pyro_unconstrained_param = self._u
            self._dense = d
        return self._dense

    def __repr__(self):
        return "LazyExpParam(shape={}, device={})".format(tuple(self.shape), self.device)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, "__name__", None)
        if name in _META or (name == "__get__" and
                             getattr(getattr(func, "__self__", None), "__name__", "") in _META_ATTRS):
            with torch._C.DisableTorchFunctionSubclass():
                return func(*args, **kwargs)
        return func(*tree_map(densify, args), **tree_map(densify, kwargs))

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        return func(*tree_map(densify, args), **tree_map(densify, kwargs or {}))


def densify(x):
    """What a native kernel (an autograd.Function, opaque to ``__torch_function__``) must be handed: the
    materialised ``exp(u)`` of a :class:`LazyExpParam`; the plain tensor inside a trace-time wrapper that keeps one
    as ``_t`` (the provenance tags of TraceGraph_ELBO); the materialised logits of a lazy linear predictor
    (pyro_b200/lazy.py) that reached a distribution other than the fused GLM routes, so that autograd sees its
    dependence on the weights; anything else unchanged."""
    if isinstance(x, LazyExpParam):
        return x.dense()
    if type(x).__name__ == "LinearPredictorTensor":
        return x.dense()
    if type(x) is not torch.Tensor and isinstance(x, torch.Tensor) and hasattr(x, "_provenance"):
        return x._t
    return x
