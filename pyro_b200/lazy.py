"""Lazy linear predictors: let an UNCHANGED model reach the fused GLM kernel.

A model such as tests/infer/mcmc/test_hmc.py:189-198 writes its likelihood as

    logits = w.squeeze(-2) @ X.T + b            # or  X @ w + b,  (X * w).sum(-1) + b,  F.linear(X, w, b)
    pyro.sample("y", dist.Bernoulli(logits=logits), obs=y)

Executed literally this materialises ``[P, N]`` logits (cuBLAS), ``[P, N]`` log-probabilities and
their gradients, which dominate the step at BASELINE config 2.  The ELBO hands latent site values
to the model as :class:`SiteValue` tensors instead; every torch operation on them runs exactly as on
a plain tensor EXCEPT a contraction with a gradient-free data matrix, which returns a
:class:`LinearPredictorTensor` -- a storage-less tensor that remembers ``(X, w, b)``.  Adding a
per-particle bias keeps it lazy; ``Bernoulli(logits=lazy)`` scores the site with ONE pass over X and
y (``b2_glm_bernoulli_logits``); any other use materialises ``X @ w + b`` on the spot, so the
semantics of arbitrary user code are unchanged.

Softmax regression has the same seam: ``X @ W.mT`` (``W.transpose(-1, -2)``, ``torch.matmul``) and
``F.linear(X, W)`` with a site value ``W[K, D]`` or ``W[P, K, D]`` give ``[N, K]`` / ``[P, N, K]`` class logits
kept as a :class:`ClassLinearPredictor`; a bias ``[K]`` or ``[P, 1, K]`` keeps them lazy, and
``Categorical(logits=lazy)`` scores the site with ``b2_glm_categorical_logits``.

Poisson regression has one more: ``torch.exp(t)`` or ``t.exp()`` of a lazy ``X @ w + b`` (a
:class:`LinearPredictor`) gives an :class:`ExpLinearPredictor`, and ``Poisson(lazy)`` scores the site with
``b2_glm_poisson_log_rate``; any other use, ``+ offset`` and ``* c`` included, materialises ``exp`` of the
eager expression, bit for bit.

Binomial regression needs one: ``Binomial(total_count, logits=lazy X @ w + b)`` scores the site with
``b2_glm_binomial_logits``; torch's constructor calls ``broadcast_all(total_count, logits)``, which keeps the logits
lazy and expands the count, and ``total_count.type_as(logits)``, which is answered without materialising them.

Linear regression needs no new seam: ``Normal(lazy X @ w + b, sigma)`` with one noise scale per particle (a
number, ``[]``, ``[1]``, ``[P, 1]``) scores the site with ``b2_glm_normal_loc``; ``broadcast_all(loc, sigma)`` of
``torch.distributions.Normal`` keeps the loc lazy and expands sigma.

Poisson matrix factorisation (the bottom layer of the sparse gamma DEF) has one more: ``torch.matmul(z, w)``,
``z @ w`` or ``torch.bmm(z, w)`` of TWO site values ``z[N, K] @ w[K, J]`` or ``z[P, N, K] @ w[P, K, J]``
(fp32, one CUDA device, 1 <= K <= 16) gives a :class:`FactorProduct`, and ``Poisson(lazy)`` scores the site with
``b2_poisson_product`` without writing the ``[P, N, J]`` rate.  Any other use, ``+`` included, materialises it.

Multilevel regression has one more: a gather of a latent table along its last dim by a gradient-free int64 ``[N]``
group index on the table's device -- ``alpha[g]`` of a ``[G]`` value, ``alpha[..., g]``, ``alpha.index_select(-1, g)``,
``torch.index_select(alpha, -1, g)``, with the table ``[G]``, ``[P, G]`` or ``[P, 1, G]`` or a view kept as a site
value -- gives a :class:`GroupGather`, and so does ``s * eta[..., g]`` with ``s`` a number or one scalar per particle
(``[]``, ``[1]``, ``[P, 1]``: the ``[P, G]`` table ``s * eta`` is formed eagerly, so autograd covers ``s``).  Added to a
lazy ``X @ w (+ b)``, before or after the bias and in either order, it becomes the predictor's group effect, and the
four families above score ``X @ w + b + alpha[g]`` with ``b2_glm_group_sum``: G more columns of the one pass over X.
Any other use of the gather, a second group effect included, materialises it exactly as torch computes it.

Varying slopes have one more: such a gather times a covariate (``beta[..., g] * X[:, c]``, either side of ``*``, with
``s * eta[..., g]`` as the gather too) is a :class:`SlopeGather` when the covariate is a gradient-free fp32 ``[N]`` view
on the table's device.  Added to a lazy ``X @ w (+ b)`` whose X has the covariate as column ``c`` (``X[:, c]``,
``X[..., c]``, ``X.select(-1, c)`` of that very X: same storage, X's row stride, ``c`` elements in), with the group
effect's index object and G, it becomes one of up to three slopes on distinct columns, in any order with the bias and
the intercept, and the four families score ``X @ w + b + alpha[g] + SUM_k beta_k[g] * X[:, c_k]`` with
``b2_glm_group_slope_sum``: G more columns per slope of the same pass.  A product with any other tensor, any other use
of the product, and a predictor with slopes but no intercept when it is scored, materialise exactly.

This is trace-time pattern matching at the seam where Pyro already passes values around (the replayed
guide value of pyro/poutine/replay_messenger.py:50-61); nothing in the model is rewritten.
"""
import torch

from ._lazyparam import LazyExpParam
from .distributions import (ClassLinearPredictor, ExpLinearPredictor, FactorProduct, GroupGather, LinearPredictor,
                            SlopeGather, _ops)

_VIEW_FUNCS = {"squeeze", "unsqueeze", "reshape", "view", "transpose", "t", "permute", "expand",
               "expand_as", "flatten", "contiguous", "__getitem__", "movedim", "swapaxes", "detach_",
               "mT", "T", "narrow", "select", "unflatten"}
_MATMUL_FUNCS = {"matmul", "__matmul__", "__rmatmul__", "mm", "mv", "linear", "inner", "bmm"}
_CLASS_MATMUL_FUNCS = {"matmul", "__matmul__", "__rmatmul__", "mm"}
_FACTOR_MATMUL_FUNCS = {"matmul", "__matmul__", "__rmatmul__", "bmm"}
# device types on which a product of two site values stays lazy: the fused Poisson kernel is CUDA only (the CPU
# tests widen this to check the lazy semantics without a GPU)
_FACTOR_DEVICE_TYPES = ("cuda",)
_ADD_FUNCS = {"add", "__add__", "__radd__", "__iadd__", "add_"}
_MUL_FUNCS = {"mul", "__mul__", "__rmul__"}
_CHEAP_TRUE = {"eq", "__eq__", "isfinite"}
_CHEAP_FALSE = {"ne", "__ne__", "isnan", "isinf"}
_META_FUNCS = {"size", "dim", "ndimension", "numel", "nelement", "__len__", "is_floating_point",
               "is_complex", "element_size", "get_device", "is_contiguous", "stride", "storage_offset",
               "__get__", "__repr__", "__str__", "__format__", "__reduce_ex__", "requires_grad_"}


def _name(func):
    return getattr(func, "__name__", None) or str(func)


def _plain(x):
    if isinstance(x, (LinearPredictorTensor, LazyExpParam)):
        return x.dense()
    if isinstance(x, SiteValue):
        # inside SiteValue.__torch_function__: a reading operation has flushed the pending draws already
        return x.as_subclass(torch.Tensor)
    if isinstance(x, (list, tuple)):
        return type(x)(_plain(v) for v in x)
    return x


def _is_data(t):
    """A gradient-free 2-d tensor that is a row-major ``[N, D]`` matrix or the transposed view of one."""
    if not isinstance(t, torch.Tensor) or isinstance(t, (SiteValue, LinearPredictorTensor, LazyExpParam)):
        return False
    if t.requires_grad or t.dim() != 2 or not t.is_floating_point():
        return False
    return True


def _row_major(t):
    """``(X[N, D] contiguous, transposed?)`` for a 2-d data operand, or None."""
    if t.is_contiguous():
        return t, False
    if t.t().is_contiguous():
        return t.t(), True
    return None


def _weights_of(w, D):
    """A site value usable as P weight vectors of length D: ``[D]``, ``[P, D]`` or ``[P, 1, D]``."""
    if w.shape[-1] != D:
        return False
    lead = w.shape[:-1]
    return all(s == 1 for s in lead[1:]) if len(lead) > 1 else True


class SiteValue(torch.Tensor):
    """The value of a latent sample site, as the model sees it.  Behaves like the plain tensor."""

    @staticmethod
    def wrap(t):
        if isinstance(t, torch.Tensor) and not isinstance(t, (SiteValue, LinearPredictorTensor)) \
                and t.is_floating_point():
            return t.as_subclass(SiteValue)
        return t

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        _ops.flush_before(func)     # a site value may be a deferred draw (distributions/_ops.py)
        name = _name(func)
        if name == "__get__":
            # a property such as ``W.mT``: name it after the attribute, so a transposed view stays a SiteValue
            name = getattr(getattr(func, "__self__", None), "__name__", name)
        if name in _MATMUL_FUNCS and not kwargs:
            lazy = _try_lazy_matmul(name, args)
            if lazy is not None:
                if isinstance(lazy, LinearPredictorTensor) and isinstance(lazy.lazy, LinearPredictor):
                    lazy._eager = _eager_call(func, args, kwargs)   # read by exp (ExpLinearPredictor)
                return lazy
        if name in ("__getitem__", "index_select") and not kwargs:
            lazy = _try_group_gather(name, args)
            if lazy is not None:
                return lazy
        if any(isinstance(a, LinearPredictorTensor) for a in args):
            return LinearPredictorTensor.__torch_function__(func, types, args, kwargs)
        with torch._C.DisableTorchFunctionSubclass():
            out = func(*_plain(args), **{k: _plain(v) for k, v in kwargs.items()})
        if name in _VIEW_FUNCS and isinstance(out, torch.Tensor) and not isinstance(out, SiteValue):
            return out.as_subclass(SiteValue)
        return out


def _eager_args(x):
    if isinstance(x, LinearPredictorTensor):
        return x.eager()
    if isinstance(x, (list, tuple)):
        return type(x)(_eager_args(v) for v in x)
    return _plain(x)


def _eager_call(func, args, kwargs):
    """The expression as the model wrote it, run on plain tensors when called."""
    def run():
        with torch._C.DisableTorchFunctionSubclass():
            return func(*_eager_args(args), **{k: _eager_args(v) for k, v in kwargs.items()})
    return run


def _try_lazy_matmul(name, args):
    """``w_view @ X.T``, ``X @ w``, ``F.linear(X, w[, b])`` with X a gradient-free data matrix."""
    if name == "linear":
        if len(args) < 2:
            return None
        Xa, wa = args[0], args[1]
        bias = args[2] if len(args) > 2 else None
        if not (_is_data(Xa) and isinstance(wa, SiteValue)):
            return None
        rm = _row_major(Xa)
        if rm is None or rm[1]:
            return None
        if wa.dim() == 2:
            # F.linear(X, W[K, D][, b[K]]) -> [N, K] class logits
            if not _class_weights_of(wa, Xa) or (bias is not None and not _class_bias_ok(bias, wa.shape[0], Xa)):
                return None
            return _make_class(rm[0], wa.mT, bias, linear=True)
        if wa.dim() != 1 or not _weights_of(wa, Xa.shape[1]):
            return None
        lp = _make(rm[0], wa, None)
        return lp if bias is None else lp + bias
    if len(args) != 2:
        return None
    a, b = args
    if name == "__rmatmul__":
        a, b = b, a
    if isinstance(a, SiteValue) and isinstance(b, SiteValue):
        return _try_factor_product(name, a, b)
    if name == "bmm":
        return None
    if isinstance(a, SiteValue) and _is_data(b):
        # w_view [..., D] @ X^T [D, N]
        rm = _row_major(b)
        if rm is None or not rm[1]:
            return None
        X = rm[0]
        if not _weights_of(a, X.shape[1]) or a.dim() > 2:
            return None
        return _make(X, a, None)
    if _is_data(a) and isinstance(b, SiteValue):
        rm = _row_major(a)
        if rm is None or rm[1]:
            return None
        if b.dim() in (2, 3) and name in _CLASS_MATMUL_FUNCS:
            # X [N, D] @ W.mT, W [K, D] or [P, K, D] -> [N, K] / [P, N, K] class logits
            if b.shape[-2] != a.shape[1] or not _class_weights_of(b.mT, a):
                return None
            return _make_class(rm[0], b, None)
        # X [N, D] @ w [D]
        if b.dim() != 1 or b.shape[0] != a.shape[1]:
            return None
        return _make(rm[0], b, None)
    return None


def _try_group_gather(name, args):
    """``alpha[g]`` (``alpha`` 1-d), ``alpha[..., g]`` or ``index_select(alpha, -1, g)`` of a site value ``[G]``,
    ``[P, G]`` or ``[P, 1, G]`` and a gradient-free int64 ``[N]`` index on its device: a lazy gather, or None."""
    if name == "__getitem__":
        if len(args) != 2:
            return None
        t, key = args
        if isinstance(key, tuple) and len(key) == 2 and key[0] is Ellipsis:
            idx = key[1]
        elif isinstance(key, torch.Tensor) and isinstance(t, torch.Tensor) and t.dim() == 1:
            idx = key
        else:
            return None
    else:
        if len(args) != 3:
            return None
        t, dim, idx = args
        if not isinstance(t, torch.Tensor) or isinstance(dim, bool) or dim not in (-1, t.dim() - 1):
            return None
    if not isinstance(t, SiteValue) or not (t.dim() in (1, 2) or (t.dim() == 3 and t.shape[1] == 1)):
        return None
    if (not isinstance(idx, torch.Tensor) or isinstance(idx, (SiteValue, LinearPredictorTensor, LazyExpParam))
            or idx.dtype != torch.int64 or idx.dim() != 1 or idx.requires_grad or idx.device != t.device):
        return None
    return LinearPredictorTensor(GroupGather(t, idx))


def _try_factor_product(name, a, b):
    """``z [N, K] @ w [K, J]`` or ``z [P, N, K] @ w [P, K, J]`` of two site values: a lazy rate, or None."""
    if name not in _FACTOR_MATMUL_FUNCS or a.dtype != torch.float32 or b.dtype != torch.float32:
        return None
    if a.device != b.device or a.device.type not in _FACTOR_DEVICE_TYPES:
        return None
    if a.dim() == 2 and b.dim() == 2 and name != "bmm":
        pass
    elif not (a.dim() == 3 and b.dim() == 3 and a.shape[0] == b.shape[0]):
        return None
    K = a.shape[-1]
    if b.shape[-2] != K or not 1 <= K <= 16:
        return None
    return LinearPredictorTensor(FactorProduct(a, b, bmm=name == "bmm"))


def _class_weights_of(W, X):
    """A site value usable as class weights for the data matrix X: [K, D] or [P, K, D], same dtype/device."""
    return (W.dim() in (2, 3) and W.shape[-1] == X.shape[1] and W.shape[-2] >= 1 and W.dtype == X.dtype
            and W.device == X.device)


def _class_bias_ok(b, K, X):
    return isinstance(b, torch.Tensor) and not isinstance(b, LinearPredictorTensor) and tuple(b.shape) == (K,) \
        and b.dtype == X.dtype and b.device == X.device


def _make_class(X, Wt, b, linear=False):
    return LinearPredictorTensor(ClassLinearPredictor(X, Wt, b, linear=linear, linear_bias=b is not None))


def _make(X, w, b):
    wp = _ops.plain_value(w) if isinstance(w, SiteValue) else w
    bp = _ops.plain_value(b) if isinstance(b, SiteValue) else b
    return LinearPredictorTensor(LinearPredictor(X, wp, bp))


class LinearPredictorTensor(torch.Tensor):
    """``X @ w^T + b`` not yet computed: metadata of a ``[P, N]`` / ``[N]`` tensor, no storage.  Wrapping a
    :class:`ClassLinearPredictor` it stands for ``[N, K]`` / ``[P, N, K]`` class logits, wrapping a
    :class:`FactorProduct` for an ``[N, J]`` / ``[P, N, J]`` product of two latent factors."""

    @staticmethod
    def __new__(cls, lazy):
        t = torch.Tensor._make_wrapper_subclass(cls, tuple(lazy.shape), dtype=lazy.dtype, device=lazy.device,
                                                requires_grad=False)
        t._lazy = lazy
        t._dense = None
        t._eager = None
        return t

    def __init__(self, lazy):
        pass

    @property
    def lazy(self):
        return self._lazy

    def dense(self):
        if self._dense is None:
            self._dense = self._lazy.dense()
        return self._dense

    def eager(self):
        """The value of the expression the model wrote, computed as it wrote it (``dense`` may contract in
        another order)."""
        return self._eager() if self._eager is not None else self.dense()

    def _with_group(self, gg):
        """This ``X @ w (+ b)`` plus the lazy gather ``gg`` as its group effect, or None: one group effect per
        predictor, an index of one value per row, and a gather that broadcasts to the predictor's shape with one
        table row, or one per particle."""
        lz = self._lazy
        if lz.group is not None or not self._fits(gg):
            return None
        if lz.slopes and (gg.index is not lz.slopes[0].index or gg.G != lz.slopes[0].G):
            return None             # the slopes that came first are by another index or G
        return LinearPredictorTensor(LinearPredictor(lz.X, lz.w, lz.b, lz.tensor_cores, group=gg, slopes=lz.slopes))

    def _fits(self, gg):
        """A gather (or slope) ``gg`` of one value per row of this predictor, of its dtype and device, that broadcasts
        to its shape with one table row, or one per particle."""
        lz = self._lazy
        if gg.index.numel() != lz.X.shape[0] or gg.dtype != lz.dtype or gg.device != lz.device:
            return False
        try:
            if torch.broadcast_shapes(gg.shape, lz.shape) != lz.shape:
                return False
        except RuntimeError:
            return False
        return gg.table.numel() // gg.G in (1, lz.P)

    def _with_slope(self, sg):
        """This ``X @ w (+ b) (+ alpha[g])`` plus the lazy slope ``sg`` as one of its varying slopes, or None: a
        covariate that is column ``c`` of the predictor's X (its storage, X's row stride, ``c`` elements past X's first
        element), at most three slopes on distinct columns, and the index object and G of the group effect or of the
        slopes already there."""
        lz = self._lazy
        X, cov = lz.X, sg.covariate
        if len(lz.slopes) >= 3 or not self._fits(sg):
            return None
        if cov.untyped_storage().data_ptr() != X.untyped_storage().data_ptr() or cov.stride(0) != X.stride(0):
            return None
        col = cov.storage_offset() - X.storage_offset()
        if not 0 <= col < X.shape[1] or any(other.col == col for other in lz.slopes):
            return None
        first = lz.group if lz.group is not None else (lz.slopes[0] if lz.slopes else None)
        if first is not None and (sg.index is not first.index or sg.G != first.G):
            return None
        return LinearPredictorTensor(LinearPredictor(lz.X, lz.w, lz.b, lz.tensor_cores, group=lz.group,
                                                     slopes=lz.slopes + (sg.with_col(col),)))

    def _times_covariate(self, c):
        """``table[..., index] * c`` as a lazy slope, or None: ``c`` a gradient-free fp32 ``[N]`` view (a column of a
        matrix is one; a tensor with storage of its own can never be a column of X) on the table's device."""
        gg = self._lazy
        if (not isinstance(c, torch.Tensor) or isinstance(c, (SiteValue, LinearPredictorTensor, LazyExpParam))
                or c.dtype != torch.float32 or gg.dtype != torch.float32 or c.dim() != 1
                or c.numel() != gg.index.numel() or c.requires_grad or c.device != gg.device or c._base is None):
            return None
        return LinearPredictorTensor(SlopeGather(gg.table, gg.index, c))

    def _scaled(self, s):
        """``s * table[..., index]`` as the gather of the table ``s * table``, or None: ``s`` a number or one scalar
        per particle (``[]``, ``[1]``, ``[P, 1]``), and a table of at most two dims."""
        gg = self._lazy
        if isinstance(s, (int, float)) and not isinstance(s, bool):
            shape = torch.Size(())
        elif (isinstance(s, torch.Tensor) and not isinstance(s, (LinearPredictorTensor, LazyExpParam))
              and s.dtype == gg.dtype and s.device == gg.device
              and ((s.numel() == 1 and s.dim() <= 2) or (s.dim() == 2 and s.shape[1] == 1))):
            shape = s.shape
            s = _ops.plain_value(s) if isinstance(s, SiteValue) else s
        else:
            return None
        try:
            tshape = torch.broadcast_shapes(shape, gg.table.shape)
            if len(tshape) > 2 or tshape[:-1] + gg.index.shape != torch.broadcast_shapes(shape, gg.shape):
                return None
        except RuntimeError:
            return None
        return LinearPredictorTensor(GroupGather(s * gg.table, gg.index))

    def _with_bias(self, b):
        lz = self._lazy
        if isinstance(lz, (GroupGather, SlopeGather)):
            if isinstance(b, LinearPredictorTensor) and isinstance(b._lazy, LinearPredictor):
                return b._with_group(lz) if isinstance(lz, GroupGather) else b._with_slope(lz)
            return None
        if isinstance(lz, LinearPredictor) and isinstance(b, LinearPredictorTensor) and isinstance(b._lazy,
                                                                                                  GroupGather):
            return self._with_group(b._lazy)
        if isinstance(lz, LinearPredictor) and isinstance(b, LinearPredictorTensor) and isinstance(b._lazy,
                                                                                                  SlopeGather):
            return self._with_slope(b._lazy)
        if isinstance(lz, (FactorProduct, ExpLinearPredictor)):
            return None
        if isinstance(lz, ClassLinearPredictor):
            if isinstance(b, LinearPredictorTensor):
                return None
            out = lz.with_bias(_ops.plain_value(b) if isinstance(b, SiteValue) else b)
            return None if out is None else LinearPredictorTensor(out)
        if lz.b is not None:
            return None
        if isinstance(b, (int, float)):
            return None
        if not isinstance(b, torch.Tensor) or isinstance(b, LinearPredictorTensor):
            return None
        bp = _ops.plain_value(b) if isinstance(b, SiteValue) else b
        # per-particle scalar: [], [1], [P], [P, 1]
        ok = bp.numel() == 1 or (lz.vectorised and bp.numel() == lz.P and
                                 tuple(bp.shape) in ((lz.P,), (lz.P, 1)) and
                                 (bp.dim() == 2 or lz.shape[-1] == lz.P))
        if lz.vectorised and bp.dim() == 1 and bp.numel() == lz.P and lz.shape[-1] != lz.P:
            ok = False          # a [P] vector broadcasts against N, not against particles
        if not ok:
            return None
        if bp.numel() == 1 and lz.P > 1:
            bp = bp.reshape(()).expand(lz.P)
        return LinearPredictorTensor(LinearPredictor(lz.X, lz.w, bp, lz.tensor_cores, group=lz.group,
                                                     slopes=lz.slopes))

    @classmethod
    def __torch_dispatch__(cls, func, types, args=(), kwargs=None):
        # only reached when an ATen call slipped past __torch_function__: materialise and run it
        from torch.utils._pytree import tree_map
        dense = lambda x: x.dense() if isinstance(x, LinearPredictorTensor) else x  # noqa: E731
        return func(*tree_map(dense, args), **tree_map(dense, kwargs or {}))

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = _name(func)
        self = next(a for a in args if isinstance(a, LinearPredictorTensor)) if any(
            isinstance(a, LinearPredictorTensor) for a in args) else None
        if self is not None:
            if name in _META_FUNCS or name in ("shape", "dtype", "device", "ndim", "layout", "is_cuda",
                                               "requires_grad", "grad_fn", "is_leaf", "names"):
                with torch._C.DisableTorchFunctionSubclass():
                    return func(*args, **kwargs)
            if name in _ADD_FUNCS and len(args) == 2 and not kwargs:
                other = args[1] if args[0] is self else args[0]
                out = self._with_bias(other)
                if out is not None:
                    if isinstance(out.lazy, LinearPredictor):
                        out._eager = _eager_call(func, args, kwargs)
                        if out.lazy.group is not None or out.lazy.slopes:
                            out.lazy.eager = out._eager      # dense() is the sum in the order the model wrote it
                    return out
            if name in _MUL_FUNCS and len(args) == 2 and not kwargs and isinstance(self._lazy, GroupGather):
                other = args[1] if args[0] is self else args[0]
                out = self._scaled(other)
                if out is None:
                    out = self._times_covariate(other)
                    if out is not None:
                        out._eager = _eager_call(func, args, kwargs)
                if out is not None:
                    return out
            # a lazy gather or slope answers nothing else: every other use materialises it
            if any(isinstance(a, LinearPredictorTensor) and isinstance(a._lazy, (GroupGather, SlopeGather))
                   for a in args):
                with torch._C.DisableTorchFunctionSubclass():
                    return func(*_plain(args), **{k: _plain(v) for k, v in kwargs.items()})
            if name == "exp" and len(args) == 1 and not kwargs and isinstance(self._lazy, LinearPredictor):
                return LinearPredictorTensor(ExpLinearPredictor(self._lazy, self.eager))
            # Poisson's rate check (constraints.nonnegative: rate >= 0) answered from the operation: exp >= 0
            if name in ("ge", "__ge__") and isinstance(self._lazy, ExpLinearPredictor) and len(args) == 2 \
                    and args[0] is self and isinstance(args[1], (int, float)) and args[1] <= 0 and not kwargs:
                return torch.ones((), dtype=torch.bool, device=self.device).expand(self.shape)
            if name in ("expand", "broadcast_to") and len(args) >= 2:
                shape = args[1] if isinstance(args[1], (tuple, list, torch.Size)) else args[1:]
                if tuple(shape) == tuple(self.shape):
                    return self
            if name == "broadcast_tensors" and all(
                    (not isinstance(a, torch.Tensor)) or tuple(a.shape) == tuple(self.shape) or a.numel() == 1
                    for a in args):
                with torch._C.DisableTorchFunctionSubclass():
                    return tuple(a if isinstance(a, LinearPredictorTensor) else a.expand(self.shape)
                                 for a in args)
            # torch.distributions.Normal(lazy X @ w + b, scale) calls broadcast_all(loc, scale): a scale that
            # broadcasts to the loc's shape ([P, 1] per particle, [N], ...) is expanded and the loc stays lazy.  The
            # expanded view remembers its operand, so the fused Normal site takes the stored scale, not a slice.
            if name == "broadcast_tensors" and isinstance(self._lazy, LinearPredictor) and not kwargs and all(
                    a is self or (isinstance(a, torch.Tensor) and not isinstance(a, LinearPredictorTensor)
                                  and a.dim() <= len(self.shape)
                                  and torch.broadcast_shapes(a.shape, self.shape) == self.shape)
                    for a in args):
                out = []
                for a in args:
                    if a is self:
                        out.append(a)
                        continue
                    plain = _plain(a)
                    with torch._C.DisableTorchFunctionSubclass():
                        v = plain.expand(self.shape)
                    v._b2_unexpanded = plain
                    out.append(v)
                return tuple(out)
            # torch.distributions.Binomial casts the broadcast total_count with ``type_as(logits)``: answered from
            # the metadata, so the logits stay lazy and the cast count keeps what it expanded
            if name == "type_as" and len(args) == 2 and args[1] is self and not kwargs \
                    and isinstance(args[0], torch.Tensor) and not isinstance(args[0], LinearPredictorTensor):
                a = args[0]
                if a.dtype == self.dtype and a.device == self.device:
                    return a
                with torch._C.DisableTorchFunctionSubclass():
                    return a.to(dtype=self.dtype, device=self.device)
            if name in ("detach", "clone", "contiguous", "float", "to") and len(args) == 1 and not kwargs:
                return self
            # distribution-argument validation (constraints.real.check): an affine image of finite
            # operands; a NaN would surface in the ELBO itself (warn_if_nan)
            # (not for exp(...): its value may be 0 or inf, so those answers are not constants; every use but the
            # rate check above materialises it)
            if (name in _CHEAP_TRUE or name in _CHEAP_FALSE) and not isinstance(self._lazy, ExpLinearPredictor):
                flag = torch.ones((), dtype=torch.bool, device=self.device) if name in _CHEAP_TRUE \
                    else torch.zeros((), dtype=torch.bool, device=self.device)
                return flag.expand(self.shape)
        with torch._C.DisableTorchFunctionSubclass():
            return func(*_plain(args), **{k: _plain(v) for k, v in kwargs.items()})


def wrap_site_values(trace):
    """Hand the latent values of a (guide) trace to the model as :class:`SiteValue` tensors.  The
    original tensor OBJECTS are remembered on the wrappers (a fused draw carries its score as a python
    attribute) and put back by :func:`unwrap_site_values`."""
    for site in trace.nodes.values():
        if site["type"] == "sample" and not site["is_observed"]:
            v = site["value"]
            w = SiteValue.wrap(v)
            if w is not v:
                w._b2_plain = v
                site["value"] = w
    return trace


def unwrap_site_values(*traces):
    for trace in traces:
        for site in trace.nodes.values():
            if site["type"] == "sample":
                v = site.get("value")
                if isinstance(v, SiteValue):
                    plain = getattr(v, "_b2_plain", None)
                    site["value"] = plain if plain is not None else _ops.plain_value(v)


def lazy_of(logits):
    """The :class:`LinearPredictor` behind a logits argument, or None."""
    if isinstance(logits, LinearPredictorTensor):
        return logits.lazy
    if isinstance(logits, LinearPredictor):
        return logits
    return None
