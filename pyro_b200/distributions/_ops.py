"""Native-backed scoring ops: thin wrappers over the C ABI plus the autograd glue.

Two entry points per family kind:

``log_prob_op``   materialised ``log_prob`` tensor with autograd (drop-in for
                  ``site["fn"].log_prob(value)``, pyro/poutine/trace_struct.py:264).  Backward is
                  one more fused kernel that consumes the upstream gradient.
``fused_site_sum``  the ELBO fast path: ONE kernel returns ``sum(scale*mask*log_prob)`` and, in the
                  same pass, the final (weight-multiplied) gradients of every operand that
                  requires grad.  Its autograd node only hands those gradients back, under the
                  contract that the upstream gradient is exactly 1 (our Trace_ELBO guarantees it).
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from .. import _native as N
from .._lazyparam import densify


def _common_shape(value, params, batch_shape=None):
    shapes = [p.shape for p in params]
    if value is not None:
        shapes.append(value.shape)
    if batch_shape is not None:
        shapes.append(torch.Size(batch_shape))
    return torch.broadcast_shapes(*shapes)


def _pad_shape(t_shape, nd):
    return (1,) * (nd - len(t_shape)) + tuple(t_shape)


def _grad_plan(t, shape):
    """How the gradient of operand ``t`` (stored shape) comes out of a kernel working on ``shape``:
    ('full', out), ('scalar', out), ('inkernel', out) -- summed to the stored shape inside the
    one-CTA kernel (small sites) -- or ('reduce', out, tmp)."""
    if t.numel() == 1 and len(shape) > 0 and _numel(shape) > 1:
        out = torch.empty(t.shape, dtype=t.dtype, device=t.device)
        return ("scalar", out, None)
    if _pad_shape(t.shape, len(shape)) == tuple(shape):
        out = torch.empty(t.shape, dtype=t.dtype, device=t.device)
        return ("full", out, None)
    out = torch.empty(t.shape, dtype=t.dtype, device=t.device)
    if _numel(shape) <= N.SITE_SMALL_N and not N.FORCE_LARGE_SITE_KERNELS:
        return ("inkernel", out, None)
    tmp = torch.empty(shape, dtype=t.dtype, device=t.device)
    return ("reduce", out, tmp)


def _numel(shape):
    n = 1
    for s in shape:
        n *= int(s)
    return n


def _plan_desc(plan, shape):
    kind, out, tmp = plan
    nd = len(shape)
    if kind == "scalar":
        d = N.b2_tensor()
        d.ptr = out.data_ptr()
        d.dtype = N._DTYPES[out.dtype]
        d.ndim = nd
        for i in range(nd):
            d.shape[i] = shape[i]
            d.stride[i] = 0
        return d
    if kind == "full":
        return N.desc(out.reshape(_pad_shape(out.shape, nd)), shape)
    if kind == "inkernel":
        return N.desc(out.reshape(_pad_shape(out.shape, nd)).expand(shape), shape)
    return N.desc(tmp, shape)


def reduce_to(src, dst):
    """dst[stored shape] = sum of src over the dims where dst is broadcast (own kernel, fixed order)."""
    shape = tuple(src.shape)
    nd = len(shape)
    dv = dst.reshape(_pad_shape(dst.shape, nd))
    sd = N.desc(src, shape)
    dd = N.desc(dv.expand(shape) if tuple(dv.shape) != shape else dv, shape)
    # column reductions split the reduced rows over CTAs and keep [splits, numel(dst)] fp64 partials
    need = min(256 + 8 * dst.numel() * 32, 64 << 20)
    ws = N.workspace(src.device, max(need, int(N.lib().b2_site_score_workspace())))
    N.check(N.lib().b2_reduce_to(ctypes.byref(sd), ctypes.byref(dd), ws.data_ptr(), ws.numel(),
                                 N.stream_ptr(src.device)), "b2_reduce_to")


def _finish_plans(plans):
    outs = []
    for plan in plans:
        if plan is None:
            outs.append(None)
            continue
        kind, out, tmp = plan
        if kind == "reduce":
            reduce_to(tmp, out)
        outs.append(out)
    return outs


def site_score(family, value, params, shape, *, mask=None, scale=1.0, upstream=None, weight=1.0,
               sum_coeff=1.0, accumulate=False, want_logprob=False, out_sum=None,
               need_dvalue=False, need_dparams=None, event_size=None, grad_like=None):
    """Launch the fused kernel for one site.  Returns (logprob | None, dvalue | None, [dparams]).
    ``grad_like[k]`` (elementwise families) overrides the tensor whose stored shape the k-th
    parameter-slot gradient is reduced to."""
    ref = params[0]
    N.require_cuda(ref, "log_prob scoring")
    dev = ref.device
    if _numel(shape) == 0:
        return _empty_site(value, params, shape, want_logprob, out_sum, accumulate, need_dvalue,
                           need_dparams)
    nd = len(shape)
    np_ = len(params)
    need_dparams = need_dparams or [False] * np_
    elementwise = event_size is None
    if elementwise:
        bshape = tuple(shape)
    else:
        bshape = tuple(shape)  # batch shape; event dims are trailing dims of each operand

    def ev_desc(t, ev_ndim):
        # descriptor over the batch dims only (event dims contiguous)
        bs = t.shape[: t.dim() - ev_ndim] if ev_ndim else t.shape
        view = t
        full = tuple(bshape) + tuple(t.shape[t.dim() - ev_ndim:]) if ev_ndim else tuple(bshape)
        view = t.expand(full) if tuple(t.shape) != full else t
        d = N.b2_tensor()
        d.ptr = view.data_ptr()
        d.dtype = N._DTYPES[view.dtype]
        d.ndim = len(bshape)
        st = view.stride()
        for i in range(len(bshape)):
            d.shape[i] = bshape[i]
            d.stride[i] = st[i] if bshape[i] != 1 else 0
        return d

    lp = torch.empty(bshape, dtype=ref.dtype, device=dev) if want_logprob else None
    ws = N.workspace(dev)
    flags = N.B2_FLAG_ACCUMULATE_SUM if accumulate else 0
    if N.FORCE_LARGE_SITE_KERNELS:
        flags |= N.B2_FLAG_SITE_LARGE
    pdesc = (N.b2_tensor * np_)()
    gdesc = (N.b2_tensor * np_)()
    if elementwise:
        vd = N.desc(value, shape) if value is not None else N.desc(None, shape)
        if value is None:
            vd.dtype = N._DTYPES[ref.dtype]
            for i in range(nd):
                vd.shape[i] = shape[i]
        for k in range(np_):
            pdesc[k] = N.desc(params[k], shape)
        md = N.desc(mask, shape) if mask is not None else None
        ud = N.desc(upstream, shape) if upstream is not None else None
        lpd = N.desc(lp, shape) if lp is not None else None
        vplan = _grad_plan(value, shape) if need_dvalue else None
        like = [(grad_like[k] if grad_like is not None and grad_like[k] is not None else params[k])
                for k in range(np_)]
        pplans = [(_grad_plan(like[k], shape) if need_dparams[k] else None) for k in range(np_)]
        gvd = _plan_desc(vplan, shape) if vplan else None
        for k in range(np_):
            if pplans[k] is not None:
                gdesc[k] = _plan_desc(pplans[k], shape)
            else:
                gdesc[k].ptr = None
                gdesc[k].ndim = nd
        code = N.lib().b2_site_score(
            family, ctypes.byref(vd), pdesc, np_, ctypes.byref(md) if md is not None else None,
            float(scale), ctypes.byref(ud) if ud is not None else None, float(weight),
            float(sum_coeff), flags, ctypes.byref(lpd) if lpd is not None else None,
            out_sum.data_ptr() if out_sum is not None else None,
            ctypes.byref(gvd) if gvd is not None else None, gdesc, ws.data_ptr(), ws.numel(),
            N.stream_ptr(dev))
        N.check(code, "b2_site_score")
        outs = _finish_plans([vplan] + pplans)
        return lp, outs[0], outs[1:]

    # ---- event families: gradients are produced full shape, then reduced if the operand was
    # batch-broadcast --------------------------------------------------------------------------------
    ev_dims = {N.DIRICHLET: (1, [1]), N.CATEGORICAL: (0, [1]), N.MVN_TRIL: (1, [1, 2])}[family]
    v_ev, p_ev = ev_dims
    vd = ev_desc(value, v_ev)
    for k in range(np_):
        pdesc[k] = ev_desc(params[k], p_ev[k])
    md = ev_desc(mask, 0) if mask is not None else None
    ud = ev_desc(upstream, 0) if upstream is not None else None
    lpd = ev_desc(lp, 0) if lp is not None else None

    def full_grad(t, ev_ndim):
        full = tuple(bshape) + tuple(t.shape[t.dim() - ev_ndim:]) if ev_ndim else tuple(bshape)
        return torch.empty(full, dtype=ref.dtype, device=dev), full

    gv_full = None
    if need_dvalue:
        gv_full, _ = full_grad(value, v_ev)
        gvd = ev_desc(gv_full, v_ev)
    else:
        gvd = None
    gp_full = [None] * np_
    for k in range(np_):
        if need_dparams[k]:
            gp_full[k], _ = full_grad(params[k], p_ev[k])
            gdesc[k] = ev_desc(gp_full[k], p_ev[k])
        else:
            gdesc[k].ptr = None
            gdesc[k].ndim = len(bshape)
    code = N.lib().b2_event_score(
        family, ctypes.byref(vd), pdesc, np_, int(event_size),
        ctypes.byref(md) if md is not None else None, float(scale),
        ctypes.byref(ud) if ud is not None else None, float(weight), float(sum_coeff), flags,
        ctypes.byref(lpd) if lpd is not None else None,
        out_sum.data_ptr() if out_sum is not None else None,
        ctypes.byref(gvd) if gvd is not None else None, gdesc, ws.data_ptr(), ws.numel(),
        N.stream_ptr(dev))
    N.check(code, "b2_event_score")

    def back_to_stored(gfull, t):
        if gfull is None:
            return None
        if tuple(gfull.shape) == tuple(t.shape):
            return gfull
        out = torch.empty(t.shape, dtype=gfull.dtype, device=dev)
        reduce_to(gfull, out)
        return out

    return lp, back_to_stored(gv_full, value), [back_to_stored(gp_full[k], params[k]) for k in range(np_)]


def _empty_site(value, params, shape, want_logprob, out_sum, accumulate, need_dvalue, need_dparams):
    """A site with zero elements: log_prob is empty, its sum and every gradient are zero."""
    ref = params[0]
    lp = torch.empty(shape, dtype=ref.dtype, device=ref.device) if want_logprob else None
    if out_sum is not None and not accumulate:
        out_sum.zero_()
    gv = torch.zeros_like(value) if need_dvalue else None
    need_dparams = need_dparams or [False] * len(params)
    gp = [torch.zeros_like(p) if need_dparams[k] else None for k, p in enumerate(params)]
    return lp, gv, gp


class _LogProbFn(torch.autograd.Function):
    """Materialised log_prob with a fused backward."""

    @staticmethod
    def forward(ctx, meta, value, *params):
        family, shape, event_size, value_is_float = meta
        ctx.meta = meta
        lp, _, _ = site_score(family, value, list(params), shape, want_logprob=True,
                              event_size=event_size)
        ctx.save_for_backward(value, *params)
        return lp

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        family, shape, event_size, value_is_float = ctx.meta
        value, *params = ctx.saved_tensors
        need_v = ctx.needs_input_grad[1] and value_is_float
        need_p = list(ctx.needs_input_grad[2:])
        gout = gout.contiguous() if not gout.is_contiguous() and gout.numel() > 0 else gout
        _, gv, gp = site_score(family, value, params, shape, upstream=gout, need_dvalue=need_v,
                               need_dparams=need_p, event_size=event_size)
        return (None, gv) + tuple(gp)


def log_prob_op(family, value, params, batch_shape, event_size=None):
    params = [densify(p) for p in params]
    value = densify(value)
    if event_size is None:
        shape = _common_shape(value, params, batch_shape)
        value_is_float = value is not None and value.is_floating_point()
    else:
        shape = torch.Size(batch_shape)
        value_is_float = value.is_floating_point()
    meta = (family, tuple(shape), event_size, value_is_float)
    return _LogProbFn.apply(meta, value, *params)


class _FusedSiteSumFn(torch.autograd.Function):
    """sum(scale*mask*log_prob) with the FINAL gradients computed in the same pass.

    With ``unit`` set the upstream gradient reaching this node is taken to be exactly 1 (the
    caller has folded its coefficient into ``weight``; pyro_b200's ELBOs and potentials guarantee
    it).  Otherwise the stored gradients are multiplied by the upstream scalar.
    """

    @staticmethod
    def forward(ctx, meta, value, *params):
        (family, shape, event_size, mask, scale, weight, sum_coeff, out_sum, accumulate, vfloat,
         unit) = meta
        ctx.unit = unit
        need_v = vfloat and value is not None and value.requires_grad
        need_p = [p.requires_grad for p in params]
        dev = params[0].device
        res = out_sum if out_sum is not None else torch.empty((), dtype=params[0].dtype, device=dev)
        _, gv, gp = site_score(family, value, list(params), shape, mask=mask, scale=scale,
                               weight=weight, sum_coeff=sum_coeff, accumulate=accumulate,
                               out_sum=res, need_dvalue=need_v, need_dparams=need_p,
                               event_size=event_size)
        ctx.grads = (gv, gp)
        return res

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        gv, gp = ctx.grads
        if not ctx.unit:
            # general autograd use: honour the upstream scalar (one small extra multiply)
            gv = gv * gout if gv is not None else None
            gp = [g * gout if g is not None else None for g in gp]
        return (None, gv) + tuple(gp)


def fused_site_sum(family, value, params, batch_shape, *, mask=None, scale=1.0, weight=1.0,
                   sum_coeff=1.0, event_size=None, assume_unit_upstream=True):
    """0-d tensor ``sum_coeff * sum(scale*mask*log_prob)`` whose backward delivers
    ``weight * d(sum)/d(operand)`` for every operand requiring grad (assuming upstream == 1)."""
    params = [densify(p) for p in params]
    value = densify(value)
    if event_size is None:
        shape = _common_shape(value, params, batch_shape)
        vfloat = value is not None and value.is_floating_point()
    else:
        shape = torch.Size(batch_shape)
        vfloat = value.is_floating_point()
    if mask is not None and mask.dtype != torch.bool:
        mask = mask.bool()
    meta = (family, tuple(shape), event_size, mask, float(scale), float(weight), float(sum_coeff),
            None, False, vfloat, bool(assume_unit_upstream))
    return _FusedSiteSumFn.apply(meta, value, *params)


# ---- fused reparameterised Normal draw (SURVEY.md 8(f) row 1) ------------------------------------
def normal_rsample_score(loc, scale, eps):
    """(z, lq): z = loc + eps*scale on eps's shape and the 0-d sum of Normal(loc, scale).log_prob(z),
    one launch (family NORMAL_RSAMPLE; replaces addcmul + the guide site's scoring kernel)."""
    shape = tuple(eps.shape)
    z = torch.empty(shape, dtype=eps.dtype, device=eps.device)
    lq = torch.empty((), dtype=eps.dtype, device=eps.device)
    if eps.numel() == 0:
        return z, lq.zero_()
    N.require_cuda(eps, "fused Normal rsample")
    nd = len(shape)
    pdesc = (N.b2_tensor * 2)()
    pdesc[0] = N.desc(loc, shape)
    pdesc[1] = N.desc(scale, shape)
    gdesc = (N.b2_tensor * 2)()
    for k in range(2):
        gdesc[k].ptr = None
        gdesc[k].ndim = nd
    vd = N.desc(eps, shape)
    zd = N.desc(z, shape)
    ws = N.workspace(eps.device)
    N.check(N.lib().b2_site_score(N.NORMAL_RSAMPLE, ctypes.byref(vd), pdesc, 2, None, 1.0, None, 1.0,
                                  1.0, 0, None, lq.data_ptr(), ctypes.byref(zd), gdesc,
                                  ws.data_ptr(), ws.numel(), N.stream_ptr(eps.device)),
            "b2_site_score[normal_rsample]")
    return z, lq


_RNG_STATE = {}


def rng_state(device):
    """Per-device {seed, launch counter, ticket} of the in-kernel Philox draws, seeded from torch's current seed
    on first use (``pyro_b200.set_rng_seed`` / ``torch.manual_seed`` before the first draw selects the
    stream).  The kernels advance the counter themselves (the ticket is the draw kernel's, left zero)."""
    key = (device.type, device.index)
    st = _RNG_STATE.get(key)
    if st is None:
        st = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=device)
        _RNG_STATE[key] = st
    return st


def reseed(seed):
    """Restart the in-kernel Philox streams (called by ``pyro_b200.set_rng_seed``)."""
    for st in _RNG_STATE.values():
        st.copy_(torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64))


def normal_rsample_philox(loc, scale, shape):
    """(z, lq, eps): the draw, the 0-d sum of its log density and the noise it used -- ONE launch, noise
    from Philox inside the kernel (b2_normal_rsample)."""
    shape = tuple(shape)
    dev, dtype = loc.device, loc.dtype
    z = torch.empty(shape, dtype=dtype, device=dev)
    eps = torch.empty(shape, dtype=dtype, device=dev)
    lq = torch.empty((), dtype=dtype, device=dev)
    ld, sd = N.desc(loc, shape), N.desc(scale, shape)
    shp = (ctypes.c_int64 * max(1, len(shape)))(*shape)
    N.check(N.lib().b2_normal_rsample(ctypes.byref(ld), ctypes.byref(sd), len(shape), shp, z.data_ptr(),
                                      eps.data_ptr(), lq.data_ptr(), rng_state(dev).data_ptr(),
                                      N.stream_ptr(dev)), "b2_normal_rsample")
    return z, lq, eps


def normal_rsample_backward(gz, eps, loc, scale, c, need_loc, need_scale):
    """Gradients of L w.r.t. (loc, scale) given gz = dL/dz and c = coefficient of sum log q(z) in L,
    reduced to the stored shapes, one launch for small sites (family NORMAL_RSAMPLE_BWD)."""
    shape = tuple(eps.shape)
    if eps.numel() == 0:
        return (torch.zeros_like(loc) if need_loc else None,
                torch.zeros_like(scale) if need_scale else None)
    from . import _const
    cten = _const(c, eps.dtype, eps.device)
    params = [eps, scale, cten]
    _, _, gp = site_score(N.NORMAL_RSAMPLE_BWD, gz, params, shape, need_dvalue=False,
                          need_dparams=[need_loc, need_scale, False],
                          grad_like=[loc, scale, None])
    return gp[0], gp[1]


def gamma_rsample(conc, rate, shape, want_grad=True):
    """``(z, dz_dconc)``: reparameterised Gamma(conc, rate) draws of ``shape`` and, with ``want_grad``, the
    derivative of every draw w.r.t. its concentration -- one launch (b2_gamma_rsample)."""
    shape = tuple(int(s) for s in shape)
    dev, dtype = conc.device, conc.dtype
    N.require_cuda(conc, "Gamma.rsample")
    z = torch.empty(shape, dtype=dtype, device=dev)
    dz = torch.empty(shape, dtype=dtype, device=dev) if want_grad else None
    cd, rd = N.desc(conc, shape), N.desc(rate, shape)
    shp = (ctypes.c_int64 * max(1, len(shape)))(*shape)
    N.check(N.lib().b2_gamma_rsample(ctypes.byref(cd), ctypes.byref(rd), len(shape), shp, z.data_ptr(),
                                     dz.data_ptr() if dz is not None else None, rng_state(dev).data_ptr(),
                                     N.stream_ptr(dev)), "b2_gamma_rsample")
    return z, dz


# ---- latent-sites block (csrc/latent.cu) -----------------------------------------------------------
def _latent_job(shape, dtype, loc=None, scale=None, log_scale=False, prior=None, z=None, eps=None, gz=None,
                out0=None, out1=None, c=0.0, pw=0.0):
    j = N.b2_latent_job()
    j.dtype = N._DTYPES[dtype]
    j.ndim = len(shape)
    j.flags = N.LATENT_LOG_SCALE if log_scale else 0
    for i, s in enumerate(shape):
        j.shape[i] = int(s)

    def view(t, strides):
        if t is None:
            return None
        v = t.expand(shape) if tuple(t.shape) != tuple(shape) else t
        st = v.stride()
        if any(abs(x) > 32767 for x in st):
            # the kernels index with 32-bit offsets: a widely strided view is packed first (its memory stays
            # valid for the launch: the caching allocator reuses it in stream order only)
            v = t.contiguous().expand(shape)
            st = v.stride()
        for i in range(len(shape)):
            strides[i] = st[i] if shape[i] != 1 else 0
        return v.data_ptr()

    j.loc = view(loc, j.loc_stride)
    j.scale = view(scale, j.scale_stride)
    if prior is not None:
        j.prior_loc = view(prior[0], j.prior_loc_stride)
        j.prior_scale = view(prior[1], j.prior_scale_stride)
    for name, t in (("z", z), ("eps", eps), ("gz", gz), ("out0", out0), ("out1", out1)):
        setattr(j, name, t.data_ptr() if t is not None else None)
    j.c = float(c)
    j.prior_weight = float(pw)
    return j


def latent_draw(loc, scale, log_scale, shape):
    """(z, lq, eps) of ONE Normal site: ``z = loc + eps*s`` with ``s = scale`` or ``exp(scale)`` (``log_scale``),
    eps from the in-kernel Philox stream, and the 0-d ``sum log Normal(z | loc, s)`` (b2_latent_normal_draw),
    launched at once (with any draws still pending before it)."""
    out = defer_latent_draw(loc, scale, log_scale, shape)
    flush_draws()
    return out


def defer_latent_draw(loc, scale, log_scale, shape):
    """:func:`latent_draw`, DEFERRED: the site joins the pending draws, which run as ONE launch (per 8 sites) at
    :func:`flush_draws`.  The returned tensors are not written yet; the caller hands z and lq out only as
    :class:`DeferredDraw` tensors, whose first read flushes, and eps is read by the draw's backward only."""
    shape = tuple(int(s) for s in shape)
    dev, dtype = loc.device, loc.dtype
    z = torch.empty(shape, dtype=dtype, device=dev)
    eps = torch.empty(shape, dtype=dtype, device=dev)
    lq = torch.empty((), dtype=dtype, device=dev)
    # the operands are read through pointers at the flush: building the job reads loc and scale through torch,
    # which flushes any pending draw they come from first
    job = _latent_job(shape, dtype, loc=loc, scale=scale, log_scale=log_scale, z=z, eps=eps, out0=lq)
    _PENDING_DRAWS.append((job, (loc, scale, z, eps, lq), dev))
    return z, lq, eps


# Draws registered by latent_draw and not launched yet: (job, tensors its pointers refer to, device).
_PENDING_DRAWS = []


def flush_draws():
    """Launch every pending draw: one b2_latent_normal_draw per run of up to 8 sites of one device and dtype, in
    the order they were drawn.  Job k of a launch uses the Philox counter the k-th one-job launch would have, so
    the values equal those of separate launches bit for bit."""
    global _PENDING_DRAWS
    if not _PENDING_DRAWS:
        return
    pending, _PENDING_DRAWS = _PENDING_DRAWS, []
    i = 0
    while i < len(pending):
        dev, dt = pending[i][2], pending[i][0].dtype
        j = i
        while j < len(pending) and j - i < N.LATENT_MAX_JOBS and pending[j][2] == dev and pending[j][0].dtype == dt:
            j += 1
        chunk = pending[i:j]
        jobs = (N.b2_latent_job * len(chunk))(*[jb for jb, _, _ in chunk])
        N.check(N.lib().b2_latent_normal_draw(jobs, len(chunk), rng_state(dev).data_ptr(), N.stream_ptr(dev)),
                "b2_latent_normal_draw")
        i = j


# tensor queries that read no element: they leave the pending draws pending
_NO_READ = {"size", "dim", "ndimension", "numel", "nelement", "__len__", "is_floating_point", "is_complex",
            "element_size", "get_device", "is_contiguous", "stride", "storage_offset", "as_subclass", "shape",
            "dtype", "device", "ndim", "layout", "is_cuda", "requires_grad", "grad_fn", "is_leaf", "names",
            "requires_grad_"}


def _func_name(func):
    name = getattr(func, "__name__", None) or str(func)
    if name == "__get__":
        name = getattr(getattr(func, "__self__", None), "__name__", name)
    return name


def flush_before(func):
    """Flush the pending draws unless ``func`` only asks for metadata."""
    if _PENDING_DRAWS and _func_name(func) not in _NO_READ:
        flush_draws()


N.before_launch = flush_draws


def plain_value(t):
    """``t`` (a site value of a lazy-aware subclass) as a plain tensor, its pending draw launched first: the plain
    alias no longer guards its reads."""
    flush_draws()
    return t.as_subclass(torch.Tensor)


class DeferredDraw(torch.Tensor):
    """The value (or 0-d score) of a deferred draw: any torch operation that can read it launches the pending
    draws first, so an unwritten value can never be read; the result is a plain tensor."""

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        flush_before(func)
        with torch._C.DisableTorchFunctionSubclass():
            return func(*args, **(kwargs or {}))


def latent_prior(items):
    """``[sum log Normal(z_k | ploc_k, pscale_k)]`` for a list of ``(z, ploc, pscale)``: value only, one launch
    per 8 sites (b2_latent_normal_prior).  Returns a list of 0-d tensors (views of one buffer)."""
    ref = items[0][0]
    out = torch.empty(len(items), dtype=ref.dtype, device=ref.device)
    for base in range(0, len(items), N.LATENT_MAX_JOBS):
        chunk = items[base:base + N.LATENT_MAX_JOBS]
        jobs = (N.b2_latent_job * len(chunk))()
        for k, (z, ploc, pscale) in enumerate(chunk):
            zc = z if z.is_contiguous() else z.contiguous()
            jobs[k] = _latent_job(tuple(z.shape), z.dtype, prior=(ploc, pscale), z=zc, out0=out[base + k])
        N.check(N.lib().b2_latent_normal_prior(jobs, len(chunk), N.stream_ptr(ref.device)),
                "b2_latent_normal_prior")
    return [out[k] for k in range(len(items))]


def latent_prior_combine(items, item_coeffs, terms, term_coeffs):
    """0-d ``sum_j item_coeffs[j] * sum log Normal(z_j | prior_j) + sum_t term_coeffs[t] * terms[t]`` in ONE launch
    (b2_latent_normal_prior_combine), or None when it does not apply (too many / too large sites, mixed dtypes)."""
    ref = items[0][0]
    if (len(items) > N.LATENT_MAX_JOBS or len(terms) > N.LATENT_MAX_TERMS
            or sum(z.numel() for z, _, _ in items) > N.LATENT_COMBINE_MAX_N
            or any(z.dtype != ref.dtype for z, _, _ in items) or any(t.dtype != ref.dtype for t in terms)):
        return None
    out = torch.empty((), dtype=ref.dtype, device=ref.device)
    jobs = (N.b2_latent_job * len(items))()
    keep = []
    for k, (z, ploc, pscale) in enumerate(items):
        zc = z if z.is_contiguous() else z.contiguous()
        keep.append(zc)
        jobs[k] = _latent_job(tuple(z.shape), z.dtype, prior=(ploc, pscale), z=zc)
    jc = (ctypes.c_double * len(items))(*[float(c) for c in item_coeffs])
    n = len(terms)
    ptrs = (ctypes.c_void_p * max(1, n))(*[t.data_ptr() for t in terms])
    tc = (ctypes.c_double * max(1, n))(*[float(c) for c in term_coeffs])
    N.check(N.lib().b2_latent_normal_prior_combine(jobs, len(items), jc, ptrs, tc, n, out.data_ptr(),
                                                   N.stream_ptr(ref.device)), "b2_latent_normal_prior_combine")
    return out


# Loss assembly handed to the likelihood call of a step's LAST model site: the fused Bernoulli GLM call computes
# what latent_prior_combine(items, item_coeffs, terms + [its own total], term_coeffs + [own_coeff]) would, in its
# finish kernel (b2_glm_bernoulli_logits_elbo), which saves that launch.  Trace_ELBO opens it around the site's
# scoring; the first GLM call inside takes it and sets ``loss``; if none does, ``loss`` stays None.
_ELBO_ASSEMBLY = None


class elbo_assembly:
    def __init__(self, items, item_coeffs, terms, term_coeffs, own_coeff):
        self.items, self.item_coeffs = items, item_coeffs
        self.terms, self.term_coeffs, self.own_coeff = terms, term_coeffs, own_coeff
        self.loss = self.total = None

    def __enter__(self):
        global _ELBO_ASSEMBLY
        self._prev, _ELBO_ASSEMBLY = _ELBO_ASSEMBLY, self
        return self

    def __exit__(self, *exc):
        global _ELBO_ASSEMBLY
        _ELBO_ASSEMBLY = self._prev
        return False


def take_elbo_assembly(device):
    """The open assembly as the ctypes arguments of b2_glm_bernoulli_logits_elbo, ``(asm, jobs, n_jobs, job_coeffs,
    terms, term_coeffs, n_terms, keep)``, or None when there is none or it does not fit one finish kernel (the
    limits of latent_prior_combine, fp32 on ``device``).  Taking it closes it for any later call."""
    global _ELBO_ASSEMBLY
    asm, _ELBO_ASSEMBLY = _ELBO_ASSEMBLY, None
    if asm is None:
        return None
    items, terms = asm.items, asm.terms
    if (not items or len(items) > N.LATENT_MAX_JOBS or len(terms) + 1 > N.LATENT_MAX_TERMS
            or sum(z.numel() for z, _, _ in items) > N.LATENT_COMBINE_MAX_N
            or any(z.dtype != torch.float32 or z.device != device for z, _, _ in items)
            or any(t.dtype != torch.float32 or t.device != device for t in terms)):
        return None
    jobs = (N.b2_latent_job * len(items))()
    keep = []
    for k, (z, ploc, pscale) in enumerate(items):
        zc = z if z.is_contiguous() else z.contiguous()
        keep.append(zc)
        jobs[k] = _latent_job(tuple(z.shape), z.dtype, prior=(ploc, pscale), z=zc)
    jc = (ctypes.c_double * len(items))(*[float(c) for c in asm.item_coeffs])
    n = len(terms) + 1
    ptrs = (ctypes.c_void_p * n)(*([t.data_ptr() for t in terms] + [None]))
    tc = (ctypes.c_double * n)(*([float(c) for c in asm.term_coeffs] + [float(asm.own_coeff)]))
    return asm, jobs, len(items), jc, ptrs, tc, n, keep


# Deferred draw-backwards: inside `deferred_latent_backward()` (Trace_ELBO wraps its autograd.backward call in it)
# the backward of a fused draw whose gradients all go straight into existing leaf `.grad` buffers only registers
# its job; the registered jobs of the pass run as ONE launch when the context closes.  (A draw that has to hand a
# gradient tensor back to the autograd engine launches at once: the engine may add to that tensor right away.)
_DEFERRED = None


class deferred_latent_backward:
    def __enter__(self):
        global _DEFERRED
        self._prev = _DEFERRED
        _DEFERRED = []
        return self

    def __exit__(self, *exc):
        global _DEFERRED
        pending, _DEFERRED = _DEFERRED, self._prev
        for base in range(0, len(pending), N.LATENT_MAX_JOBS):
            chunk = pending[base:base + N.LATENT_MAX_JOBS]
            jobs = (N.b2_latent_job * len(chunk))(*[j for j, _, _ in chunk])
            N.check(N.lib().b2_latent_normal_backward(jobs, len(chunk), N.stream_ptr(chunk[0][2])),
                    "b2_latent_normal_backward")
        return False


SLOT_LEAVES = set()   # id() of the leaves whose gradient went straight into their .grad (read by SVI's capture)


def _grad_slot(t):
    """A leaf whose ``.grad`` already exists (a replicated step keeps the gradients as views of the all-reduce
    payload; an eager step keeps the buffers the optimiser zeroed): the backward kernel can add into it and the
    autograd engine is told there is nothing left to accumulate -- no AccumulateGrad launch per parameter."""
    g = t.grad if t.is_leaf and t.requires_grad else None
    if g is not None and g.is_contiguous() and g.shape == t.shape and g.dtype == t.dtype and not g.requires_grad:
        return g
    return None


def latent_backward(gz, eps, z, loc, scale, log_scale, c, prior, need_loc, need_scale, accumulate=False):
    """Gradients of the loss w.r.t. ``(loc, scale | log scale)`` of a fused draw: ``gz`` = dL/dz from the
    consumers of z, ``c`` = coefficient of ``sum log q(z)``, ``prior`` = ``(ploc, pscale, weight)`` of a Normal
    prior whose ``weight * d log p(z)/dz`` joins ``gz`` here; reduced to the stored shapes, one launch.  With
    ``accumulate``, an operand that is a leaf with an existing ``.grad`` gets its gradient ADDED there by the
    kernel and None is returned in its place."""
    shape = tuple(eps.shape)
    if eps.numel() == 0:
        return (torch.zeros_like(loc) if need_loc else None, torch.zeros_like(scale) if need_scale else None)
    dev, dtype = eps.device, eps.dtype
    if gz is not None and (tuple(gz.shape) != shape or not gz.is_contiguous()):
        gz = gz.expand(shape).contiguous()
    flags_acc = 0
    gloc = gscale = None
    ret_loc = ret_scale = True
    if need_loc:
        slot = _grad_slot(loc) if accumulate else None
        if slot is not None:
            gloc, ret_loc, flags_acc = slot, False, flags_acc | N.LATENT_ACC_OUT0
            SLOT_LEAVES.add(id(loc))
        else:
            gloc = torch.empty(loc.shape, dtype=dtype, device=dev)
    slot = _grad_slot(scale) if (accumulate and need_scale and scale.is_contiguous()) else None
    if slot is not None:
        SLOT_LEAVES.add(id(scale))
    if not scale.is_contiguous():
        scale = scale.contiguous()      # the kernel writes d/dscale with the strides it reads scale with
    if need_scale:
        if slot is not None:
            gscale, ret_scale, flags_acc = slot, False, flags_acc | N.LATENT_ACC_OUT1
        else:
            gscale = torch.empty(scale.shape, dtype=dtype, device=dev)
    pr = (prior[0], prior[1]) if prior is not None else None
    # loc itself is not read in the backward pass: its slot carries the (contiguous) layout of d/dloc
    job = _latent_job(shape, dtype, loc=gloc, scale=scale, log_scale=log_scale, prior=pr, z=z, eps=eps, gz=gz,
                      out0=gloc, out1=gscale, c=c, pw=prior[2] if prior is not None else 0.0)
    job.flags |= flags_acc
    if _DEFERRED is not None and (not need_loc or not ret_loc) and (not need_scale or not ret_scale):
        # every wanted gradient is ADDED into an existing .grad by the kernel (order-independent on the stream)
        # and nothing is handed back to the engine, so the launch can wait for the other draws of this backward
        # pass; the job's pointers stay valid through the tensors kept alongside it
        _DEFERRED.append((job, (gz, eps, z, scale, gloc, gscale, pr), dev))
        return (gloc if ret_loc else None), (gscale if ret_scale else None)
    jobs = (N.b2_latent_job * 1)(job)
    N.check(N.lib().b2_latent_normal_backward(jobs, 1, N.stream_ptr(dev)), "b2_latent_normal_backward")
    return (gloc if ret_loc else None), (gscale if ret_scale else None)


def elbo_combine(terms, coeffs):
    """0-d ``sum_i coeffs[i] * terms[i]`` of 0-d device tensors in ONE launch (b2_elbo_combine)."""
    ref = terms[0]
    N.require_cuda(ref, "ELBO assembly")
    n = len(terms)
    if n > 32:
        return torch.dot(torch.stack([t.reshape(()) for t in terms]),
                         torch.tensor(coeffs, dtype=ref.dtype, device=ref.device))
    out = torch.empty((), dtype=ref.dtype, device=ref.device)
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in terms])
    cs = (ctypes.c_double * n)(*[float(c) for c in coeffs])
    N.check(N.lib().b2_elbo_combine(ptrs, cs, n, N._DTYPES[ref.dtype], out.data_ptr(),
                                    N.stream_ptr(ref.device)), "b2_elbo_combine")
    return out
