// site_score.cu -- host side of b2_site_score: validate, coalesce dims, pick a kernel, launch.
#include <string.h>

#include "site_score.cuh"

namespace b2 {

namespace {

struct OpView {
  const b2_tensor* t;
  int64_t st[B2_MAX_DIMS];
  bool present;
};

inline bool is_float_dtype(int d) { return d == B2_F32 || d == B2_F64; }

// classify an output's stride pattern on the common shape: 1 full, 2 scalar (summed over
// everything), 3 summed over the dims where its stride is 0 (the operand's stored shape)
int out_mode(const int64_t* shape, const int64_t* st, int ndim) {
  bool any_zero = false, any_nonzero = false;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] == 1) continue;
    if (st[d] == 0) any_zero = true; else any_nonzero = true;
  }
  if (any_zero && any_nonzero) return 3;
  return any_zero ? 2 : 1;
}

}  // namespace

int dispatch_site(int family, int dtype, bool grad, const SiteArgs& a, int kind, cudaStream_t s) {
  if (family < 0 || family >= kNumElementwise) return B2_ERR_BAD_FAMILY;
  if (family <= kPoisson) return dispatch_site_a(family, dtype, grad, a, kind, s);
  if (family <= kHalfNormal) return dispatch_site_b(family, dtype, grad, a, kind, s);
  if (family <= kNormalRsampleBwd) return dispatch_site_c(family, dtype, grad, a, kind, s);
  return dispatch_site_d(family, dtype, grad, a, kind, s);
}

static const int kFamilyNumParams[kNumElementwise] = {2, 1, 2, 2, 1, 2, 1, 1, 2, 1, 1, 2, 4, 4, 2, 3, 2, 2};

}  // namespace b2

using namespace b2;

extern "C" size_t b2_site_score_workspace(void) { return kReduceWorkspaceBytes; }

extern "C" int b2_site_score(int family, const b2_tensor* value, const b2_tensor* params,
                             int n_params, const b2_tensor* mask, double scale,
                             const b2_tensor* upstream, double weight, double sum_coeff, int flags,
                             b2_tensor* out_logprob, void* out_sum, b2_tensor* out_dvalue,
                             b2_tensor* out_dparams, void* workspace, size_t workspace_bytes,
                             void* stream) {
  if (family < 0 || family >= kNumElementwise) return B2_ERR_BAD_FAMILY;
  if (!value || !params) return B2_ERR_NULL;
  if (n_params != kFamilyNumParams[family]) return B2_ERR_BAD_SHAPE;
  if (!workspace || workspace_bytes < kReduceWorkspaceBytes) return B2_ERR_WORKSPACE;
  const int dtype = value->dtype;
  if (!is_float_dtype(dtype)) return B2_ERR_BAD_DTYPE;
  const int nd = value->ndim;
  if (nd < 0 || nd > B2_MAX_DIMS) return B2_ERR_BAD_SHAPE;

  // gather all operands on the common shape
  const b2_tensor* ins[3 + B2_MAX_PARAMS];
  const b2_tensor* outs[2 + B2_MAX_PARAMS];
  int n_in = 0, n_out = 0;
  ins[n_in++] = value;
  for (int k = 0; k < n_params; ++k) ins[n_in++] = &params[k];
  const int i_mask = mask && mask->ptr ? n_in : -1;
  if (i_mask >= 0) ins[n_in++] = mask;
  const int i_up = upstream && upstream->ptr ? n_in : -1;
  if (i_up >= 0) ins[n_in++] = upstream;
  outs[n_out++] = out_logprob && out_logprob->ptr ? out_logprob : nullptr;
  outs[n_out++] = out_dvalue && out_dvalue->ptr ? out_dvalue : nullptr;
  for (int k = 0; k < n_params; ++k)
    outs[n_out++] = out_dparams && out_dparams[k].ptr ? &out_dparams[k] : nullptr;

  int64_t n = 1;
  for (int d = 0; d < nd; ++d) {
    if (value->shape[d] < 0) return B2_ERR_BAD_SHAPE;
    n *= value->shape[d];
  }
  for (int i = 0; i < n_in; ++i) {
    if (!ins[i]->ptr && !(i == 0 && family >= kKLNormalNormal)) return B2_ERR_NULL;
    if (ins[i]->ndim != nd) return B2_ERR_BAD_SHAPE;
    const int want = (i == i_mask) ? B2_U8 : dtype;
    if (ins[i]->ptr && ins[i]->dtype != want) return B2_ERR_BAD_DTYPE;
  }
  for (int i = 0; i < n_out; ++i)
    if (outs[i]) {
      if (outs[i]->ndim != nd) return B2_ERR_BAD_SHAPE;
      if (outs[i]->dtype != dtype) return B2_ERR_BAD_DTYPE;
    }

  SiteArgs a;
  memset(&a, 0, sizeof(a));
  a.n = n;
  a.scale = scale;
  a.weight = weight;
  a.scale32 = (float)scale;
  a.f032 = (float)(weight * scale);
  a.sum_coeff = sum_coeff;
  a.flags = flags;
  a.out_sum = out_sum;
  a.partials = ws_partials(workspace);
  a.ticket = ws_ticket(workspace);

  // output modes (checked on the un-coalesced shape)
  int modes[2 + B2_MAX_PARAMS];
  for (int i = 0; i < n_out; ++i) {
    modes[i] = 0;
    if (!outs[i]) continue;
    int m = out_mode(value->shape, outs[i]->stride, nd);
    // partial reductions are fused only by the one-CTA kernel; larger sites get a full-shape
    // gradient from the caller and reduce it with b2_reduce_to
    if (m == 3 && (n > kSmallN || (flags & B2_FLAG_SITE_LARGE))) return B2_ERR_UNSUPPORTED_REDUCTION;
    if (i == 0 && m != 1 && n > 1) return B2_ERR_BAD_SHAPE;  // log_prob output is always full
    modes[i] = m;
  }
  bool grad = false;
  for (int i = 1; i < n_out; ++i) grad = grad || modes[i] != 0;

  if (n == 0) {
    // empty site: sum is 0, scalar grads are 0; nothing to launch except the tiny writes.
    // Handle by launching the generic kernel with n = 0 (it only runs the finish step).
  }

  // ---- coalesce dims: drop size-1 dims, merge (d, d+1) when every operand is jointly
  // contiguous-or-broadcast across them --------------------------------------------------------
  int64_t shp[B2_MAX_DIMS];
  int64_t ist[3 + B2_MAX_PARAMS][B2_MAX_DIMS];
  int64_t ost[2 + B2_MAX_PARAMS][B2_MAX_DIMS];
  int cd = 0;
  for (int d = 0; d < nd; ++d) {
    if (value->shape[d] == 1) continue;
    shp[cd] = value->shape[d];
    for (int i = 0; i < n_in; ++i) ist[i][cd] = ins[i]->ptr ? ins[i]->stride[d] : 0;
    for (int i = 0; i < n_out; ++i)
      ost[i][cd] = (outs[i] && (modes[i] == 1 || modes[i] == 3)) ? outs[i]->stride[d] : 0;
    ++cd;
  }
  // merge from the right
  for (int d = cd - 2; d >= 0; --d) {
    bool ok = true;
    for (int i = 0; i < n_in && ok; ++i) ok = ist[i][d] == ist[i][d + 1] * shp[d + 1];
    for (int i = 0; i < n_out && ok; ++i) ok = ost[i][d] == ost[i][d + 1] * shp[d + 1];
    if (ok) {
      shp[d] *= shp[d + 1];
      for (int i = 0; i < n_in; ++i) ist[i][d] = ist[i][d + 1];
      for (int i = 0; i < n_out; ++i) ost[i][d] = ost[i][d + 1];
      for (int e = d + 1; e < cd - 1; ++e) {
        shp[e] = shp[e + 1];
        for (int i = 0; i < n_in; ++i) ist[i][e] = ist[i][e + 1];
        for (int i = 0; i < n_out; ++i) ost[i][e] = ost[i][e + 1];
      }
      --cd;
    }
  }
  if (cd > kMaxD) return B2_ERR_BAD_SHAPE;
  if (cd == 0) {
    cd = 1;
    shp[0] = (n == 0) ? 0 : 1;
    for (int i = 0; i < n_in; ++i) ist[i][0] = 0;
    for (int i = 0; i < n_out; ++i) ost[i][0] = 0;
  }
  a.ndim = cd;
  for (int d = 0; d < cd; ++d) a.shape[d] = shp[d];

  auto fill_in = [&](Opnd& o, int i) {
    o.ptr = ins[i]->ptr;
    for (int d = 0; d < cd; ++d) o.st[d] = ist[i][d];
  };
  fill_in(a.x, 0);
  for (int k = 0; k < n_params; ++k) fill_in(a.p[k], 1 + k);
  if (i_mask >= 0) fill_in(a.mask, i_mask);
  if (i_up >= 0) fill_in(a.up, i_up);
  auto fill_out = [&](OutOpnd& o, int i) {
    o.mode = modes[i];
    o.ptr = outs[i] ? outs[i]->ptr : nullptr;
    for (int d = 0; d < cd; ++d) o.st[d] = ost[i][d];
  };
  fill_out(a.lp, 0);
  fill_out(a.gx, 1);
  for (int k = 0; k < n_params; ++k) fill_out(a.gp[k], 2 + k);

  // ---- small sites: one CTA, one launch ----------------------------------------------------------
  if (n > 0 && n <= kSmallN && !(flags & B2_FLAG_SITE_LARGE)) {
    a.scratch = a.partials;  // a single CTA needs no cross-CTA partials; reuse them as the slabs
    return dispatch_site(family, dtype, grad, a, kSiteSmall, reinterpret_cast<cudaStream_t>(stream));
  }

  // ---- vector path eligibility -----------------------------------------------------------------
  const int V = (dtype == B2_F32) ? 4 : 2;
  bool vec = (cd <= 2) && n > 0;
  int64_t R = 1, C = 1;
  if (vec) {
    C = shp[cd - 1];
    R = (cd == 2) ? shp[0] : 1;
    if (C % V != 0) vec = false;
  }
  auto vec_ok = [&](const void* ptr, const int64_t* st, bool is_mask) {
    if (!ptr) return true;
    const int64_t sc = st[cd - 1];
    const int64_t sr = (cd == 2) ? st[0] : 0;
    if (sc != 0 && sc != 1) return false;
    if (is_mask) return true;  // masks are read bytewise
    if (sc == 1) {
      if (reinterpret_cast<uintptr_t>(ptr) % 16 != 0) return false;
      if (sr % V != 0) return false;
    }
    return true;
  };
  if (vec) {
    for (int i = 0; i < n_in && vec; ++i) vec = vec_ok(ins[i]->ptr, ist[i], i == i_mask);
    for (int i = 0; i < n_out && vec; ++i)
      if (outs[i] && modes[i] == 1) {
        vec = vec_ok(outs[i]->ptr, ost[i], false) && ost[i][cd - 1] == 1;
      }
  }
  if (vec) {
    // kernel reads st[0] = row stride, st[1] = column stride
    auto to2 = [&](int64_t* st) {
      const int64_t sc = st[cd - 1];
      const int64_t sr = (cd == 2) ? st[0] : 0;
      st[0] = sr;
      st[1] = sc;
    };
    to2(a.x.st);
    for (int k = 0; k < n_params; ++k) to2(a.p[k].st);
    to2(a.mask.st);
    to2(a.up.st);
    to2(a.lp.st);
    to2(a.gx.st);
    for (int k = 0; k < n_params; ++k) to2(a.gp[k].st);
    a.R = R;
    a.C = C;
    const int64_t CV = C / V;
    int lg = 0;
    while (lg < 8 && ((int64_t)1 << lg) < CV) ++lg;
    a.tx_log2 = lg;
  }
  return dispatch_site(family, dtype, grad, a, vec ? kSiteVec : kSiteGen,
                       reinterpret_cast<cudaStream_t>(stream));
}
