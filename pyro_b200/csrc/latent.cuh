// latent.cuh -- the device form of a latent-site job (b2_latent_job) and its index math, shared by the latent-sites
// kernels (latent.cu) and the GLM finish kernel, which scores the value-only Normal priors of a step while it
// assembles the loss (glm.cu).
#pragma once
#include <stdint.h>

#include "b2_common.cuh"

namespace b2 {

struct LatentJob {
  int ndim;
  unsigned n;
  unsigned shape[kMaxD];
  int st_loc[kMaxD], st_scale[kMaxD], st_ploc[kMaxD], st_pscale[kMaxD];
  int flags;
  const void* loc;
  const void* scale;    // scale, or log(scale) with B2_LATENT_LOG_SCALE
  const void* ploc;     // prior (may be null)
  const void* pscale;
  void* z;              // [shape] contiguous (draw: out; prior / backward: in)
  void* eps;            // [shape] contiguous (draw: out; backward: in)
  const void* gz;       // backward: dL/dz [shape] contiguous, may be null (= 0)
  void* out0;           // draw: sum log q (0-d); prior: sum log p (0-d); backward: d/dloc (stored shape)
  void* out1;           // backward: d/dscale or d/dlog_scale (stored shape)
  double c, pw;         // backward: coefficient of d(sum log q)/d(.), weight of the prior's d log p/dz
};
struct LatentArgs {
  LatentJob job[B2_LATENT_MAX_JOBS];
  unsigned long long* state;
};

__device__ __forceinline__ void unravel(const LatentJob& j, unsigned i, int& ol, int& os, int& opl, int& ops) {
  unsigned rem = i;
  ol = os = opl = ops = 0;
  for (int d = j.ndim - 1; d >= 0; --d) {
    const unsigned sd = j.shape[d];
    const unsigned q = rem / sd;
    const int idx = (int)(rem - q * sd);
    rem = q;
    ol += idx * j.st_loc[d];
    os += idx * j.st_scale[d];
    opl += idx * j.st_ploc[d];
    ops += idx * j.st_pscale[d];
  }
}

static inline int fill_job(LatentJob& j, const b2_latent_job& h, int dtype) {
  if (h.ndim < 0 || h.ndim > kMaxD) return B2_ERR_BAD_SHAPE;
  j.ndim = h.ndim;
  int64_t n = 1;
  for (int d = 0; d < kMaxD; ++d) {
    j.shape[d] = 1;
    j.st_loc[d] = j.st_scale[d] = j.st_ploc[d] = j.st_pscale[d] = 0;
  }
  for (int d = 0; d < h.ndim; ++d) {
    if (h.shape[d] <= 0) return B2_ERR_BAD_SHAPE;
    // offsets are 32-bit in the kernels (a site has <= 65 536 elements, but an operand may be a strided view)
    const int64_t lim = INT32_MAX / B2_RSAMPLE_MAX_N;
    if (h.loc_stride[d] > lim || h.loc_stride[d] < -lim || h.scale_stride[d] > lim || h.scale_stride[d] < -lim ||
        h.prior_loc_stride[d] > lim || h.prior_loc_stride[d] < -lim || h.prior_scale_stride[d] > lim ||
        h.prior_scale_stride[d] < -lim)
      return B2_ERR_TOO_LARGE;
    j.shape[d] = (unsigned)h.shape[d];
    n *= h.shape[d];
    j.st_loc[d] = (int)h.loc_stride[d];
    j.st_scale[d] = (int)h.scale_stride[d];
    j.st_ploc[d] = (int)h.prior_loc_stride[d];
    j.st_pscale[d] = (int)h.prior_scale_stride[d];
  }
  if (n <= 0 || n > B2_RSAMPLE_MAX_N) return B2_ERR_TOO_LARGE;
  if (h.dtype != dtype) return B2_ERR_BAD_DTYPE;
  j.n = (unsigned)n;
  j.flags = h.flags;
  j.loc = h.loc;
  j.scale = h.scale;
  j.ploc = h.prior_loc;
  j.pscale = h.prior_scale;
  j.z = h.z;
  j.eps = h.eps;
  j.gz = h.gz;
  j.out0 = h.out0;
  j.out1 = h.out1;
  j.c = h.c;
  j.pw = h.prior_weight;
  return B2_OK;
}

static inline int fill_args(LatentArgs& a, const b2_latent_job* jobs, int n_jobs, int& dtype, unsigned& nmax) {
  if (!jobs) return B2_ERR_NULL;
  if (n_jobs < 1 || n_jobs > B2_LATENT_MAX_JOBS) return B2_ERR_BAD_SHAPE;
  dtype = jobs[0].dtype;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_BAD_DTYPE;
  nmax = 0;
  for (int k = 0; k < n_jobs; ++k) {
    const int code = fill_job(a.job[k], jobs[k], dtype);
    if (code != B2_OK) return code;
    if (a.job[k].n > nmax) nmax = a.job[k].n;
  }
  a.state = nullptr;
  return B2_OK;
}

// Job flag set by the host for the backward (never by a caller): loc and scale are summed over the same broadcast
// positions, so latent_backward_kernel reduces both in one pass.  That holds when every dim of more than one
// element is broadcast (stride 0) in both operands or in neither.
constexpr int kLatentSameReduction = 1 << 16;

static inline bool latent_same_reduction(const LatentJob& j) {
  for (int d = 0; d < j.ndim; ++d)
    if (j.shape[d] > 1 && (j.st_loc[d] == 0) != (j.st_scale[d] == 0)) return false;
  return true;
}

// threads of a one-CTA-per-job launch whose largest job has nmax elements
static inline int threads_for(unsigned nmax) { return nmax >= 1024 ? 1024 : (int)((nmax + 31) / 32 * 32); }

}  // namespace b2
