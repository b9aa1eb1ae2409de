// glm_poisson_tc.cu -- Hopper fused Poisson-regression (log link) likelihood kernels: for up to 64 weight vectors
// (particles) per CTA slab, ONE pass over X[N,D] and the counts y[N] gives
//   l_pn    = x_n.w_p + b_p
//   sum_p   = SUM_n ( y_n l_pn - exp(l_pn) - lgamma(y_n + 1) )     torch/distributions/poisson.py, log(rate) = l
//   dW_p    = weight * SUM_n (y_n - exp(l_pn)) x_n,   db_p = weight * SUM_n (y_n - exp(l_pn))
// It replaces the model's `X @ w + b`, `exp`, Poisson(rate).log_prob, the site sum and the autograd backward of
// all of them, which write and re-read the [P, N] log-rate, rate, log_prob and gradient tensors.
//
// The tile loops are the GLM ones with the Poisson family of glm_tc_common.cuh (fp32 labels as for Bernoulli;
// the epilogue takes one ex2 per logit and writes g = y - e^l rounded to nearest TF32 as GEMM 2's register
// operand): glm_tile_pipeline at D = 32 (TMA tiles, glm_tc.cu) and glm_flat_pipeline at every other D in
// 1..128 (bulk-copied tiles, glm_flat_tc.cuh).  Their precision policy: W always split hi + lo, X split too
// under SPLIT_X; unlike theirs, GEMM 1 starts from zero and the epilogue adds the bias, rounded to nearest
// (the tensor cores' truncating accumulation biases a log-rate held from the first k-step; see poisson_epilogue).
//
// SUM lgamma(y + 1) depends on y alone: after its tile loop each CTA sums it in fp64 over the rows of its own
// tiles (read again from L2, outside the wgmma pipeline) and subtracts it from each particle's fp64 lp sum before
// rounding that to its fp32 partial (Poisson in glm_tc_common.cuh).  At counts of 100 a row's y l - e^l is about
// +360 nats and its lp about -3, so the cancellation happens before anything is rounded at the scale of the
// terms.  Every sum has a fixed order; no float atomics, and a call is still two launches (kernel + finish).
//
// Overflow: above l = 88.72 e^l is +inf in fp32.  Such a row's lp and g are -inf (y l - inf, y - inf), so sum_p
// is -inf and db is -inf * weight; dW is non-finite (inf, or NaN where the row's x is zero or infinities of
// both signs meet).  The materialised path gives sum_p = NaN where the count is positive (xlogy(y, inf) - inf).
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {

namespace tcpr {

using namespace tc;

// D = 32.  SPLIT_X = false (default): W split hi/lo, X rounded to nearest.  SPLIT_X = true: X split as well.
template <bool SPLIT_X>
__global__ void __launch_bounds__(tile32::kThreads, 1)
glm_poisson_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const float* __restrict__ y, const float* __restrict__ W, const float* __restrict__ bvec,
                      int64_t N, int P, float* __restrict__ partials) {
  tile32::glm_tile_pipeline<Poisson, SPLIT_X>(map_x, map_y, W, bvec, N, P, 1, partials, nullptr, nullptr, y);
}

// every other D in 1..128, padded to DC atoms of 32 columns
template <int DC, bool SPLIT_X>
__global__ void __launch_bounds__(tcf::Cfg<DC>::kThreads, 1)
glm_poisson_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                           const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials) {
  tcf::glm_flat_pipeline<Poisson, DC, SPLIT_X>(X, y, W, bvec, N, D, P, partials);
}

// with a group effect: D + G columns, X split (X rounded to TF32: glm_group.cu)
template <int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_poisson_group_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                            const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                            const int32_t* __restrict__ groups, int G) {
  tcf::glm_flat_pipeline<Poisson, DC, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, GlmGroups{groups, G});
}

// with varying slopes as well (S > 0): D + G (1 + S) columns, X split
template <int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_poisson_slope_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                            const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                            GlmGroups grp) {
  tcf::glm_flat_pipeline<Poisson, DC, true, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, grp);
}

int launch(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
           float* partials, int gx, bool split_x, cudaStream_t s, GlmGroups grp) {
  const dim3 grid = slab_grid(gx, P);
  if (grp.idx && !split_x)
    return launch_glm_group_rn(B2_GLM_POISSON, X, y, nullptr, false, W, b, N, D, P, partials, gx, s, grp);
  if (grp.idx)
    return glm_dispatch_dc<1>(D + grp.cols(), true, [&](auto dc, auto) {
      using C = tcf::Cfg<decltype(dc)::value, true>;
      constexpr int kDC = decltype(dc)::value;
      if (grp.S)
        return launch_tc(glm_poisson_slope_tc_kernel<kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, W, b, N, D,
                         P, partials, grp);
      return launch_tc(glm_poisson_group_tc_kernel<kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, W, b, N, D, P,
                       partials, grp.idx, grp.G);
    });
  if (D == 32) {
    using namespace tile32;
    CUtensorMap mx, my;
    if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Poisson::kYType)) return B2_ERR_LAUNCH;
    constexpr uint32_t kSmemBytes = Smem32<Poisson::kYBytes>::kBytes;
    return split_x ? launch_tc(glm_poisson_tc_kernel<true>, grid, dim3(kThreads), kSmemBytes, s, mx, my, y, W, b, N,
                               P, partials)
                   : launch_tc(glm_poisson_tc_kernel<false>, grid, dim3(kThreads), kSmemBytes, s, mx, my, y, W, b, N,
                               P, partials);
  }
  return glm_dispatch_dc<1>(D, split_x, [&](auto dc, auto sx) {
    using C = tcf::Cfg<decltype(dc)::value>;
    return launch_tc(glm_poisson_flat_tc_kernel<decltype(dc)::value, decltype(sx)::value>, grid, dim3(C::kThreads),
                     C::kSmemBytes, s, X, y, W, b, N, D, P, partials);
  });
}

}  // namespace tcpr
}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_poisson_workspace(int64_t N, int D, int P) { return glm_row_workspace(N, D, P); }

int b2::glm_poisson_log_rate(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                             double scale, double weight, double sum_coeff, int flags, float* out_sum_p,
                             float* out_total, float* out_dW, float* out_db, void* workspace, size_t workspace_bytes,
                             cudaStream_t s, GlmGroups grp) {
  int rc = glm_row_check(X, y, W, false, N, D, P, false, flags, workspace, workspace_bytes, grp);
  if (rc != B2_OK) return rc;
  const int Da = D + grp.cols();
  const GlmRowWorkspace w = glm_row_areas(workspace, N, Da, P);
  rc = tcpr::launch(X, y, W, b, N, D, P, w.partials, w.gx, glm_split_x(flags, N), s, grp);
  if (rc != 0) return rc;
  launch_glm_finish(w.partials, w.ticket, w.gx, P, 1, Da, scale, weight, sum_coeff, flags, out_sum_p, out_total,
                    out_dW, out_db, s);
  count_launch(2);
  return check_launch();
}

extern "C" int b2_glm_poisson_log_rate(const float* X, const float* y, const float* W, const float* b, int64_t N,
                                       int D, int P, double scale, double weight, double sum_coeff, int flags,
                                       float* out_sum_p, float* out_total, float* out_dW, float* out_db,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  return glm_poisson_log_rate(X, y, W, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                              out_db, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), {});
}
