// glm_binomial_tc.cu -- Hopper fused Binomial-regression (logit link) likelihood kernels: for up to 64 weight
// vectors (particles) per CTA slab, ONE pass over X[N,D], the successes y[N] and the trial counts m (one count for
// every row, or m[N]) gives
//   l_pn    = x_n.w_p + b_p
//   sum_p   = SUM_n ( y_n l_pn - m_n softplus(l_pn) - log C(m_n, y_n) )    pyro/distributions/torch.py Binomial
//   dW_p    = weight * SUM_n (y_n - m_n sigmoid(l_pn)) x_n,   db_p = weight * SUM_n (y_n - m_n sigmoid(l_pn))
// It replaces the model's `X @ w + b`, Binomial(m, logits).log_prob, the site sum and the autograd backward of
// all of them, which write and re-read the [P, N] logits, log_prob and gradient tensors.  It is the logistic
// kernel with a weight per row: at m = 1 it scores what b2_glm_bernoulli_logits scores.
//
// The tile loops are the GLM ones with the Binomial family of glm_tc_common.cuh: glm_tile_pipeline at D = 32 (TMA
// tiles, glm_tc.cu) and glm_flat_pipeline at every other D in 1..128 (bulk-copied tiles, glm_flat_tc.cuh; D < 32
// padded to two atoms, see launch).  Per-row
// trial counts arrive next to y, on the same mbarrier, straight from the caller's [N] tensor; one count for every
// row is read once per call from device memory.  The epilogue reads y and m from shared memory and takes ex2, rcp
// and lg2 per logit (see binomial_epilogue).
// Precision policy of the Poisson kernels: W always split hi + lo, X split too under SPLIT_X; GEMM 1 starts from
// zero and the epilogue adds the bias, rounded to nearest (see poisson_epilogue); g rounded to nearest TF32.
//
// SUM log C(m, y) = -SUM [lgamma(y + 1) + lgamma(m - y + 1) - lgamma(m + 1)] depends on the data alone: after its
// tile loop each CTA sums it in fp64 over the rows of its own tiles (read again from L2, outside the wgmma
// pipeline) and adds it to each particle's fp64 lp sum before rounding that to its fp32 partial (Binomial in
// glm_tc_common.cuh): at m = 1000 a row's y l - m softplus(l) is about -690 nats and its lp a few.  Every sum has
// a fixed order; no float atomics, and a call is two launches (kernel + finish).
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {

namespace tcbi {

using namespace tc;

// D = 32.  SPLIT_X = false (default): W split hi/lo, X rounded to nearest.  SPLIT_X = true: X split as well.
// ROW: per-row trial counts (map_m); else the one count trials[0].
template <bool ROW, bool SPLIT_X>
__global__ void __launch_bounds__(tile32::kThreads, 1)
glm_binomial_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                       const __grid_constant__ CUtensorMap map_m, const float* __restrict__ y,
                       const float* __restrict__ trials, const float* __restrict__ W,
                       const float* __restrict__ bvec, int64_t N, int P, float* __restrict__ partials) {
  tile32::glm_tile_pipeline<Binomial<ROW>, SPLIT_X>(map_x, map_y, W, bvec, N, P, 1, partials, &map_m, trials, y);
}

// every other D in 1..128, padded to DC atoms of 32 columns
template <bool ROW, int DC, bool SPLIT_X>
__global__ void __launch_bounds__(tcf::Cfg<DC>::kThreads, 1)
glm_binomial_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y,
                            const float* __restrict__ trials, const float* __restrict__ W,
                            const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials) {
  tcf::glm_flat_pipeline<Binomial<ROW>, DC, SPLIT_X>(X, y, W, bvec, N, D, P, partials, trials);
}

// with a group effect: D + G columns, X split (X rounded to TF32: glm_group.cu)
template <bool ROW, int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_binomial_group_tc_kernel(const float* __restrict__ X, const float* __restrict__ y,
                             const float* __restrict__ trials, const float* __restrict__ W,
                             const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                             const int32_t* __restrict__ groups, int G) {
  tcf::glm_flat_pipeline<Binomial<ROW>, DC, true, true>(X, y, W, bvec, N, D, P, partials, trials, GlmGroups{groups, G});
}

// with varying slopes as well (S > 0): D + G (1 + S) columns, X split
template <bool ROW, int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_binomial_slope_tc_kernel(const float* __restrict__ X, const float* __restrict__ y,
                             const float* __restrict__ trials, const float* __restrict__ W,
                             const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                             GlmGroups grp) {
  tcf::glm_flat_pipeline<Binomial<ROW>, DC, true, true, true>(X, y, W, bvec, N, D, P, partials, trials, grp);
}

template <bool ROW>
int launch(const float* X, const float* y, const float* m, const float* W, const float* b, int64_t N, int D, int P,
           float* partials, int gx, bool split_x, cudaStream_t s, GlmGroups grp) {
  const dim3 grid = slab_grid(gx, P);
  // D + G < 32 runs the two-atom loop too (see below)
  if (grp.idx && !split_x)
    return launch_glm_group_rn(B2_GLM_BINOMIAL, X, y, m, ROW, W, b, N, D, P, partials, gx, s, grp);
  if (grp.idx)
    return glm_dispatch_dc<2>(D + grp.cols(), true, [&](auto dc, auto) {
      using C = tcf::Cfg<decltype(dc)::value, true>;
      constexpr int kDC = decltype(dc)::value;
      if (grp.S)
        return launch_tc(glm_binomial_slope_tc_kernel<ROW, kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, m,
                         W, b, N, D, P, partials, grp);
      return launch_tc(glm_binomial_group_tc_kernel<ROW, kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, m, W,
                       b, N, D, P, partials, grp.idx, grp.G);
    });
  if (D == 32) {
    using namespace tile32;
    using Fam = Binomial<ROW>;
    CUtensorMap mx, my, mm;
    if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Fam::kYType)) return B2_ERR_LAUNCH;
    if (ROW ? !encode_label_map(&mm, m, N, Fam::kYType) : false) return B2_ERR_LAUNCH;
    if (!ROW) mm = my;                           // not read
    constexpr uint32_t kSmemBytes = Smem32<Fam::kYBytes>::kBytes;
    return split_x ? launch_tc(glm_binomial_tc_kernel<ROW, true>, grid, dim3(kThreads), kSmemBytes, s, mx, my, mm, y,
                               m, W, b, N, P, partials)
                   : launch_tc(glm_binomial_tc_kernel<ROW, false>, grid, dim3(kThreads), kSmemBytes, s, mx, my, mm, y,
                               m, W, b, N, P, partials);
  }
  // D < 32 runs the two-atom loop (two warpgroups, 255 registers): with one atom and four warpgroups the
  // 128-register cap made this epilogue spill
  return glm_dispatch_dc<2>(D, split_x, [&](auto dc, auto sx) {
    using C = tcf::Cfg<decltype(dc)::value>;
    return launch_tc(glm_binomial_flat_tc_kernel<ROW, decltype(dc)::value, decltype(sx)::value>, grid,
                     dim3(C::kThreads), C::kSmemBytes, s, X, y, m, W, b, N, D, P, partials);
  });
}

}  // namespace tcbi
}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_binomial_workspace(int64_t N, int D, int P) { return glm_row_workspace(N, D, P); }

int b2::glm_binomial_logits(const float* X, const float* y, const float* trials, int trials_per_row, const float* W,
                            const float* b, int64_t N, int D, int P, double scale, double weight, double sum_coeff,
                            int flags, float* out_sum_p, float* out_total, float* out_dW, float* out_db,
                            void* workspace, size_t workspace_bytes, cudaStream_t s, GlmGroups grp) {
  const bool bad_trials = (trials_per_row != 0 && trials_per_row != 1) ||
                          (trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0);
  int rc = glm_row_check(X, y, W, !trials, N, D, P, bad_trials, flags, workspace, workspace_bytes, grp);
  if (rc != B2_OK) return rc;
  const int Da = D + grp.cols();
  const GlmRowWorkspace w = glm_row_areas(workspace, N, Da, P);
  const bool split_x = glm_split_x(flags, N);
  rc = trials_per_row ? tcbi::launch<true>(X, y, trials, W, b, N, D, P, w.partials, w.gx, split_x, s, grp)
                      : tcbi::launch<false>(X, y, trials, W, b, N, D, P, w.partials, w.gx, split_x, s, grp);
  if (rc != 0) return rc;
  launch_glm_finish(w.partials, w.ticket, w.gx, P, 1, Da, scale, weight, sum_coeff, flags, out_sum_p, out_total,
                    out_dW, out_db, s);
  count_launch(2);
  return check_launch();
}

extern "C" int b2_glm_binomial_logits(const float* X, const float* y, const float* trials, int trials_per_row,
                                      const float* W, const float* b, int64_t N, int D, int P, double scale,
                                      double weight, double sum_coeff, int flags, float* out_sum_p,
                                      float* out_total, float* out_dW, float* out_db, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  return glm_binomial_logits(X, y, trials, trials_per_row, W, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p,
                             out_total, out_dW, out_db, workspace, workspace_bytes,
                             reinterpret_cast<cudaStream_t>(stream), {});
}
