// glm_normal_tc.cu -- Hopper fused linear-regression (Gaussian likelihood) kernels: for up to 64 weight vectors
// (particles) per CTA slab, ONE pass over X[N,D] and y[N] gives the sufficient statistics
//   l_pn  = x_n.w_p + b_p,   r_pn = y_n - l_pn
//   S_p   = SUM_n r_pn^2,    G_p = SUM_n r_pn [x_n | 1]
// and glm_finish_kernel (glm.cu) applies the noise scale sigma_p of each particle in fp64:
//   sum_p = -S_p / (2 sigma_p^2) - N (log sigma_p + log(2 pi) / 2)      torch/distributions/normal.py log_prob
//   dW_p  = weight * SUM_n r_pn x_n / sigma_p^2,   db_p = weight * SUM_n r_pn / sigma_p^2
//   dsigma_p = weight * (S_p / sigma_p^3 - N / sigma_p)
// (scale multiplies all of them).  It replaces the model's `X @ w + b`, Normal(loc, sigma).log_prob, the site
// sum and the autograd backward of all of them, which write and re-read the [P, N] loc, log_prob and gradient
// tensors.  sigma never enters the tile loop, so a constant, a learned or a latent sigma of any per-particle
// shape run the same kernel, and the epilogue takes no MUFU op at all.
//
// The tile loops are the GLM ones with the Normal family of glm_tc_common.cuh (fp32 labels as for Bernoulli;
// the epilogue writes g = r rounded to nearest TF32 as GEMM 2's register operand and adds r^2 to the lp slot):
// glm_tile_pipeline at D = 32 (TMA tiles, glm_tc.cu) and glm_flat_pipeline at every other D in 1..128
// (bulk-copied tiles, glm_flat_tc.cuh).  As for Poisson, GEMM 1 starts from zero and the epilogue adds the bias,
// rounded to nearest.
//
// Precision policy: W AND X are always split hi + lo (3xTF32; only the SPLIT_X instantiations exist, and
// B2_FLAG_GLM_3XTF32 changes nothing here).  The other families score a nonlinear function of l whose gradient
// averages the TF32 rounding of X away; here the scored quantity is the residual itself, and a rounding error
// delta of l does not average out of S = SUM (r + delta)^2: it adds SUM delta^2.  With X rounded to TF32, delta
// is about 2^-12 |x.w|, which at sigma = 0.01 |l| biases S by about 1e-3 relative.  So every l is fp32-exact
// up to the tensor cores' truncating accumulation: at 4 DC k-steps of three products each, the residual carries
// a shift of a few ulp of |x.w| toward zero, which reaches sum_p as SUM (r / sigma^2) delta and so grows as
// 1 / sigma^2.  Measured on an H100 at N = 1e6 against fp64 (y = X w* + 3 + sigma* eps, rms(X w*) = 1): sum_p
// within 2.4e-5 of the size of its terms at sigma* = 0.005 (6.1e-6 at 0.05), but dsigma 1e-3 .. 1.7e-3 of
// max N / sigma at sigma* = 0.005 (4.3e-3 at D = 1), about 1e-5 of the largest dsigma there; DESIGN.md section 4
// has the figures.  Per-k-block accumulators added with round-to-nearest would remove the shift, at 32 more
// accumulator registers per k-block.  g = r rounded to nearest TF32 (single-pass GEMM 2).
//
// Every sum has a fixed order; no float atomics, and a call is two launches (kernel + finish).
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {

namespace tcn {

using namespace tc;

// D = 32, X split hi / lo
__global__ void __launch_bounds__(tile32::kThreads, 1)
glm_normal_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                     const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int P,
                     float* __restrict__ partials) {
  tile32::glm_tile_pipeline<Normal, true>(map_x, map_y, W, bvec, N, P, 1, partials);
}

// every other D in 1..128, padded to DC atoms of 32 columns, X split hi / lo
template <int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC>::kThreads, 1)
glm_normal_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                          const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials) {
  tcf::glm_flat_pipeline<Normal, DC, true>(X, y, W, bvec, N, D, P, partials);
}

// with a group effect: D + G columns
template <int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_normal_group_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                           const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                           const int32_t* __restrict__ groups, int G) {
  tcf::glm_flat_pipeline<Normal, DC, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, GlmGroups{groups, G});
}

// with varying slopes as well (S > 0): D + G (1 + S) columns
template <int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_normal_slope_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                           const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                           GlmGroups grp) {
  tcf::glm_flat_pipeline<Normal, DC, true, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, grp);
}

int launch(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
           float* partials, int gx, cudaStream_t s, GlmGroups grp) {
  const dim3 grid = slab_grid(gx, P);
  if (grp.idx)
    return glm_dispatch_dc<1>(D + grp.cols(), true, [&](auto dc, auto) {
      using C = tcf::Cfg<decltype(dc)::value, true>;
      constexpr int kDC = decltype(dc)::value;
      if (grp.S)
        return launch_tc(glm_normal_slope_tc_kernel<kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, W, b, N, D,
                         P, partials, grp);
      return launch_tc(glm_normal_group_tc_kernel<kDC>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y, W, b, N, D, P,
                       partials, grp.idx, grp.G);
    });
  if (D == 32) {
    using namespace tile32;
    CUtensorMap mx, my;
    if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Normal::kYType)) return B2_ERR_LAUNCH;
    return launch_tc(glm_normal_tc_kernel, grid, dim3(kThreads), Smem32<Normal::kYBytes>::kBytes, s, mx, my, W, b, N,
                     P, partials);
  }
  // X is always split: there is one instantiation per DC
  return glm_dispatch_dc<1>(D, true, [&](auto dc, auto) {
    using C = tcf::Cfg<decltype(dc)::value>;
    return launch_tc(glm_normal_flat_tc_kernel<decltype(dc)::value>, grid, dim3(C::kThreads), C::kSmemBytes, s, X, y,
                     W, b, N, D, P, partials);
  });
}

}  // namespace tcn
}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_normal_workspace(int64_t N, int D, int P) { return glm_row_workspace(N, D, P); }

int b2::glm_normal_loc(const float* X, const float* y, const float* W, const float* b, const float* sigma,
                       int sigma_stride, int64_t N, int D, int P, double scale, double weight, double sum_coeff,
                       int flags, float* out_sum_p, float* out_total, float* out_dW, float* out_db, float* out_dsigma,
                       void* workspace, size_t workspace_bytes, cudaStream_t s, GlmGroups grp) {
  int rc = glm_row_check(X, y, W, !sigma, N, D, P, sigma_stride != 0 && sigma_stride != 1, flags, workspace,
                         workspace_bytes, grp);
  if (rc != B2_OK) return rc;
  const int Da = D + grp.cols();
  const GlmRowWorkspace w = glm_row_areas(workspace, N, Da, P);
  rc = tcn::launch(X, y, W, b, N, D, P, w.partials, w.gx, s, grp);
  if (rc != 0) return rc;
  launch_glm_finish(w.partials, w.ticket, w.gx, P, 1, Da, scale, weight, sum_coeff, flags, out_sum_p, out_total,
                    out_dW, out_db, s, sigma, sigma_stride, N, out_dsigma);
  count_launch(2);
  return check_launch();
}

extern "C" int b2_glm_normal_loc(const float* X, const float* y, const float* W, const float* b,
                                 const float* sigma, int sigma_stride, int64_t N, int D, int P, double scale,
                                 double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                                 float* out_dW, float* out_db, float* out_dsigma, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return glm_normal_loc(X, y, W, b, sigma, sigma_stride, N, D, P, scale, weight, sum_coeff, flags, out_sum_p,
                        out_total, out_dW, out_db, out_dsigma, workspace, workspace_bytes,
                        reinterpret_cast<cudaStream_t>(stream), {});
}
