// glm_flat_tc.cu -- Hopper fused logistic-regression likelihood kernel for any feature count D in 1..128
// (every D without a fused kernel of its own: glm_tc.cu takes D = 32, glm.cu's SIMT kernel D in {4, 8, 16}).
//
// Same contract as glm_bernoulli_tc_kernel (glm_tc.cu): ONE pass over X[N,D] and y[N] gives, for up to 64
// weight vectors (particles) per CTA slab, sum_n log Bernoulli(y_n | logits = x_n.w_p + b_p), dW and db, as
// CTA partials [gridDim.x][P][D + 2] that glm_finish_kernel adds in a fixed order.  The tile loop, its
// layout, budget and precision policy are glm_flat_pipeline (glm_flat_tc.cuh) with the Bernoulli family of
// glm_tc_common.cuh: the epilogue of glm_tc.cu.
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {
namespace tcf {

template <int DC, bool SPLIT_X>
__global__ void __launch_bounds__(Cfg<DC>::kThreads, 1)
glm_bernoulli_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                             const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials) {
  glm_flat_pipeline<Bernoulli, DC, SPLIT_X>(X, y, W, bvec, N, D, P, partials);
}

// with a group effect: D + G columns, X split (X rounded to TF32: glm_group.cu)
template <int DC>
__global__ void __launch_bounds__(Cfg<DC, true>::kThreads, 1)
glm_bernoulli_group_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                              const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                              const int32_t* __restrict__ groups, int G) {
  glm_flat_pipeline<Bernoulli, DC, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, GlmGroups{groups, G});
}

// with varying slopes as well (S > 0): D + G (1 + S) columns, X split
template <int DC>
__global__ void __launch_bounds__(Cfg<DC, true>::kThreads, 1)
glm_bernoulli_slope_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                              const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                              GlmGroups grp) {
  glm_flat_pipeline<Bernoulli, DC, true, true, true>(X, y, W, bvec, N, D, P, partials, nullptr, grp);
}

}  // namespace tcf

// ---- host side -------------------------------------------------------------------------------------------
// The caller (b2_glm_bernoulli_logits) has checked 1 <= D <= 128 (D + G with groups), N < 2^31 and 16-byte
// aligned X and y.
int launch_glm_flat_tc(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                       float* partials, int gx, bool split_x, cudaStream_t s, GlmGroups grp) {
  if (grp.idx && !split_x)
    return launch_glm_group_rn(B2_GLM_BERNOULLI, X, y, nullptr, false, W, b, N, D, P, partials, gx, s, grp);
  if (grp.idx)
    return glm_dispatch_dc<1>(D + grp.cols(), true, [&](auto dc, auto) {
      using C = tcf::Cfg<decltype(dc)::value, true>;
      constexpr int kDC = decltype(dc)::value;
      if (grp.S)
        return launch_tc(tcf::glm_bernoulli_slope_tc_kernel<kDC>, tc::slab_grid(gx, P), dim3(C::kThreads),
                         C::kSmemBytes, s, X, y, W, b, N, D, P, partials, grp);
      return launch_tc(tcf::glm_bernoulli_group_tc_kernel<kDC>, tc::slab_grid(gx, P), dim3(C::kThreads),
                       C::kSmemBytes, s, X, y, W, b, N, D, P, partials, grp.idx, grp.G);
    });
  return glm_dispatch_dc<1>(D, split_x, [&](auto dc, auto sx) {
    using C = tcf::Cfg<decltype(dc)::value>;
    return launch_tc(tcf::glm_bernoulli_flat_tc_kernel<decltype(dc)::value, decltype(sx)::value>,
                     tc::slab_grid(gx, P), dim3(C::kThreads), C::kSmemBytes, s, X, y, W, b, N, D, P, partials);
  });
}

}  // namespace b2
