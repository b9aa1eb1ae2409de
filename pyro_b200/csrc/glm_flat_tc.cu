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

namespace b2 {
namespace tcf {

template <int DC, bool SPLIT_X>
__global__ void __launch_bounds__(Cfg<DC>::kThreads, 1)
glm_bernoulli_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                             const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials) {
  glm_flat_pipeline<Bernoulli, DC, SPLIT_X>(X, y, W, bvec, N, D, P, partials);
}

template <int DC, bool SPLIT_X>
void launch_one(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                float* partials, int gx, cudaStream_t s) {
  using C = Cfg<DC>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_bernoulli_flat_tc_kernel<DC, SPLIT_X>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)C::kSmemBytes);
    attr_set = true;
  }
  dim3 grid((unsigned)gx, (unsigned)((P + kM - 1) / kM), 1);
  launch_pdl(glm_bernoulli_flat_tc_kernel<DC, SPLIT_X>, grid, dim3(C::kThreads), (size_t)C::kSmemBytes, s,
             X, y, W, b, N, D, P, partials);
}

}  // namespace tcf

// ---- host side -------------------------------------------------------------------------------------------
// The caller (b2_glm_bernoulli_logits) has checked 1 <= D <= 128, N < 2^31 and 16-byte aligned X and y.
void launch_glm_flat_tc(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                        float* partials, int gx, bool split_x, cudaStream_t s) {
  using namespace tcf;
  switch ((D + 31) / 32) {
    case 1: (split_x ? launch_one<1, true> : launch_one<1, false>)(X, y, W, b, N, D, P, partials, gx, s); break;
    case 2: (split_x ? launch_one<2, true> : launch_one<2, false>)(X, y, W, b, N, D, P, partials, gx, s); break;
    case 3: (split_x ? launch_one<3, true> : launch_one<3, false>)(X, y, W, b, N, D, P, partials, gx, s); break;
    default: (split_x ? launch_one<4, true> : launch_one<4, false>)(X, y, W, b, N, D, P, partials, gx, s); break;
  }
}

}  // namespace b2
