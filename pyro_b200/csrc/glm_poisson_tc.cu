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
// SUM lgamma(y + 1) depends on y alone: after its tile loop each CTA of particle slab 0 sums it over the rows
// of its own tiles (read again from L2, outside the wgmma pipeline) into one more partial, and glm_finish_kernel
// subtracts the sum of those partials from every particle's sum.  Every sum has a fixed order; no float
// atomics, and a call is still two launches (kernel + finish).
//
// Overflow: above l = 88.72 e^l is +inf in fp32.  Such a row's lp and g are -inf (y l - inf, y - inf), so sum_p
// is -inf and db is -inf * weight; dW is non-finite (inf, or NaN where the row's x is zero or infinities of
// both signs meet).  The materialised path gives sum_p = NaN where the count is positive (xlogy(y, inf) - inf).
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "glm_flat_tc.cuh"

namespace b2 {

// glm.cu / glm_tc.cu
void launch_glm_finish(const float* partials, unsigned int* ticket, int gx, int P, int K, int D, double scale,
                       double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                       float* out_dW, float* out_db, const float* lg, cudaStream_t s);
int glm_tc_grid_x(int64_t N);

namespace tcpr {

using namespace tc;

// lg[blockIdx.x] = SUM lgamma(y_n + 1) over the rows of the CTA's tiles (blockIdx.x, blockIdx.x + gridDim.x,
// ...), in a fixed order; called by every thread of a CTA of slab 0 after its tile loop
template <int NT>
__device__ __forceinline__ void lgamma_partial(const float* __restrict__ y, int64_t N, float* __restrict__ lg) {
  __shared__ float red[NT / 32];
  const int64_t ntiles = (N + kRows - 1) / kRows;
  const int nt = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < (int64_t)nt * kRows; i += NT) {
    const int64_t n = (blockIdx.x + (i / kRows) * (int64_t)gridDim.x) * kRows + i % kRows;
    if (n < N) s += ValueAux<kPoisson, float, false>::make(__ldg(y + n)).lgx;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int w = 0; w < NT / 32; ++w) v += red[w];
    lg[blockIdx.x] = v;
  }
}

// D = 32.  SPLIT_X = false (default): W split hi/lo, X rounded to nearest.  SPLIT_X = true: X split as well.
template <bool SPLIT_X>
__global__ void __launch_bounds__(tile32::kThreads, 1)
glm_poisson_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const float* __restrict__ y, const float* __restrict__ W, const float* __restrict__ bvec,
                      int64_t N, int P, float* __restrict__ partials, float* __restrict__ lg) {
  tile32::glm_tile_pipeline<Poisson, SPLIT_X>(map_x, map_y, W, bvec, N, P, 1, partials);
  if (blockIdx.y == 0) lgamma_partial<tile32::kThreads>(y, N, lg);
}

// every other D in 1..128, padded to DC atoms of 32 columns
template <int DC, bool SPLIT_X>
__global__ void __launch_bounds__(tcf::Cfg<DC>::kThreads, 1)
glm_poisson_flat_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                           const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                           float* __restrict__ lg) {
  tcf::glm_flat_pipeline<Poisson, DC, SPLIT_X>(X, y, W, bvec, N, D, P, partials);
  if (blockIdx.y == 0) lgamma_partial<tcf::Cfg<DC>::kThreads>(y, N, lg);
}

template <bool SPLIT_X>
int launch_32(const float* X, const float* y, const float* W, const float* b, int64_t N, int P, float* partials,
              float* lg, int gx, cudaStream_t s) {
  using namespace tile32;
  CUtensorMap mx, my;
  if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Poisson::kYType)) return B2_ERR_LAUNCH;
  constexpr uint32_t kSmemBytes = Smem32<Poisson::kYBytes>::kBytes;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_poisson_tc_kernel<SPLIT_X>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)kSmemBytes);
    attr_set = true;
  }
  dim3 grid((unsigned)gx, (unsigned)((P + kM - 1) / kM), 1);
  launch_pdl(glm_poisson_tc_kernel<SPLIT_X>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, y, W, b, N, P,
             partials, lg);
  return 0;
}

template <int DC, bool SPLIT_X>
int launch_flat(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                float* partials, float* lg, int gx, cudaStream_t s) {
  using C = tcf::Cfg<DC>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_poisson_flat_tc_kernel<DC, SPLIT_X>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)C::kSmemBytes);
    attr_set = true;
  }
  dim3 grid((unsigned)gx, (unsigned)((P + kM - 1) / kM), 1);
  launch_pdl(glm_poisson_flat_tc_kernel<DC, SPLIT_X>, grid, dim3(C::kThreads), (size_t)C::kSmemBytes, s, X, y, W,
             b, N, D, P, partials, lg);
  return 0;
}

template <bool SPLIT_X>
int launch(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
           float* partials, float* lg, int gx, cudaStream_t s) {
  switch ((D + 31) / 32) {
    case 1: return launch_flat<1, SPLIT_X>(X, y, W, b, N, D, P, partials, lg, gx, s);
    case 2: return launch_flat<2, SPLIT_X>(X, y, W, b, N, D, P, partials, lg, gx, s);
    case 3: return launch_flat<3, SPLIT_X>(X, y, W, b, N, D, P, partials, lg, gx, s);
    default: return launch_flat<4, SPLIT_X>(X, y, W, b, N, D, P, partials, lg, gx, s);
  }
}

}  // namespace tcpr
}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_poisson_workspace(int64_t N, int D, int P) {
  // [ticket, 256 B] + CTA partials [gx][P][D + 2] + one [P] row for the per-particle sums + lgamma partials [gx]
  if (N < 1 || D < 1 || D > 128 || P < 1) return 256;
  const size_t gx = (size_t)glm_tc_grid_x(N);
  return 256 + (gx * (size_t)P * (size_t)(D + 2) + (size_t)P + gx) * sizeof(float);
}

extern "C" int b2_glm_poisson_log_rate(const float* X, const float* y, const float* W, const float* b, int64_t N,
                                       int D, int P, double scale, double weight, double sum_coeff, int flags,
                                       float* out_sum_p, float* out_total, float* out_dW, float* out_db,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  if (!X || !y || !W) return B2_ERR_NULL;
  if (N <= 0 || P <= 0 || D < 1 || D > 128) return B2_ERR_BAD_SHAPE;
  // the tiles arrive by TMA / bulk copies (16-byte aligned sources, 32-bit row coordinates); there is no fp32
  // SIMT kernel for this family
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (flags & B2_FLAG_GLM_FP32) return B2_ERR_BAD_SHAPE;
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_glm_poisson_workspace(N, D, P)) return B2_ERR_WORKSPACE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int gx = glm_tc_grid_x(N);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
  float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  float* lg = partials + (size_t)gx * P * (D + 2) + P;
  // the precision policy of b2_glm_bernoulli_logits: below 64 Ki rows the incoherent X rounding has not
  // averaged out yet -> X split as well
  const bool split_x = (flags & B2_FLAG_GLM_3XTF32) || N < 65536;
  int rc;
  if (D == 32)
    rc = split_x ? tcpr::launch_32<true>(X, y, W, b, N, P, partials, lg, gx, s)
                 : tcpr::launch_32<false>(X, y, W, b, N, P, partials, lg, gx, s);
  else
    rc = split_x ? tcpr::launch<true>(X, y, W, b, N, D, P, partials, lg, gx, s)
                 : tcpr::launch<false>(X, y, W, b, N, D, P, partials, lg, gx, s);
  if (rc != 0) return rc;
  launch_glm_finish(partials, ticket, gx, P, 1, D, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                    out_db, lg, s);
  count_launch(2);
  return check_launch();
}
