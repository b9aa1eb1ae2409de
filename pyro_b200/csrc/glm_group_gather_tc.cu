// glm_group_gather_tc.cu -- the likelihood kernels of a regression whose group effect is too wide for the one-hot
// columns of the contraction (D + G (1 + S) > 128): glm_flat_pipeline's GATHER mode (glm_flat_tc.cuh), GEMM 1 and
// GEMM 2 over X's D columns, the group term alpha[g_n] + SUM_k beta_k[g_n] X[n, c_k] added to GEMM 1's logits on
// the CUDA cores from group-major tables, and the group gradients summed over runs of rows of equal g (the rows
// sorted by group).  Used by b2_glm_potential (glm_potential.cu), which always runs 3xTF32, and by
// b2_glm_group_gather_sum (glm_group.cu), the SVI site sum: X is split here.
//
// One kernel per family (Bernoulli, Poisson, Normal) and atom count DC of D; S is read at run time.  A call is the
// kernel and glm_finish_kernel (D wide), with no host sync.  There is no Binomial kernel: instantiated on this
// pipeline, it scored the tile before a partial last tile with that tile's zeroed labels whenever the partial tile
// was not the first of its warpgroup's range (b off by the sum of the lost 64 labels, at N = 33 793 .. 250 001, and
// exact at N a multiple of 64 or with the partial tile first in its range).  Only Binomial keeps a tile's labels in
// shared memory, in two alternating slots, until its epilogue; the three families here read theirs into registers
// before the refill, and their results at those N are exact (tests/test_glm_many_groups_potential.py).
#include <cuda.h>

#include "b2_common.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {

namespace tcg {

using namespace tc;

template <class Fam, int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, false, true>::kThreads, 1)
glm_group_gather_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ W,
                           const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                           const __grid_constant__ GlmGather ga) {
  tcf::glm_flat_pipeline<Fam, DC, true, false, false, true>(X, y, W, bvec, N, D, P, partials, nullptr, {}, ga);
}

template <class Fam>
int launch(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P, float* partials,
           int gx, cudaStream_t s, const GlmGather& ga) {
  return glm_dispatch_dc<1>(D, true, [&](auto dc, auto) {
    constexpr int kDC = decltype(dc)::value;
    using C = tcf::Cfg<kDC, false, true>;
    return launch_tc(glm_group_gather_tc_kernel<Fam, kDC>, slab_grid(gx, P), dim3(C::kThreads), C::kSmemBytes, s, X,
                     y, W, b, N, D, P, partials, ga);
  });
}

}  // namespace tcg

// the kernel's own warpgroup count, through the dispatch that launches it
int glm_gather_ranges(int64_t N, int D) {
  return glm_tc_grid_x(N) * glm_dispatch_dc<1>(D, true, [](auto dc, auto) {
           return tcf::Cfg<decltype(dc)::value, false, true>::kWG;
         });
}

int glm_gather_likelihood(int kind, const float* X, const float* y, const float* W, const float* b,
                          const float* sigma, int sigma_stride, float* dsigma, int64_t N, int D, int P, double scale,
                          double weight, double sum_coeff, int flags, float* sum_p, float* total, float* dW, float* db,
                          void* workspace, cudaStream_t s, const GlmGather& ga) {
  using namespace tc;
  const GlmRowWorkspace w = glm_row_areas(workspace, N, D, P);
  int rc;
  switch (kind) {
    case B2_GLM_BERNOULLI: rc = tcg::launch<Bernoulli>(X, y, W, b, N, D, P, w.partials, w.gx, s, ga); break;
    case B2_GLM_POISSON: rc = tcg::launch<Poisson>(X, y, W, b, N, D, P, w.partials, w.gx, s, ga); break;
    case B2_GLM_NORMAL: rc = tcg::launch<Normal>(X, y, W, b, N, D, P, w.partials, w.gx, s, ga); break;
    default: return B2_ERR_BAD_SHAPE;
  }
  if (rc != 0) return rc;
  if (kind == B2_GLM_NORMAL)
    launch_glm_finish(w.partials, w.ticket, w.gx, P, 1, D, scale, weight, sum_coeff, flags, sum_p, total, dW, db, s,
                      sigma, sigma_stride, N, dsigma);
  else
    launch_glm_finish(w.partials, w.ticket, w.gx, P, 1, D, scale, weight, sum_coeff, flags, sum_p, total, dW, db, s);
  count_launch(2);
  return check_launch();
}

}  // namespace b2
