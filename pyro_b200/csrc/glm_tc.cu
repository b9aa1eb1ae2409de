// glm_tc.cu -- Hopper fused logistic-regression likelihood kernel (BASELINE config 2):
// TMA tile loads completing on mbarriers, wgmma with register accumulators, persistent CTAs.
//
// Same contract as glm_bernoulli_kernel (glm.cu): ONE pass over X[N,32] and y[N] gives, for up to 64
// weight vectors (particles) per CTA slab, sum_n log Bernoulli(y_n | logits = x_n.w_p + b_p), dW and
// db.  It replaces (reference, per SVI step): the user model's `w @ X.T + b`, then
// torch/distributions/bernoulli.py:121-125 (log_prob), pyro/poutine/trace_struct.py:264-278 (.sum())
// and the autograd backward of all three.
//
// Per 64-row tile (one persistent CTA per SM, tiles round-robin over CTAs, and inside a CTA round-robin
// over its four warpgroups; each warpgroup owns a whole tile):
//
//   split    the warpgroup rounds its X tile to nearest TF32 in place (SPLIT_X: X_hi / X_lo split) and
//            writes the transposed X^T[d][n] (plus 8 rows of ones) as the K-major B operand of GEMM 2, with
//            n permuted inside each group of 8 rows (kt_pos) to match the register layout of g.
//   GEMM 1   D1^T[p, n] = sum_d W[p, d] X[n, d] + b[p]    wgmma m64n64k8, K = 32, A = W, B = the X tile
//            (both K-major as they sit in shared memory), accumulator = bias.
//            W is split hi + lo, two TF32 MMAs per k-step -- the rounding of W is the only error of a
//            TF32 GEMM 1 that is COHERENT over rows (it shifts all N logits of a particle the same way
//            and survives the N-term sums); X is rounded to nearest (incoherent, averages as 1/sqrt(N)).
//            SPLIT_X splits X as well (a third MMA per k-step; every logit exact to ~1e-6).
//   epilogue each thread holds 2 particles x 16 rows of D1^T in registers, evaluates lp = y*l - softplus(l),
//            g = y - sigmoid(l) (2 MUFU per element plus one lg2 per particle and tile on the product of the
//            softplus denominators, in batches so part of the MUFU latency is covered inside the warp), keeps
//            its two per-particle lp sums in registers and rounds g to nearest TF32.  g stays in the
//            registers: it is already the A fragment of GEMM 2.  Only the last, partial tile masks rows.
//   GEMM 2   [dW | db][p, :] += sum_n g[p, n] [X | 1][n, :]   wgmma m64n40k8, K = 64, A from registers:
//            single-pass TF32 on round-to-nearest operands (unbiased; |err| <= 2^-11 sum|g x|).  The
//            accumulator stays in registers for the whole kernel; GEMM 2 of a tile is committed and left
//            running while the warpgroup waits for its next tile (the wait sits at the top of the tile
//            loop), and the warpgroups of a CTA overlap each other's phases.
//
// No ordinary instruction writes a wgmma accumulator between the start and the end of a wgmma pipeline
// stage: ptxas would serialise every wgmma of the kernel (C7515).  So GEMM 2's accumulator is started by
// the first k-step of the warpgroup's first tile with scale-d = 0 rather than zeroed, and the g registers
// are pinned before wgmma.fence.  tests/test_glm_tc_sass.py checks the SASS for this.
//
// TF32 wgmma operands must be K-major, so the split pass transposes X once per tile in shared memory.
// Every shared-memory operand tile is K-major SWIZZLE_128B (the layout TMA writes natively for the X tile).
//
// 512 threads = four warpgroups and no producer warp, so each scheduler has four warps to switch between
// while MUFU results are pending; that caps the kernel at 128 registers per thread.  Each warpgroup double-buffers its own X/y tiles:
// one thread issues the TMA load of tile j+2 into the stage of tile j as soon as GEMM 1 has read it (an
// mbarrier per stage counts the transaction bytes); X^T and X_lo are private to each warpgroup.
//
// Determinism: every CTA writes its partials once (warpgroups summed in a fixed order); glm_finish_kernel
// adds the CTA partials in a fixed order.
//
// The tile loop is glm_tile_pipeline (glm_tc_common.cuh), which the softmax kernel of glm_categorical_tc.cu
// runs as well, with the Bernoulli family of glm_tc_common.cuh: fp32 labels and the epilogue above.
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "glm_tc_common.cuh"

namespace b2 {
namespace tc {

using namespace tile32;

// SPLIT_X = false (default): W split hi/lo, X rounded to nearest.  SPLIT_X = true: full 3xTF32, X split
// hi/lo as well.
template <bool SPLIT_X>
__global__ void __launch_bounds__(kThreads, 1)
glm_bernoulli_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                        const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int P,
                        float* __restrict__ partials) {
  glm_tile_pipeline<Bernoulli, SPLIT_X>(map_x, map_y, W, bvec, N, P, 1, partials);
}

}  // namespace tc

// ---- host side -------------------------------------------------------------------------------------------
int glm_tc_grid_x(int64_t N) {
  const int64_t ntiles = (N + tc::kRows - 1) / tc::kRows;
  int64_t gx = kNumSMs;
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  return (int)gx;
}

// returns 0 on success, a negative B2_ERR code when the TMA path cannot be used for these operands
int launch_glm_tc(const float* X, const float* y, const float* W, const float* b, int64_t N, int P,
                  float* partials, int gx, bool split_x, cudaStream_t s) {
  using namespace tc;
  using namespace tc::tile32;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (N >= (int64_t)1 << 31) return B2_ERR_TOO_LARGE;
  CUtensorMap mx, my;
  if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Bernoulli::kYType)) return B2_ERR_LAUNCH;
  constexpr uint32_t kSmemBytes = Smem32<Bernoulli::kYBytes>::kBytes;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_bernoulli_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    cudaFuncSetAttribute(glm_bernoulli_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    attr_set = true;
  }
  dim3 grid((unsigned)gx, (unsigned)((P + kM - 1) / kM), 1);
  if (split_x)
    launch_pdl(glm_bernoulli_tc_kernel<true>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, W, b, N, P, partials);
  else
    launch_pdl(glm_bernoulli_tc_kernel<false>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, W, b, N, P, partials);
  return 0;
}

}  // namespace b2
