// glm_potential.cu -- HMC / NUTS potential energy of Bayesian logistic, softmax and Poisson regression for C
// chains.
//
//   U[c]    = -( SUM_n log p(y_n | logits_cn) + SUM log Normal(w; 0, s_w) + SUM log Normal(b; 0, s_b) )
//   grad[c] = dU / dz[c]                                           (in z's layout)
//
// The likelihood and its gradient come from the fused GLM kernels (glm.cu / glm_tc.cu for Bernoulli,
// glm_categorical_tc.cu for Categorical, glm_poisson_tc.cu for Poisson, the D = 32 ones on the tile pipeline
// of glm_tc_common.cuh, and glm_finish_kernel of glm.cu for all three) with their particle axis set to the chains, so X is read once per
// evaluation for every chain together.  One evaluation is a fixed launch sequence with no host sync (CUDA
// graph capturable):
//   1. glm_potential_pack_kernel    z's weight / bias columns -> the contiguous [C, K*D] / [C, K] operands
//                                   (z's rows also hold the other site, so their stride is not the kernels')
//   2. the GLM kernel + its finish  weight = -1: dW, db are d(-loglik)/dW, d(-loglik)/db; sum_p = loglik
//   3. glm_potential_finish_kernel  adds the Normal prior value and gradient, one warp per chain, fp64
//                                   accumulation in a fixed order, and writes U and grad
// The GLM kernels always run with B2_FLAG_GLM_3XTF32 here: every logit is fp32-exact, so the sampler
// targets the posterior of the data as given, not of X rounded to TF32.
#include <math.h>

#include "b2_common.cuh"

namespace b2 {

__global__ void __launch_bounds__(256) glm_potential_pack_kernel(const float* __restrict__ z, int64_t C,
                                                                 int64_t Dz, int64_t w_off, int64_t b_off,
                                                                 int KD, int Kb, float* __restrict__ Wp,
                                                                 float* __restrict__ bp) {
  const int64_t per = KD + Kb;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * per) return;
  const int64_t c = i / per;
  const int64_t j = i - c * per;
  if (j < KD) Wp[c * KD + j] = z[c * Dz + w_off + j];
  else bp[c * Kb + (j - KD)] = z[c * Dz + b_off + (j - KD)];
}

__global__ void __launch_bounds__(256) glm_potential_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const double iw = 1.0 / (s_w * s_w);
  const double ib = Kb ? 1.0 / (s_b * s_b) : 0.0;
  const float* zc = z + c * Dz;
  float* gc = grad + c * Dz;
  double qw = 0.0, qb = 0.0;  // SUM w^2 / s_w^2, SUM b^2 / s_b^2
  for (int j = lane; j < KD; j += 32) {
    const double v = (double)zc[w_off + j];
    qw += v * v * iw;
    gc[w_off + j] = (float)((double)dW[c * KD + j] + v * iw);
  }
  for (int j = lane; j < Kb; j += 32) {
    const double v = (double)zc[b_off + j];
    qb += v * v * ib;
    gc[b_off + j] = (float)((double)db[c * Kb + j] + v * ib);
  }
  qw = warp_sum(qw);
  qb = warp_sum(qb);
  if (lane == 0) {
    constexpr double kHalfLog2Pi = 0.91893853320467274178;
    double u = -(double)sum_p[c] + 0.5 * qw + (double)KD * (log(s_w) + kHalfLog2Pi);
    if (Kb) u += 0.5 * qb + (double)Kb * (log(s_b) + kHalfLog2Pi);
    U[c] = (float)u;
  }
}

// workspace areas, each 256-byte aligned: [GLM kernel workspace][Wp][bp][dW][db][sum_p]
struct GlmPotentialLayout {
  size_t glm, wp, bp, dw, db, sum_p, total;
};

inline size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }

inline GlmPotentialLayout glm_potential_layout(int kind, int64_t N, int D, int K, int64_t C) {
  GlmPotentialLayout L;
  const size_t KD = (size_t)K * D, c = (size_t)C;
  L.glm = 0;
  size_t off = round256(kind == B2_GLM_BERNOULLI ? b2_glm_workspace(N, D, (int)C)
                        : kind == B2_GLM_POISSON ? b2_glm_poisson_workspace(N, D, (int)C)
                                                 : b2_glm_categorical_workspace(N, D, K, (int)C));
  L.wp = off; off += round256(c * KD * sizeof(float));
  L.bp = off; off += round256(c * K * sizeof(float));
  L.dw = off; off += round256(c * KD * sizeof(float));
  L.db = off; off += round256(c * K * sizeof(float));
  L.sum_p = off; off += round256(c * sizeof(float));
  L.total = off;
  return L;
}

inline bool glm_potential_in_scope(int kind, int64_t N, int D, int K, int64_t C) {
  if (N < 1 || C < 1 || C >= ((int64_t)1 << 31)) return false;
  if (kind == B2_GLM_BERNOULLI) return K == 1 && (D == 4 || D == 8 || D == 16 || D == 32);
  if (kind == B2_GLM_CATEGORICAL) return D == 32 && K >= 2 && K <= 16;
  if (kind == B2_GLM_POISSON) return K == 1 && D >= 1 && D <= 128;
  return false;
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_potential_workspace(int kind, int64_t N, int D, int K, int64_t C) {
  if (!glm_potential_in_scope(kind, N, D, K, C)) return 256;
  return glm_potential_layout(kind, N, D, K, C).total;
}

extern "C" int b2_glm_potential(int kind, const float* X, const void* y, int64_t N, int D, int K, int has_bias,
                                const float* z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, double s_w,
                                double s_b, float* U, float* grad, void* workspace, size_t workspace_bytes,
                                void* stream) {
  if (!X || !y || !z || !U || !grad) return B2_ERR_NULL;
  if (!glm_potential_in_scope(kind, N, D, K, C)) return B2_ERR_BAD_SHAPE;
  const int KD = K * D, Kb = has_bias ? K : 0;
  // z's row is exactly the weight block and the bias block, neither overlapping nor out of the row
  if (Dz != (int64_t)KD + Kb || w_off < 0 || w_off + KD > Dz) return B2_ERR_BAD_SHAPE;
  if (has_bias && (b_off < 0 || b_off + Kb > Dz || (b_off < w_off + KD && w_off < b_off + Kb)))
    return B2_ERR_BAD_SHAPE;
  if (!(s_w > 0.0) || (has_bias && !(s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  const GlmPotentialLayout L = glm_potential_layout(kind, N, D, K, C);
  if (!workspace || workspace_bytes < L.total) return B2_ERR_WORKSPACE;
  char* ws = reinterpret_cast<char*>(workspace);
  float* Wp = reinterpret_cast<float*>(ws + L.wp);
  float* bp = has_bias ? reinterpret_cast<float*>(ws + L.bp) : nullptr;
  float* dW = reinterpret_cast<float*>(ws + L.dw);
  float* db = has_bias ? reinterpret_cast<float*>(ws + L.db) : nullptr;
  float* sum_p = reinterpret_cast<float*>(ws + L.sum_p);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  const int64_t npack = C * (KD + Kb);
  glm_potential_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(z, C, Dz, w_off, b_off, KD, Kb, Wp, bp);
  count_launch(1);
  int rc = check_launch();
  if (rc != 0) return rc;
  const size_t glm_bytes = L.wp - L.glm;
  if (kind == B2_GLM_BERNOULLI)
    rc = b2_glm_bernoulli_logits(X, static_cast<const float*>(y), Wp, bp, N, D, (int)C, 1.0, -1.0, 1.0,
                                 B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws + L.glm, glm_bytes, stream);
  else if (kind == B2_GLM_POISSON)
    rc = b2_glm_poisson_log_rate(X, static_cast<const float*>(y), Wp, bp, N, D, (int)C, 1.0, -1.0, 1.0,
                                 B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws + L.glm, glm_bytes, stream);
  else
    rc = b2_glm_categorical_logits(X, static_cast<const int64_t*>(y), Wp, bp, N, D, K, (int)C, 1.0, -1.0, 1.0,
                                   B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws + L.glm, glm_bytes, stream);
  if (rc != 0) return rc;
  glm_potential_finish_kernel<<<(unsigned)((C * 32 + 255) / 256), 256, 0, s>>>(
      z, C, Dz, w_off, b_off, KD, Kb, s_w, s_b, sum_p, dW, db, U, grad);
  count_launch(1);
  return check_launch();
}
