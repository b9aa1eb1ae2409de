// glm_group.cu -- the site sum of a regression with a varying intercept by group, for P particles (SVI):
//   eta[p,n] = <X[n,:], W[p,:]> + b[p] + alpha[p, g[n]]
// scored by one pass of the kind's fused likelihood kernel over [X | onehot(g)] (glm_flat_tc.cuh GROUPS): the
// group effect is G more columns of the contraction, so X is read once and no [P, N] tensor is written, and the
// extra columns D .. D+G-1 of dW are d/dalpha.  Three launches with no host sync (CUDA graph capturable):
//   1. glm_group_sum_pack_kernel   each particle's [w | alpha] row into the workspace (a stride-0 operand is
//                                  shared by every particle)
//   2. the kind's group kernel     Bernoulli, Poisson, Binomial: X split or rounded to TF32 by glm_split_x, as their
//                                  plain kernels; Normal: X split
//   3. glm_finish_kernel           D + G wide
// With S varying slopes by group as well (b2_glm_group_slope_sum),
//   eta[p,n] = <X[n,:], W[p,:]> + b[p] + alpha[p, g[n]] + SUM_k beta_k[p, g[n]] X[n, c_k]
// is the same pass over [X | onehot(g) | X[:, c_1] onehot(g) | ..] (glm_flat_tc.cuh SLOPES), D + G (1 + S) columns
// whose last S G columns of dW are d/dbeta_k; glm_group_slope_pack_kernel packs [w | alpha | beta_1 .. beta_S] and
// the slope kernels take the group kernels' place, with the same precision policy.
// The group and slope kernels with X rounded to TF32 (glm_group_rn_tc_kernel, glm_group_slope_rn_tc_kernel) live
// here; the X-split ones, which the potentials use too, stay with their families.
#include <cuda.h>

#include "b2_common.cuh"
#include "glm_flat_tc.cuh"
#include "glm_host.cuh"

namespace b2 {

// glm_flat_pipeline with a group effect (D + G columns), X rounded to nearest TF32 (SPLIT_X = false): the one-hot
// columns are exact in TF32 either way.  trials: Binomial's counts, null for the other families.
template <class Fam, int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_group_rn_tc_kernel(const float* __restrict__ X, const float* __restrict__ y, const float* __restrict__ trials,
                       const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int D, int P,
                       float* __restrict__ partials, const int32_t* __restrict__ groups, int G) {
  tcf::glm_flat_pipeline<Fam, DC, false, true>(X, y, W, bvec, N, D, P, partials, trials, GlmGroups{groups, G});
}

// with varying slopes as well (grp.S > 0): D + G (1 + S) columns, X and the slope columns (X's own values) rounded
// to nearest TF32
template <class Fam, int DC>
__global__ void __launch_bounds__(tcf::Cfg<DC, true>::kThreads, 1)
glm_group_slope_rn_tc_kernel(const float* __restrict__ X, const float* __restrict__ y,
                             const float* __restrict__ trials, const float* __restrict__ W,
                             const float* __restrict__ bvec, int64_t N, int D, int P, float* __restrict__ partials,
                             GlmGroups grp) {
  tcf::glm_flat_pipeline<Fam, DC, false, true, true>(X, y, W, bvec, N, D, P, partials, trials, grp);
}

// MinDC: Binomial runs D + G (1 + S) < 32 on the two-atom loop, as its plain kernels do (glm_binomial_tc.cu)
template <class Fam, int MinDC>
int launch_group_rn(const float* X, const float* y, const float* m, const float* W, const float* b, int64_t N, int D,
                    int P, float* partials, int gx, cudaStream_t s, GlmGroups grp) {
  return glm_dispatch_dc<MinDC>(D + grp.cols(), false, [&](auto dc, auto) {
    using C = tcf::Cfg<decltype(dc)::value, true>;
    constexpr int kDC = decltype(dc)::value;
    if (grp.S)
      return launch_tc(glm_group_slope_rn_tc_kernel<Fam, kDC>, tc::slab_grid(gx, P), dim3(C::kThreads),
                       C::kSmemBytes, s, X, y, m, W, b, N, D, P, partials, grp);
    return launch_tc(glm_group_rn_tc_kernel<Fam, kDC>, tc::slab_grid(gx, P), dim3(C::kThreads), C::kSmemBytes, s, X,
                     y, m, W, b, N, D, P, partials, grp.idx, grp.G);
  });
}

int launch_glm_group_rn(int kind, const float* X, const float* y, const float* m, bool row_trials, const float* W,
                        const float* b, int64_t N, int D, int P, float* partials, int gx, cudaStream_t s,
                        GlmGroups grp) {
  switch (kind) {
    case B2_GLM_BERNOULLI: return launch_group_rn<tc::Bernoulli, 1>(X, y, m, W, b, N, D, P, partials, gx, s, grp);
    case B2_GLM_POISSON: return launch_group_rn<tc::Poisson, 1>(X, y, m, W, b, N, D, P, partials, gx, s, grp);
    case B2_GLM_BINOMIAL:
      return row_trials ? launch_group_rn<tc::Binomial<true>, 2>(X, y, m, W, b, N, D, P, partials, gx, s, grp)
                        : launch_group_rn<tc::Binomial<false>, 2>(X, y, m, W, b, N, D, P, partials, gx, s, grp);
    default: return B2_ERR_BAD_SHAPE;
  }
}

__global__ void __launch_bounds__(256) glm_group_sum_pack_kernel(const float* __restrict__ W, int64_t w_stride,
                                                                 const float* __restrict__ alpha, int64_t a_stride,
                                                                 int P, int D, int G, float* __restrict__ Wp) {
  const int Da = D + G;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)P * Da) return;
  const int64_t p = i / Da;
  const int j = (int)(i - p * Da);
  Wp[i] = j < D ? W[p * w_stride + j] : alpha[p * a_stride + (j - D)];
}

// [w | alpha | beta_1 .. beta_S] per particle: the S = 0 layout of glm_group_sum_pack_kernel with the slope tables
// after alpha (a stride-0 table is shared by every particle)
__global__ void __launch_bounds__(256)
glm_group_slope_pack_kernel(const float* __restrict__ W, int64_t w_stride, const float* __restrict__ alpha,
                            int64_t a_stride, b2_glm_slope_tables sl, int P, int D, int G, float* __restrict__ Wp) {
  const int Da = D + G * (1 + sl.S);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)P * Da) return;
  const int64_t p = i / Da;
  const int j = (int)(i - p * Da);
  if (j < D) {
    Wp[i] = W[p * w_stride + j];
    return;
  }
  // block k: alpha (k = 0) or beta_k, chosen by selects (an indexed read of the parameter struct needs a stack frame)
  const int k = (j - D) / G, jg = j - D - k * G;
  const float* t = k == 0 ? alpha : k == 1 ? sl.beta[0] : k == 2 ? sl.beta[1] : sl.beta[2];
  const int64_t st = k == 0 ? a_stride : k == 1 ? sl.beta_stride[0] : k == 2 ? sl.beta_stride[1] : sl.beta_stride[2];
  Wp[i] = t[p * st + jg];
}

inline bool glm_group_sum_kind(int kind) {
  return kind == B2_GLM_BERNOULLI || kind == B2_GLM_POISSON || kind == B2_GLM_NORMAL || kind == B2_GLM_BINOMIAL;
}

// workspace: [the likelihood call's workspace, D + G wide][Wp [P][D + G]], each 256-byte aligned
inline size_t glm_group_sum_lik_bytes(int kind, int64_t N, int Da, int P) {
  const size_t b = kind == B2_GLM_BERNOULLI ? b2_glm_workspace(N, Da, P) : glm_row_workspace(N, Da, P);
  return (b + 255) & ~(size_t)255;
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_group_sum_workspace(int kind, int64_t N, int D, int G, int P) {
  if (!glm_group_sum_kind(kind) || N < 1 || D < 1 || G < 1 || D + G > 128 || P < 1) return 256;
  const int Da = D + G;
  return glm_group_sum_lik_bytes(kind, N, Da, P) + (((size_t)P * Da * sizeof(float) + 255) & ~(size_t)255);
}

extern "C" size_t b2_glm_group_slope_sum_workspace(int kind, int64_t N, int D, int G, int S, int P) {
  if (!glm_group_sum_kind(kind) || N < 1 || D < 1 || G < 1 || S < 1 || S > 3 || P < 1 || D + G * (1 + S) > 128)
    return 256;
  const int Da = D + G * (1 + S);
  return glm_group_sum_lik_bytes(kind, N, Da, P) + (((size_t)P * Da * sizeof(float) + 255) & ~(size_t)255);
}

extern "C" int b2_glm_group_sum(int kind, const float* X, const float* y, const float* trials, int trials_per_row,
                                const float* sigma, int sigma_stride, const int32_t* groups, int G, const float* W,
                                int64_t w_stride, const float* alpha, int64_t alpha_stride, const float* b, int64_t N,
                                int D, int P, double scale, double weight, double sum_coeff, int flags,
                                float* out_sum_p, float* out_total, float* out_dW, float* out_db, float* out_dsigma,
                                void* workspace, size_t workspace_bytes, void* stream) {
  if (!X || !y || !groups || !W || !alpha) return B2_ERR_NULL;
  if ((kind == B2_GLM_BINOMIAL && !trials) || (kind == B2_GLM_NORMAL && !sigma)) return B2_ERR_NULL;
  if (!glm_group_sum_kind(kind)) return B2_ERR_BAD_SHAPE;
  if (N <= 0 || P <= 0 || D < 1 || G < 1 || D + G > 128) return B2_ERR_BAD_SHAPE;
  if ((w_stride != 0 && w_stride < D) || (alpha_stride != 0 && alpha_stride < G)) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_NORMAL && sigma_stride != 0 && sigma_stride != 1) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row != 0 && trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(groups) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (flags & B2_FLAG_GLM_FP32) return B2_ERR_BAD_SHAPE;   // the group kernels are tensor-core only
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_glm_group_sum_workspace(kind, N, D, G, P)) return B2_ERR_WORKSPACE;

  const int Da = D + G;
  const size_t lik_bytes = glm_group_sum_lik_bytes(kind, N, Da, P);
  float* Wp = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + lik_bytes);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int64_t npack = (int64_t)P * Da;
  glm_group_sum_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(W, w_stride, alpha, alpha_stride, P, D,
                                                                            G, Wp);
  count_launch(1);
  int rc = check_launch();
  if (rc != 0) return rc;
  GlmGroups grp;
  grp.idx = groups;
  grp.G = G;
  switch (kind) {
    case B2_GLM_BERNOULLI:
      return glm_bernoulli_logits(X, y, Wp, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                                  out_db, workspace, lik_bytes, s, grp);
    case B2_GLM_POISSON:
      return glm_poisson_log_rate(X, y, Wp, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                                  out_db, workspace, lik_bytes, s, grp);
    case B2_GLM_NORMAL:
      return glm_normal_loc(X, y, Wp, b, sigma, sigma_stride, N, D, P, scale, weight, sum_coeff, flags, out_sum_p,
                            out_total, out_dW, out_db, out_dsigma, workspace, lik_bytes, s, grp);
    default:
      return glm_binomial_logits(X, y, trials, trials_per_row, Wp, b, N, D, P, scale, weight, sum_coeff, flags,
                                 out_sum_p, out_total, out_dW, out_db, workspace, lik_bytes, s, grp);
  }
}

extern "C" int b2_glm_group_slope_sum(int kind, const float* X, const float* y, const float* trials,
                                      int trials_per_row, const float* sigma, int sigma_stride,
                                      const int32_t* groups, int G, const float* W, int64_t w_stride,
                                      const float* alpha, int64_t alpha_stride, const b2_glm_slope_tables* slopes,
                                      const float* b, int64_t N, int D, int P, double scale, double weight,
                                      double sum_coeff, int flags, float* out_sum_p, float* out_total, float* out_dW,
                                      float* out_db, float* out_dsigma, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  if (!X || !y || !groups || !W || !alpha || !slopes) return B2_ERR_NULL;
  if ((kind == B2_GLM_BINOMIAL && !trials) || (kind == B2_GLM_NORMAL && !sigma)) return B2_ERR_NULL;
  const b2_glm_slope_tables sl = *slopes;
  if (sl.S < 1 || sl.S > 3) return B2_ERR_BAD_SHAPE;
  for (int k = 0; k < sl.S; ++k)
    if (!sl.beta[k]) return B2_ERR_NULL;
  if (!glm_group_sum_kind(kind)) return B2_ERR_BAD_SHAPE;
  if (N <= 0 || P <= 0 || D < 1 || G < 1 || D + G * (1 + sl.S) > 128) return B2_ERR_BAD_SHAPE;
  if ((w_stride != 0 && w_stride < D) || (alpha_stride != 0 && alpha_stride < G)) return B2_ERR_BAD_SHAPE;
  for (int k = 0; k < sl.S; ++k) {
    if (sl.col[k] < 0 || sl.col[k] >= D || (sl.beta_stride[k] != 0 && sl.beta_stride[k] < G)) return B2_ERR_BAD_SHAPE;
    for (int j = 0; j < k; ++j)
      if (sl.col[j] == sl.col[k]) return B2_ERR_BAD_SHAPE;
  }
  if (kind == B2_GLM_NORMAL && sigma_stride != 0 && sigma_stride != 1) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row != 0 && trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(groups) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (flags & B2_FLAG_GLM_FP32) return B2_ERR_BAD_SHAPE;   // the slope kernels are tensor-core only
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_glm_group_slope_sum_workspace(kind, N, D, G, sl.S, P))
    return B2_ERR_WORKSPACE;

  const int Da = D + G * (1 + sl.S);
  const size_t lik_bytes = glm_group_sum_lik_bytes(kind, N, Da, P);
  float* Wp = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + lik_bytes);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int64_t npack = (int64_t)P * Da;
  glm_group_slope_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(W, w_stride, alpha, alpha_stride, sl,
                                                                              P, D, G, Wp);
  count_launch(1);
  int rc = check_launch();
  if (rc != 0) return rc;
  GlmGroups grp;
  grp.idx = groups;
  grp.G = G;
  grp.S = sl.S;
  for (int k = 0; k < sl.S; ++k) grp.col[k] = sl.col[k];
  switch (kind) {
    case B2_GLM_BERNOULLI:
      return glm_bernoulli_logits(X, y, Wp, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                                  out_db, workspace, lik_bytes, s, grp);
    case B2_GLM_POISSON:
      return glm_poisson_log_rate(X, y, Wp, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                                  out_db, workspace, lik_bytes, s, grp);
    case B2_GLM_NORMAL:
      return glm_normal_loc(X, y, Wp, b, sigma, sigma_stride, N, D, P, scale, weight, sum_coeff, flags, out_sum_p,
                            out_total, out_dW, out_db, out_dsigma, workspace, lik_bytes, s, grp);
    default:
      return glm_binomial_logits(X, y, trials, trials_per_row, Wp, b, N, D, P, scale, weight, sum_coeff, flags,
                                 out_sum_p, out_total, out_dW, out_db, workspace, lik_bytes, s, grp);
  }
}
