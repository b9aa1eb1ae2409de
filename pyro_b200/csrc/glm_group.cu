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
// Past 128 columns (b2_glm_group_gather_sum, rows sorted by group, G <= 65536) the group effect is gathered instead
// (glm_flat_tc.cuh GATHER, glm_group_gather_tc.cu): four launches with no host sync,
//   1. glm_group_gather_sum_pack_kernel    W's rows into Wp [P][D], the group-major tables tab [1 + S][G][cp] of
//                                          alpha and beta_k, and gsum zeroed
//   2. the kind's gather kernel            Bernoulli, Poisson, Normal: X split
//   3. glm_finish_kernel                   D wide, with the caller's scale, weight, sum_coeff and flags
//   4. glm_group_gather_sum_finish_kernel  each group's run sums (gsum, and the slots of the runs that cross the
//                                          kernel's ranges) times the finish's factor into out_dT [1 + S][P][G]
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

// b2_glm_group_gather_sum's pack: blocks [0, nbw) write Wp [P][D] from W's rows; each later block one tile of the
// group-major tables, tab[k][a][c] = the value of group a in table k (alpha for k = 0, else beta_k) for particle c
// (0 for c >= P, a stride-0 table shared by every particle), 32 groups by 64 particles read along a and written
// along c through shared memory, and the same tile of gsum zeroed (every call: a graph replay needs it too).
__global__ void __launch_bounds__(256)
glm_group_gather_sum_pack_kernel(const float* __restrict__ W, int64_t w_stride, const float* __restrict__ alpha,
                                 int64_t a_stride, b2_glm_slope_tables sl, int P, int D, int G, int cp, int nbw,
                                 float* __restrict__ Wp, float* __restrict__ tab, float* __restrict__ gsum) {
  if ((int)blockIdx.x < nbw) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)P * D) return;
    const int64_t p = i / D;
    Wp[i] = W[p * w_stride + (i - p * D)];
    return;
  }
  __shared__ float tr[64][33];
  const int ga = (G + 31) / 32, gc = cp / 64;
  const int b = (int)blockIdx.x - nbw, k = b / (ga * gc), r = b - k * ga * gc, a0 = (r / gc) * 32, c0 = (r % gc) * 64;
  // table k, chosen by selects (an indexed read of the parameter struct needs a stack frame)
  const float* t = k == 0 ? alpha : k == 1 ? sl.beta[0] : k == 2 ? sl.beta[1] : sl.beta[2];
  const int64_t st = k == 0 ? a_stride : k == 1 ? sl.beta_stride[0] : k == 2 ? sl.beta_stride[1] : sl.beta_stride[2];
#pragma unroll
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int c = i >> 5, a = i & 31;
    tr[c][a] = c0 + c < P && a0 + a < G ? t[(int64_t)(c0 + c) * st + a0 + a] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int a = i >> 6, c = i & 63;
    if (a0 + a < G) {
      const int64_t e = ((int64_t)k * G + a0 + a) * cp + c0 + c;
      tab[e] = tr[c][a];
      gsum[e] = 0.f;
    }
  }
}

// b2_glm_group_gather_sum's group finish: CTA (x, y, z) writes out_dT[k][c][g] for table k = z, the 32 groups from
// g0 = 32 x and the 64 particles from c0 = 64 y.  Warp w takes groups g0 + 4w .. g0 + 4w + 3, lanes particles c0 +
// lane and c0 + lane + 32, so every read of gsum and of a slot is 32 consecutive floats.  A group's value is its gsum
// entry plus, in slot (row) order and fp64, every slot that carries its key: the warp finds its first slot by a
// 32-way search on the slot orders, then takes the slots 32 keys at a time until one orders past its groups.  Times
// fac (weight * scale) and 1 / sigma_c^2 (Normal) as glm_finish_kernel scales dW, transposed through shared memory,
// and written along g.  Any nonzero status makes every value NaN, and CTA 0 sets out_total and out_sum_p to NaN
// (this kernel runs after glm_finish_kernel, which wrote them).
__global__ void __launch_bounds__(256)
glm_group_gather_sum_finish_kernel(const GlmGatherFinish gf, int G, int P, const float* __restrict__ sigma,
                                   int sigma_stride, double fac, float* __restrict__ out_dT,
                                   float* __restrict__ out_total, float* __restrict__ out_sum_p) {
  constexpr unsigned kAll = 0xffffffffu;
  const float kNaN = __int_as_float(0x7fc00000);
  __shared__ float tr[64][33];
  const int k = blockIdx.z, g0 = blockIdx.x * 32, c0 = blockIdx.y * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int st = 0;
  for (int q = threadIdx.x; q < gf.Q; q += 256) st |= gf.status[q];
  const bool bad = __syncthreads_or(st) != 0;
  if (bad && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    if (threadIdx.x == 0 && out_total) *out_total = kNaN;
    if (out_sum_p)
      for (int p = threadIdx.x; p < P; p += 256) out_sum_p[p] = kNaN;
  }
  const int gw = g0 + 4 * warp;
  double acc[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      acc[j][h] = !bad && gw + j < G ? (double)gf.gsum[((int64_t)k * G + gw + j) * gf.cp + c0 + lane + 32 * h] : 0.0;
  if (!bad && gw < G) {
    const int64_t ntiles = (gf.N + 63) / 64;
    const int ne = 2 * gf.Q;
    // the first slot whose order is >= gw lies in [lo, hi]; each round narrows that to one of 32 steps
    int lo = 0, hi = ne;
    while (lo < hi) {
      const int step = (hi - lo + 31) >> 5;
      const int e = min(lo + (lane + 1) * step - 1, hi - 1);
      const unsigned m = __ballot_sync(kAll, gather_slot_order(gf, e, ntiles) >= gw);
      if (m == 0) {
        lo = hi;
      } else {
        const int j = __ffs(m) - 1;
        hi = min(lo + (j + 1) * step - 1, hi - 1);
        lo += j * step;
      }
    }
    for (int e0 = hi; e0 < ne; e0 += 32) {
      const int e = e0 + lane;
      const bool in = e < ne && gather_slot_order(gf, e, ntiles) < gw + 4;
      const int key = in ? gather_slot_key(gf, e, ntiles) : -1;
      const unsigned m = ~__ballot_sync(kAll, in);
      const int n = m ? __ffs(m) - 1 : 32;     // the slots e0 .. e0 + n - 1 order within the warp's groups
      for (int i = 0; i < n; ++i) {
        const int j = __shfl_sync(kAll, key, i) - gw;
        if ((unsigned)j < 4u) {
          const float* sv = gf.slots + ((int64_t)(e0 + i) * 4 + k) * gf.cp + c0 + lane;
          const double v0 = (double)sv[0], v1 = (double)sv[32];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            if (j == jj) {
              acc[jj][0] += v0;
              acc[jj][1] += v1;
            }
        }
      }
      if (n < 32) break;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int p = lane + 32 * h, c = c0 + p;
    double f = fac;
    if (sigma != nullptr && c < P) {
      const double sg = (double)sigma[(int64_t)c * sigma_stride];
      f = fac * (1.0 / (sg * sg));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) tr[p][4 * warp + j] = bad ? kNaN : (float)(f * acc[j][h]);
  }
  __syncthreads();
#pragma unroll
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int p = i >> 5, gl = i & 31;
    if (c0 + p < P && g0 + gl < G) out_dT[((int64_t)k * P + c0 + p) * G + g0 + gl] = tr[p][gl];
  }
}

inline bool glm_group_sum_kind(int kind) {
  return kind == B2_GLM_BERNOULLI || kind == B2_GLM_POISSON || kind == B2_GLM_NORMAL || kind == B2_GLM_BINOMIAL;
}

// workspace: [the likelihood call's workspace, D + G wide][Wp [P][D + G]], each 256-byte aligned
inline size_t glm_group_sum_lik_bytes(int kind, int64_t N, int Da, int P) {
  const size_t b = kind == B2_GLM_BERNOULLI ? b2_glm_workspace(N, Da, P) : glm_row_workspace(N, Da, P);
  return (b + 255) & ~(size_t)255;
}

// b2_glm_group_gather_sum's workspace, each area 256-byte aligned: [glm_row_workspace(N, D, P)][Wp P x D]
// [tab (1 + S) G cp][gsum (1 + S) G cp][slots Q 2 4 cp][status Q], cp = P rounded up to 64 and Q the gather kernel's
// ranges (glm_gather_ranges, the dispatch that launches it)
struct GlmGatherSumLayout {
  size_t wp, tab, gsum, slots, status, total;
  int cp, Q;
};

inline GlmGatherSumLayout glm_gather_sum_layout(int64_t N, int D, int G, int S, int P) {
  auto r256 = [](size_t b) { return (b + 255) & ~(size_t)255; };
  GlmGatherSumLayout L;
  L.cp = (P + 63) / 64 * 64;
  L.Q = glm_gather_ranges(N, D);
  const size_t table = (size_t)(1 + S) * G * L.cp * sizeof(float);
  size_t off = r256(glm_row_workspace(N, D, P));
  L.wp = off; off += r256((size_t)P * D * sizeof(float));
  L.tab = off; off += r256(table);
  L.gsum = off; off += r256(table);
  L.slots = off; off += r256((size_t)L.Q * 2 * 4 * L.cp * sizeof(float));
  L.status = off; off += r256((size_t)L.Q * sizeof(int));
  L.total = off;
  return L;
}

inline bool glm_gather_sum_kind(int kind) {
  return kind == B2_GLM_BERNOULLI || kind == B2_GLM_POISSON || kind == B2_GLM_NORMAL;
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

extern "C" size_t b2_glm_group_gather_sum_workspace(int kind, int64_t N, int D, int G, int S, int P) {
  if (!glm_gather_sum_kind(kind) || N < 1 || N >= ((int64_t)1 << 31) || D < 1 || D > 128 || G < 1 || G > 65536 ||
      S < 0 || S > 3 || P < 1)
    return 256;
  return glm_gather_sum_layout(N, D, G, S, P).total;
}

extern "C" int b2_glm_group_gather_sum(int kind, const float* X, const float* y, const float* sigma, int sigma_stride,
                                       const int32_t* groups, int G, const float* W, int64_t w_stride,
                                       const float* alpha, int64_t alpha_stride, const b2_glm_slope_tables* slopes,
                                       const float* b, int64_t N, int D, int P, double scale, double weight,
                                       double sum_coeff, int flags, float* out_sum_p, float* out_total,
                                       float* out_dW, float* out_db, float* out_dsigma, float* out_dT,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  if (!X || !y || !groups || !W || !alpha || !out_dT) return B2_ERR_NULL;
  if (kind == B2_GLM_NORMAL && !sigma) return B2_ERR_NULL;
  b2_glm_slope_tables sl = {};
  if (slopes) {
    sl = *slopes;
    if (sl.S < 0 || sl.S > 3) return B2_ERR_BAD_SHAPE;
    for (int k = 0; k < sl.S; ++k)
      if (!sl.beta[k]) return B2_ERR_NULL;
  }
  if (!glm_gather_sum_kind(kind)) return B2_ERR_BAD_SHAPE;   // Binomial and Categorical have no gather kernel
  if (N <= 0 || P <= 0 || D < 1 || D > 128 || G < 1 || G > 65536) return B2_ERR_BAD_SHAPE;
  if ((w_stride != 0 && w_stride < D) || (alpha_stride != 0 && alpha_stride < G)) return B2_ERR_BAD_SHAPE;
  for (int k = 0; k < sl.S; ++k) {
    if (sl.col[k] < 0 || sl.col[k] >= D || (sl.beta_stride[k] != 0 && sl.beta_stride[k] < G)) return B2_ERR_BAD_SHAPE;
    for (int j = 0; j < k; ++j)
      if (sl.col[j] == sl.col[k]) return B2_ERR_BAD_SHAPE;
  }
  if (kind == B2_GLM_NORMAL && sigma_stride != 0 && sigma_stride != 1) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(groups) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (flags & B2_FLAG_GLM_FP32) return B2_ERR_BAD_SHAPE;   // the gather kernels are tensor-core only
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_glm_group_gather_sum_workspace(kind, N, D, G, sl.S, P))
    return B2_ERR_WORKSPACE;

  const GlmGatherSumLayout L = glm_gather_sum_layout(N, D, G, sl.S, P);
  char* ws = reinterpret_cast<char*>(workspace);
  float* Wp = reinterpret_cast<float*>(ws + L.wp);
  GlmGather ga;
  ga.idx = groups;
  ga.G = G;
  ga.S = sl.S;
  for (int k = 0; k < sl.S; ++k) ga.col[k] = sl.col[k];
  ga.cp = L.cp;
  float* tab = reinterpret_cast<float*>(ws + L.tab);
  ga.tab = tab;
  ga.gsum = reinterpret_cast<float*>(ws + L.gsum);
  ga.slots = reinterpret_cast<float*>(ws + L.slots);
  ga.status = reinterpret_cast<int*>(ws + L.status);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int nbw = (int)(((int64_t)P * D + 255) / 256);
  const int nbt = (1 + sl.S) * ((G + 31) / 32) * (L.cp / 64);
  glm_group_gather_sum_pack_kernel<<<(unsigned)(nbw + nbt), 256, 0, s>>>(W, w_stride, alpha, alpha_stride, sl, P, D,
                                                                         G, L.cp, nbw, Wp, tab, ga.gsum);
  count_launch(1);
  int rc = check_launch();
  if (rc != 0) return rc;
  const bool normal = kind == B2_GLM_NORMAL;
  rc = glm_gather_likelihood(kind, X, y, Wp, b, normal ? sigma : nullptr, sigma_stride, normal ? out_dsigma : nullptr,
                             N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW, out_db, ws, s, ga);
  if (rc != 0) return rc;
  const GlmGatherFinish gf = {ga.gsum, ga.slots, ga.status, groups, L.cp, L.Q, N};
  glm_group_gather_sum_finish_kernel<<<dim3((unsigned)((G + 31) / 32), (unsigned)(L.cp / 64), (unsigned)(1 + sl.S)),
                                       256, 0, s>>>(gf, G, P, normal ? sigma : nullptr, sigma_stride, weight * scale,
                                                    out_dT, out_total, out_sum_p);
  count_launch(1);
  return check_launch();
}
