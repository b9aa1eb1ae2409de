// glm_categorical_tc.cu -- Hopper fused softmax-regression likelihood kernel: one pass over X[N,32] and
// the labels y[N] gives, for P weight matrices W[p] in R^{K x 32} (2 <= K <= 16) and biases b[p] in R^K,
//   l[p,n,k]  = <x_n, W[p,k,:]> + b[p,k],   lse[p,n] = logsumexp_k l[p,n,k]
//   sum_p[p]  = SUM_n ( l[p,n,y_n] - lse[p,n] )                 (torch/distributions/categorical.py log_prob)
//   g[p,n,k]  = [k == y_n] - softmax_k(l[p,n,:])
//   dW[p,k,:] = weight * SUM_n g[p,n,k] x_n,     db[p,k] = weight * SUM_n g[p,n,k]
// It replaces the user model's `X @ W.mT + b`, Categorical(logits).log_prob, the site sum and the autograd
// backward of all three, which together write and re-read [P, N, K] tensors.
//
// The Bernoulli kernel of glm_tc.cu with a class axis: both run the D = 32 tile pipeline of glm_tc_common.cuh
// with the same precision policy and determinism argument (see glm_tc.cu), and glm_finish_kernel (glm.cu)
// adds the CTA partials.  This file gives the softmax family of the pipeline.  What differs:
//
//   rows     the 64 rows of GEMM 1's M slab are (particle, class) pairs: each particle's K classes take KP
//            consecutive rows, KP = the next power of two >= K in {2, 4, 8, 16}, so a slab holds 64 / KP
//            particles.  Padding rows (class >= K, or a particle past P) have zero weights and bias.
//   softmax  wgmma fragment row m = 16 w4 + gid + 8h and 16 % KP == 0, so a thread's class is
//            (gid + 8h) % KP: the logsumexp of a column is an in-thread pair (KP = 16) plus log2(min(KP, 8))
//            shfl.xor steps over lanes 4 / 8 / 16.  Padding classes enter the max as -inf, so their
//            exponential is exactly 0 and so is their g: they add nothing to any sum or gradient.
//   labels   int64, TMA-loaded next to the X tile.  The thread that owns class y_n of a column adds l[y_n];
//            the class-0 thread subtracts lse once per (particle, row), or adds NaN when y_n is outside
//            [0, K).  A label is only ever compared, never used as an index.
//   slabs    P * KP > 64 takes several slabs (blockIdx.y).  The grid is sized so that every slab is resident
//            at once and all walk the X tiles in the same order: X comes from HBM about once and the other
//            slabs read it from L2.
//
// MUFU work: every thread issues one ex2 per logit it holds and one rcp and one lg2 per (particle, row) it
// holds (the lg2 is issued by the whole warp, though only the class-0 lanes use it).  That is 2 MUFU ops per
// padded logit for KP = 16 (a thread's two rows are one particle) and 3 for KP <= 8: P * N * KP * (2 | 3).
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "glm_tc_common.cuh"

namespace b2 {

// launches glm_finish_kernel (glm.cu) over the partials [gx][P][K (D + 1) + 1]
void launch_glm_finish(const float* partials, unsigned int* ticket, int gx, int P, int K, int D, double scale,
                       double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                       float* out_dW, float* out_db, const float* lg, cudaStream_t s);

namespace tcc {

using namespace tc;
using namespace tc::tile32;

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// max / sum over the KP rows of one particle held by the lanes 4 gid + t4 of a warp (lane bits 2..4)
template <int KP>
__device__ __forceinline__ float class_max(float v) {
#pragma unroll
  for (int o = 4; o < 4 * (KP < 16 ? KP : 8); o <<= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int KP>
__device__ __forceinline__ float class_sum(float v) {
#pragma unroll
  for (int o = 4; o < 4 * (KP < 16 ? KP : 8); o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the softmax family of the D = 32 tile pipeline: KP GEMM 1 rows per particle, int64 labels
template <int KP>
struct Softmax {
  static_assert(KP == 2 || KP == 4 || KP == 8 || KP == 16, "class padding");
  static constexpr bool kBiasInEpilogue = false;
  static constexpr int kKP = KP;
  static constexpr uint32_t kYBytes = kRows * 8;  // 512 B of int64 labels
  static constexpr CUtensorMapDataType kYType = CU_TENSOR_MAP_DATA_TYPE_INT64;
  using Labels = int[16];                         // labels of the thread's rows n = 8j + 2 t4 + e, -1 outside [0, K)
  static __device__ __forceinline__ void read_labels(const uint8_t* ys, int t4, int K, Labels& yl) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const longlong2 v = reinterpret_cast<const longlong2*>(ys)[4 * j + t4];
      yl[2 * j] = ((unsigned long long)v.x < (unsigned long long)K) ? (int)v.x : -1;
      yl[2 * j + 1] = ((unsigned long long)v.y < (unsigned long long)K) ? (int)v.y : -1;
    }
  }
  // softmax over the class rows, lp sums and g, all in registers
  static __device__ __forceinline__ void epilogue(const float (&acc1)[32], const Labels& yl, const int (&cls)[2],
                                                  int K, int64_t row0, int64_t N, int t4, float (&lpa)[2],
                                                  uint32_t (&g)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float l[2][2], lm[2][2], mx[2][2], ex[2][2], sm_[2][2];
#pragma unroll
      for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          l[e][h] = acc1[4 * j + 2 * h + e];
          lm[e][h] = (cls[h] < K) ? l[e][h] : -INFINITY;
        }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (KP == 16) {
          mx[e][0] = mx[e][1] = class_max<KP>(fmaxf(lm[e][0], lm[e][1]));
        } else {
          mx[e][0] = class_max<KP>(lm[e][0]);
          mx[e][1] = class_max<KP>(lm[e][1]);
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int h = 0; h < 2; ++h) ex[e][h] = ex2f((lm[e][h] - mx[e][h]) * kLog2e);   // padding: ex2(-inf) = 0
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (KP == 16) {
          sm_[e][0] = sm_[e][1] = class_sum<KP>(ex[e][0] + ex[e][1]);
        } else {
          sm_[e][0] = class_sum<KP>(ex[e][0]);
          sm_[e][1] = class_sum<KP>(ex[e][1]);
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = yl[2 * j + e];
        const bool rv = row0 + 8 * j + 2 * t4 + e < N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float inv = rcpf(sm_[e][h]);
          const float gg = ((c == cls[h]) ? 1.f : 0.f) - ex[e][h] * inv;
          g[4 * j + 2 * h + e] = __float_as_uint(tf32_rn(rv ? gg : 0.f));
          float lp = (c == cls[h]) ? l[e][h] : 0.f;
          if (cls[h] == 0 && (KP < 16 || h == 0)) {
            const float lse = fmaf(lg2f(sm_[e][h]), kLn2, mx[e][h]);
            lp -= (c >= 0) ? lse : __int_as_float(0x7fffffff);
          }
          lpa[h] += rv ? lp : 0.f;
        }
      }
    }
  }
};

template <int KP, bool SPLIT_X>
__global__ void __launch_bounds__(kThreads, 1)
glm_categorical_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                          const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int P, int K,
                          float* __restrict__ partials) {
  glm_tile_pipeline<Softmax<KP>, SPLIT_X>(map_x, map_y, W, bvec, N, P, K, partials);
}

inline int class_pad(int K) { return K <= 2 ? 2 : K <= 4 ? 4 : K <= 8 ? 8 : 16; }

// CTAs per slab: every slab resident at once (one CTA per SM), at most one CTA per tile
inline int grid_x(int64_t N, int K, int P) {
  const int64_t ntiles = (N + kRows - 1) / kRows;
  const int slabs = (P + kM / class_pad(K) - 1) / (kM / class_pad(K));
  int64_t gx = kNumSMs / slabs;
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  return (int)gx;
}

template <int KP, bool SPLIT_X>
void launch(const CUtensorMap& mx, const CUtensorMap& my, const float* W, const float* b, int64_t N, int P, int K,
            float* partials, int gx, cudaStream_t s) {
  constexpr uint32_t kSmemBytes = Smem32<Softmax<KP>::kYBytes>::kBytes;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_categorical_tc_kernel<KP, SPLIT_X>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)kSmemBytes);
    attr_set = true;
  }
  constexpr int PPS = kM / KP;
  dim3 grid((unsigned)gx, (unsigned)((P + PPS - 1) / PPS), 1);
  launch_pdl(glm_categorical_tc_kernel<KP, SPLIT_X>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, W, b, N,
             P, K, partials);
}

template <bool SPLIT_X>
void launch_split(int KP, const CUtensorMap& mx, const CUtensorMap& my, const float* W, const float* b, int64_t N,
                  int P, int K, float* partials, int gx, cudaStream_t s) {
  switch (KP) {
    case 2: launch<2, SPLIT_X>(mx, my, W, b, N, P, K, partials, gx, s); break;
    case 4: launch<4, SPLIT_X>(mx, my, W, b, N, P, K, partials, gx, s); break;
    case 8: launch<8, SPLIT_X>(mx, my, W, b, N, P, K, partials, gx, s); break;
    default: launch<16, SPLIT_X>(mx, my, W, b, N, P, K, partials, gx, s); break;
  }
}

}  // namespace tcc
}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_categorical_workspace(int64_t N, int D, int K, int P) {
  // [ticket, 256 B] + CTA partials [gx][P][K (D + 1) + 1] + one [P] row for the per-particle sums
  if (N < 1 || D < 1 || K < 1 || P < 1) return 256;
  const size_t S = (size_t)K * (size_t)(D + 1) + 1;
  return 256 + ((size_t)tcc::grid_x(N, K, P) * (size_t)P * S + (size_t)P) * sizeof(float);
}

extern "C" int b2_glm_categorical_logits(const float* X, const int64_t* y, const float* W, const float* b, int64_t N,
                                         int D, int K, int P, double scale, double weight, double sum_coeff,
                                         int flags, float* out_sum_p, float* out_total, float* out_dW, float* out_db,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  using namespace tcc;
  if (!X || !y || !W) return B2_ERR_NULL;
  if (N < 1 || N >= ((int64_t)1 << 31) || P < 1 || D != kD || K < 2 || K > 16) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (!workspace || workspace_bytes < b2_glm_categorical_workspace(N, D, K, P)) return B2_ERR_WORKSPACE;
  CUtensorMap mx, my;
  if (!encode_x_map(&mx, X, N) || !encode_label_map(&my, y, N, Softmax<2>::kYType)) return B2_ERR_LAUNCH;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int gx = grid_x(N, K, P);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
  float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  // same precision policy as b2_glm_bernoulli_logits: below 64 Ki rows X is split hi + lo as well
  const bool split_x = (flags & B2_FLAG_GLM_3XTF32) || N < 65536;
  if (split_x)
    launch_split<true>(class_pad(K), mx, my, W, b, N, P, K, partials, gx, s);
  else
    launch_split<false>(class_pad(K), mx, my, W, b, N, P, K, partials, gx, s);
  launch_glm_finish(partials, ticket, gx, P, K, kD, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                    out_db, nullptr, s);
  count_launch(2);
  return check_launch();
}
