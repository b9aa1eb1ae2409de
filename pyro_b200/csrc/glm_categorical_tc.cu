// glm_categorical_tc.cu -- Hopper fused softmax-regression likelihood kernel: one pass over X[N,32] and
// the labels y[N] gives, for P weight matrices W[p] in R^{K x 32} (2 <= K <= 16) and biases b[p] in R^K,
//   l[p,n,k]  = <x_n, W[p,k,:]> + b[p,k],   lse[p,n] = logsumexp_k l[p,n,k]
//   sum_p[p]  = SUM_n ( l[p,n,y_n] - lse[p,n] )                 (torch/distributions/categorical.py log_prob)
//   g[p,n,k]  = [k == y_n] - softmax_k(l[p,n,:])
//   dW[p,k,:] = weight * SUM_n g[p,n,k] x_n,     db[p,k] = weight * SUM_n g[p,n,k]
// It replaces the user model's `X @ W.mT + b`, Categorical(logits).log_prob, the site sum and the autograd
// backward of all three, which together write and re-read [P, N, K] tensors.
//
// The Bernoulli kernel of glm_tc.cu with a class axis; the tile pipeline, the precision policy and the
// determinism argument are the same (see there).  What differs:
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
namespace tcc {

using namespace tc;

constexpr int kRows = 64;                       // rows per tile = N of GEMM 1 = K of GEMM 2
constexpr int kD = 32;
constexpr int kM = 64;                          // (particle, class) rows per slab
constexpr int kWG = 4;                          // warpgroups
constexpr int kStages = 2 * kWG;                // two X/y stages per warpgroup
constexpr int kThreads = kWG * 128;

constexpr uint32_t kTile = kRows * kD * 4;      // 8 KB X tile
constexpr uint32_t kYBytes = kRows * 8;         // 512 B of int64 labels
constexpr uint32_t kXtBlock = (kD + 8) * 128;   // X^T k-block: 32 rows of d + 8 rows of ones, 32 n each (5 KB)

constexpr uint32_t WG_XT = 0;
constexpr uint32_t WG_XLO = WG_XT + 2 * kXtBlock;
constexpr uint32_t kWGBytes = WG_XLO + kTile;
constexpr uint32_t OFF_X = 0;
constexpr uint32_t OFF_Y = OFF_X + kStages * kTile;
constexpr uint32_t OFF_WHI = OFF_Y + kStages * kYBytes;   // [m 64][32 d] SW128, 8 KB
constexpr uint32_t OFF_WLO = OFF_WHI + 8192;
constexpr uint32_t OFF_WG = OFF_WLO + 8192;
constexpr uint32_t OFF_BAR = OFF_WG + kWG * kWGBytes;
constexpr uint32_t kSmemBytes = OFF_BAR + 256 + 1024;   // + slack for the 1024-byte alignment
static_assert(kSmemBytes <= 232448, "shared memory budget");
static_assert(OFF_WHI % 1024 == 0 && kWGBytes % 1024 == 0 && kXtBlock % 1024 == 0, "operand alignment");
static_assert((kWG * kM * 33 + kWG * kM) * 4 <= kStages * kTile, "reduction scratch");

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

// wgmma accumulator fragment (m64nN, f32): thread (warp w4 of the warpgroup, lane = 4 gid + t4) holds
// d[4j + 2h + e] = D[16 w4 + gid + 8h][8j + 2 t4 + e].
template <int KP, bool SPLIT_X>
__global__ void __launch_bounds__(kThreads, 1)
glm_categorical_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                          const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int P, int K,
                          float* __restrict__ partials) {
  static_assert(KP == 2 || KP == 4 || KP == 8 || KP == 16, "class padding");
  constexpr int PPS = kM / KP;                  // particles per slab
  pdl_enter();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + OFF_BAR;
  auto bar_full = [&](int s) { return bar0 + 8u * (uint32_t)s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int slab = blockIdx.y;
  const int64_t ntiles = (N + kRows - 1) / kRows;
  const int nt = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);
  const int S = K * (kD + 1) + 1;               // partials per particle: [K][dW 32 | db], sum

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(bar_full(s), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  {
    float* whi = reinterpret_cast<float*>(sm + OFF_WHI);
    float* wlo = reinterpret_cast<float*>(sm + OFF_WLO);
    for (int e = tid; e < kM * kD; e += kThreads) {
      const int m = e >> 5, d = e & 31;
      const int gp = slab * PPS + m / KP, k = m % KP;
      const float w = (gp < P && k < K) ? W[((int64_t)gp * K + k) * kD + d] : 0.f;
      const float hi = tf32_trunc(w);
      const int off = m * 32 + ((((d >> 2) ^ (m & 7)) << 2) | (d & 3));
      whi[off] = hi;
      wlo[off] = w - hi;
    }
    for (int e = tid; e < kWG * 2 * 256; e += kThreads) {
      const int g = e >> 9, kb = (e >> 8) & 1, w = e & 255;
      reinterpret_cast<float*>(sm + OFF_WG + g * kWGBytes + WG_XT + kb * kXtBlock + kD * 128)[w] = 1.f;
    }
  }
  fence_proxy_async();
  __syncthreads();

  float lpa[2] = {0.f, 0.f};                   // lp sums of the thread's two rows
  float acc2[20];                              // [dW | db] of the slab's rows; started with scale-d = 0
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), w4 = warp & 3, t = tid & 127;
  const int gid = lane >> 2, t4 = lane & 3;
  // the thread's two rows m = 16 w4 + gid + 8h: class (gid + 8h) % KP of particle slab * PPS + m / KP
  int cls[2];
  float bias[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = 16 * w4 + gid + 8 * h;
    const int gp = slab * PPS + m / KP;
    cls[h] = m % KP;
    bias[h] = (bvec != nullptr && gp < P && cls[h] < K) ? bvec[(int64_t)gp * K + cls[h]] : 0.f;
  }

  {
    uint8_t* my = sm + OFF_WG + wg * kWGBytes;
    const uint32_t my_s = base + OFF_WG + wg * kWGBytes;
    const uint64_t d_whi = desc_sw128(base + OFF_WHI), d_wlo = desc_sw128(base + OFF_WLO);
    const uint64_t d_xlo = desc_sw128(my_s + WG_XLO);
    auto load = [&](int it, int s) {
      const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
      mbar_expect_tx(bar_full(s), kTile + kYBytes);
      tma_load_2d(base + OFF_X + s * kTile, &map_x, 0, (int)(tile * kRows), bar_full(s));
      tma_load_1d(base + OFF_Y + s * kYBytes, &map_y, (int)(tile * kRows), bar_full(s));
    };
    if (t == 0)
      for (int k = 0; k < 2 && wg + k * kWG < nt; ++k) load(wg + k * kWG, 2 * wg + k);
    for (int k = 0, it = wg; it < nt; ++k, it += kWG) {
      const int s = 2 * wg + (k & 1);
      const int64_t row0 = (blockIdx.x + (int64_t)it * gridDim.x) * kRows;
      mbar_wait(bar_full(s), (uint32_t)(k >> 1) & 1u);
      wgmma_wait0();
      fence_regs(acc2);
      // ---- split / transposition pass (as in glm_tc.cu) ------------------------------------------------
      {
        const int r = t >> 1, hh = t & 1, rk = kt_pos(r);
        float4* xs = reinterpret_cast<float4*>(sm + OFF_X + s * kTile);
        float4* xl = reinterpret_cast<float4*>(my + WG_XLO);
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          const int c = hh * 4 + c4;
          const int idx = r * 8 + (c ^ (r & 7));
          const float4 v = xs[idx];
          const float x[4] = {v.x, v.y, v.z, v.w};
          float xr[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) xr[q] = tf32_rn(x[q]);
          if (SPLIT_X) {
            float h[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) h[q] = tf32_trunc(x[q]);
            xs[idx] = make_float4(h[0], h[1], h[2], h[3]);
            xl[idx] = make_float4(x[0] - h[0], x[1] - h[1], x[2] - h[2], x[3] - h[3]);
          } else {
            xs[idx] = make_float4(xr[0], xr[1], xr[2], xr[3]);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int d = c * 4 + q;
            reinterpret_cast<float*>(my + WG_XT + (rk >> 5) * kXtBlock)[d * 32 + (((((rk & 31) >> 2) ^ (d & 7)) << 2) |
                                                                                  (rk & 3))] = xr[q];
          }
        }
      }
      // labels of the thread's rows n = 8j + 2 t4 + e, -1 outside [0, K); read before the refill
      int yl[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const longlong2 v = reinterpret_cast<const longlong2*>(sm + OFF_Y + s * kYBytes)[4 * j + t4];
        yl[2 * j] = ((unsigned long long)v.x < (unsigned long long)K) ? (int)v.x : -1;
        yl[2 * j + 1] = ((unsigned long long)v.y < (unsigned long long)K) ? (int)v.y : -1;
      }
      fence_proxy_async();
      wg_bar(1 + wg);
      // ---- GEMM 1: logits L^T[(p, k), n] = W X^T + b ---------------------------------------------------
      float acc1[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc1[i] = bias[(i >> 1) & 1];
      wgmma_fence();
      const uint64_t d_x = desc_sw128(base + OFF_X + s * kTile);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        wgmma_n64_tf32(acc1, d_whi + 2 * k, d_x + 2 * k);
        wgmma_n64_tf32(acc1, d_wlo + 2 * k, d_x + 2 * k);
        if (SPLIT_X) wgmma_n64_tf32(acc1, d_whi + 2 * k, d_xlo + 2 * k);
      }
      wgmma_commit();
      wgmma_wait0();
      fence_regs(acc1);
      if (t == 0 && it + 2 * kWG < nt) load(it + 2 * kWG, s);
      // ---- epilogue: softmax over the class rows, lp sums and g, all in registers -------------------------
      uint32_t g[32];                          // indexed like acc1
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
      // ---- GEMM 2: [dW | db] += g [X | 1], g from registers --------------------------------------------
      fence_regs(g);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t a[4] = {g[4 * j], g[4 * j + 2], g[4 * j + 1], g[4 * j + 3]};
        wgmma_n40_tf32_ra(acc2, a, desc_sw128(my_s + WG_XT + (j >> 2) * kXtBlock) + 2 * (j & 3), it != wg || j != 0);
      }
      wgmma_commit();
    }
    wgmma_wait0();
    fence_regs(acc2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v = lpa[h];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      lpa[h] = v;
    }
  }
  // ---- CTA results through shared memory (the X ring is idle now), fixed summation order -----------------
  __syncthreads();
  float* red2 = reinterpret_cast<float*>(sm + OFF_X);     // [kWG][64 m][33]
  float* redlp = red2 + kWG * kM * 33;                    // [kWG][64 m]
  {
#pragma unroll
    for (int j = 0; j < 5; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 16 * w4 + gid + 8 * h, c = 8 * j + 2 * t4 + e;
          if (c <= kD) red2[(wg * kM + m) * 33 + c] = acc2[4 * j + 2 * h + e];
        }
    if (t4 == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) redlp[wg * kM + 16 * w4 + gid + 8 * h] = lpa[h];
    }
  }
  __syncthreads();
  const int nwg = nt < kWG ? nt : kWG;         // warpgroups that had a tile
  for (int e = tid; e < kM * 33; e += kThreads) {
    const int m = e / 33, c = e - 33 * m;
    const int gp = slab * PPS + m / KP, k = m % KP;
    if (gp < P && k < K) {
      float v = 0.f;
      for (int q = 0; q < nwg; ++q) v += red2[(q * kM + m) * 33 + c];
      partials[((int64_t)blockIdx.x * P + gp) * S + k * (kD + 1) + c] = v;
    }
  }
  if (tid < PPS && slab * PPS + tid < P) {
    float v = 0.f;
    for (int q = 0; q < nwg; ++q)
      for (int k = 0; k < KP; ++k) v += redlp[q * kM + tid * KP + k];
    partials[((int64_t)blockIdx.x * P + slab * PPS + tid) * S + K * (kD + 1)] = v;
  }
}

// Fixed-order sum of the CTA partials, one warp per entry of the [P][K (33) + 1] table; applies weight and
// scale.  The last of the P sum warps also totals sum_p (ticket), as glm_finish_kernel does.
__global__ void __launch_bounds__(256) glm_categorical_finish_kernel(const float* __restrict__ partials, int nblocks,
                                                                     int P, int K, double scale, double weight,
                                                                     float* __restrict__ sum_p,
                                                                     float* __restrict__ out_dW,
                                                                     float* __restrict__ out_db, double sum_coeff,
                                                                     int flags, float* __restrict__ out_total,
                                                                     unsigned int* __restrict__ ticket) {
  pdl_enter();
  const int S = K * (kD + 1) + 1;
  const int total = P * S;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= total) return;
  double s = 0.0;
  for (int bl = lane; bl < nblocks; bl += 32) s += (double)partials[(int64_t)bl * total + e];
  s = warp_sum(s);
  const int p = e / S, r = e - p * S;
  if (r < K * (kD + 1)) {
    const int k = r / (kD + 1), c = r - k * (kD + 1);
    if (lane == 0) {
      if (c < kD) {
        if (out_dW) out_dW[((int64_t)p * K + k) * kD + c] = (float)(weight * scale * s);
      } else if (out_db) {
        out_db[(int64_t)p * K + k] = (float)(weight * scale * s);
      }
    }
    return;
  }
  unsigned int t = 0;
  if (lane == 0) {
    sum_p[p] = (float)(scale * s);
    if (out_total) {
      __threadfence();
      t = atomicAdd(ticket, 1u);
    }
  }
  if (!out_total) return;
  t = __shfl_sync(0xffffffffu, t, 0);
  if (t != (unsigned)(P - 1)) return;
  __threadfence();
  double acc = 0.0;
  for (int q = lane; q < P; q += 32) acc += (double)__ldcg(sum_p + q);
  acc = warp_sum(acc);
  if (lane == 0) {
    const double v = sum_coeff * acc;
    *out_total = (flags & B2_FLAG_ACCUMULATE_SUM) ? (float)((double)*out_total + v) : (float)v;
    *ticket = 0u;
  }
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
  tc::EncodeTiledFn enc = tc::encode_fn();
  if (enc == nullptr) return B2_ERR_LAUNCH;
  CUtensorMap mx, my;
  {
    const cuuint64_t dims[2] = {(cuuint64_t)kD, (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)kD * 4};
    const cuuint32_t box[2] = {(cuuint32_t)kD, (cuuint32_t)kRows};
    const cuuint32_t estr[2] = {1, 1};
    if (enc(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(X), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B2_ERR_LAUNCH;
  }
  {
    const cuuint64_t dims[1] = {(cuuint64_t)N};
    const cuuint64_t strides[1] = {0};
    const cuuint32_t box[1] = {(cuuint32_t)kRows};
    const cuuint32_t estr[1] = {1};
    if (enc(&my, CU_TENSOR_MAP_DATA_TYPE_INT64, 1, const_cast<int64_t*>(y), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B2_ERR_LAUNCH;
  }
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
  const int S = K * (kD + 1) + 1;
  float* sum_p = out_sum_p ? out_sum_p : partials + (size_t)gx * P * S;
  const int total = P * S;
  launch_pdl(glm_categorical_finish_kernel, dim3((total + 7) / 8), dim3(256), 0, s, partials, gx, P, K, scale, weight,
             sum_p, out_dW, out_db, sum_coeff, flags, out_total, ticket);
  count_launch(2);
  return check_launch();
}
