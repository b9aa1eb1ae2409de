// poisson_product_tc.cu -- Hopper fused Poisson matrix-factorisation likelihood: for P particles with
// factors A[p] in R^{N x K} and B[p] in R^{K x J} (1 <= K <= 16) and shared counts x[N, J],
//   rate[p,n,j] = SUM_k A[p,n,k] B[p,k,j]
//   sum_p[p]    = SUM_{n,j} ( xlogy(x, rate) - rate - lgamma(x + 1) )      (torch/distributions/poisson.py)
//   G[p,n,j]    = x / rate - 1                                              (d log p / d rate)
//   dA[p]       = weight * scale * G[p] B[p]^T,     dB[p] = weight * scale * A[p]^T G[p]
// It replaces the model's `torch.matmul(z, w)`, Poisson(rate).log_prob, the site sum and the autograd backward
// of all three, which together write and re-read several [P, N, J] tensors; here no [P, N, J] value leaves the
// registers and shared memory of the CTA that computes it.
//
// Decomposition.  One CTA (one warpgroup) per particle and group of S consecutive 64-column blocks of J; for
// each block it keeps B's columns in shared memory and walks N in 64-row tiles.  Everything runs "transposed",
// with the J block as the 64 wgmma rows:
//   GEMM 1   rate^T[j, n] = B^T[j, :] A[n, :]^T            m64n64k8 x 2 k-steps x 3 (split, below)
//   epilogue lp and G per element on the register accumulator; G^T stays in registers, G goes to shared memory
//   GEMM 2   dB^T[j, :] += G^T[j, n] A[n, :]               m64n16k8 x 8 x 3, G^T as the register A operand
//                                                          (kt_pos order)
//   GEMM 3   dA[n, :]    = G[n, j] B[:, j]^T               m64n16k8 x 8 x 3, both operands in shared memory
// dB of a block accumulates in registers over the whole row walk and is written once.  dA of a tile is
// complete over the block's 64 columns; the CTA adds its S blocks into one partial in global memory (the same
// thread re-reads what it wrote), and poisson_product_finish_kernel sums the partials of the CTAs in a fixed
// order.  A (60-byte rows for K = 15, not a legal TMA stride) and B are tiny and loaded with ordinary loads;
// x is read from L2 straight into registers by the thread that owns each element.
//
// Precision.  A rounding error of A[n,k] is shared by a whole row of 4096 rates and one of B[k,j] by a whole
// column, so unlike data x weights neither averages out: both are split hi + lo and GEMM 1 takes three
// products (hi.hi + hi.lo + lo.hi), every rate fp32-exact.  The gradient contractions are split the same way
// (G, A and B hi + lo, three products): G = x / rate - 1 has both signs and a few large entries where the rate
// is small, so dA and dB are sums with heavy cancellation, and with one operand rounded to TF32 their error
// was measured at 2-6e-4 of the largest gradient (K = 15, N = 320, J = 4096), against 1e-6 split.
//
// Value-only terms.  SUM lgamma(x + 1) depends on x alone: the CTAs of particle 0 evaluate it once per call
// and the finish subtracts it from every particle's sum.  Where x == 0 the log term is dropped (lp = -rate)
// and G = 0 * rcp(rate) - 1 is -1, or NaN at rate == 0, exactly as in the generic Poisson kernel (kPoisson).
// The epilogue is branch-free and issues 2 MUFU ops (lg2, rcp) per element whatever x is: zero counts are
// scattered over the lanes of a warp, so skipping them per lane would not save a warp's issue slots.
// A non-finite G makes every factor gradient it enters non-finite, as on the materialised path; an entry the
// materialised path gives as +-inf can be NaN here, where a split product multiplies G = +inf by the zero low
// part of a factor value that TF32 represents exactly (inf * 0).
#include <stdlib.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "glm_tc_common.cuh"

namespace b2 {
namespace tcp {

using namespace tc;

constexpr int kT = 64;                   // rows of an N tile = columns of a J block
constexpr int kKP = 16;                  // K padded
constexpr int kThreads = 128;
constexpr int kMaxS = 8;                 // J blocks per CTA

constexpr uint32_t OFF_BT = 0;           // B^T [64 j][hi k 0..15 | lo k 0..15] SW128, 8 KB
constexpr uint32_t OFF_A = 8192;         // A tile [64 n][hi | lo] SW128, 8 KB
constexpr uint32_t OFF_AT = 16384;       // A^T hi, lo: 2 x 2 blocks [16 k][32 n] (n in kt_pos order), 2 KB each
constexpr uint32_t OFF_BS = 24576;       // B hi, lo: 2 x 2 blocks [16 k][32 j], 2 KB each
constexpr uint32_t OFF_G = 32768;        // G hi, lo: 2 x 2 blocks [64 n][32 j], 8 KB each
constexpr uint32_t OFF_RED = 65536;      // 2 x 4 floats
constexpr uint32_t kSmemBytes = OFF_RED + 64 + 1024;   // + slack for the 1024-byte alignment
static_assert(OFF_AT % 1024 == 0 && OFF_BS % 1024 == 0 && OFF_G % 1024 == 0, "operand alignment");

constexpr float kLn2 = 0.6931471805599453f;

// wgmma accumulator fragment (m64nN, f32): thread (warp w4, lane = 4 gid + t4) holds
// d[4i + 2h + e] = D[16 w4 + gid + 8h][8i + 2 t4 + e].
__global__ void __launch_bounds__(kThreads, 3)
poisson_product_tc_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ x,
                          int64_t N, int K, int64_t J, int S, float gscale, float* __restrict__ part_dA,
                          float* __restrict__ part_lp, float* __restrict__ part_lg, float* __restrict__ out_dB) {
  pdl_enter();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  float* bt = reinterpret_cast<float*>(sm + OFF_BT);
  float* as = reinterpret_cast<float*>(sm + OFF_A);
  float* at = reinterpret_cast<float*>(sm + OFF_AT);
  float* bs = reinterpret_cast<float*>(sm + OFF_BS);
  float* gs = reinterpret_cast<float*>(sm + OFF_G);
  float* red = reinterpret_cast<float*>(sm + OFF_RED);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int w4 = warp, gid = lane >> 2, t4 = lane & 3;
  const int p = blockIdx.y, G = gridDim.x;
  const int64_t NK = N * K;
  const float* Ap = A + (int64_t)p * NK;
  const float* Bp = B + (int64_t)p * K * J;
  const int ntiles = (int)((N + kT - 1) / kT);
  const uint64_t d_bt = desc_sw128(base + OFF_BT), d_a = desc_sw128(base + OFF_A);
  float* pdA = part_dA + ((int64_t)p * G + blockIdx.x) * NK;

  float lpa = 0.f, lga = 0.f;
  for (int s = 0; s < S; ++s) {
    const int64_t j0 = ((int64_t)blockIdx.x * S + s) * kT;
    if (j0 >= J) break;
    __syncthreads();                                   // the previous block's operands are no longer read
    // ---- B block: B^T hi | lo for GEMM 1, B hi and lo for GEMM 3; zero past K and J ---------------------------
    for (int e = tid; e < kT * kKP; e += kThreads) {
      const int k = e & 15, jl = e >> 4;
      const float v = (k < K && j0 + jl < J) ? Bp[(int64_t)k * J + j0 + jl] : 0.f;
      const float hi = tf32_trunc(v);
      bt[sw128(jl, k)] = hi;
      bt[sw128(jl, 16 + k)] = v - hi;
      bs[(jl >> 5) * 512 + sw128(k, jl & 31)] = hi;
      bs[(2 + (jl >> 5)) * 512 + sw128(k, jl & 31)] = v - hi;
    }
    float accB[8];                                     // dB^T[j, k] of the block; started with scale-d = 0
    for (int t = 0; t < ntiles; ++t) {
      const int64_t n0 = (int64_t)t * kT;
      // rows and columns of the tile inside [0, N) x [0, J): only the last row tile and column block are partial
      const int nrem = (int)(N - n0 < kT ? N - n0 : kT);
      const int jrem = (int)(J - j0 < kT ? J - j0 : kT);
      // ---- counts of the thread's elements (n = n0 + 8i + 2 t4 + e, j = j0 + 16 w4 + gid + 8h), from L2; a
      // masked element loads x[0] (branch-free, so all 32 loads are in flight at once) and is zeroed ----------
      float xv[32];
      const float* xb = x + (n0 + 2 * t4) * J + j0 + 16 * w4 + gid;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const bool v = 8 * i + 2 * t4 + e < nrem && 16 * w4 + gid + 8 * h < jrem;
            const float xx = __ldg(v ? xb + (8 * i + e) * J + 8 * h : x);
            xv[4 * i + 2 * h + e] = v ? xx : 0.f;
          }
      // ---- this tile's dA partial so far (added to below), loaded early to hide the latency -----------------
      float prev[8];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t n = n0 + 16 * w4 + gid + 8 * h;
            const int k = 8 * i + 2 * t4 + e;
            prev[4 * i + 2 * h + e] = (s != 0 && n < N && k < K) ? pdA[n * K + k] : 0.f;
          }
      // ---- A tile: hi | lo for GEMM 1, A^T hi and lo (kt_pos order) for GEMM 2; zero past K and N -------------
      for (int e = tid; e < kT * kKP; e += kThreads) {
        const int k = e & 15, nl = e >> 4;
        const float v = (k < K && n0 + nl < N) ? Ap[(n0 + nl) * K + k] : 0.f;
        const float hi = tf32_trunc(v);
        as[sw128(nl, k)] = hi;
        as[sw128(nl, 16 + k)] = v - hi;
        const int rk = kt_pos(nl);
        at[(rk >> 5) * 512 + sw128(k, rk & 31)] = hi;
        at[(2 + (rk >> 5)) * 512 + sw128(k, rk & 31)] = v - hi;
      }
      fence_proxy_async();
      __syncthreads();
      // ---- GEMM 1: rate^T = B^T A^T, fp32-exact (k-steps 0, 1 are hi, 2, 3 lo) ------------------------------
      float acc1[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        wgmma_n64_tf32(acc1, d_bt + 2 * k, d_a + 2 * k);
        wgmma_n64_tf32(acc1, d_bt + 2 * k, d_a + 4 + 2 * k);
        wgmma_n64_tf32(acc1, d_bt + 4 + 2 * k, d_a + 2 * k);
      }
      wgmma_commit();
      wgmma_wait0();
      fence_regs(acc1);
      // ---- epilogue: lp and G in registers (hi + lo); G also to shared memory for GEMM 3 --------------------
      uint32_t ghi[32], glo[32];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int q = 4 * i + 2 * h + e;
            const int nl = 8 * i + 2 * t4 + e, jl = 16 * w4 + gid + 8 * h;
            const float r = acc1[q], xx = xv[q];
            const float lp = (xx != 0.f) ? fmaf(xx * kLn2, lg2f(r), -r) : -r;
            const float gg = fmaf(xx, rcpf(r), -1.f);
            const bool v = nl < nrem && jl < jrem;
            lpa += v ? lp : 0.f;
            const float gv = v ? gg : 0.f;
            // lo = 0 for a non-finite G (+inf at rate == 0 with x > 0), not inf - inf = NaN
            const float hi = tf32_trunc(gv), lo = (hi - hi == 0.f) ? gv - hi : 0.f;
            ghi[q] = __float_as_uint(hi);
            glo[q] = __float_as_uint(lo);
            gs[(jl >> 5) * 2048 + sw128(nl, jl & 31)] = hi;
            gs[(2 + (jl >> 5)) * 2048 + sw128(nl, jl & 31)] = lo;
          }
      fence_proxy_async();
      __syncthreads();
      // ---- GEMM 2: dB^T += G^T A (G^T from registers); GEMM 3: dA tile = G B^T; hi.hi + hi.lo + lo.hi ---------
      float accA[8];
      fence_regs(ghi);
      fence_regs(glo);
      wgmma_fence();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t a[4] = {ghi[4 * i], ghi[4 * i + 2], ghi[4 * i + 1], ghi[4 * i + 3]};
        const uint32_t b[4] = {glo[4 * i], glo[4 * i + 2], glo[4 * i + 1], glo[4 * i + 3]};
        const uint64_t d_hi = desc_sw128(base + OFF_AT + (i >> 2) * 2048) + 2 * (i & 3);
        const uint64_t d_lo = desc_sw128(base + OFF_AT + (2 + (i >> 2)) * 2048) + 2 * (i & 3);
        wgmma_tf32_ra<16>(accB, a, d_hi, t != 0 || i != 0);
        wgmma_tf32_ra<16>(accB, a, d_lo, 1);
        wgmma_tf32_ra<16>(accB, b, d_hi, 1);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint64_t g_hi = desc_sw128(base + OFF_G + (i >> 2) * 8192) + 2 * (i & 3);
        const uint64_t g_lo = desc_sw128(base + OFF_G + (2 + (i >> 2)) * 8192) + 2 * (i & 3);
        const uint64_t b_hi = desc_sw128(base + OFF_BS + (i >> 2) * 2048) + 2 * (i & 3);
        const uint64_t b_lo = desc_sw128(base + OFF_BS + (2 + (i >> 2)) * 2048) + 2 * (i & 3);
        wgmma_n16_tf32(accA, g_hi, b_hi, i != 0);
        wgmma_n16_tf32(accA, g_hi, b_lo, 1);
        wgmma_n16_tf32(accA, g_lo, b_hi, 1);
      }
      wgmma_commit();
      wgmma_wait0();
      fence_regs(accA);
      fence_regs(accB);
      // ---- dA tile into the CTA's partial: stored by the first block, added by the others -------------------
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t n = n0 + 16 * w4 + gid + 8 * h;
            const int k = 8 * i + 2 * t4 + e;
            if (n < N && k < K) pdA[n * K + k] = prev[4 * i + 2 * h + e] + accA[4 * i + 2 * h + e];
          }
    }
    // ---- dB of the block, final ------------------------------------------------------------------------------
    if (out_dB != nullptr) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t j = j0 + 16 * w4 + gid + 8 * h;
            const int k = 8 * i + 2 * t4 + e;
            if (j < J && k < K) out_dB[((int64_t)p * K + k) * J + j] = gscale * accB[4 * i + 2 * h + e];
          }
    }
    // ---- SUM lgamma(x + 1) over the block, once per call (particle 0's CTAs) ---------------------------------
    if (p == 0) {
      for (int64_t e = tid; e < N * (kT / 4); e += kThreads) {
        const int64_t n = e >> 4, j = j0 + 4 * (e & 15);
        if (j < J) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(x + n * J + j));
          lga += ValueAux<kPoisson, float, false>::make(v.x).lgx + ValueAux<kPoisson, float, false>::make(v.y).lgx +
                 ValueAux<kPoisson, float, false>::make(v.z).lgx + ValueAux<kPoisson, float, false>::make(v.w).lgx;
        }
      }
    }
  }
  // ---- CTA sums, fixed order -----------------------------------------------------------------------------------
  lpa = warp_sum(lpa);
  lga = warp_sum(lga);
  __syncthreads();
  if (lane == 0) {
    red[warp] = lpa;
    red[4 + warp] = lga;
  }
  __syncthreads();
  if (tid == 0) {
    part_lp[(int64_t)p * G + blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
    if (p == 0) part_lg[blockIdx.x] = (red[4] + red[5]) + (red[6] + red[7]);
  }
}

// Fixed-order sums of the CTA partials: one thread per dA entry, then one per particle sum.  The last particle
// thread to finish (ticket) totals sum_p, as glm_finish_kernel does.
__global__ void __launch_bounds__(256) poisson_product_finish_kernel(
    const float* __restrict__ part_dA, const float* __restrict__ part_lp, const float* __restrict__ part_lg, int G,
    int P, int64_t NK, double scale, double weight, float* __restrict__ sum_p, float* __restrict__ out_dA,
    double sum_coeff, int flags, float* __restrict__ out_total, unsigned int* __restrict__ ticket) {
  pdl_enter();
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nA = out_dA != nullptr ? (int64_t)P * NK : 0;
  if (e < nA) {
    const int64_t p = e / NK, r = e - p * NK;
    double s = 0.0;
    for (int b = 0; b < G; ++b) s += (double)part_dA[(p * G + b) * NK + r];
    out_dA[e] = (float)(weight * scale * s);
    return;
  }
  const int64_t q = e - nA;
  if (q >= P) return;
  double lg = 0.0, s = 0.0;
  for (int b = 0; b < G; ++b) lg += (double)part_lg[b];
  for (int b = 0; b < G; ++b) s += (double)part_lp[q * G + b];
  sum_p[q] = (float)(scale * (s - lg));
  if (!out_total) return;
  __threadfence();
  const unsigned int t = atomicAdd(ticket, 1u);
  if (t != (unsigned)(P - 1)) return;
  __threadfence();
  double acc = 0.0;
  for (int i = 0; i < P; ++i) acc += (double)__ldcg(sum_p + i);
  const double v = sum_coeff * acc;
  *out_total = (flags & B2_FLAG_ACCUMULATE_SUM) ? (float)((double)*out_total + v) : (float)v;
  *ticket = 0u;
}

// J blocks per CTA: enough CTAs for about two waves at three CTAs per SM, at most kMaxS blocks each (fewer
// partials of dA to write and sum)
inline int blocks_per_cta(int64_t J, int P) {
  const int64_t nb = (J + kT - 1) / kT;
  int64_t s = (int64_t)P * nb / (2 * 3 * kNumSMs);
  if (s < 1) s = 1;
  if (s > kMaxS) s = kMaxS;
  return (int)s;
}
inline int cta_groups(int64_t J, int P) {
  const int64_t nb = (J + kT - 1) / kT;
  const int s = blocks_per_cta(J, P);
  return (int)((nb + s - 1) / s);
}

}  // namespace tcp
}  // namespace b2

using namespace b2;

static bool poisson_product_shape_ok(int64_t N, int K, int64_t J, int P) {
  return N >= 1 && N < ((int64_t)1 << 31) && K >= 1 && K <= 16 && J >= 1 && J < ((int64_t)1 << 31) && J % 4 == 0 &&
         P >= 1 && P <= 65535 && N * J < ((int64_t)1 << 40);
}

extern "C" size_t b2_poisson_product_workspace(int64_t N, int K, int64_t J, int P) {
  // [ticket, 256 B] + dA partials [P][G][N][K] + lp partials [P][G] + lgamma partials [G] + a [P] row for sum_p
  if (!poisson_product_shape_ok(N, K, J, P)) return 256;
  const size_t G = (size_t)tcp::cta_groups(J, P);
  return 256 + ((size_t)P * G * (size_t)N * (size_t)K + (size_t)P * G + G + (size_t)P) * sizeof(float);
}

extern "C" int b2_poisson_product(const float* A, const float* B, const float* x, int64_t N, int K, int64_t J, int P,
                                  double scale, double weight, double sum_coeff, int flags, float* out_sum_p,
                                  float* out_total, float* out_dA, float* out_dB, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  using namespace tcp;
  if (!A || !B || !x) return B2_ERR_NULL;
  if (!poisson_product_shape_ok(N, K, J, P)) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(x) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (!workspace || workspace_bytes < b2_poisson_product_workspace(N, K, J, P)) return B2_ERR_WORKSPACE;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(poisson_product_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    attr_set = true;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int S = blocks_per_cta(J, P), G = cta_groups(J, P);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
  float* part_dA = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  float* part_lp = part_dA + (size_t)P * G * N * K;
  float* part_lg = part_lp + (size_t)P * G;
  float* sum_p = out_sum_p ? out_sum_p : part_lg + G;
  const float gscale = (float)(weight * scale);
  launch_pdl(poisson_product_tc_kernel, dim3((unsigned)G, (unsigned)P, 1), dim3(kThreads), (size_t)kSmemBytes, s,
             A, B, x, N, K, J, S, gscale, part_dA, part_lp, part_lg, out_dB);
  const int64_t total = (out_dA ? (int64_t)P * N * K : 0) + P;
  launch_pdl(poisson_product_finish_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s,
             (const float*)part_dA, (const float*)part_lp, (const float*)part_lg, G, P, N * K, scale, weight, sum_p,
             out_dA, sum_coeff, flags, out_total, ticket);
  count_launch(2);
  return check_launch();
}
