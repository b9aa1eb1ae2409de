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
#include <cuda.h>
#include <stdlib.h>

#include "b2_common.cuh"
#include "glm_tc_common.cuh"

namespace b2 {
namespace tc {

constexpr int kRows = 64;                       // rows per tile = M of one wgmma
constexpr int kD = 32;
constexpr int kP = 64;
constexpr int kWG = 4;                          // warpgroups
constexpr int kStages = 2 * kWG;                // two X/y stages per warpgroup
constexpr int kThreads = kWG * 128;

constexpr uint32_t kTile = kRows * kD * 4;      // 8 KB X tile
constexpr uint32_t kYBytes = kRows * 4;         // 256 B of y
constexpr uint32_t kXtBlock = (kD + 8) * 128;   // X^T k-block: 32 rows of d + 8 rows of ones, 32 n each (5 KB)

// per-warpgroup region
constexpr uint32_t WG_XT = 0;                       // X^T  [kb 2][c 40][32 n] fp32, n permuted (see kt_pos)
constexpr uint32_t WG_XLO = WG_XT + 2 * kXtBlock;   // X_lo [n 64][32 d] fp32 (SPLIT_X)
constexpr uint32_t kWGBytes = WG_XLO + kTile;
// CTA layout (every operand region 1024-byte aligned: the 128-byte swizzle pattern is taken from address bits)
constexpr uint32_t OFF_X = 0;
constexpr uint32_t OFF_Y = OFF_X + kStages * kTile;
constexpr uint32_t OFF_WHI = OFF_Y + 2048;          // [p 64][32 d] SW128, 8 KB
constexpr uint32_t OFF_WLO = OFF_WHI + 8192;
constexpr uint32_t OFF_WG = OFF_WLO + 8192;
constexpr uint32_t OFF_BAR = OFF_WG + kWG * kWGBytes;
constexpr uint32_t kSmemBytes = OFF_BAR + 256 + 1024;   // + slack for the 1024-byte alignment
static_assert(kStages * kYBytes <= 2048 && kSmemBytes <= 232448, "shared memory budget");
static_assert(kWGBytes % 1024 == 0 && kXtBlock % 1024 == 0, "operand alignment");
// the final reduction reuses the X ring: [kWG][64 p][33] + [kWG][64 p] floats
static_assert((kWG * kP * 33 + kWG * kP) * 4 <= kStages * kTile, "reduction scratch");

// SPLIT_X = false (default): W split hi/lo, X rounded to nearest.  SPLIT_X = true: full 3xTF32, X split
// hi/lo as well.
//
// wgmma accumulator fragment (m64nN, f32): thread (warp w4 of the warpgroup, lane = 4 gid + t4) holds
// d[4j + 2h + e] = D[16 w4 + gid + 8h][8j + 2 t4 + e].
template <bool SPLIT_X>
__global__ void __launch_bounds__(kThreads, 1)
glm_bernoulli_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                        const float* __restrict__ W, const float* __restrict__ bvec, int64_t N, int P,
                        float* __restrict__ partials) {
  pdl_enter();   // lets glm_finish_kernel be resident (blocked in its griddepcontrol.wait) before this kernel ends
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + OFF_BAR;
  auto bar_full = [&](int s) { return bar0 + 8u * (uint32_t)s; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int slab = blockIdx.y;
  const int64_t ntiles = (N + kRows - 1) / kRows;
  // tiles handled by this CTA: blockIdx.x, blockIdx.x + gridDim.x, ...
  const int nt = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);

  // ---- one-time setup --------------------------------------------------------------------------------
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(bar_full(s), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  {
    // weight tiles (generic-proxy writes, made visible to the tensor cores below)
    float* whi = reinterpret_cast<float*>(sm + OFF_WHI);
    float* wlo = reinterpret_cast<float*>(sm + OFF_WLO);
    for (int e = tid; e < kP * kD; e += kThreads) {
      const int p = e >> 5, d = e & 31;
      const int gp = slab * kP + p;
      const float w = (gp < P) ? W[(int64_t)gp * kD + d] : 0.f;
      const float hi = tf32_trunc(w);
      const int off = p * 32 + ((((d >> 2) ^ (p & 7)) << 2) | (d & 3));   // float index, 128B swizzle
      whi[off] = hi;
      wlo[off] = w - hi;
    }
    // rows 32..39 of every X^T buffer are ones: GEMM 2 then yields db in column 32 of its accumulator
    for (int e = tid; e < kWG * 2 * 256; e += kThreads) {
      const int g = e >> 9, kb = (e >> 8) & 1, w = e & 255;
      reinterpret_cast<float*>(sm + OFF_WG + g * kWGBytes + WG_XT + kb * kXtBlock + kD * 128)[w] = 1.f;
    }
  }
  fence_proxy_async();
  __syncthreads();

  float lpa[2] = {0.f, 0.f};                   // lp sums of the thread's two particles
  // GEMM 2 accumulator [p][c]: dW in c < 32, db in c = 32.  Never written by ordinary instructions before
  // the tile loop (that serialises every wgmma, C7515): the warpgroup's first GEMM 2 k-step starts it with
  // scale-d = 0, and a warpgroup without a tile is left out of the CTA reduction.
  float acc2[20];
  // warp-uniform by construction (a shuffle result), so the tile loop is not a divergent branch to ptxas
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), w4 = warp & 3, t = tid & 127;
  const int gid = lane >> 2, t4 = lane & 3;

  {
    // =========================== consumer warpgroups ====================================================
    uint8_t* my = sm + OFF_WG + wg * kWGBytes;
    const uint32_t my_s = base + OFF_WG + wg * kWGBytes;
    const uint64_t d_whi = desc_sw128(base + OFF_WHI), d_wlo = desc_sw128(base + OFF_WLO);
    const uint64_t d_xlo = desc_sw128(my_s + WG_XLO);
    float bias[2];                             // of particles 16 w4 + gid + 8h
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gp = slab * kP + 16 * w4 + gid + 8 * h;
      bias[h] = (bvec != nullptr && gp < P) ? bvec[gp] : 0.f;
    }
    // tile it -> X/y stage; one thread of the warpgroup issues the loads
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
      // GEMM 2 of this warpgroup's previous tile has finished reading X^T and the g registers
      wgmma_wait0();
      fence_regs(acc2);
      // ---- split / transposition pass ------------------------------------------------------------------
      // Thread t owns the 16-byte chunk c (d = 4c .. 4c+3) of the four rows n = 8 q8 + 2i + e (i = 0..3):
      // kt_pos puts them at the consecutive k = 8 q8 + 4e + i, so after a 4x4 transpose in registers each d
      // is one 16-byte store into X^T.  The eight lanes of a quarter-warp (one phase of a 16-byte access)
      // take the eight (q8 & 3, e) and eight distinct chunks, chosen so that the 16-byte bank groups of both
      // the X loads (c ^ (n & 7)) and the X^T stores ((2 (q8 & 3) + e) ^ (d & 7)) are all different.
      {
        const int lam = t & 7, mu = t >> 3;
        const int e = lam & 1, q8 = ((mu >> 3) << 2) | (lam >> 1);
        const int c = (((lam & 1) << 2) | (lam >> 1)) ^ (mu & 7);
        float4* xs = reinterpret_cast<float4*>(sm + OFF_X + s * kTile);
        float4* xl = reinterpret_cast<float4*>(my + WG_XLO);
        float xr[4][4];                        // [i][q] = X[8 q8 + 2i + e][4c + q] rounded to nearest TF32
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = 8 * q8 + 2 * i + e;
          const int idx = r * 8 + (c ^ (r & 7));      // 16-byte chunk holding d = 4c .. 4c+3 of row r
          const float4 v = xs[idx];
          const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) xr[i][q] = tf32_rn(x[q]);
          if (SPLIT_X) {
            float h[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) h[q] = tf32_trunc(x[q]);
            xs[idx] = make_float4(h[0], h[1], h[2], h[3]);
            xl[idx] = make_float4(x[0] - h[0], x[1] - h[1], x[2] - h[2], x[3] - h[3]);
          } else {
            xs[idx] = make_float4(xr[i][0], xr[i][1], xr[i][2], xr[i][3]);
          }
        }
        // X^T[d][k]: k-block k >> 5, 16-byte chunk ((k & 31) >> 2) ^ (d & 7), element k & 3 (= i here)
        const int kc = 2 * (q8 & 3) + e;
        float4* xt = reinterpret_cast<float4*>(my + WG_XT + (q8 >> 2) * kXtBlock);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int d = 4 * c + q;
          xt[d * 8 + (kc ^ (d & 7))] = make_float4(xr[0][q], xr[1][q], xr[2][q], xr[3][q]);
        }
      }
      float2 yr[8];                            // y of the thread's rows n = 8j + 2 t4 + e, read before the refill
#pragma unroll
      for (int j = 0; j < 8; ++j) yr[j] = reinterpret_cast<const float2*>(sm + OFF_Y + s * kYBytes)[4 * j + t4];
      fence_proxy_async();
      wg_bar(1 + wg);
      // ---- GEMM 1: logits D1^T[p, n] = W X^T + b, accumulator initialised with the bias ---------------
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
      // GEMM 1 has read the X stage and y is in registers: refill the stage with tile it + 2 kWG
      if (t == 0 && it + 2 * kWG < nt) load(it + 2 * kWG, s);
      // ---- epilogue: lp sums and g, both in registers; the row mask only in the last, partial tile ------
      uint32_t g[32];                          // indexed like acc1
      float lin[2], prod[2];
      if (row0 + kRows > N)
        epilogue<true>(acc1, yr, row0, N, t4, lin, prod, g);
      else
        epilogue<false>(acc1, yr, row0, N, t4, lin, prod, g);
#pragma unroll
      for (int h = 0; h < 2; ++h) lpa[h] += fmaf(lg2f(prod[h]), -0.6931471805599453f, lin[h]);
      // ---- GEMM 2: [dW | db] += g [X | 1], g from registers, left running while the next tile is waited for
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
  float* red2 = reinterpret_cast<float*>(sm + OFF_X);     // [kWG][64 p][33]
  float* redlp = red2 + kWG * kP * 33;                    // [kWG][64 p]
  {
#pragma unroll
    for (int j = 0; j < 5; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int p = 16 * w4 + gid + 8 * h, c = 8 * j + 2 * t4 + e;
          if (c <= kD) red2[(wg * kP + p) * 33 + c] = acc2[4 * j + 2 * h + e];
        }
    if (t4 == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) redlp[wg * kP + 16 * w4 + gid + 8 * h] = lpa[h];
    }
  }
  __syncthreads();
  if (tid < kP) {
    const int gp = slab * kP + tid;
    if (gp < P) {
      float* o = partials + ((int64_t)blockIdx.x * P + gp) * (kD + 2);
      for (int c = 0; c <= kD; ++c) {          // dW[0..31], db
        float v = 0.f;
        for (int g = 0; g < kWG && g < nt; ++g) v += red2[(g * kP + tid) * 33 + c];
        o[c] = v;
      }
      float v = 0.f;
      for (int g = 0; g < kWG && g < nt; ++g) v += redlp[g * kP + tid];
      o[kD + 1] = v;
    }
  }
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
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) return B2_ERR_LAUNCH;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (N >= (int64_t)1 << 31) return B2_ERR_TOO_LARGE;
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
    if (enc(&my, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, const_cast<float*>(y), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B2_ERR_LAUNCH;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(glm_bernoulli_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    cudaFuncSetAttribute(glm_bernoulli_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    attr_set = true;
  }
  dim3 grid((unsigned)gx, (unsigned)((P + kP - 1) / kP), 1);
  if (split_x)
    launch_pdl(glm_bernoulli_tc_kernel<true>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, W, b, N, P, partials);
  else
    launch_pdl(glm_bernoulli_tc_kernel<false>, grid, dim3(kThreads), (size_t)kSmemBytes, s, mx, my, W, b, N, P, partials);
  return 0;
}

}  // namespace b2
