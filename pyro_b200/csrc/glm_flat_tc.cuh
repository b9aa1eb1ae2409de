// glm_flat_tc.cuh -- the any-D tile loop of the Hopper GLM likelihood kernels: glm_flat_pipeline<Fam, DC,
// SPLIT_X> runs one likelihood family (glm_tc_common.cuh: Bernoulli for glm_flat_tc.cu, Poisson for
// glm_poisson_tc.cu) for any feature count D in 1..128.
//
// Same contract as the D = 32 tile pipeline (glm_tc_common.cuh): ONE pass over X[N,D] and y[N] gives, for up
// to 64 weight vectors (particles) per CTA slab, sum_n lp(y_n | l_n = x_n.w_p + b_p), dW and db, as CTA
// partials [gridDim.x][P][D + 2] that glm_finish_kernel adds in a fixed order.
//
// D is padded to DC = ceil(D / 32) swizzle atoms of 32 columns (KD = 32 DC).  A 2-D TMA load needs a row
// stride that is a multiple of 16 bytes, which 4 D mostly is not; but the 64 rows of a tile are one
// contiguous block of 256 D bytes, 16-byte aligned when X is.  So each tile arrives by ONE 1-D bulk copy
// (cp.async.bulk, completing on an mbarrier) into an unswizzled [64][D] landing buffer, and its y the same
// way.  The last tile's byte count need not be a multiple of 16: the thread that issues the copies writes
// its last (< 4) floats, and the y of rows past N as zeros, with ordinary loads and stores first, so nothing
// is read past the end of X or y.
//
// Per 64-row tile (persistent CTAs, tiles round-robin over CTAs and inside a CTA over its warpgroups):
//
//   split    the warpgroup reads the landing buffer and writes the padded SWIZZLE_128B GEMM 1 operand
//            (X rounded to nearest TF32, or X_hi / X_lo under SPLIT_X) and the transposed X^T (rows kt_pos
//            permuted like glm_tc.cu, plus 8 rows of ones) that is GEMM 2's B operand.  Columns d >= D and
//            rows past N are written as exact zeros: a landing buffer that was never written, or that holds
//            another tile, may hold NaN bit patterns, and 0 * NaN = NaN.  Then the landing buffer is refilled
//            with the warpgroup's next tile, which arrives while this tile is contracted.
//   GEMM 1   D1^T[p, n] = sum_d W[p, d] X[n, d] + b[p]    wgmma m64n64k8 over 4 DC k-steps, W split hi + lo.
//   epilogue the family's tile_epilogue (glm_tc_common.cuh): lp sums and g = dlp/dl rounded to TF32, in
//            registers; only the last, partial tile masks rows.
//   GEMM 2   [dW | db][p, :] += sum_n g[p, n] [X | 1][n, :]   wgmma m64n(KD + 8)k8, A = g from registers;
//            db is accumulator column KD.  Committed and left running while the next tile is waited for.
//
// Precision policy of glm_tc.cu: W always split, X split under SPLIT_X, g rounded to nearest TF32.
//
// Budget: at DC = 4 one warpgroup holds W hi + lo (64 KB), X hi + lo (64 KB), X^T (34 KB) and a landing tile
// (32 KB), and its GEMM 2 accumulator alone takes 68 registers.  So DC = 1 runs four warpgroups per CTA (the
// 128-register cap of glm_tc.cu), DC = 2 two and DC >= 3 one, each with a single landing stage.
//
// Determinism: every CTA writes its partials once (warpgroups summed in a fixed order); no float atomics.
#pragma once
#include <cuda.h>

#include "b2_common.cuh"
#include "glm_tc_common.cuh"

namespace b2 {
namespace tcf {

using namespace tc;

template <int DC>
struct Cfg {
  static constexpr int kKD = 32 * DC;                          // padded feature count
  static constexpr int kN2 = kKD + 8;                          // GEMM 2 width: dW columns, db, 7 unused
  static constexpr int kWG = DC == 1 ? 4 : DC == 2 ? 2 : 1;    // warpgroups per CTA
  static constexpr int kThreads = 128 * kWG;
  static constexpr uint32_t kOp = DC * 8192u;                  // [DC atoms][64 rows][32] fp32, SW128
  static constexpr uint32_t kXtBlock = kN2 * 128u;             // X^T k-block: KD + 8 rows of 32 n
  // per-warpgroup region
  static constexpr uint32_t WG_XOP = 0;                        // GEMM 1 operand: rounded X or X_hi
  static constexpr uint32_t WG_XLO = WG_XOP + kOp;             // X_lo (SPLIT_X)
  static constexpr uint32_t WG_XT = WG_XLO + kOp;              // X^T [kb 2][c KD + 8][32 n], n permuted (kt_pos)
  static constexpr uint32_t WG_LAND = WG_XT + 2 * kXtBlock;    // landing buffer [64][D], unswizzled
  static constexpr uint32_t WG_Y = WG_LAND + kOp;              // y [64]
  static constexpr uint32_t kWGBytes = WG_Y + 1024;
  // CTA layout (operand regions 1024-byte aligned: the 128-byte swizzle pattern is taken from address bits)
  static constexpr uint32_t OFF_WHI = 0;                       // [DC][p 64][32] SW128
  static constexpr uint32_t OFF_WLO = OFF_WHI + kOp;
  static constexpr uint32_t OFF_WG = OFF_WLO + kOp;
  static constexpr uint32_t OFF_BAR = OFF_WG + kWG * kWGBytes;
  static constexpr uint32_t kSmemBytes = OFF_BAR + 64 + 1024;  // + slack for the 1024-byte alignment
  // the final reduction reuses the warpgroup regions: [kWG][64 p][KD + 1] + [kWG][64 p] floats
  static constexpr int kRS = kKD + 1;
  static_assert(kSmemBytes <= 232448, "shared memory budget");
  static_assert(kXtBlock % 1024 == 0 && kWGBytes % 1024 == 0, "operand alignment");
  static_assert((kWG * kM * kRS + kWG * kM) * 4 <= kWG * kWGBytes, "reduction scratch");
};

// one 1-D bulk copy global -> shared, completing `bytes` (a non-zero multiple of 16) on the mbarrier
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// wgmma accumulator fragment (m64nN, f32): thread (warp w4 of the warpgroup, lane = 4 gid + t4) holds
// d[4j + 2h + e] = D[16 w4 + gid + 8h][8j + 2 t4 + e].
template <class Fam, int DC, bool SPLIT_X>
__device__ __forceinline__ void glm_flat_pipeline(const float* __restrict__ X, const float* __restrict__ y,
                                                  const float* __restrict__ W, const float* __restrict__ bvec,
                                                  int64_t N, int D, int P, float* __restrict__ partials) {
  using C = Cfg<DC>;
  constexpr int kKD = C::kKD, kWG = C::kWG;
  pdl_enter();   // lets glm_finish_kernel be resident (blocked in its griddepcontrol.wait) before this kernel ends
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int slab = blockIdx.y;
  const int64_t ntiles = (N + kRows - 1) / kRows;
  // tiles handled by this CTA: blockIdx.x, blockIdx.x + gridDim.x, ...
  const int nt = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);

  // ---- one-time setup --------------------------------------------------------------------------------
  if (tid == 0) {
    for (int s = 0; s < kWG; ++s) mbar_init(base + C::OFF_BAR + 8u * (uint32_t)s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // weight tiles, zero in the padding columns d >= D, and the ones rows of X^T
  stage_w_and_ones<1, kKD, C::kThreads>(reinterpret_cast<float*>(sm + C::OFF_WHI),
                                        reinterpret_cast<float*>(sm + C::OFF_WLO), sm + C::OFF_WG + C::WG_XT,
                                        C::kWGBytes, W, slab, P, 1, D);
  fence_proxy_async();
  __syncthreads();

  float lpa[2] = {0.f, 0.f};                   // lp sums of the thread's two particles
  // GEMM 2 accumulator [p][c]: dW in c < D, db in c = KD.  Started by the warpgroup's first GEMM 2 k-step
  // with scale-d = 0, never written by ordinary instructions before the tile loop (C7515, see glm_tc.cu).
  float acc2[C::kN2 / 2];
  // warp-uniform by construction (a shuffle result), so the tile loop is not a divergent branch to ptxas
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), w4 = warp & 3, t = tid & 127;
  const int gid = lane >> 2, t4 = lane & 3;

  {
    uint8_t* my = sm + C::OFF_WG + wg * C::kWGBytes;
    const uint32_t my_s = base + C::OFF_WG + wg * C::kWGBytes;
    const uint32_t bar = base + C::OFF_BAR + 8u * (uint32_t)wg;
    float* land = reinterpret_cast<float*>(my + C::WG_LAND);
    float* ys = reinterpret_cast<float*>(my + C::WG_Y);
    float bias[2];                             // of particles 16 w4 + gid + 8h
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gp = slab * kM + 16 * w4 + gid + 8 * h;
      bias[h] = (bvec != nullptr && gp < P) ? bvec[gp] : 0.f;
    }
    // tile it -> landing buffer; one thread of the warpgroup issues the loads
    auto load = [&](int it) {
      const int64_t row0 = (blockIdx.x + (int64_t)it * gridDim.x) * kRows;
      const int rows = (int)(N - row0 < kRows ? N - row0 : kRows);
      const uint32_t xb = (uint32_t)(rows * D) * 4u, yb = (uint32_t)rows * 4u;
      const uint32_t xbulk = xb & ~15u, ybulk = yb & ~15u;
      if (rows < kRows || xbulk != xb) {       // the last tile: its remainder and zeros for y past N
        const float* xsrc = X + row0 * D;
        for (uint32_t i = xbulk / 4; i < xb / 4; ++i) land[i] = xsrc[i];
        for (int i = (int)(ybulk / 4); i < kRows; ++i) ys[i] = (i < rows) ? y[row0 + i] : 0.f;
      }
      // the arrive releases the ordinary stores above to the warpgroup's mbar_wait
      mbar_expect_tx(bar, xbulk + ybulk);
      if (xbulk) bulk_load(my_s + C::WG_LAND, X + row0 * D, xbulk, bar);
      if (ybulk) bulk_load(my_s + C::WG_Y, y + row0, ybulk, bar);
    };
    if (t == 0 && wg < nt) load(wg);
    for (int k = 0, it = wg; it < nt; ++k, it += kWG) {
      const int64_t row0 = (blockIdx.x + (int64_t)it * gridDim.x) * kRows;
      const int rows = (int)(N - row0 < kRows ? N - row0 : kRows);
      mbar_wait(bar, (uint32_t)k & 1u);
      // GEMM 2 of this warpgroup's previous tile has finished reading X^T and the g registers
      wgmma_wait0();
      fence_regs(acc2);
      // ---- split pass, once per 32-column atom, with the thread mapping of the D = 32 pipeline
      // (glm_tc_common.cuh): columns d >= D and rows past N are exact zeros --------------------------------
      {
        const int lam = t & 7, mu = t >> 3;
        const int e = lam & 1, q8 = ((mu >> 3) << 2) | (lam >> 1);
        const int c = (((lam & 1) << 2) | (lam >> 1)) ^ (mu & 7);
        const int kc = 2 * (q8 & 3) + e;
        float4* xs = reinterpret_cast<float4*>(my + C::WG_XOP);
        float4* xl = reinterpret_cast<float4*>(my + C::WG_XLO);
        float4* xt = reinterpret_cast<float4*>(my + C::WG_XT + (q8 >> 2) * C::kXtBlock);
#pragma unroll
        for (int a = 0; a < DC; ++a) {
          float xr[4][4];                      // [i][q] = X[8 q8 + 2i + e][32 a + 4c + q] rounded to TF32
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = 8 * q8 + 2 * i + e;
            const int idx = a * 512 + r * 8 + (c ^ (r & 7));
            float x[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int d = 32 * a + 4 * c + q;
              const float v = land[r * D + min(d, D - 1)];
              x[q] = (d < D && r < rows) ? v : 0.f;
              xr[i][q] = tf32_rn(x[q]);
            }
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
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int d = 32 * a + 4 * c + q;
            xt[d * 8 + (kc ^ (d & 7))] = make_float4(xr[0][q], xr[1][q], xr[2][q], xr[3][q]);
          }
        }
      }
      typename Fam::Labels yr;                 // read before the refill
      Fam::read_labels(reinterpret_cast<const uint8_t*>(ys), t4, 1, yr);
      fence_proxy_async();
      wg_bar(1 + wg);
      // the landing buffer is free: the warpgroup's next tile arrives while this one is contracted
      if (t == 0 && it + kWG < nt) load(it + kWG);
      float acc1[32];
      if constexpr (Fam::kBiasInEpilogue) {
        const float zero[2] = {0.f, 0.f};
        gemm1<DC, SPLIT_X>(acc1, zero, base + C::OFF_WHI, base + C::OFF_WLO, my_s + C::WG_XOP, my_s + C::WG_XLO);
      } else {
        gemm1<DC, SPLIT_X>(acc1, bias, base + C::OFF_WHI, base + C::OFF_WLO, my_s + C::WG_XOP, my_s + C::WG_XLO);
      }
      uint32_t g[32];                          // indexed like acc1
      if constexpr (Fam::kBiasInEpilogue)
        Fam::tile_epilogue(acc1, bias, yr, row0, N, t4, rows < kRows, lpa, g);
      else
        Fam::tile_epilogue(acc1, yr, row0, N, t4, rows < kRows, lpa, g);
      // left running while the next tile is waited for
      gemm2<C::kN2>(acc2, g, my_s + C::WG_XT, it == wg);
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
  // CTA results through the warpgroup regions, idle now
  cta_partials<1, C::kN2, C::kThreads>(reinterpret_cast<float*>(sm + C::OFF_WG), acc2, lpa, wg, nt, slab, P, 1, D,
                                       partials);
}

}  // namespace tcf
}  // namespace b2
