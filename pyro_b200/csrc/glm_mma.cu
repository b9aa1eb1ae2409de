// glm_mma.cu -- tensor-core version of the fused logistic-regression likelihood kernel.
//
// Same contract as glm_bernoulli_kernel (glm.cu): one pass over X[N,D] and y[N] gives, per particle,
// sum_n log Bernoulli(y_n | logits), dW and db.  The two contractions run on the tensor cores with
// TF32 operands and fp32 accumulation (mma.sync.m16n8k8):
//
//   GEMM 1 (per 8-row tile)  L^T[p, r] = sum_d W[p, d] X[r, d]        M = particles, N = rows, K = D
//   elementwise              g = y - sigmoid(l),  lp = y*l - softplus(l)   on the accumulator
//                            fragment, in registers
//   GEMM 2                   dW[p, d] += sum_r g[p, r] X[r, d]        M = particles, N = D, K = rows
//
// GEMM 1 is computed TRANSPOSED so that its accumulator fragment (c0..c3 = particles {g, g+8} x rows
// {2t, 2t+1}) is, register for register, the A fragment GEMM 2 needs once the 8 rows of the tile are
// taken in the order (0,2,4,6,1,3,5,7): no shuffles, no shared-memory round trip (the trick
// flash-attention uses between Q K^T and P V).  The B fragments of both GEMMs are read from the same
// shared-memory X tile (row pitch 36 floats: both access patterns are bank-conflict free).
//
// This is the legacy tensor-core path (B2_FLAG_GLM_MMA_SYNC); the default for D == 32 is the
// wgmma/TMA kernel of glm_tc.cu.  Both are bounded by the SFU work of the epilogue (3 MUFU per
// (row, particle)) rather than by the contractions.
//
// Precision: TF32 operands (10-bit mantissa, round-to-nearest) perturb each logit by ~1e-3 relative;
// the errors are unbiased and average out over the N-term sums.  The fp32 SIMT kernel in glm.cu stays available (flag B2_GLM_FP32).
#include <cuda_pipeline.h>

#include "b2_common.cuh"
#include "b2_math.cuh"

namespace b2 {

constexpr int kMmaTileRows = 64;                 // rows staged per CTA iteration
constexpr int kMmaPitch = 36;                    // floats per staged row (32 + 4 pad)
constexpr int kMmaWarps = 8;                     // 4 row groups x 2 particle halves
constexpr int kMmaParticles = 64;                // particles per CTA (blockIdx.y slabs)

// fp32 -> tf32 with round-to-nearest (ties away), done with two integer ALU ops.  cvt.rna.tf32.f32
// executes on the same 16-lane pipe as MUFU; at 3 conversions per (row, particle) it doubled the
// load of the pipe that bounds this kernel.
__device__ __forceinline__ uint32_t to_tf32(float x) {
  return (__float_as_uint(x) + 0x1000u) & 0xffffe000u;
}

// D(16x8, f32) += A(16x8, tf32, row) * B(8x8, tf32, col)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float lg2_ftz(float x) {
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// D must be 32 (four k-steps / four n-tiles of 8).
__global__ void __launch_bounds__(256, 2) glm_bernoulli_mma_kernel(const float* __restrict__ X,
                                                                   const float* __restrict__ y,
                                                                   const float* __restrict__ W,
                                                                   const float* __restrict__ b, int64_t N,
                                                                   int P, float* __restrict__ partials) {
  constexpr int D = 32;
  __shared__ __align__(16) float xs[2][kMmaTileRows * kMmaPitch];
  __shared__ float ys[2][kMmaTileRows];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int half = warp & 1;        // which 32 particles of the 64-particle slab
  const int rgroup = warp >> 1;     // which 16 rows of every 64-row tile
  const int pbase = blockIdx.y * kMmaParticles + half * 32;

  // ---- W fragments (A operand of GEMM 1), constant for the whole kernel ------------------------------
  uint32_t wa[2][4][4];
  float bias[2][2];
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int p0 = pbase + m * 16 + g, p1 = p0 + 8;
    bias[m][0] = (b && p0 < P) ? b[p0] : 0.f;
    bias[m][1] = (b && p1 < P) ? b[p1] : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int d0 = k * 8 + t, d1 = d0 + 4;
      wa[m][k][0] = to_tf32(p0 < P ? W[(int64_t)p0 * D + d0] : 0.f);
      wa[m][k][1] = to_tf32(p1 < P ? W[(int64_t)p1 * D + d0] : 0.f);
      wa[m][k][2] = to_tf32(p0 < P ? W[(int64_t)p0 * D + d1] : 0.f);
      wa[m][k][3] = to_tf32(p1 < P ? W[(int64_t)p1 * D + d1] : 0.f);
    }
  }
  float dw[2][4][4];   // [m-tile][n-tile over D][c0..c3]
  float sum[2][2], db[2][2];
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    sum[m][0] = sum[m][1] = db[m][0] = db[m][1] = 0.f;
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int i = 0; i < 4; ++i) dw[m][n][i] = 0.f;
  }

  const int64_t ntiles = (N + kMmaTileRows - 1) / kMmaTileRows;
  auto stage = [&](int buf, int64_t tile) {
    const int64_t row0 = tile * kMmaTileRows;
    const int rows = (int)((N - row0 < kMmaTileRows) ? (N - row0) : kMmaTileRows);
    // 64 rows x 8 chunks of 16 B; thread i copies chunk (i & 7) of row (i >> 3), two passes
    for (int i = tid; i < kMmaTileRows * 8; i += 256) {
      const int r = i >> 3, c = i & 7;
      float* dst = &xs[buf][r * kMmaPitch + c * 4];
      if (r < rows) __pipeline_memcpy_async(dst, X + (row0 + r) * D + c * 4, 16);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < kMmaTileRows) {
      if (tid < rows) __pipeline_memcpy_async(&ys[buf][tid], y + row0 + tid, 4);
      else ys[buf][tid] = 0.f;
    }
    __pipeline_commit();
  };

  int64_t tile = blockIdx.x;
  int buf = 0;
  if (tile < ntiles) stage(0, tile);
  for (; tile < ntiles; tile += gridDim.x) {
    const int64_t next = tile + gridDim.x;
    if (next < ntiles) stage(buf ^ 1, next);
    else __pipeline_commit();
    __pipeline_wait_prior(1);
    __syncthreads();
    const int64_t row0 = tile * kMmaTileRows;
    const int rows = (int)((N - row0 < kMmaTileRows) ? (N - row0) : kMmaTileRows);
    const float* xt = xs[buf];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {              // two 8-row n-tiles per row group
      const int r0 = rgroup * 16 + nt * 8;
      if (r0 >= rows) break;
      // ---- B fragments of GEMM 1: X[r0 + g][8k + t], X[r0 + g][8k + t + 4] ------------------------
      uint32_t xb[4][2];
      const float* xrow = xt + (r0 + g) * kMmaPitch;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        xb[k][0] = to_tf32(xrow[k * 8 + t]);
        xb[k][1] = to_tf32(xrow[k * 8 + t + 4]);
      }
      // ---- B fragments of GEMM 2: X[r0 + 2t][8n + g], X[r0 + 2t + 1][8n + g] ----------------------
      uint32_t xc[4][2];
      const float* xr2 = xt + (r0 + 2 * t) * kMmaPitch;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        xc[n][0] = to_tf32(xr2[n * 8 + g]);
        xc[n][1] = to_tf32(xr2[kMmaPitch + n * 8 + g]);
      }
      const float y0 = ys[buf][r0 + 2 * t], y1 = ys[buf][r0 + 2 * t + 1];
      // rows beyond the end of the data (last tile only) are masked by a 0/1 weight
      const float v0 = (r0 + 2 * t) < rows ? 1.f : 0.f, v1 = (r0 + 2 * t + 1) < rows ? 1.f : 0.f;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        // logits^T fragment: c0 = (p = g, r = 2t), c1 = (g, 2t+1), c2 = (g+8, 2t), c3 = (g+8, 2t+1)
        float c[4] = {bias[m][0], bias[m][0], bias[m][1], bias[m][1]};
#pragma unroll
        for (int k = 0; k < 4; ++k) mma_tf32(c, wa[m][k], xb[k][0], xb[k][1]);
        float gv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float l = c[i];
          const float yy = (i & 1) ? y1 : y0;
          const float vw = (i & 1) ? v1 : v0;
          // e = exp(-|l|) in (0, 1]; SFU ops issued directly (ftz forms: no denormal fix-up code)
          const float e = ex2_ftz(-1.4426950408889634f * fabsf(l));
          const float den = 1.f + e;
          float inv;
          asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(den));
          const float sp = fmaf(lg2_ftz(den), 0.6931471805599453f, fmaxf(l, 0.f));
          const float sg = (l >= 0.f) ? inv : e * inv;
          const float lp = vw * fmaf(yy, l, -sp);
          const float gg = vw * (yy - sg);
          sum[m][i >> 1] += lp;
          db[m][i >> 1] += gg;
          gv[i] = gg;
        }
        // A fragment of GEMM 2 with the row order (0,2,4,6,1,3,5,7):
        //   a0 = G[g][k=t]   -> row 2t   = c0      a1 = G[g+8][k=t]   -> c2
        //   a2 = G[g][k=t+4] -> row 2t+1 = c1      a3 = G[g+8][k=t+4] -> c3
        const uint32_t ga[4] = {to_tf32(gv[0]), to_tf32(gv[2]), to_tf32(gv[1]), to_tf32(gv[3])};
#pragma unroll
        for (int n = 0; n < 4; ++n) mma_tf32(dw[m][n], ga, xc[n][0], xc[n][1]);
      }
    }
    __syncthreads();
    buf ^= 1;
  }
  __pipeline_wait_prior(0);
  __syncthreads();

  // ---- reduce: lanes t (rows) by shuffles, row groups through shared memory -----------------------------
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float s = sum[m][h], d = db[m][h];
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      sum[m][h] = s;
      db[m][h] = d;
    }
  // table[rgroup][particle (64)][D + 2]
  float* table = &xs[0][0];  // 2 * 64 * 36 = 4608 floats available; need 4 * 64 * 34 = 8704 -> two passes
  float* out = partials + (int64_t)blockIdx.x * P * (D + 2);
  for (int pass = 0; pass < 2; ++pass) {
    // pass 0: row groups 0,1 -> table; pass 1: row groups 2,3 -> accumulate into registers of groups 0,1
    __syncthreads();
    if ((rgroup >> 1) == 1 - pass) {
      // writers: in pass 0 groups 2,3 park their values; in pass 1 groups 0,1 (already merged) write
      const int slot = rgroup & 1;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int pl0 = half * 32 + m * 16 + g, pl1 = pl0 + 8;
        float* t0 = table + ((slot * 64 + pl0) * (D + 2));
        float* t1 = table + ((slot * 64 + pl1) * (D + 2));
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          t0[n * 8 + 2 * t] = dw[m][n][0];
          t0[n * 8 + 2 * t + 1] = dw[m][n][1];
          t1[n * 8 + 2 * t] = dw[m][n][2];
          t1[n * 8 + 2 * t + 1] = dw[m][n][3];
        }
        if (t == 0) {
          t0[D] = db[m][0]; t0[D + 1] = sum[m][0];
          t1[D] = db[m][1]; t1[D + 1] = sum[m][1];
        }
      }
    }
    __syncthreads();
    if (pass == 0 && (rgroup >> 1) == 0) {
      // groups 0,1 absorb groups 2,3 (slot = rgroup & 1 pairs 0<-2, 1<-3)
      const int slot = rgroup & 1;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int pl0 = half * 32 + m * 16 + g, pl1 = pl0 + 8;
        const float* t0 = table + ((slot * 64 + pl0) * (D + 2));
        const float* t1 = table + ((slot * 64 + pl1) * (D + 2));
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          dw[m][n][0] += t0[n * 8 + 2 * t];
          dw[m][n][1] += t0[n * 8 + 2 * t + 1];
          dw[m][n][2] += t1[n * 8 + 2 * t];
          dw[m][n][3] += t1[n * 8 + 2 * t + 1];
        }
        db[m][0] += t0[D]; sum[m][0] += t0[D + 1];
        db[m][1] += t1[D]; sum[m][1] += t1[D + 1];
      }
    }
  }
  __syncthreads();
  // table now holds slots 0 (groups 0+2) and 1 (groups 1+3): add them in a fixed order and write
  for (int e = tid; e < kMmaParticles * (D + 2); e += 256) {
    const int pl = e / (D + 2);
    const int p = blockIdx.y * kMmaParticles + pl;
    if (p < P) out[(int64_t)p * (D + 2) + (e - pl * (D + 2))] = table[e] + table[kMmaParticles * (D + 2) + e];
  }
}

}  // namespace b2

namespace b2 {
int glm_mma_grid_x(int64_t N) {
  const int64_t ntiles = (N + kMmaTileRows - 1) / kMmaTileRows;
  int64_t gx = (int64_t)kNumSMs * 2;
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  return (int)gx;
}
void launch_glm_mma(const float* X, const float* y, const float* W, const float* b, int64_t N, int P,
                    float* partials, int gx, cudaStream_t s) {
  dim3 grid((unsigned)gx, (unsigned)((P + kMmaParticles - 1) / kMmaParticles), 1);
  glm_bernoulli_mma_kernel<<<grid, 256, 0, s>>>(X, y, W, b, N, P, partials);
}
}  // namespace b2
