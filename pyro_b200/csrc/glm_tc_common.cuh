// glm_tc_common.cuh -- device helpers shared by the Hopper wgmma kernels (glm_tc.cu, glm_flat_tc.cu,
// glm_categorical_tc.cu, poisson_product_tc.cu): mbarriers, TMA tile loads, SWIZZLE_128B operand
// descriptors, the TF32 wgmma wrappers, MUFU wrappers and TF32 rounding, the Bernoulli epilogue, and the
// host-side tensor-map encoder.
#pragma once
#include <cuda.h>

#include "b2_common.cuh"

namespace b2 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// The retry loop lives inside the asm block: a C++ loop around try_wait is a divergent branch to ptxas, and
// wgmma accumulators live across a divergent path make it serialise every wgmma of the kernel (C7520).
// After 2^26 failed tries it traps: a protocol bug must not hang the device.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
      "mov.u32 n, 0;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 67108864;\n\t"
      "@p bra.uni WAIT;\n\t"
      "trap;\n"
      "DONE:\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const CUtensorMap* map, int c0, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void wg_bar(int id) {   // named barrier of one warpgroup (ids 1..kWG)
  asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory");
}

// wgmma shared-memory matrix descriptor: start address >> 4 in [0,14), leading byte offset >> 4 in [16,30)
// (unused for swizzled K-major operands), stride byte offset >> 4 in [32,46) (8-row groups are 1024 bytes
// apart), layout type in [62,64) (1 = SWIZZLE_128B).  A k-step inside the 128-byte atom adds 32 bytes (+2).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from touching accumulator registers while an asynchronous wgmma owns them
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// pins register A operands before wgmma.fence (a definition after it makes ptxas insert warpgroup.arrive)
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// D[64 x 64] += A[64 x 8] B[64 x 8]^T, TF32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_n64_tf32(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1)
      : "memory");
}
// D[64 x 40] = A[64 x 8] B[40 x 8]^T (+ D when acc != 0), TF32, A from registers: thread (warp w4 of the
// warpgroup, lane = 4 gid + t4) passes a[i] = A[16 w4 + gid + 8 (i & 1)][t4 + 4 (i >> 1)]
__device__ __forceinline__ void wgmma_n40_tf32_ra(float (&d)[20], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %25, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n40k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, "
      "{%20, %21, %22, %23}, %24, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

// D[64 x 16] = A[64 x 8] B[16 x 8]^T (+ D when acc != 0), TF32, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_n16_tf32(float (&d)[8], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(acc)
      : "memory");
}
// D[64 x 16] = A[64 x 8] B[16 x 8]^T (+ D when acc != 0), TF32, A from registers (layout of wgmma_n40_tf32_ra)
__device__ __forceinline__ void wgmma_n16_tf32_ra(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

// float offset of element (row, col), col < 32, in a K-major SWIZZLE_128B operand of 32-float rows
__device__ __forceinline__ int sw128(int row, int col) {
  return row * 32 + ((((col >> 2) ^ (row & 7)) << 2) | (col & 3));
}

__device__ __forceinline__ float ex2f(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float lg2f(float x) {
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float rcpf(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ float tf32_rn(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

// Position of tile row n in GEMM 2's k order.  GEMM 1's accumulator gives a thread the rows n = 8j + 2 t4 + e
// (e = 0, 1) of k-block j, and the register A operand of GEMM 2 takes them as k = t4 + 4e; X^T is stored in
// that order, so g never leaves the registers.
__device__ __forceinline__ int kt_pos(int n) { return (n & ~7) | ((n & 7) >> 1) | ((n & 1) << 2); }

// ---- Bernoulli epilogue of the logistic-regression kernels (glm_tc.cu, glm_flat_tc.cu) ----------------------
constexpr int kEpiBatch = 4;                    // logits of one particle per epilogue batch (8 fits, no faster)

// lp = y*l - softplus(l) = y*l - max(l, 0) - ln(1 + e^-|l|).  The epilogue sums the linear part per tile and
// multiplies the denominators den = 1 + e^-|l| instead of taking a logarithm of each: den is in (1, 2], so
// the product of a thread's 16 rows of one particle is at most 2^16, and one lg2 per particle and tile
// replaces 16.  Rounding: each of the 15 products adds at most 2^-24 relative, at most 15 * 2^-24 = 9e-7
// nats per 16 logits, no worse than the sixteen lg2.approx results it replaces (about 1e-7 nats each).
//
// One batch of B logits of one particle, stage by stage: each MUFU result is consumed a stage (>= B
// instructions) after it was issued, and the four warps per scheduler cover the rest of the MUFU latency.
// Returns the sum of y*l - max(l, 0) over the batch, multiplies the batch's den into prod and writes
// g = y - sigmoid(l) rounded to nearest TF32.  MASK weights the linear part and g with vw (0 for rows past
// N) and gives a masked row the factor 1 exactly.
template <bool MASK, int B>
__device__ __forceinline__ float epi_batch(const float* lr, const float* y, const float* vw, float& prod,
                                           uint32_t* g) {
  float e[B], den[B], inv[B], f[B], lp[B];
#pragma unroll
  for (int j = 0; j < B; ++j) e[j] = ex2f(-1.4426950408889634f * fabsf(lr[j]));
#pragma unroll
  for (int j = 0; j < B; ++j) den[j] = 1.f + e[j];
#pragma unroll
  for (int j = 0; j < B; ++j) inv[j] = rcpf(den[j]);
#pragma unroll
  for (int j = 0; j < B; ++j) f[j] = MASK ? fmaf(vw[j], e[j], 1.f) : den[j];
#pragma unroll
  for (int j = 0; j < B; ++j) {
    const float l = lr[j];
    lp[j] = fmaf(y[j], l, -fmaxf(l, 0.f));
    const float sg = (l >= 0.f) ? inv[j] : e[j] * inv[j];
    float gg = y[j] - sg;
    if (MASK) {
      lp[j] *= vw[j];
      gg *= vw[j];
    }
    g[j] = __float_as_uint(tf32_rn(gg));
  }
#pragma unroll
  for (int w = 1; w < B; w *= 2)
#pragma unroll
    for (int j = 0; j < B; j += 2 * w) {
      lp[j] += lp[j + w];
      f[j] *= f[j + w];
    }
  prod *= f[0];
  return lp[0];
}

// The epilogue of one tile: the linear lp sums lin[h] and den products prod[h] of the thread's two particles
// (16 rows each), and g indexed like acc1.  MASK (the last, partial tile only) zeroes rows past N.
template <bool MASK>
__device__ __forceinline__ void epilogue(const float (&acc1)[32], const float2 (&yr)[8], int64_t row0, int64_t N,
                                         int t4, float (&lin)[2], float (&prod)[2], uint32_t (&g)[32]) {
  constexpr int B = kEpiBatch;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    prod[h] = 1.f;
#pragma unroll
    for (int q = 0; q < 16 / B; ++q) {         // k-blocks j = B/2 q .. B/2 q + B/2 - 1
      float l[B], yy[B], vw[B];
      uint32_t gb[B];
#pragma unroll
      for (int i = 0; i < B; ++i) {
        const int j = B / 2 * q + (i >> 1), e = i & 1;
        l[i] = acc1[4 * j + 2 * h + e];
        yy[i] = e ? yr[j].y : yr[j].x;
        vw[i] = MASK ? ((row0 + 8 * j + 2 * t4 + e < N) ? 1.f : 0.f) : 1.f;
      }
      const float s = epi_batch<MASK, B>(l, yy, vw, prod[h], gb);
      lin[h] = q ? lin[h] + s : s;
#pragma unroll
      for (int i = 0; i < B; ++i) g[4 * (B / 2 * q + (i >> 1)) + 2 * h + (i & 1)] = gb[i];
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace tc
}  // namespace b2
