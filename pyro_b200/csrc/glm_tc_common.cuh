// glm_tc_common.cuh -- device helpers shared by the Hopper wgmma kernels (glm_tc.cu, glm_flat_tc.cu,
// glm_categorical_tc.cu, glm_poisson_tc.cu, glm_normal_tc.cu, glm_binomial_tc.cu, poisson_product_tc.cu): mbarriers,
// TMA tile loads, SWIZZLE_128B operand descriptors, the TF32 wgmma wrappers, MUFU wrappers and TF32 rounding, the
// Bernoulli, Poisson, Normal and Binomial epilogues and families, the stages of the GLM tile pipeline and the D = 32 pipeline itself, and the
// host-side tensor-map encoders.
#pragma once
#include <cuda.h>

#include "b2_common.cuh"
#include "b2_math.cuh"

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

// D[64 x N] = A[64 x 8] B[N x 8]^T (+ D when acc != 0), TF32, A from registers, B K-major in shared memory:
// thread (warp w4 of the warpgroup, lane = 4 gid + t4) passes a[i] = A[16 w4 + gid + 8 (i & 1)][t4 + 4 (i >> 1)]
template <int N>
__device__ __forceinline__ void wgmma_tf32_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b, int acc);
template <>
__device__ __forceinline__ void wgmma_tf32_ra<16>(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<40>(float (&d)[20], const uint32_t (&a)[4], uint64_t b, int acc) {
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
template <>
__device__ __forceinline__ void wgmma_tf32_ra<72>(float (&d)[36], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %41, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n72k8.f32.tf32.tf32 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20,"
      "%21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35"
      "}, {%36, %37, %38, %39}, %40, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<104>(float (&d)[52], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %57, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n104k8.f32.tf32.tf32 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20,"
      "%21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39,"
      "%40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51"
      "}, {%52, %53, %54, %55}, %56, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<136>(float (&d)[68], const uint32_t (&a)[4], uint64_t b, int acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %73, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n136k8.f32.tf32.tf32 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20,"
      "%21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39,"
      "%40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58,"
      "%59, %60, %61, %62, %63, %64, %65, %66, %67"
      "}, {%68, %69, %70, %71}, %72, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67])
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

constexpr int kRows = 64;                       // rows per tile = N of GEMM 1 = K of GEMM 2
constexpr int kM = 64;                          // GEMM 1 rows per slab

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

// The Bernoulli epilogue with its lp update: lpa[h] += the lp sum of particle h over the tile, one lg2 each.
// Only the last, partial tile (last) takes the row mask.
__device__ __forceinline__ void bernoulli_epilogue(const float (&acc1)[32], const float2 (&yr)[8], int64_t row0,
                                                   int64_t N, int t4, bool last, float (&lpa)[2],
                                                   uint32_t (&g)[32]) {
  float lin[2], prod[2];
  if (last)
    epilogue<true>(acc1, yr, row0, N, t4, lin, prod, g);
  else
    epilogue<false>(acc1, yr, row0, N, t4, lin, prod, g);
#pragma unroll
  for (int h = 0; h < 2; ++h) lpa[h] += fmaf(lg2f(prod[h]), -0.6931471805599453f, lin[h]);
}

// ---- Poisson epilogue of the log-link regression kernels (glm_poisson_tc.cu) -------------------------------
// lp = y*l - e^l (the parameter-free -lgamma(y + 1) is summed once per call, not here) and g = y - e^l rounded
// to nearest TF32: ONE MUFU op (ex2) per logit.  MASK (the last, partial tile only) zeroes rows past N.
// Above l = 88.72 e^l is +inf: lp and g are then -inf, never NaN.
// lpa is fp64 (see Poisson): a row's y*l - e^l is hundreds of nats at counts of 100 and cancels against lgamma(y + 1)
// to a few, so the sum over a thread's tiles must not round at the scale of the terms; the 16 rows of one tile are
// still summed in fp32.
// The bias is added here, rounded to nearest, not carried by GEMM 1's accumulator: the tensor cores truncate
// each fp32 accumulation, and from an accumulator of |b| (a log-rate of a few units) every k-step shifts l
// toward zero by about half an ulp of b.  That shift enters the sum as SUM (y - e^l) dl, which does not cancel
// for a particle away from the data's optimum: at counts of mean 100 and b off by 0.05 it cost 2.3e-5 of
// sum_p at D = 100 (48 accumulation steps), against 7.5e-6 at D = 32 (12 steps).
template <bool MASK>
__device__ __forceinline__ void poisson_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                 const float2 (&yr)[8], int64_t row0, int64_t N, int t4,
                                                 double (&lpa)[2], uint32_t (&g)[32]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s[2] = {0.f, 0.f};                    // two chains of adds (k-blocks j even / odd)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e;
        const float l = acc1[i] + bias[h], yy = e ? yr[j].y : yr[j].x;
        const float ex = ex2f(1.4426950408889634f * l);
        float lp = fmaf(yy, l, -ex), gg = yy - ex;
        if (MASK) {
          const bool v = row0 + 8 * j + 2 * t4 + e < N;
          lp = v ? lp : 0.f;
          gg = v ? gg : 0.f;
        }
        s[j & 1] += lp;
        g[i] = __float_as_uint(tf32_rn(gg));
      }
    lpa[h] += (double)(s[0] + s[1]);
  }
}

// ---- Normal epilogue of the linear-regression kernels (glm_normal_tc.cu) -----------------------------------
// The residual r = y - l with l = acc1 + b (the bias added here, rounded to nearest, as in poisson_epilogue):
// lpa accumulates the sufficient statistic S = SUM r^2 and g = r, rounded to nearest TF32, is GEMM 2's register
// operand.  sigma never enters the tile loop: glm_finish_kernel applies it per particle in fp64, so the epilogue
// takes no MUFU op at all.  MASK (the last, partial tile only) zeroes rows past N.
template <bool MASK>
__device__ __forceinline__ void normal_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                const float2 (&yr)[8], int64_t row0, int64_t N, int t4,
                                                float (&lpa)[2], uint32_t (&g)[32]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s[2] = {0.f, 0.f};                    // two chains of adds (k-blocks j even / odd)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e;
        const float yy = e ? yr[j].y : yr[j].x;
        float r = yy - (acc1[i] + bias[h]);
        if (MASK) r = (row0 + 8 * j + 2 * t4 + e < N) ? r : 0.f;
        s[j & 1] = fmaf(r, r, s[j & 1]);
        g[i] = __float_as_uint(tf32_rn(r));
      }
    lpa[h] += s[0] + s[1];
  }
}

// ---- Binomial epilogue of the aggregated logistic-regression kernels (glm_binomial_tc.cu) -------------------
// lp = y*l - m*softplus(l) (the parameter-free log binomial coefficient is summed once per call, not here) and
// g = y - m*sigmoid(l) rounded to nearest TF32, for y successes out of m trials: ex2, rcp and lg2 per logit.  The
// linear part is y*l for l < 0 and (y - m)*l otherwise, exact for integer counts.  y and m are read from shared
// memory here (ROW: one m per row, else the count mc of every row).  The bias is added here and lpa is fp64, as in
// poisson_epilogue.  MASK (the last, partial tile only) zeroes rows past N.
// (The running product of epi_batch, one lg2 per particle and tile for one count of every row, made the 128-register
// kernels spill.)
template <bool MASK, bool ROW>
__device__ __forceinline__ void binomial_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                  const float2* yr, const float2* mr, float mc, int64_t row0,
                                                  int64_t N, int t4, double (&lpa)[2], uint32_t (&g)[32]) {
  // k-block outermost: the labels of a k-block serve both particles of the thread and are dead after it
  float s[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 y2 = yr[4 * j], m2 = ROW ? mr[4 * j] : make_float2(mc, mc);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e;
        const float l = acc1[i] + bias[h], yy = e ? y2.y : y2.x, m = e ? m2.y : m2.x;
        const float ex = ex2f(-1.4426950408889634f * fabsf(l));
        const float den = 1.f + ex, inv = rcpf(den);
        const float sg = (l >= 0.f) ? inv : ex * inv;
        float lp = fmaf(-0.6931471805599453f * m, lg2f(den), (l >= 0.f ? yy - m : yy) * l);
        float gg = fmaf(-m, sg, yy);
        if (MASK) {
          const bool v = row0 + 8 * j + 2 * t4 + e < N;
          lp = v ? lp : 0.f;
          gg = v ? gg : 0.f;
        }
        s[h] += lp;
        g[i] = __float_as_uint(tf32_rn(gg));
      }
  }
  lpa[0] += (double)s[0];
  lpa[1] += (double)s[1];
}

// SUM f(n) over the rows n < N of the CTA's tiles (blockIdx.x, blockIdx.x + gridDim.x, ...), in fp64 and a fixed
// order; called by every thread of the CTA, each of which gets the sum
template <int NT, class F>
__device__ __forceinline__ double cta_row_sum(int64_t N, F f) {
  __shared__ double red[NT / 32];
  const int64_t ntiles = (N + kRows - 1) / kRows;
  const int nt = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < (int64_t)nt * kRows; i += NT) {
    const int64_t n = (blockIdx.x + (i / kRows) * (int64_t)gridDim.x) * kRows + i % kRows;
    if (n < N) s += f(n);
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double v = 0.0;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) v += red[w];
  return v;
}

// SUM f(n) over the rows r0 <= n < r1 (one contiguous span of the CTA's rows), as cta_row_sum
template <int NT, class F>
__device__ __forceinline__ double span_row_sum(int64_t r0, int64_t r1, F f) {
  __shared__ double red[NT / 32];
  double s = 0.0;
  for (int64_t n = r0 + threadIdx.x; n < r1; n += NT) s += f(n);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double v = 0.0;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) v += red[w];
  return v;
}

// ---- likelihood families of the GLM tile pipelines ----------------------------------------------------------
// Fam is the likelihood family: kBiasInEpilogue (the bias is added by the epilogue, which then takes it after
// acc1, instead of starting GEMM 1's accumulator), kKP (GEMM 1 rows per particle), kYBytes (labels of one
// tile), kYType (their TMA type), Labels (a thread's labels of one tile), read_labels(stage, t4, K, labels) and epilogue(acc1, labels,
// cls, K, row0, N, t4, lpa, g), which writes g (indexed like acc1, rounded to TF32) and adds the tile's lp sums
// of the thread's two rows to lpa; the any-D tile loop (glm_flat_tc.cuh) calls tile_epilogue(acc1, labels,
// row0, N, t4, last, lpa, g) instead.  kTrials (Binomial only) adds a second label operand, the trial counts:
// one device value for every row (kConstTrials) or one per row (kRowTrials, loaded next to y on the same
// mbarrier); read_trials(stage + 256, t4, m, labels) then completes the labels.  LpAcc is the type of the lp sums
// lpa.  kDataTerm families (Poisson, Binomial) leave a parameter-free term of each row's lp out of the tile loop:
// data_term<NT>(y, trials, N) is its fp64 sum over the CTA's rows, which cta_partials subtracts from every
// particle's fp64 lp sum before rounding it to the fp32 partial.  So the partial is of the size of the lp sum, not
// of its terms, and glm_finish_kernel adds no data term.
enum : int { kNoTrials = 0, kConstTrials = 1, kRowTrials = 2 };

// logistic regression: one GEMM 1 row per particle, fp32 labels y
struct Bernoulli {
  static constexpr int kTrials = kNoTrials;
  using LpAcc = float;
  static constexpr bool kDataTerm = false;
  static constexpr bool kBiasInEpilogue = false;  // GEMM 1's accumulator starts at the bias
  static constexpr int kKP = 1;
  static constexpr uint32_t kYBytes = kRows * 4;  // 256 B of y
  static constexpr CUtensorMapDataType kYType = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  using Labels = float2[8];                       // y of the thread's rows n = 8j + 2 t4 + e
  static __device__ __forceinline__ void read_labels(const uint8_t* ys, int t4, int, Labels& y) {
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = reinterpret_cast<const float2*>(ys)[4 * j + t4];
  }
  // lp sums and g, both in registers; the row mask only in the last, partial tile
  static __device__ __forceinline__ void epilogue(const float (&acc1)[32], const Labels& y, const int (&)[2], int,
                                                  int64_t row0, int64_t N, int t4, float (&lpa)[2],
                                                  uint32_t (&g)[32]) {
    bernoulli_epilogue(acc1, y, row0, N, t4, row0 + kRows > N, lpa, g);
  }
  // the same for the any-D tile loop (glm_flat_tc.cuh), which knows whether its tile is the last
  static __device__ __forceinline__ void tile_epilogue(const float (&acc1)[32], const Labels& y, int64_t row0,
                                                       int64_t N, int t4, bool last, float (&lpa)[2],
                                                       uint32_t (&g)[32]) {
    bernoulli_epilogue(acc1, y, row0, N, t4, last, lpa, g);
  }
};

// Poisson regression (log link): the labels of Bernoulli, fp32 counts y
// (GEMM 1 starts from zero and the epilogue adds the bias, see poisson_epilogue); the data term is SUM lgamma(y + 1)
struct Poisson : Bernoulli {
  static constexpr bool kBiasInEpilogue = true;
  using LpAcc = double;
  static constexpr bool kDataTerm = true;
  // SPAN: over the rows [r0, r1) instead of the CTA's round-robin tiles
  template <int NT, bool SPAN = false>
  static __device__ __forceinline__ double data_term(const float* __restrict__ y, const float*, int64_t N,
                                                     int64_t r0 = 0, int64_t r1 = 0) {
    auto f = [&](int64_t n) { return log_factorial_f64(__ldg(y + n)); };
    if constexpr (SPAN) return span_row_sum<NT>(r0, r1, f);
    else return cta_row_sum<NT>(N, f);
  }
  static __device__ __forceinline__ void tile_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                       const Labels& y, int64_t row0, int64_t N, int t4, bool last,
                                                       double (&lpa)[2], uint32_t (&g)[32]) {
    if (last)
      poisson_epilogue<true>(acc1, bias, y, row0, N, t4, lpa, g);
    else
      poisson_epilogue<false>(acc1, bias, y, row0, N, t4, lpa, g);
  }
  static __device__ __forceinline__ void epilogue(const float (&acc1)[32], const float (&bias)[2], const Labels& y,
                                                  const int (&)[2], int, int64_t row0, int64_t N, int t4,
                                                  double (&lpa)[2], uint32_t (&g)[32]) {
    tile_epilogue(acc1, bias, y, row0, N, t4, row0 + kRows > N, lpa, g);
  }
};

// linear regression (Gaussian likelihood): the labels of Bernoulli, fp32 y; lpa holds SUM (y - l)^2, not lp
// (GEMM 1 starts from zero and the epilogue adds the bias, see normal_epilogue)
struct Normal : Bernoulli {
  static constexpr bool kBiasInEpilogue = true;
  static __device__ __forceinline__ void tile_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                       const Labels& y, int64_t row0, int64_t N, int t4, bool last,
                                                       float (&lpa)[2], uint32_t (&g)[32]) {
    if (last)
      normal_epilogue<true>(acc1, bias, y, row0, N, t4, lpa, g);
    else
      normal_epilogue<false>(acc1, bias, y, row0, N, t4, lpa, g);
  }
  static __device__ __forceinline__ void epilogue(const float (&acc1)[32], const float (&bias)[2], const Labels& y,
                                                  const int (&)[2], int, int64_t row0, int64_t N, int t4,
                                                  float (&lpa)[2], uint32_t (&g)[32]) {
    tile_epilogue(acc1, bias, y, row0, N, t4, row0 + kRows > N, lpa, g);
  }
};

// Binomial regression (logit link): fp32 successes y and trial counts m, one for every row (ROW = false, a
// device value read once per call) or one per row (ROW: [N] fp32, loaded next to y).  GEMM 1 starts from zero
// and the epilogue adds the bias, see binomial_epilogue.  The data term is -SUM log C(m, y).
template <bool ROW>
struct Binomial : Bernoulli {
  static constexpr int kTrials = ROW ? kRowTrials : kConstTrials;
  static constexpr bool kBiasInEpilogue = true;
  using LpAcc = double;
  static constexpr bool kDataTerm = true;
  template <int NT>
  static __device__ __forceinline__ double data_term(const float* __restrict__ y, const float* __restrict__ trials,
                                                     int64_t N) {
    const float mc = ROW ? 0.f : __ldg(trials);
    const double lgm = ROW ? 0.0 : log_factorial_f64(mc);
    return cta_row_sum<NT>(N, [&](int64_t n) {
      const float yv = __ldg(y + n), m = ROW ? __ldg(trials + n) : mc;
      return (log_factorial_f64(yv) + log_factorial_f64(m - yv)) - (ROW ? log_factorial_f64(m) : lgm);
    });
  }
  static constexpr uint32_t kYBytes = (ROW ? 2 : 1) * kRows * 4;   // y, then the trials of the tile
  // The labels stay in shared memory until the epilogue reads them (y and m of the thread's rows n = 8j + 2 t4 + e
  // at y[4j], m[4j]): held in registers across GEMM 1 they made the 128-register kernels spill.  So the tile
  // pipelines keep a tile's labels in place until its epilogue is done: glm_tile_pipeline refills a stage one
  // tile later, glm_flat_pipeline alternates two label slots.
  struct Labels {
    const float2* y;
    const float2* m;                            // ROW only
    float mc;                                   // the trial count of every row (ROW = false)
  };
  static __device__ __forceinline__ void read_labels(const uint8_t* ys, int t4, int, Labels& lab) {
    lab.y = reinterpret_cast<const float2*>(ys) + t4;
  }
  static __device__ __forceinline__ void read_trials(const uint8_t* ms, int t4, float mc, Labels& lab) {
    lab.m = reinterpret_cast<const float2*>(ms) + t4;
    lab.mc = mc;
  }
  static __device__ __forceinline__ void tile_epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                       const Labels& lab, int64_t row0, int64_t N, int t4,
                                                       bool last, double (&lpa)[2], uint32_t (&g)[32]) {
    if (last)
      binomial_epilogue<true, ROW>(acc1, bias, lab.y, lab.m, lab.mc, row0, N, t4, lpa, g);
    else
      binomial_epilogue<false, ROW>(acc1, bias, lab.y, lab.m, lab.mc, row0, N, t4, lpa, g);
  }
  static __device__ __forceinline__ void epilogue(const float (&acc1)[32], const float (&bias)[2],
                                                  const Labels& lab, const int (&)[2], int, int64_t row0,
                                                  int64_t N, int t4, double (&lpa)[2], uint32_t (&g)[32]) {
    tile_epilogue(acc1, bias, lab, row0, N, t4, row0 + kRows > N, lpa, g);
  }
};

// ---- stages of the GLM tile pipeline (glm_tc.cu, glm_categorical_tc.cu, glm_flat_tc.cu) ---------------------
//
// GEMM 1's M = 64 rows of a CTA slab are particles (KP = 1) or (particle, class) pairs: each particle's K
// classes take KP consecutive rows, so row m is class m % KP of particle slab * (64 / KP) + m / KP.
//
// wgmma accumulator fragment (m64nN, f32): thread (warp w4 of the warpgroup, lane = 4 gid + t4) holds
// d[4j + 2h + e] = D[16 w4 + gid + 8h][8j + 2 t4 + e].

// W hi / lo, the A operands of GEMM 1: [KD / 32 atoms][m 64][32] SW128, zero for a particle past P, a class
// past K and a column past D (generic-proxy writes; the caller makes them visible to the tensor cores).  And
// rows KD .. KD+7 of both X^T k-blocks of each of the NT / 128 warpgroups (wg_bytes apart) are ones: GEMM 2
// then yields db in column KD of its accumulator.
template <int KP, int KD, int NT>
__device__ __forceinline__ void stage_w_and_ones(float* whi, float* wlo, uint8_t* xt0, uint32_t wg_bytes,
                                                 const float* W, int slab, int P, int K, int D) {
  for (int e = threadIdx.x; e < kM * KD; e += NT) {
    const int m = e / KD, d = e - m * KD;
    const int gp = slab * (kM / KP) + m / KP, k = m % KP;
    const float w = (gp < P && k < K && d < D) ? W[((int64_t)gp * K + k) * D + d] : 0.f;
    const float hi = tf32_trunc(w);
    const int off = (d >> 5) * 2048 + sw128(m, d & 31);
    whi[off] = hi;
    wlo[off] = w - hi;
  }
  for (int e = threadIdx.x; e < NT / 128 * 2 * 256; e += NT) {
    const int g = e >> 9, kb = (e >> 8) & 1, w = e & 255;
    reinterpret_cast<float*>(xt0 + g * wg_bytes + kb * (KD + 8) * 128 + KD * 128)[w] = 1.f;
  }
}

// GEMM 1: logits D1^T[m, n] = W X^T + b over DC atoms (8 KB apart), accumulator initialised with the bias of
// the thread's rows.  W is split hi + lo, two TF32 MMAs per k-step; SPLIT_X adds X_lo as a third.
template <int DC, bool SPLIT_X>
__device__ __forceinline__ void gemm1(float (&acc1)[32], const float (&bias)[2], uint32_t whi, uint32_t wlo,
                                      uint32_t x, uint32_t xlo) {
#pragma unroll
  for (int i = 0; i < 32; ++i) acc1[i] = bias[(i >> 1) & 1];
  wgmma_fence();
#pragma unroll
  for (int a = 0; a < DC; ++a) {
    const uint64_t d_whi = desc_sw128(whi + a * 8192), d_wlo = desc_sw128(wlo + a * 8192);
    const uint64_t d_x = desc_sw128(x + a * 8192), d_xlo = desc_sw128(xlo + a * 8192);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      wgmma_n64_tf32(acc1, d_whi + 2 * k, d_x + 2 * k);
      wgmma_n64_tf32(acc1, d_wlo + 2 * k, d_x + 2 * k);
      if (SPLIT_X) wgmma_n64_tf32(acc1, d_whi + 2 * k, d_xlo + 2 * k);
    }
  }
  wgmma_commit();
  wgmma_wait0();
  fence_regs(acc1);
}

// GEMM 2: [dW | db] += g [X | 1] with g (indexed like acc1) from registers and X^T from its two k-blocks of N2
// rows at xt; committed and left running.  The warpgroup's first tile starts the accumulator with scale-d = 0:
// an ordinary write to it inside a wgmma pipeline stage would serialise every wgmma of the kernel (C7515).
template <int N2>
__device__ __forceinline__ void gemm2(float (&acc2)[N2 / 2], uint32_t (&g)[32], uint32_t xt, bool first) {
  fence_regs(g);
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t a[4] = {g[4 * j], g[4 * j + 2], g[4 * j + 1], g[4 * j + 3]};
    wgmma_tf32_ra<N2>(acc2, a, desc_sw128(xt + (j >> 2) * N2 * 128) + 2 * (j & 3), !first || j != 0);
  }
  wgmma_commit();
}

// CTA results through the idle shared memory red, in a fixed summation order: [NT / 128][64 m][KD + 1] GEMM 2
// accumulators (dW in columns < D, db in column KD) and [NT / 128][64 m] lp sums of type A (lpa already summed
// over the four lanes of a row), then each row summed over the warpgroups that had a tile.  The CTA's partials are
// [P][K (D + 1) + 1]: per class dW[0..D-1] and db, then the particle's lp sum, less dterm (fp64 lp sums only).
template <int KP, int N2, int NT, typename A>
__device__ __forceinline__ void cta_partials(float* red, const float (&acc2)[N2 / 2], const A (&lpa)[2], int wg,
                                             int nt, int slab, int P, int K, int D, float* partials,
                                             double dterm = 0.0) {
  constexpr int KD = N2 - 8, kWG = NT / 128;
  const int tid = threadIdx.x, w4 = (tid >> 5) & 3, gid = (tid & 31) >> 2, t4 = tid & 3;
  float* red2 = red;
  A* redlp = reinterpret_cast<A*>(red2 + kWG * kM * (KD + 1));   // 8-byte aligned: kM * (KD + 1) is even
  __syncthreads();
#pragma unroll
  for (int j = 0; j < N2 / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int m = 16 * w4 + gid + 8 * h, c = 8 * j + 2 * t4 + e;
        if (c < D || c == KD) red2[(wg * kM + m) * (KD + 1) + c] = acc2[4 * j + 2 * h + e];
      }
  if (t4 == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) redlp[wg * kM + 16 * w4 + gid + 8 * h] = lpa[h];
  }
  __syncthreads();
  const int nwg = nt < kWG ? nt : kWG;
  const int S = K * (D + 1) + 1;
  for (int e = tid; e < kM * (D + 1); e += NT) {
    const int m = e / (D + 1), c = e - (D + 1) * m;
    const int gp = slab * (kM / KP) + m / KP, k = m % KP;
    if (gp < P && k < K) {
      float v = 0.f;
      for (int q = 0; q < nwg; ++q) v += red2[(q * kM + m) * (KD + 1) + (c < D ? c : KD)];
      partials[((int64_t)blockIdx.x * P + gp) * S + k * (D + 1) + c] = v;
    }
  }
  if (tid < kM / KP && slab * (kM / KP) + tid < P) {
    A v = 0;
    for (int q = 0; q < nwg; ++q)
      for (int k = 0; k < KP; ++k) v += redlp[q * kM + tid * KP + k];
    if constexpr (sizeof(A) == 8) v -= dterm;
    partials[((int64_t)blockIdx.x * P + slab * (kM / KP) + tid) * S + K * (D + 1)] = (float)v;
  }
}

// ---- the D = 32 tile pipeline (glm_tc.cu: Bernoulli, glm_categorical_tc.cu: softmax) -----------------------
//
// ONE pass over X[N,32] and the labels y[N] gives, for each CTA slab of 64 GEMM 1 rows, the lp sums and the
// [dW | db] sums as CTA partials for glm_finish_kernel.  Per 64-row tile: split pass, GEMM 1, the family's
// epilogue, GEMM 2; the stages, the TMA ring and the register budget are described in glm_tc.cu.
namespace tile32 {

constexpr int kD = 32;
constexpr int kWG = 4;                          // warpgroups
constexpr int kStages = 2 * kWG;                // two X / label stages per warpgroup
constexpr int kThreads = kWG * 128;
constexpr uint32_t kTile = kRows * kD * 4;      // 8 KB X tile
constexpr uint32_t kXtBlock = (kD + 8) * 128;   // X^T k-block: 32 rows of d + 8 rows of ones, 32 n each (5 KB)
// per-warpgroup region
constexpr uint32_t WG_XT = 0;                       // X^T  [kb 2][c 40][32 n] fp32, n permuted (see kt_pos)
constexpr uint32_t WG_XLO = WG_XT + 2 * kXtBlock;   // X_lo [n 64][32 d] fp32 (SPLIT_X)
constexpr uint32_t kWGBytes = WG_XLO + kTile;

// CTA layout (every operand region 1024-byte aligned: the 128-byte swizzle pattern is taken from address bits)
template <uint32_t kYBytes>
struct Smem32 {
  static constexpr uint32_t OFF_X = 0;
  static constexpr uint32_t OFF_Y = OFF_X + kStages * kTile;
  static constexpr uint32_t OFF_WHI = OFF_Y + kStages * kYBytes;   // [m 64][32 d] SW128, 8 KB
  static constexpr uint32_t OFF_WLO = OFF_WHI + 8192;
  static constexpr uint32_t OFF_WG = OFF_WLO + 8192;
  static constexpr uint32_t OFF_BAR = OFF_WG + kWG * kWGBytes;
  static constexpr uint32_t kBytes = OFF_BAR + 256 + 1024;   // + slack for the 1024-byte alignment
  static_assert(kBytes <= 232448, "shared memory budget");
  static_assert(OFF_WHI % 1024 == 0 && kWGBytes % 1024 == 0 && kXtBlock % 1024 == 0, "operand alignment");
  // the final reduction reuses the X ring: [kWG][64 m][33] floats + [kWG][64 m] lp sums (at most fp64)
  static_assert(kWG * kM * 33 * 4 + kWG * kM * 8 <= kStages * kTile, "reduction scratch");
};

// Fam is the likelihood family (Bernoulli, Poisson, Normal, Binomial above, Softmax of glm_categorical_tc.cu).
// Binomial only: map_m is the trials' label map (kRowTrials), trials the trial counts (one device count for
// kConstTrials).  y, the labels in global memory, is read by the data term of kDataTerm families only.
template <class Fam, bool SPLIT_X>
__device__ __forceinline__ void glm_tile_pipeline(const CUtensorMap& map_x, const CUtensorMap& map_y,
                                                  const float* W, const float* bvec, int64_t N, int P, int K,
                                                  float* partials, const CUtensorMap* map_m = nullptr,
                                                  const float* trials = nullptr, const float* y = nullptr) {
  using L = Smem32<Fam::kYBytes>;
  constexpr int KP = Fam::kKP;
  constexpr uint32_t kYBytes = Fam::kYBytes;
  pdl_launch_dependents();   // lets glm_finish_kernel be resident (blocked in its griddepcontrol.wait) early
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + L::OFF_BAR;
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
  __syncthreads();
  // warp-uniform by construction (a shuffle result), so the tile loop is not a divergent branch to ptxas
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), w4 = warp & 3, t = tid & 127;
  // tile it -> X / label stage; one thread of the warpgroup issues the loads
  auto load = [&](int it, int s) {
    const int64_t tile = blockIdx.x + (int64_t)it * gridDim.x;
    mbar_expect_tx(bar_full(s), kTile + kYBytes);
    tma_load_2d(base + L::OFF_X + s * kTile, &map_x, 0, (int)(tile * kRows), bar_full(s));
    tma_load_1d(base + L::OFF_Y + s * kYBytes, &map_y, (int)(tile * kRows), bar_full(s));
    if constexpr (Fam::kTrials == kRowTrials)
      tma_load_1d(base + L::OFF_Y + s * kYBytes + kRows * 4, map_m, (int)(tile * kRows), bar_full(s));
  };
  // Each warpgroup's first two X / label tiles are requested BEFORE griddepcontrol.wait, so they stream while the
  // predecessor (the step's draw kernel, on a CTA or two) finishes.  Sound because no native kernel that can
  // precede a GLM launch writes X or the labels: the draws write site values, the pack kernels of glm_potential.cu
  // write W and b only, and a predecessor launched without PDL never lets this kernel start early.  W, the bias
  // and everything else a predecessor may write are read after the wait.
  if (t == 0)
    for (int k = 0; k < 2 && wg + k * kWG < nt; ++k) load(wg + k * kWG, 2 * wg + k);
  pdl_wait();
  stage_w_and_ones<KP, kD, kThreads>(reinterpret_cast<float*>(sm + L::OFF_WHI),
                                     reinterpret_cast<float*>(sm + L::OFF_WLO), sm + L::OFF_WG + WG_XT, kWGBytes,
                                     W, slab, P, K, kD);
  fence_proxy_async();
  __syncthreads();

  typename Fam::LpAcc lpa[2] = {0, 0};         // lp sums of the thread's two rows
  // GEMM 2 accumulator [m][c]: dW in c < 32, db in c = 32.  Never written by ordinary instructions before
  // the tile loop (C7515): the warpgroup's first GEMM 2 k-step starts it with scale-d = 0, and a warpgroup
  // without a tile is left out of the CTA reduction.
  float acc2[20];
  const int gid = lane >> 2, t4 = lane & 3;
  // the thread's two rows m = 16 w4 + gid + 8h: class (gid + 8h) % KP of particle slab * 64 / KP + m / KP
  int cls[2];
  float bias[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = 16 * w4 + gid + 8 * h;
    const int gp = slab * (kM / KP) + m / KP;
    cls[h] = m % KP;
    bias[h] = (bvec != nullptr && gp < P && cls[h] < K) ? bvec[(int64_t)gp * K + cls[h]] : 0.f;
  }
  float mconst = 0.f;                          // Binomial with one trial count for every row
  if constexpr (Fam::kTrials == kConstTrials) mconst = *trials;

  {
    uint8_t* my = sm + L::OFF_WG + wg * kWGBytes;
    const uint32_t my_s = base + L::OFF_WG + wg * kWGBytes;
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
        float4* xs = reinterpret_cast<float4*>(sm + L::OFF_X + s * kTile);
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
      typename Fam::Labels lab;                // read before the refill
      Fam::read_labels(sm + L::OFF_Y + s * kYBytes, t4, K, lab);
      if constexpr (Fam::kTrials != kNoTrials)
        Fam::read_trials(sm + L::OFF_Y + s * kYBytes + kRows * 4, t4, mconst, lab);
      fence_proxy_async();
      wg_bar(1 + wg);
      // Binomial reads its labels from the stage in the epilogue: the stage of the previous tile, whose epilogue
      // every thread of the warpgroup has now finished, is refilled here instead of after GEMM 1
      if constexpr (Fam::kTrials != kNoTrials)
        if (t == 0 && k > 0 && it + kWG < nt) load(it + kWG, s ^ 1);
      float acc1[32];
      if constexpr (Fam::kBiasInEpilogue) {
        const float zero[2] = {0.f, 0.f};
        gemm1<1, SPLIT_X>(acc1, zero, base + L::OFF_WHI, base + L::OFF_WLO, base + L::OFF_X + s * kTile,
                          my_s + WG_XLO);
      } else {
        gemm1<1, SPLIT_X>(acc1, bias, base + L::OFF_WHI, base + L::OFF_WLO, base + L::OFF_X + s * kTile,
                          my_s + WG_XLO);
      }
      // GEMM 1 has read the X stage and the labels are in registers: refill the stage with tile it + 2 kWG
      if constexpr (Fam::kTrials == kNoTrials)
        if (t == 0 && it + 2 * kWG < nt) load(it + 2 * kWG, s);
      uint32_t g[32];
      if constexpr (Fam::kBiasInEpilogue)
        Fam::epilogue(acc1, bias, lab, cls, K, row0, N, t4, lpa, g);
      else
        Fam::epilogue(acc1, lab, cls, K, row0, N, t4, lpa, g);
      // left running while the next tile is waited for
      gemm2<kD + 8>(acc2, g, my_s + WG_XT, it == wg);
    }
    wgmma_wait0();
    fence_regs(acc2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      auto v = lpa[h];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      lpa[h] = v;
    }
  }
  double dterm = 0.0;
  if constexpr (Fam::kDataTerm) dterm = Fam::template data_term<kThreads>(y, trials, N);
  cta_partials<KP, kD + 8, kThreads>(reinterpret_cast<float*>(sm + L::OFF_X), acc2, lpa, wg, nt, slab, P, K, kD,
                                     partials, dterm);
}

}  // namespace tile32

// ---- host side ------------------------------------------------------------------------------------------------
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

// X[N, 32] fp32 in 64-row boxes, SWIZZLE_128B: the tile as the D = 32 pipeline's GEMM 1 reads it.  False
// when the driver cannot encode it.
inline bool encode_x_map(CUtensorMap* m, const float* X, int64_t N) {
  EncodeTiledFn enc = encode_fn();
  const cuuint64_t dims[2] = {32, (cuuint64_t)N};
  const cuuint64_t strides[1] = {32 * 4};
  const cuuint32_t box[2] = {32, (cuuint32_t)kRows};
  const cuuint32_t estr[2] = {1, 1};
  return enc != nullptr &&
         enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(X), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the labels y[N] of element type `type` in 64-row boxes
inline bool encode_label_map(CUtensorMap* m, const void* y, int64_t N, CUtensorMapDataType type) {
  EncodeTiledFn enc = encode_fn();
  const cuuint64_t dims[1] = {(cuuint64_t)N};
  const cuuint64_t strides[1] = {0};
  const cuuint32_t box[1] = {(cuuint32_t)kRows};
  const cuuint32_t estr[1] = {1};
  return enc != nullptr &&
         enc(m, type, 1, const_cast<void*>(y), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// gx CTAs for each slab of kM particles
inline dim3 slab_grid(int gx, int P) { return dim3((unsigned)gx, (unsigned)((P + kM - 1) / kM), 1); }

}  // namespace tc
}  // namespace b2
