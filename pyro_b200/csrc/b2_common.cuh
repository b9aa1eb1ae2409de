// b2_common.cuh -- shared device helpers: vector loads, block reductions with a deterministic
// cross-CTA finish, launch bookkeeping.
#pragma once
#include <stdlib.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pyro_b200.h"

namespace b2 {

constexpr int kMaxD = 6;          // dims kept after host-side coalescing
constexpr int kNumSMs = 132;      // H100 SXM
constexpr int kMaxRed = 8;        // reduction slots per launch (sum, dvalue, dparams[4], spare)
constexpr int kMaxPartialBlocks = 8192;

extern int64_t g_launch_count;  // defined in api.cu
inline void count_launch(int n = 1) { g_launch_count += n; }

// ---- programmatic dependent launch -------------------------------------------------------------------
// The small kernels of an SVI step run one after the other from a cold L2 (the step streams 132 MB through it),
// so each of them spends most of its few microseconds on launch latency and on fetching its own code.  A kernel
// launched with the programmatic-stream-serialization attribute may start while its predecessor in the stream is
// still running, provided the predecessor allowed it (griddepcontrol.launch_dependents); it then blocks in
// griddepcontrol.wait until the predecessor has COMPLETED and its memory is visible.  Both instructions sit at the
// very top of the kernels below, so only launch + code fetch overlap, never a data access.  Captured into a CUDA
// graph the dependency becomes a programmatic edge.  B2_PDL=0 in the environment launches the plain way.
#if defined(__CUDACC__)
__device__ __forceinline__ void pdl_enter() {
#if __CUDA_ARCH__ >= 900
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
inline bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("B2_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

inline int check_launch() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? B2_OK : B2_ERR_LAUNCH;
}

// ---- 16-byte vectors --------------------------------------------------------------------------
template <typename T>
struct VecOf;
template <>
struct VecOf<float> {
  using type = float4;
  static constexpr int N = 4;
};
template <>
struct VecOf<double> {
  using type = double2;
  static constexpr int N = 2;
};

template <typename T>
struct Pack {
  T v[VecOf<T>::N];
};

// N-element vector type of T (N * sizeof(T) <= 16)
template <typename T, int N>
struct VecN;
template <>
struct VecN<float, 4> { using type = float4; };
template <>
struct VecN<float, 2> { using type = float2; };
template <>
struct VecN<double, 2> { using type = double2; };
template <>
struct VecN<double, 1> { using type = double; };

// streaming load (read-once data): evict-first in L1/L2
template <typename T>
__device__ __forceinline__ Pack<T> ld_stream(const T* p) {
  using VT = typename VecOf<T>::type;
  union {
    VT v;
    Pack<T> k;
  } u;
  u.v = __ldcs(reinterpret_cast<const VT*>(p));
  return u.k;
}
// cached load (data re-read by other rows / CTAs)
template <typename T>
__device__ __forceinline__ Pack<T> ld_keep(const T* p) {
  using VT = typename VecOf<T>::type;
  union {
    VT v;
    Pack<T> k;
  } u;
  u.v = __ldg(reinterpret_cast<const VT*>(p));
  return u.k;
}
template <typename T>
__device__ __forceinline__ void st_stream(T* p, const Pack<T>& k) {
  using VT = typename VecOf<T>::type;
  union {
    VT v;
    Pack<T> k;
  } u;
  u.k = k;
  __stcs(reinterpret_cast<VT*>(p), u.v);
}

// ---- reductions -------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum NRED per-thread values over the CTA; result valid in thread 0.  smem: NRED * 32 doubles.
template <int NRED>
__device__ __forceinline__ void block_sum(double (&v)[NRED], double* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int k = 0; k < NRED; ++k) {
    double w = warp_sum(v[k]);
    if (lane == 0) smem[k * 32 + warp] = w;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) {
      double w = (lane < nwarps) ? smem[k * 32 + lane] : 0.0;
      w = warp_sum(w);
      v[k] = w;
    }
  }
  __syncthreads();
}

// Deterministic grid finish: every CTA stores its NRED block sums; the last CTA to arrive
// (ticket counter) adds all partials in a fixed order and calls `fin(k, total)` from thread 0.
// `ticket` must be zero on entry and is reset to zero by the last CTA.
template <int NRED, typename Fin>
__device__ __forceinline__ void grid_finish(double (&v)[NRED], double* partials,
                                            unsigned int* ticket, double* smem, Fin fin) {
  __shared__ bool is_last;
  const unsigned int nblocks = gridDim.x * gridDim.y * gridDim.z;
  const unsigned int bid = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
  block_sum<NRED>(v, smem);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) partials[(size_t)k * kMaxPartialBlocks + bid] = v[k];
    __threadfence();
    const unsigned int t = atomicAdd(ticket, 1u);
    is_last = (t == nblocks - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double tot[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) {
    double s = 0.0;
    for (unsigned int i = threadIdx.x; i < nblocks; i += blockDim.x)
      s += __ldcg(&partials[(size_t)k * kMaxPartialBlocks + i]);
    tot[k] = s;
  }
  block_sum<NRED>(tot, smem);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) fin(k, tot[k]);
    *ticket = 0u;
    __threadfence();
  }
}

// workspace layout shared by the reducing kernels: [ticket (256 B)] [partials kMaxRed x kMaxPartialBlocks doubles]
constexpr size_t kReduceWorkspaceBytes = 256 + sizeof(double) * kMaxRed * kMaxPartialBlocks;
inline unsigned int* ws_ticket(void* ws) { return reinterpret_cast<unsigned int*>(ws); }
inline double* ws_partials(void* ws) {
  return reinterpret_cast<double*>(reinterpret_cast<char*>(ws) + 256);
}

}  // namespace b2
