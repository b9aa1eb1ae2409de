// glm_host.cuh -- host plumbing shared by the GLM likelihood entry points (glm.cu, glm_tc.cu, glm_flat_tc.cu,
// glm_categorical_tc.cu, glm_poisson_tc.cu, glm_normal_tc.cu, glm_binomial_tc.cu) and poisson_product_tc.cu: the
// tensor-core kernel launcher, the dispatch from D to the atom count of glm_flat_pipeline, the precision policy, the
// finish launch, and the checks and workspace of the per-row entry points (Poisson, Normal, Binomial).
#pragma once
#include <type_traits>

#include "b2_common.cuh"

namespace b2 {

// A varying intercept by group (glm_flat_pipeline's GROUPS): idx[N] is the int32 group of each row, 16-byte
// aligned, and G the number of groups; no group effect when idx is null.  With one, a likelihood call runs the flat
// pipeline at D + G columns whatever D is: W, dW, the CTA partials and the workspace are D + G wide, and dW's
// columns D .. D+G-1 are the derivatives with respect to the group effects.  S (0..3) varying slopes by group add G
// columns each: slope k's columns D + kG + j (k = 1..S) hold X[n, col[k - 1]] where g_n == j, so the call is
// D + G (1 + S) wide and dW's slope columns are the derivatives with respect to the slopes.
struct GlmGroups {
  const int32_t* idx = nullptr;
  int G = 0;
  int S = 0;
  int col[3] = {0, 0, 0};
  // the synthesised columns of the contraction, G (1 + S); none without a group effect
  __host__ __device__ int cols() const { return idx ? G * (1 + S) : 0; }
};

// A gathered group effect (glm_flat_pipeline's GATHER, for more groups than the contraction has columns): the same
// X @ w + b + alpha[g] + SUM_k beta_k[g] X[n, col[k]], with idx sorted, but the group term added to GEMM 1's logits
// from the group-major tables tab [1 + S][G][cp] (cp >= P chains, a multiple of 64) and the group gradients summed
// over the rows of each group (run sums): gsum [1 + S][G][cp] for a group inside one warpgroup's range of tiles (the
// caller zeroes it first), slots [Q][2][4][cp] for the first and last run of warpgroup q's range, status [Q] with bit
// 0 for an index outside [0, G) and bit 1 for a descending pair.  Q = gx * (warpgroups per CTA).
struct GlmGather {
  const int32_t* idx = nullptr;
  int G = 0;
  int S = 0;
  int col[3] = {0, 0, 0};
  int cp = 0;
  const float* tab = nullptr;
  float* gsum = nullptr;
  float* slots = nullptr;
  int* status = nullptr;
};

// warpgroup q's contiguous range of tiles [t0, t1) among Q for ntiles tiles (GATHER); rows [64 t0, min(64 t1, N))
__host__ __device__ inline void gather_tiles(int q, int Q, int64_t ntiles, int64_t& t0, int64_t& t1) {
  t0 = (int64_t)q * ntiles / Q;
  t1 = (int64_t)(q + 1) * ntiles / Q;
}

// The finishes' view of a gathered call (b2_glm_potential's and b2_glm_group_gather_sum's): each group's run sums
// (1 + S blocks) end up in gsum[k][g][c].  A group inside one warpgroup's range is there already (and an empty one 0,
// from the pack); a group that the first or last run of a range reaches is in the at most 2 Q slots, in row order,
// and its value is the sum of the slots that carry its key (gather_slot_key).  status[Q] as in GlmGather.
struct GlmGatherFinish {
  float* gsum;
  const float* slots;
  const int* status;
  const int32_t* idx;
  int cp, Q;
  int64_t N;
};

// The group key of slot e (0 <= e < 2 Q) of a gathered call, range e / 2 having the tiles [t0, t1), t0 < t1: slot
// 2q is the first run of range q, slot 2q + 1 its last run if that is another group; -1 for a slot without a run (a
// range of one run) and for a negative index.  The keys ascend along the slots for sorted rows; any rows are read
// in bounds.
__device__ __forceinline__ int gather_run_key(const GlmGatherFinish& gf, int e, int64_t t0, int64_t t1) {
  const int f = gf.idx[t0 * 64], l = gf.idx[(t1 * 64 < gf.N ? t1 * 64 : gf.N) - 1];
  const int key = (e & 1) == 0 ? f : (f != l ? l : -1);
  return key < -1 ? -1 : key;
}

// the key of slot e over ntiles tiles, -1 for an empty range too
__device__ __forceinline__ int gather_slot_key(const GlmGatherFinish& gf, int e, int64_t ntiles) {
  int64_t t0, t1;
  gather_tiles(e >> 1, gf.Q, ntiles, t0, t1);
  return t0 < t1 ? gather_run_key(gf, e, t0, t1) : -1;
}

// The group at the row that places slot e among the slots, run or not: the first row of range e / 2 for even e, its
// last row for odd e, and the first for both slots of an empty range (clamped to the last row of the data).  These
// rows never descend along the slots, so for sorted rows the orders ascend, and a slot with a run has its key
// (gather_slot_key) as its order: b2_glm_group_gather_sum's finish finds a group's slots by binary search on them.
__device__ __forceinline__ int gather_slot_order(const GlmGatherFinish& gf, int e, int64_t ntiles) {
  int64_t t0, t1;
  gather_tiles(e >> 1, gf.Q, ntiles, t0, t1);
  int64_t r = (e & 1) && t1 > t0 ? (t1 * 64 < gf.N ? t1 * 64 : gf.N) - 1 : t0 * 64;
  if (r > gf.N - 1) r = gf.N - 1;
  return gf.idx[r];
}

// The potential's bookkeeping for chain c (one warp): the slots are summed by group key with a segmented scan of the
// warp in fp64 over 32 slots at a time, and written over their groups' entries of gsum.  Returns whether any range
// saw an index outside [0, G) or a descending pair (status).
__device__ __forceinline__ bool gather_fixup(const GlmGatherFinish& gf, int G, int S, int64_t c, int lane) {
  constexpr unsigned kAll = 0xffffffffu;
  int st = 0;
  for (int q = lane; q < gf.Q; q += 32) st |= gf.status[q];
  st = __reduce_or_sync(kAll, st);
  const int64_t ntiles = (gf.N + 63) / 64;
  const int ne = 2 * gf.Q;
  double carry[4] = {0.0, 0.0, 0.0, 0.0};
  int ckey = -1;
  for (int e0 = 0; e0 < ne; e0 += 32) {
    const int e = e0 + lane;
    int key = -1;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    if (e < ne) {
      int64_t t0, t1;
      gather_tiles(e >> 1, gf.Q, ntiles, t0, t1);
      if (t0 < t1) {
        key = gather_run_key(gf, e, t0, t1);
        if (key >= 0)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k <= S) v[k] = (double)gf.slots[((int64_t)e * 4 + k) * gf.cp + c];
      }
    }
    // a slot without a run takes the key before it (they ascend) and adds nothing
    if (lane == 0 && ckey > key) key = ckey;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(kAll, key, o);
      if (lane >= o && u > key) key = u;
    }
    // the previous chunk's last segment is complete when this chunk starts with another key
    if (lane == 0 && key != ckey && (unsigned)ckey < (unsigned)G)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k <= S) gf.gsum[((int64_t)k * G + ckey) * gf.cp + c] = (float)carry[k];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int ko = __shfl_up_sync(kAll, key, o);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double vo = __shfl_up_sync(kAll, v[k], o);
        if (lane >= o && ko == key) v[k] += vo;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (key == ckey) v[k] += carry[k];
    const int knext = __shfl_down_sync(kAll, key, 1);
    if (lane < 31 && knext != key && (unsigned)key < (unsigned)G)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k <= S) gf.gsum[((int64_t)k * G + key) * gf.cp + c] = (float)v[k];
    ckey = __shfl_sync(kAll, key, 31);
#pragma unroll
    for (int k = 0; k < 4; ++k) carry[k] = __shfl_sync(kAll, v[k], 31);
  }
  if (lane == 0 && (unsigned)ckey < (unsigned)G)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k <= S) gf.gsum[((int64_t)k * G + ckey) * gf.cp + c] = (float)carry[k];
  __syncwarp();
  return st != 0;
}

// ---- glm.cu ----
// The second launch of every GLM likelihood call: glm_finish_kernel over the CTA partials [gx][P][K (D + 1) + 1].
// The Normal noise scale sigma[p * sigma_stride] with n = N rows and out_dsigma are optional.  The per-particle sums
// go to out_sum_p, or without one to the [P] row of the workspace after the partials.
void launch_glm_finish(const float* partials, unsigned int* ticket, int gx, int P, int K, int D, double scale,
                       double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                       float* out_dW, float* out_db, cudaStream_t s, const float* sigma = nullptr,
                       int sigma_stride = 0, int64_t n = 0, float* out_dsigma = nullptr);

// ---- glm_tc.cu ----
// CTAs per particle slab of the tensor-core tile loops: one per SM, at most one per 64-row tile
int glm_tc_grid_x(int64_t N);
// Bernoulli at D = 32 on glm_tile_pipeline; 0 or a negative B2_ERR code
int launch_glm_tc(const float* X, const float* y, const float* W, const float* b, int64_t N, int P,
                  float* partials, int gx, bool split_x, cudaStream_t s);
// cudaFuncAttributeMaxDynamicSharedMemorySize = bytes for kernel on the current device, set once per (kernel,
// device, under a lock; false when CUDA refuses it
bool set_max_dynamic_smem(const void* kernel, int bytes);

// b2_glm_bernoulli_logits with an optional group effect
int glm_bernoulli_logits(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                         double scale, double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                         float* out_dW, float* out_db, void* workspace, size_t workspace_bytes, cudaStream_t s,
                         GlmGroups grp);

// ---- glm_flat_tc.cu ----
// Bernoulli at every other D in 1..128 on glm_flat_pipeline, and at every D with a group effect
int launch_glm_flat_tc(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                       float* partials, int gx, bool split_x, cudaStream_t s, GlmGroups grp = {});

// ---- glm_poisson_tc.cu, glm_normal_tc.cu, glm_binomial_tc.cu ----
// b2_glm_poisson_log_rate, b2_glm_normal_loc and b2_glm_binomial_logits with an optional group effect
int glm_poisson_log_rate(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                         double scale, double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                         float* out_dW, float* out_db, void* workspace, size_t workspace_bytes, cudaStream_t s,
                         GlmGroups grp);
int glm_normal_loc(const float* X, const float* y, const float* W, const float* b, const float* sigma,
                   int sigma_stride, int64_t N, int D, int P, double scale, double weight, double sum_coeff, int flags,
                   float* out_sum_p, float* out_total, float* out_dW, float* out_db, float* out_dsigma,
                   void* workspace, size_t workspace_bytes, cudaStream_t s, GlmGroups grp);
int glm_binomial_logits(const float* X, const float* y, const float* trials, int trials_per_row, const float* W,
                        const float* b, int64_t N, int D, int P, double scale, double weight, double sum_coeff,
                        int flags, float* out_sum_p, float* out_total, float* out_dW, float* out_db, void* workspace,
                        size_t workspace_bytes, cudaStream_t s, GlmGroups grp);

// ---- glm_group_gather_tc.cu ----
// The run-sum ranges Q of a gathered call: CTAs times the warpgroups of the kernel that D dispatches to
int glm_gather_ranges(int64_t N, int D);
// The likelihood call of kind B2_GLM_BERNOULLI, B2_GLM_POISSON or B2_GLM_NORMAL with a gathered group effect (any
// other kind: B2_ERR_BAD_SHAPE), X split (every logit fp32-exact): the kind's gather kernel and glm_finish_kernel,
// D wide, with the finish's scale, weight, sum_coeff, flags, total and noise scale sigma[p * sigma_stride] (Normal).
// The run sums of ga are d loglik / d T_k before the finish's factor (weight * scale, and 1 / sigma_p^2 for Normal).
// workspace: glm_row_workspace(N, D, P) bytes.
int glm_gather_likelihood(int kind, const float* X, const float* y, const float* W, const float* b,
                          const float* sigma, int sigma_stride, float* dsigma, int64_t N, int D, int P, double scale,
                          double weight, double sum_coeff, int flags, float* sum_p, float* total, float* dW, float* db,
                          void* workspace, cudaStream_t s, const GlmGather& ga);

// ---- glm_group.cu ----
// The group kernel of kind B2_GLM_BERNOULLI, B2_GLM_POISSON or B2_GLM_BINOMIAL (row_trials: per-row counts m) with X
// rounded to nearest TF32, for the family launchers when glm_split_x is false; the X-split group kernels stay with
// their families.
int launch_glm_group_rn(int kind, const float* X, const float* y, const float* m, bool row_trials, const float* W,
                        const float* b, int64_t N, int D, int P, float* partials, int gx, cudaStream_t s,
                        GlmGroups grp);

// Launch of a kernel that needs more than 48 KB of dynamic shared memory: 0, or B2_ERR_LAUNCH when its
// shared-memory limit could not be raised.
template <typename... KArgs, typename... Args>
int launch_tc(void (*kernel)(KArgs...), dim3 grid, dim3 block, uint32_t smem, cudaStream_t s, Args... args) {
  if (!set_max_dynamic_smem(reinterpret_cast<const void*>(kernel), (int)smem)) return B2_ERR_LAUNCH;
  launch_pdl(kernel, grid, block, (size_t)smem, s, args...);
  return 0;
}

// Precision policy of the tensor-core tile loops: W is always split hi + lo; below 64 Ki rows the incoherent
// rounding of X to TF32 has not averaged out yet, so X is split as well (and whenever B2_FLAG_GLM_3XTF32 asks).
inline bool glm_split_x(int flags, int64_t N) { return (flags & B2_FLAG_GLM_3XTF32) || N < 65536; }

// f(std::integral_constant<int, DC>, std::integral_constant<bool, split_x>) for the glm_flat_pipeline
// instantiation that holds D: D padded to DC atoms of 32 columns, at least MinDC of them (D <= 128, so DC <= 4).
// Only DC >= MinDC are instantiated.
template <int MinDC, int DC = MinDC, class F>
int glm_dispatch_dc(int D, bool split_x, F&& f) {
  if constexpr (DC < 4) {
    if ((D + 31) / 32 > DC) return glm_dispatch_dc<MinDC, DC + 1>(D, split_x, f);
  }
  return split_x ? f(std::integral_constant<int, DC>{}, std::true_type{})
                 : f(std::integral_constant<int, DC>{}, std::false_type{});
}

// ---- the per-row entry points: b2_glm_poisson_log_rate, b2_glm_normal_loc, b2_glm_binomial_logits ----
// workspace: [ticket, 256 B][CTA partials gx * P * (D + 2)][one [P] row for the per-particle sums]
inline size_t glm_row_workspace(int64_t N, int D, int P) {
  if (N < 1 || D < 1 || D > 128 || P < 1) return 256;
  const size_t gx = (size_t)glm_tc_grid_x(N);
  return 256 + (gx * (size_t)P * (size_t)(D + 2) + (size_t)P) * sizeof(float);
}

struct GlmRowWorkspace {
  int gx;
  unsigned int* ticket;
  float* partials;
};

inline GlmRowWorkspace glm_row_areas(void* workspace, int64_t N, int D, int P) {
  GlmRowWorkspace w;
  w.gx = glm_tc_grid_x(N);
  w.ticket = reinterpret_cast<unsigned int*>(workspace);
  w.partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  return w;
}

// The argument checks of the per-row entry points, in order; null_operand and bad_operand are the family's own
// (a null sigma or trial-count pointer; a bad sigma_stride, trials_per_row or trial-count alignment).  The tiles
// arrive by TMA / bulk copies (16-byte aligned sources, 32-bit row coordinates), and these families have no fp32
// SIMT kernel.  With a group effect D + G columns must fit and the workspace is theirs.
inline int glm_row_check(const float* X, const float* y, const float* W, bool null_operand, int64_t N, int D, int P,
                         bool bad_operand, int flags, const void* workspace, size_t workspace_bytes,
                         GlmGroups grp = {}) {
  if (!X || !y || !W || null_operand) return B2_ERR_NULL;
  const int Da = D + grp.cols();
  if (N <= 0 || P <= 0 || D < 1 || Da > 128 || bad_operand) return B2_ERR_BAD_SHAPE;
  if (grp.idx && (grp.G < 1 || reinterpret_cast<uintptr_t>(grp.idx) % 16 != 0)) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (flags & B2_FLAG_GLM_FP32) return B2_ERR_BAD_SHAPE;
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < glm_row_workspace(N, Da, P)) return B2_ERR_WORKSPACE;
  return B2_OK;
}

}  // namespace b2
