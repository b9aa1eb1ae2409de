// glm_flat_tc.cuh -- the any-D tile loop of the Hopper GLM likelihood kernels: glm_flat_pipeline<Fam, DC,
// SPLIT_X> runs one likelihood family (glm_tc_common.cuh: Bernoulli for glm_flat_tc.cu, Poisson for
// glm_poisson_tc.cu, Normal for glm_normal_tc.cu, Binomial for glm_binomial_tc.cu) for any feature count D in 1..128.
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
// Budget: at DC = 4 one warpgroup holds W hi + lo (64 KB), X hi + lo (64 KB), X^T (34 KB), a landing tile
// (32 KB), 1 KB of labels and with GROUPS 1 KB of group indices (197 KB in all), and its GEMM 2 accumulator alone takes 68 registers.  So DC = 1 runs four warpgroups per CTA (the
// 128-register cap of glm_tc.cu), DC = 2 two and DC >= 3 one, each with a single landing stage.
//
// Group columns (GROUPS, a varying intercept alpha[g_n] by group): X @ w + b + alpha[g] is [X | onehot(g)] @
// [w ; alpha] + b, so the kernel runs at D_aug = D + G (<= 128) with G synthesised columns.  The group index g[N]
// (int32) is bulk-copied next to y into its own 1 KB region; the landing buffer keeps X's stride D, and the split
// pass writes column D + j of a row as 1 when g_n == j and 0 otherwise, in X (exact in TF32: X_lo is zero) and in
// X^T, so GEMM 1 gathers alpha and GEMM 2's dW columns D .. D+G-1 are the segment sums d loglik / d alpha_g.
// W, the partials and the finish are D_aug wide.  A row whose index is outside [0, G) gets NaN in every group
// column, so the likelihood and the group columns of dW come out NaN rather than silently dropping the row.  (The
// other gradients need not: the epilogues clamp a logit before they take its gradient.)
//
// Varying slopes (GROUPS and SLOPES, GlmGroups::S > 0 read at run time; the S = 0 kernels are built without them): X @ w + b + alpha[g] + SUM_k beta_k[g] x_{c_k} is
// [X | onehot(g) | x_{c_1} onehot(g) | ..] @ [w ; alpha ; beta_1 ; ..] + b, D_aug = D + G (1 + S).  Slope k's
// column D + kG + j of a row is its covariate X[n, c_k], read from the landing buffer row the split pass is on,
// when g_n == j and 0 otherwise.  It is split hi + lo and transposed into X^T as X's own columns are, so GEMM 1's
// logits stay fp32-exact under SPLIT_X and GEMM 2's columns D + kG .. D + (k+1)G - 1 are d loglik / d beta_k.  A
// row with an index outside [0, G) gets NaN in the slope columns too.
//
// Gathered group effects (GATHER, for more groups than the contraction has columns): X @ w + b + alpha[g] + SUM_k
// beta_k[g] x_{c_k} with GEMM 1 and GEMM 2 over X's D columns only, as the plain kernels; W, dW and the partials are
// D wide.  The group term e[n, p] = T_0[g_n][p] + SUM_k T_k[g_n][p] X[n, c_k] (GlmGather::tab, group-major [1 + S][G]
// tables of the chains' values, so a row's 64 chains are one 256-byte line) is built in fp32 into the warpgroup's
// [64 rows][64 chains] shared area while the tile's g and covariates are still in shared memory, and added to GEMM
// 1's accumulators before the family's epilogue, so every logit stays fp32-exact and no epilogue changes.  The same
// area then takes the tile's residuals (TF32-rounded, as GEMM 2 takes them), and the group gradients are run sums
// of them over rows of equal g: the rows must be sorted by group.  Each warpgroup takes a contiguous range of tiles
// (gather_range) and walks its rows in order, one thread per chain and block; a run that starts after the range's
// first row and ends before its last is written once to the group-gradient table GlmGather::gsum [1 + S][G][cp]; the
// range's first run goes to slot 0 and its last (if another) to slot 1 of GlmGather::slots [Q][2][4][cp], which the
// potential's finish adds in row order.  GlmGather::status[q] gets bit 0 for an index outside [0, G) (its rows get a
// NaN term, and no table entry is written for it) and bit 1 for a descending pair, checked across ranges too.
//
// Determinism: every CTA writes its partials once (warpgroups summed in a fixed order); no float atomics.
#pragma once
#include <cuda.h>

#include "b2_common.cuh"
#include "glm_host.cuh"
#include "glm_tc_common.cuh"

namespace b2 {
namespace tcf {

using namespace tc;

template <int DC, bool GROUPS = false, bool GATHER = false>
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
  static constexpr uint32_t WG_Y = WG_LAND + kOp;              // y [64] (Binomial: two slots of y, trials)
  static constexpr uint32_t WG_G = WG_Y + 1024;                // group index [64] int32 (GROUPS, GATHER)
  static constexpr uint32_t WG_E = WG_G + 1024;                // GATHER: [64 n][64 p] fp32 group term, then residuals
  static constexpr uint32_t kWGBytes = WG_G + (GROUPS ? 1024 : 0) + (GATHER ? 1024 + 16384 : 0);
  // CTA layout (operand regions 1024-byte aligned: the 128-byte swizzle pattern is taken from address bits)
  static constexpr uint32_t OFF_WHI = 0;                       // [DC][p 64][32] SW128
  static constexpr uint32_t OFF_WLO = OFF_WHI + kOp;
  static constexpr uint32_t OFF_WG = OFF_WLO + kOp;
  static constexpr uint32_t OFF_BAR = OFF_WG + kWG * kWGBytes;
  static constexpr uint32_t kSmemBytes = OFF_BAR + 64 + 1024;  // + slack for the 1024-byte alignment
  // the final reduction reuses the warpgroup regions: [kWG][64 p][KD + 1] floats + [kWG][64 p] lp sums (at most
  // fp64)
  static constexpr int kRS = kKD + 1;
  static_assert(kSmemBytes <= 232448, "shared memory budget");
  static_assert(kXtBlock % 1024 == 0 && kWGBytes % 1024 == 0, "operand alignment");
  static_assert(kWG * kM * kRS * 4 + kWG * kM * 8 <= kWG * kWGBytes, "reduction scratch");
};

// one 1-D bulk copy global -> shared, completing `bytes` (a non-zero multiple of 16) on the mbarrier
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// GATHER: the [64 n][64 p] shared area of a warpgroup holds entry (n, p) at n * 64 + (p ^ 8 ((n >> 1) & 3)), so
// that both the accumulator fragment (acc1[i], term_at) and a warp's row of 64 chains are free of bank conflicts
__device__ __forceinline__ int term_at(int i, int w4, int gid, int t4) {
  const int n = 8 * (i >> 2) + 2 * t4 + (i & 1), p = 16 * w4 + gid + 8 * ((i >> 1) & 1);
  return n * kM + (p ^ (t4 << 3));
}

// GATHER: the tile's group term e[n, p] = T_0[g_n][p] + SUM_k T_k[g_n][p] X[n, c_k] into et, from the landing
// buffer and the group indices before they are refilled; warp w4 builds rows 16 w4 .. 16 w4 + 15, each lane two
// chains.  An index outside [0, G) gives NaN, rows past the tile's end 0.
__device__ __forceinline__ void gather_term(const GlmGather& ga, const float* land, const int32_t* gs, float* et,
                                            int D, int rows, int slab, int w4, int lane) {
  const int64_t cb = (int64_t)slab * kM + 2 * lane;
#pragma unroll 4
  for (int i = 0; i < 16; ++i) {
    const int r = 16 * w4 + i;
    float2 e = make_float2(0.f, 0.f);
    if (r < rows) {
      const int gi = gs[r];
      if ((unsigned)gi < (unsigned)ga.G) {
        const float* tr = ga.tab + (int64_t)gi * ga.cp + cb;
        e = *reinterpret_cast<const float2*>(tr);
#pragma unroll
        for (int k = 0; k < 3; ++k)
          if (k < ga.S) {
            const float x = land[r * D + ga.col[k]];
            const float2 v = *reinterpret_cast<const float2*>(tr + (int64_t)(k + 1) * ga.G * ga.cp);
            e.x = fmaf(v.x, x, e.x);
            e.y = fmaf(v.y, x, e.y);
          }
      } else {
        e = make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
      }
    }
    reinterpret_cast<float2*>(et + r * kM)[lane ^ (((r >> 1) & 3) << 2)] = e;
  }
}

// GATHER: one thread's walk over its warpgroup's range of rows in order, for chain ch and the group effect's blocks
// k0 = kb and k1 = kb + 2 (thread t: kb = t >> 6; block 0 the intercept, block k slope k, k <= S): the run sums
// SUM r[n, ch] (times X[n, c] for a slope) over each run of equal g.  open is 0 before the range's first row, 1
// while its first run is open and 2 after.
struct GatherWalk {
  int q, k0, k1, c0, c1;                       // c0, c1: the blocks' covariate columns, -1 for none
  int64_t ch;
  int cur, open, stat;
  float s0, s1;
  __device__ __forceinline__ void init(const GlmGather& ga, int qi, int t, int slab) {
    const int kb = t >> 6;
    q = qi;
    k0 = kb;
    k1 = kb + 2;
    c0 = kb == 1 ? ga.col[0] : -1;
    c1 = kb == 0 ? (ga.S >= 2 ? ga.col[1] : -1) : (ga.S >= 3 ? ga.col[2] : -1);
    ch = (int64_t)slab * kM + (t & 63);
    cur = open = stat = 0;
    s0 = s1 = 0.f;
  }
  // the open run's sums: where 0 / 1 the range's first / last slot, 2 the table (a valid group only)
  __device__ __forceinline__ void flush(const GlmGather& ga, int where) {
    float *d0, *d1;
    if (where < 2) {
      float* b = ga.slots + (int64_t)(2 * q + where) * 4 * ga.cp + ch;
      d0 = b + (int64_t)k0 * ga.cp;
      d1 = b + (int64_t)k1 * ga.cp;
    } else {
      if ((unsigned)cur >= (unsigned)ga.G) return;
      d0 = ga.gsum + ((int64_t)k0 * ga.G + cur) * ga.cp + ch;
      d1 = ga.gsum + ((int64_t)k1 * ga.G + cur) * ga.cp + ch;
    }
    *d0 = s0;
    if (k1 <= ga.S) *d1 = s1;
  }
  // the tile's rows row0 .. row0 + rows - 1, residuals in et
  __device__ __forceinline__ void tile(const GlmGather& ga, const float* et, const float* __restrict__ X, int D,
                                       int64_t row0, int rows) {
    if (k0 > ga.S) return;
    const int p = (int)(ch & 63);
#pragma unroll 4
    for (int n = 0; n < rows; ++n) {
      const int64_t row = row0 + n;
      const int gn = __ldg(ga.idx + row);
      const float r = et[n * kM + (p ^ (((n >> 1) & 3) << 3))];
      const float x0 = c0 >= 0 ? __ldg(X + row * D + c0) : 1.f;
      const float x1 = c1 >= 0 ? __ldg(X + row * D + c1) : 0.f;
      if ((unsigned)gn >= (unsigned)ga.G) stat |= 1;
      if (open == 0) {
        if (row > 0 && __ldg(ga.idx + row - 1) > gn) stat |= 2;
        open = 1;
      } else if (gn != cur) {
        flush(ga, open == 1 ? 0 : 2);
        if (gn < cur) stat |= 2;
        open = 2;
        s0 = s1 = 0.f;
      }
      cur = gn;
      s0 = fmaf(r, x0, s0);
      s1 = fmaf(r, x1, s1);
    }
  }
  // the range's last run, and its status (one thread of the first slab)
  __device__ __forceinline__ void finish(const GlmGather& ga, int slab, int t) {
    if (k0 <= ga.S && open) flush(ga, open == 1 ? 0 : 1);
    if (t == 0 && slab == 0) ga.status[q] = stat;
  }
};

// wgmma accumulator fragment (m64nN, f32): thread (warp w4 of the warpgroup, lane = 4 gid + t4) holds
// d[4j + 2h + e] = D[16 w4 + gid + 8h][8j + 2 t4 + e].
// Binomial only (glm_tc_common.cuh): trials are the per-row counts [N] (kRowTrials, bulk-copied behind y) or
// the one count of every row (kConstTrials).
// GROUPS: grp.idx[N] the group index of each row, grp.G groups and (SLOPES) grp.S slopes on X's columns grp.col;
// W is [P][D + G (1 + S)], the partials [gx][P][D + G (1 + S) + 2].  Without SLOPES, S is 0.
// GATHER: the group effect of ga (P <= ga.cp), W and the partials D wide.
template <class Fam, int DC, bool SPLIT_X, bool GROUPS = false, bool SLOPES = false, bool GATHER = false>
__device__ __forceinline__ void glm_flat_pipeline(const float* __restrict__ X, const float* __restrict__ y,
                                                  const float* __restrict__ W, const float* __restrict__ bvec,
                                                  int64_t N, int D, int P, float* __restrict__ partials,
                                                  const float* __restrict__ trials = nullptr,
                                                  GlmGroups grp = {}, GlmGather ga = {}) {
  static_assert(!(GATHER && GROUPS), "one group-effect route per kernel");
  using C = Cfg<DC, GROUPS, GATHER>;
  constexpr int kKD = C::kKD, kWG = C::kWG;
  constexpr bool kIdx = GROUPS || GATHER;      // the tiles bring their group indices
  const int32_t* __restrict__ groups = GATHER ? ga.idx : grp.idx;
  const int G = grp.G;
  const int Da = GROUPS ? D + (SLOPES ? grp.cols() : G) : D;   // columns of the contraction
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
                                        C::kWGBytes, W, slab, P, 1, Da);
  fence_proxy_async();
  __syncthreads();

  typename Fam::LpAcc lpa[2] = {0, 0};         // lp sums of the thread's two particles
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
    int32_t* gs = reinterpret_cast<int32_t*>(my + C::WG_G);   // GROUPS, GATHER only
    // the warpgroup's tiles: it = it0, it0 + kStep, .. < itn, tile row0_of(it); GATHER: the contiguous range of tiles
    // [tb, tb + itn) of warpgroup q, the others round-robin over the CTAs and then the CTA's warpgroups
    const int q = blockIdx.x * kWG + wg;
    int64_t tb = 0, te = 0;
    if constexpr (GATHER) gather_tiles(q, gridDim.x * kWG, ntiles, tb, te);
    const int it0 = GATHER ? 0 : wg, itn = GATHER ? (int)(te - tb) : nt;
    constexpr int kStep = GATHER ? 1 : kWG;
    auto row0_of = [&](int it) -> int64_t {
      if constexpr (GATHER) return (tb + it) * kRows;
      else return (blockIdx.x + (int64_t)it * gridDim.x) * kRows;
    };
    float bias[2];                             // of particles 16 w4 + gid + 8h
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gp = slab * kM + 16 * w4 + gid + 8 * h;
      bias[h] = (bvec != nullptr && gp < P) ? bvec[gp] : 0.f;
    }
    // Binomial keeps the labels of two tiles, slot k & 1 of y [64] + trials [64] each, because its epilogue reads
    // them from shared memory while the next tile lands
    constexpr bool kRowM = Fam::kTrials == kRowTrials;
    float mconst = 0.f;                        // the one trial count (kConstTrials)
    if constexpr (Fam::kTrials == kConstTrials) mconst = *trials;
    // tile it -> landing buffer; one thread of the warpgroup issues the loads
    auto load = [&](int it) {
      const int64_t row0 = row0_of(it);
      const int rows = (int)(N - row0 < kRows ? N - row0 : kRows);
      const uint32_t xb = (uint32_t)(rows * D) * 4u, yb = (uint32_t)rows * 4u;
      const uint32_t xbulk = xb & ~15u, ybulk = yb & ~15u;
      const int yo = Fam::kTrials != kNoTrials ? (((it - it0) / kStep) & 1) * 2 * kRows : 0;
      if (rows < kRows || xbulk != xb) {       // the last tile: its remainder and zeros for y past N
        const float* xsrc = X + row0 * D;
        for (uint32_t i = xbulk / 4; i < xb / 4; ++i) land[i] = xsrc[i];
        for (int i = (int)(ybulk / 4); i < kRows; ++i) ys[yo + i] = (i < rows) ? y[row0 + i] : 0.f;
        if constexpr (kRowM)
          for (int i = (int)(ybulk / 4); i < kRows; ++i) ys[yo + kRows + i] = (i < rows) ? trials[row0 + i] : 0.f;
        if constexpr (kIdx)
          for (int i = (int)(ybulk / 4); i < kRows; ++i) gs[i] = (i < rows) ? groups[row0 + i] : 0;
      }
      // the arrive releases the ordinary stores above to the warpgroup's mbar_wait
      mbar_expect_tx(bar, xbulk + ((kRowM ? 2 : 1) + (kIdx ? 1 : 0)) * ybulk);
      if (xbulk) bulk_load(my_s + C::WG_LAND, X + row0 * D, xbulk, bar);
      if (ybulk) bulk_load(my_s + C::WG_Y + 4 * yo, y + row0, ybulk, bar);
      if constexpr (kRowM)
        if (ybulk) bulk_load(my_s + C::WG_Y + 4 * (yo + kRows), trials + row0, ybulk, bar);
      if constexpr (kIdx)
        if (ybulk) bulk_load(my_s + C::WG_G, groups + row0, ybulk, bar);
    };
    // GATHER: the walk over the range's rows (one thread per chain p and blocks kb, kb + 2 of the group effect)
    float* et = reinterpret_cast<float*>(my + C::WG_E);
    GatherWalk walk;
    if constexpr (GATHER) walk.init(ga, q, t, slab);
    if (t == 0 && it0 < itn) load(it0);
    for (int k = 0, it = it0; it < itn; ++k, it += kStep) {
      const int64_t row0 = row0_of(it);
      const int rows = (int)(N - row0 < kRows ? N - row0 : kRows);
      mbar_wait(bar, (uint32_t)k & 1u);
      // GEMM 2 of this warpgroup's previous tile has finished reading X^T and the g registers
      wgmma_wait0();
      fence_regs(acc2);
      // ---- split pass, once per 32-column atom, with the thread mapping of the D = 32 pipeline
      // (glm_tc_common.cuh): columns d >= D (GROUPS: d >= D_aug) and rows past N are exact zeros -------------
      {
        const int lam = t & 7, mu = t >> 3;
        const int e = lam & 1, q8 = ((mu >> 3) << 2) | (lam >> 1);
        const int c = (((lam & 1) << 2) | (lam >> 1)) ^ (mu & 7);
        const int kc = 2 * (q8 & 3) + e;
        float4* xs = reinterpret_cast<float4*>(my + C::WG_XOP);
        float4* xl = reinterpret_cast<float4*>(my + C::WG_XLO);
        float4* xt = reinterpret_cast<float4*>(my + C::WG_XT + (q8 >> 2) * C::kXtBlock);
        // GROUPS: the intercept column of each of the thread's rows, the covariates of its slope columns (k G
        // further on), and the value of its other group columns (0, or NaN in every group column for an index
        // outside [0, G): its intercept column is then far enough below 0 that no column matches)
        int gcol[4];
        float goff[4], gx[4][3];
        if constexpr (GROUPS) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = 8 * q8 + 2 * i + e;
            const int gi = gs[r];
            const bool ok = (unsigned)gi < (unsigned)G;
            gcol[i] = ok ? D + gi : (SLOPES ? -512 : -1);
            goff[i] = ok ? 0.f : __int_as_float(0x7fc00000);
            if constexpr (SLOPES) {
#pragma unroll
              for (int k = 0; k < 3; ++k) gx[i][k] = k < grp.S ? land[r * D + grp.col[k]] : 0.f;
            }
          }
        }
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
              if constexpr (SLOPES) {
                const int o = d - gcol[i];     // k G in slope k's column of the row's group, 0 in its intercept's
                const float gv = o == 0 ? 1.f : o == G ? gx[i][0] : o == 2 * G ? gx[i][1] : o == 3 * G ? gx[i][2]
                                                                                                      : goff[i];
                x[q] = (d < Da && r < rows) ? (d < D ? v : gv) : 0.f;
              } else if constexpr (GROUPS) {
                x[q] = (d < Da && r < rows) ? (d < D ? v : (d == gcol[i] ? 1.f : goff[i])) : 0.f;
              }
              else
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
      if constexpr (GATHER) gather_term(ga, land, gs, et, D, rows, slab, w4, lane);
      typename Fam::Labels yr;                 // read before the refill
      if constexpr (Fam::kTrials != kNoTrials) {
        const float* slot = ys + (k & 1) * 2 * kRows;
        Fam::read_labels(reinterpret_cast<const uint8_t*>(slot), t4, 1, yr);
        Fam::read_trials(reinterpret_cast<const uint8_t*>(slot + kRows), t4, mconst, yr);
      } else {
        Fam::read_labels(reinterpret_cast<const uint8_t*>(ys), t4, 1, yr);
      }
      fence_proxy_async();
      wg_bar(1 + wg);
      // the landing buffer is free: the warpgroup's next tile arrives while this one is contracted
      if (t == 0 && it + kStep < itn) load(it + kStep);
      float acc1[32];
      if constexpr (Fam::kBiasInEpilogue) {
        const float zero[2] = {0.f, 0.f};
        gemm1<DC, SPLIT_X>(acc1, zero, base + C::OFF_WHI, base + C::OFF_WLO, my_s + C::WG_XOP, my_s + C::WG_XLO);
      } else {
        gemm1<DC, SPLIT_X>(acc1, bias, base + C::OFF_WHI, base + C::OFF_WLO, my_s + C::WG_XOP, my_s + C::WG_XLO);
      }
      if constexpr (GATHER) {
#pragma unroll
        for (int i = 0; i < 32; ++i) acc1[i] += et[term_at(i, w4, gid, t4)];
      }
      uint32_t g[32];                          // indexed like acc1
      if constexpr (Fam::kBiasInEpilogue)
        Fam::tile_epilogue(acc1, bias, yr, row0, N, t4, rows < kRows, lpa, g);
      else
        Fam::tile_epilogue(acc1, yr, row0, N, t4, rows < kRows, lpa, g);
      if constexpr (GATHER) {
#pragma unroll
        for (int i = 0; i < 32; ++i) et[term_at(i, w4, gid, t4)] = __uint_as_float(g[i]);
      }
      // left running while the next tile is waited for
      gemm2<C::kN2>(acc2, g, my_s + C::WG_XT, it == it0);
      if constexpr (GATHER) {
        wg_bar(1 + wg);                        // every residual of the tile is in et
        walk.tile(ga, et, X, D, row0, rows);
        wg_bar(1 + wg);                        // et is free for the next tile's term
      }
    }
    wgmma_wait0();
    fence_regs(acc2);
    if constexpr (GATHER) {
      walk.finish(ga, slab, t);
      if (itn == 0) {                          // a warpgroup without tiles adds zeros to the CTA's partials
#pragma unroll
        for (int i = 0; i < C::kN2 / 2; ++i) acc2[i] = 0.f;
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      auto v = lpa[h];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      lpa[h] = v;
    }
  }
  double dterm = 0.0;
  if constexpr (Fam::kDataTerm) {
    if constexpr (GATHER) {                    // the CTA's rows are its warpgroups' ranges, one contiguous span
      int64_t t0, t1, u0, u1;
      gather_tiles(blockIdx.x * kWG, gridDim.x * kWG, ntiles, t0, u0);
      gather_tiles(blockIdx.x * kWG + kWG - 1, gridDim.x * kWG, ntiles, u1, t1);
      dterm = Fam::template data_term<C::kThreads, true>(y, trials, N, t0 * kRows, min(t1 * kRows, N));
    } else {
      dterm = Fam::template data_term<C::kThreads>(y, trials, N);
    }
  }
  // CTA results through the warpgroup regions, idle now (GATHER: every warpgroup, a tileless one with zeros)
  cta_partials<1, C::kN2, C::kThreads>(reinterpret_cast<float*>(sm + C::OFF_WG), acc2, lpa, wg, GATHER ? kWG : nt,
                                       slab, P, 1, Da, partials, dterm);
}

}  // namespace tcf
}  // namespace b2
