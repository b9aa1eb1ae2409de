// site_score.cuh -- fused log_prob + score kernels for elementwise families.
//
// One pass over the operands produces: the (scaled, masked) log_prob tensor if wanted, its sum,
// and the gradient w.r.t. value and every parameter, either full shape or summed to a scalar.
// Replaces the ATen chains behind pyro/poutine/trace_struct.py:248-328 (see pyro_b200.h).
//
// Two kernels:
//   site_vec_kernel  -- operands collapse to [R, C] with unit or zero inner stride; 16-byte
//                       vector loads/stores, 2 vectors in flight per operand per thread,
//                       no integer division in the loop.  This is the HBM-roofline kernel.
//   site_gen_kernel  -- any strides up to kMaxD dims; one element per thread iteration.
#pragma once
#include <stdlib.h>
#include "b2_common.cuh"
#include "b2_math.cuh"

namespace b2 {

struct Opnd {
  const void* ptr;
  int64_t st[kMaxD];
};
struct OutOpnd {
  void* ptr;
  int64_t st[kMaxD];
  int mode;  // 0 = not wanted, 1 = full shape, 2 = scalar (sum over everything),
             // 3 = summed over the dims where st == 0 (small kernel only)
};

struct SiteArgs {
  int ndim;
  int64_t shape[kMaxD];
  int64_t n;
  Opnd x;
  Opnd p[B2_MAX_PARAMS];
  Opnd mask;  // uint8
  Opnd up;    // upstream gradient (same dtype as value)
  OutOpnd lp;
  OutOpnd gx;
  OutOpnd gp[B2_MAX_PARAMS];
  double scale, weight, sum_coeff;
  float scale32, f032;  // (float)scale and (float)(weight*scale): fp32 kernels read these straight from the
                        // constant bank (the compiler re-converted the doubles PER ELEMENT: F2F.F32.F64)
  int flags;
  void* out_sum;
  double* partials;
  unsigned int* ticket;
  // vector path
  int64_t R, C;
  int tx_log2;  // threads along the column-vector axis = 1 << tx_log2 (block is 256 threads)
  // small path: scratch for mode-3 outputs, (2 + NP) slabs of n elements
  void* scratch;
};

constexpr int kSiteGen = 0, kSiteVec = 1, kSiteSmall = 2;
constexpr int64_t kSmallN = B2_SITE_SMALL_N;  // sites up to this many elements take the one-CTA kernel
constexpr int kSmallThreads = 1024;
static_assert((1 + B2_MAX_PARAMS) * kSmallN * sizeof(double) <= sizeof(double) * kMaxRed * kMaxPartialBlocks,
              "mode-3 slabs must fit in the partials region of the reduce workspace");

template <typename T>
__device__ __forceinline__ T site_scale(const SiteArgs& a) {
  return sizeof(T) == 4 ? (T)a.scale32 : (T)a.scale;
}
template <typename T>
__device__ __forceinline__ T site_f0(const SiteArgs& a) {
  return sizeof(T) == 4 ? (T)a.f032 : (T)(a.weight * a.scale);
}

template <typename T>
__device__ __forceinline__ void finish_outputs(const SiteArgs& a, int k, double tot) {
  constexpr int NPmax = B2_MAX_PARAMS;
  if (k == 0) {
    if (a.out_sum) {
      T* o = reinterpret_cast<T*>(a.out_sum);
      const double s = a.sum_coeff * tot;
      *o = (a.flags & B2_FLAG_ACCUMULATE_SUM) ? (T)((double)*o + s) : (T)s;
    }
  } else if (k == 1) {
    if (a.gx.mode == 2) *reinterpret_cast<T*>(a.gx.ptr) = (T)tot;
  } else if (k - 2 < NPmax) {
    if (a.gp[k - 2].mode == 2) *reinterpret_cast<T*>(a.gp[k - 2].ptr) = (T)tot;
  }
}

// ------------------------------------------------------------------------------------------------
// Vector kernel.  Block = 256 threads arranged TX x TY (TX = 1 << tx_log2 column-vector lanes,
// TY rows).  grid.x tiles column vectors, grid.y tiles rows; both grid-strided.
// Inner loop: U vectors per operand are loaded back to back (no predicates, no per-element
// branches), then evaluated, then stored; a one-vector tail loop handles the remainder.
// An operand is either a vector along the columns (column stride 1) or one scalar per row
// (column stride 0, loaded once per row).  MASKUP adds the optional mask / upstream operands.
// ------------------------------------------------------------------------------------------------
template <int FAM, typename T, bool GRAD, bool MASKUP, int NVEC>
struct VecBody {
  static constexpr int NP = FamilyTraits<FAM>::kNumParams;
  static constexpr bool HASV = FamilyTraits<FAM>::kHasValue;
  static constexpr int V = VecOf<T>::N;
  static constexpr int NRED = GRAD ? 2 + NP : 1;

  // operand classes, fixed for the launch: vector along columns (column stride 1) or one scalar
  // per row; row-invariant (row stride 0) vectors are loaded once per column chunk and reused
  // for every row (e.g. the observations y[N] scored against logits[P, N])
  bool x_vec, p_vec[NP], x_inv, p_inv[NP];
  T scale, f0;
  // per-row state
  const T* xr;
  const T* pr[NP];
  const T* ur;
  const uint8_t* mr;
  T* lpr;
  T* gxr;
  T* gpr[NP];
  T xs, ps[NP], us;
  bool u_vec, m_vec;
  bool want_dx;  // somebody reads the value gradient (a latent site); observed sites skip its extra SFU work
  // operand registers (invariant ones persist across rows)
  Pack<T> xv[NVEC], pv[NVEC][NP];
  // value-only term of a row-invariant value (b2_math.cuh ValueAux): once per column, not per row
  using VA = ValueAux<FAM, T, GRAD>;
  typename VA::type xa[VA::kHas ? NVEC : 1][VA::kHas ? V : 1];

  __device__ __forceinline__ void load_invariant(const T* xbase, const T* const (&pbase)[NP],
                                                 int64_t cv, int64_t cstep) {
#pragma unroll
    for (int u = 0; u < NVEC; ++u) {
      const int64_t c = (cv + u * cstep) * V;
      if (HASV && x_vec && x_inv) {
        xv[u] = ld_keep(xbase + c);
        if (VA::kHas) {
#pragma unroll
          for (int j = 0; j < V; ++j) xa[VA::kHas ? u : 0][VA::kHas ? j : 0] = VA::make(xv[u].v[j]);
        }
      }
#pragma unroll
      for (int k = 0; k < NP; ++k)
        if (p_vec[k] && p_inv[k]) pv[u][k] = ld_keep(pbase[k] + c);
    }
  }

  __device__ __forceinline__ void run(int64_t cv, int64_t cstep, T (&acc)[NRED]) {
    Pack<T> uv[NVEC];
    uint32_t mbits[NVEC];
#pragma unroll
    for (int u = 0; u < NVEC; ++u) {
      const int64_t c = (cv + u * cstep) * V;
      if (HASV && x_vec && !x_inv) xv[u] = ld_stream(xr + c);
#pragma unroll
      for (int k = 0; k < NP; ++k)
        if (p_vec[k] && !p_inv[k]) pv[u][k] = ld_stream(pr[k] + c);
      if (MASKUP) {
        if (ur && u_vec) uv[u] = ld_stream(ur + c);
        mbits[u] = 0xffffffffu;
        if (mr) {
          mbits[u] = 0;
#pragma unroll
          for (int j = 0; j < V; ++j) mbits[u] |= (mr[m_vec ? c + j : 0] != 0 ? 1u : 0u) << j;
        }
      }
    }
    // one-scalar-per-row operands are spread into the operand registers ONCE per row here; selecting
    // `p_vec ? vector : scalar` per element re-derived the predicate from the constant bank every time
    // (LDC + 2 ISETP + FSEL per operand per element: ~12 of Gamma's 75 instructions per element)
    if (HASV && !x_vec) {
#pragma unroll
      for (int u = 0; u < NVEC; ++u)
#pragma unroll
        for (int j = 0; j < V; ++j) xv[u].v[j] = xs;
    }
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      if (!p_vec[k]) {
#pragma unroll
        for (int u = 0; u < NVEC; ++u)
#pragma unroll
          for (int j = 0; j < V; ++j) pv[u][k].v[j] = ps[k];
      }
    }
#pragma unroll
    for (int u = 0; u < NVEC; ++u) {
      const int64_t c = (cv + u * cstep) * V;
      Pack<T> lpv, gxv, gpv[NP];
#pragma unroll
      for (int j = 0; j < V; ++j) {
        T pl[NP];
#pragma unroll
        for (int k = 0; k < NP; ++k) pl[k] = pv[u][k].v[j];
        const T xe = HASV ? xv[u].v[j] : (T)0;
        ElemOut<T> o;
        o.want_dx = want_dx;
        if constexpr (VA::kHas) {
          if (x_vec && x_inv) Eval<FAM, T, GRAD>::run_aux(xe, xa[u][j], pl, o);
          else Eval<FAM, T, GRAD>::run(xe, pl, o);
        } else {
          Eval<FAM, T, GRAD>::run(xe, pl, o);
        }
        T slp = o.lp * scale;
        T f = f0;
        if (MASKUP) {
          const bool m = (mbits[u] >> j) & 1u;
          slp = m ? slp : (T)0;
          f = m ? f0 : (T)0;
          if (ur) f *= u_vec ? uv[u].v[j] : us;
        }
        lpv.v[j] = slp;
        acc[0] += slp;
        if (GRAD) {
          T gxe = f * o.dx;
          if (MASKUP) gxe = (f == (T)0) ? (T)0 : gxe;  // masked-out NaNs must not leak
          gxv.v[j] = gxe;
          acc[1] += gxe;
#pragma unroll
          for (int k = 0; k < NP; ++k) {
            T g = f * o.dp[k];
            if (MASKUP) g = (f == (T)0) ? (T)0 : g;
            gpv[k].v[j] = g;
            acc[2 + k] += g;
          }
        }
      }
      if (lpr) st_stream(lpr + c, lpv);
      if (GRAD) {
        if (gxr) st_stream(gxr + c, gxv);
#pragma unroll
        for (int k = 0; k < NP; ++k)
          if (gpr[k]) st_stream(gpr[k] + c, gpv[k]);
      }
    }
  }

  // all rows of this thread for one column chunk
  __device__ __forceinline__ void chunk(const SiteArgs& a, int64_t cv, int64_t cstep, int ty, int TY,
                                        T (&acc)[NRED]) {
    const T* xbase = HASV ? reinterpret_cast<const T*>(a.x.ptr) : nullptr;
    const T* pbase[NP];
#pragma unroll
    for (int k = 0; k < NP; ++k) pbase[k] = reinterpret_cast<const T*>(a.p[k].ptr);
    load_invariant(xbase, pbase, cv, cstep);
    for (int64_t r = (int64_t)blockIdx.y * TY + ty; r < a.R; r += (int64_t)gridDim.y * TY) {
      xr = HASV ? xbase + r * a.x.st[0] : nullptr;
      xs = (HASV && !x_vec) ? __ldg(xr) : (T)0;
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        pr[k] = pbase[k] + r * a.p[k].st[0];
        ps[k] = p_vec[k] ? (T)0 : __ldg(pr[k]);
      }
      if (MASKUP) {
        ur = a.up.ptr ? reinterpret_cast<const T*>(a.up.ptr) + r * a.up.st[0] : nullptr;
        us = (ur && !u_vec) ? __ldg(ur) : (T)1;
        mr = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr) + r * a.mask.st[0] : nullptr;
      }
      lpr = a.lp.mode == 1 ? reinterpret_cast<T*>(a.lp.ptr) + r * a.lp.st[0] : nullptr;
      gxr = (GRAD && a.gx.mode == 1) ? reinterpret_cast<T*>(a.gx.ptr) + r * a.gx.st[0] : nullptr;
#pragma unroll
      for (int k = 0; k < NP; ++k)
        gpr[k] = (GRAD && a.gp[k].mode == 1) ? reinterpret_cast<T*>(a.gp[k].ptr) + r * a.gp[k].st[0] : nullptr;
      run(cv, cstep, acc);
    }
  }

  __device__ __forceinline__ void init(const SiteArgs& a) {
    x_vec = a.x.st[1] == 1;
    x_inv = a.x.st[0] == 0 && a.R > 1;
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      p_vec[k] = a.p[k].st[1] == 1;
      p_inv[k] = a.p[k].st[0] == 0 && a.R > 1;
    }
    scale = site_scale<T>(a);
    f0 = site_f0<T>(a);
    want_dx = a.gx.mode != 0;
    ur = nullptr;
    mr = nullptr;
    us = (T)1;
    u_vec = MASKUP && a.up.st[1] == 1;
    m_vec = MASKUP && a.mask.st[1] == 1;
  }
};

// Vectors in flight per operand per thread.  Forward-only fp32 kernels of the cheap families are pure streams: 4
// vectors.  Kernels that also write gradients carry more live registers, and the lgamma families (Gamma, Beta,
// Poisson) are bound by instruction issue, not by loads in flight: 2 vectors (4 would only cost registers).
template <int FAM, typename T, bool GRAD>
struct VecUnroll {
  static constexpr bool kHeavy = (FAM == kGamma || FAM == kBeta || FAM == kPoisson);
  static constexpr int U = (sizeof(T) == 4 && !GRAD && !kHeavy) ? 4 : 2;
  static constexpr int kMinBlocks = (sizeof(T) == 8 && GRAD) ? 2 : 3;
};

// Loop nest: column chunks outermost (U vectors per thread, then a one-vector tail), rows inside.
template <int FAM, typename T, bool GRAD, bool MASKUP>
__global__ void __launch_bounds__(256, VecUnroll<FAM, T, GRAD>::kMinBlocks) site_vec_kernel(const SiteArgs a) {
  constexpr int U = VecUnroll<FAM, T, GRAD>::U;
  constexpr int NP = FamilyTraits<FAM>::kNumParams;
  constexpr int V = VecOf<T>::N;
  constexpr int NRED = GRAD ? 2 + NP : 1;

  const int TX = 1 << a.tx_log2;
  const int tx = threadIdx.x & (TX - 1);
  const int ty = threadIdx.x >> a.tx_log2;
  const int TY = 256 >> a.tx_log2;
  const int64_t CV = a.C / V;
  const int64_t cstep = (int64_t)gridDim.x * TX;

  T acc[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) acc[k] = (T)0;

  int64_t cv = (int64_t)blockIdx.x * TX + tx;
  {
    VecBody<FAM, T, GRAD, MASKUP, U> body;
    body.init(a);
    for (; cv + (U - 1) * cstep < CV; cv += U * cstep) body.chunk(a, cv, cstep, ty, TY, acc);
  }
  {
    VecBody<FAM, T, GRAD, MASKUP, 1> tail;
    tail.init(a);
    for (; cv < CV; cv += cstep) tail.chunk(a, cv, cstep, ty, TY, acc);
  }

  __shared__ double smem[NRED * 32];
  double red[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) red[k] = (double)acc[k];
  grid_finish<NRED>(red, a.partials, a.ticket, smem,
                    [&](int k, double tot) { finish_outputs<T>(a, k, tot); });
}

// ------------------------------------------------------------------------------------------------
// Generic kernel: arbitrary strides, one element per loop trip.
// ------------------------------------------------------------------------------------------------
template <int FAM, typename T, bool GRAD>
__global__ void __launch_bounds__(256) site_gen_kernel(const SiteArgs a) {
  constexpr int NP = FamilyTraits<FAM>::kNumParams;
  constexpr bool HASV = FamilyTraits<FAM>::kHasValue;
  constexpr int NRED = GRAD ? 2 + NP : 1;
  const T f0 = site_f0<T>(a);
  const T scale = site_scale<T>(a);
  T acc[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) acc[k] = (T)0;

  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t rem = i;
    int64_t ox = 0, om = 0, ou = 0, olp = 0, ogx = 0;
    int64_t op[NP > 0 ? NP : 1], ogp[NP > 0 ? NP : 1];
#pragma unroll
    for (int k = 0; k < NP; ++k) op[k] = ogp[k] = 0;
    for (int d = a.ndim - 1; d >= 0; --d) {
      const int64_t q = rem / a.shape[d];
      const int64_t idx = rem - q * a.shape[d];
      rem = q;
      ox += idx * a.x.st[d];
      om += idx * a.mask.st[d];
      ou += idx * a.up.st[d];
      olp += idx * a.lp.st[d];
      ogx += idx * a.gx.st[d];
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        op[k] += idx * a.p[k].st[d];
        ogp[k] += idx * a.gp[k].st[d];
      }
    }
    T pl[NP > 0 ? NP : 1];
#pragma unroll
    for (int k = 0; k < NP; ++k) pl[k] = reinterpret_cast<const T*>(a.p[k].ptr)[op[k]];
    const T xv = HASV ? reinterpret_cast<const T*>(a.x.ptr)[ox] : (T)0;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    ElemOut<T> o;
    o.want_dx = a.gx.mode != 0;
    Eval<FAM, T, GRAD>::run(xv, pl, o);
    const T slp = m ? o.lp * scale : (T)0;
    acc[0] += slp;
    if (a.lp.mode == 1) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    if (GRAD) {
      T f = m ? f0 : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      const T gxe = m ? f * o.dx : (T)0;
      acc[1] += gxe;
      if (a.gx.mode == 1) reinterpret_cast<T*>(a.gx.ptr)[ogx] = gxe;
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        const T g = m ? f * o.dp[k] : (T)0;
        acc[2 + k] += g;
        if (a.gp[k].mode == 1) reinterpret_cast<T*>(a.gp[k].ptr)[ogp[k]] = g;
      }
    }
  }
  __shared__ double smem[NRED * 32];
  double red[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) red[k] = (double)acc[k];
  grid_finish<NRED>(red, a.partials, a.ticket, smem,
                    [&](int k, double tot) { finish_outputs<T>(a, k, tot); });
}

// ------------------------------------------------------------------------------------------------
// Small kernel: sites of at most kSmallN elements (every latent site of the BASELINE SVI configs:
// [P, D] weights, [P] biases) are launch-latency bound, so ONE CTA does everything in one launch --
// the elementwise pass, the scalar sums, and the reduction of each parameter gradient to the
// parameter's STORED shape (mode 3), which the large kernels leave to a follow-up b2_reduce_to.
// Mode-3 gradients go through a scratch slab (common shape, row major); after a CTA barrier one
// warp per stored element sums its broadcast positions in a fixed order (deterministic).
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void small_reduce_out(const SiteArgs& a, const OutOpnd& o, const T* slab) {
  // dims with st != 0 index the output; dims with st == 0 are summed.  n <= kSmallN, so every
  // index fits 32 bits (64-bit integer division is a ~100-instruction dependent chain on the GPU).
  unsigned cst[kMaxD], shp[kMaxD];
  unsigned m = 1;
  {
    unsigned c = 1;
    for (int d = a.ndim - 1; d >= 0; --d) {
      shp[d] = (unsigned)a.shape[d];
      cst[d] = c;
      c *= shp[d];
      if (o.st[d] != 0) m *= shp[d];
    }
  }
  const unsigned n = (unsigned)a.n;
  const unsigned q = n / m;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  T* out = reinterpret_cast<T*>(o.ptr);
  for (unsigned j = warp; j < m; j += nwarps) {
    unsigned rem = j, base = 0;
    int64_t off = 0;
    for (int d = a.ndim - 1; d >= 0; --d) {
      if (o.st[d] == 0) continue;
      const unsigned qq = rem / shp[d];
      const unsigned idx = rem - qq * shp[d];
      rem = qq;
      base += idx * cst[d];
      off += (int64_t)idx * o.st[d];
    }
    double s = 0.0;
    for (unsigned t = lane; t < q; t += 32) {
      unsigned r2 = t, flat = base;
      for (int d = a.ndim - 1; d >= 0; --d) {
        if (o.st[d] != 0) continue;
        const unsigned qq = r2 / shp[d];
        flat += (r2 - qq * shp[d]) * cst[d];
        r2 = qq;
      }
      s += (double)slab[flat];
    }
    s = warp_sum(s);
    if (lane == 0) out[off] = (T)s;
  }
}

template <int FAM, typename T, bool GRAD>
__global__ void __launch_bounds__(kSmallThreads) site_small_kernel(const SiteArgs a) {
  constexpr int NP = FamilyTraits<FAM>::kNumParams;
  constexpr bool HASV = FamilyTraits<FAM>::kHasValue;
  constexpr int NRED = GRAD ? 2 + NP : 1;
  const T f0 = site_f0<T>(a);
  const T scale = site_scale<T>(a);
  T acc[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) acc[k] = (T)0;
  T* slab = reinterpret_cast<T*>(a.scratch);
  const unsigned n = (unsigned)a.n;

  for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
    unsigned rem = i;
    int64_t ox = 0, om = 0, ou = 0, olp = 0, ogx = 0;
    int64_t op[NP > 0 ? NP : 1], ogp[NP > 0 ? NP : 1];
#pragma unroll
    for (int k = 0; k < NP; ++k) op[k] = ogp[k] = 0;
    for (int d = a.ndim - 1; d >= 0; --d) {
      const unsigned sd = (unsigned)a.shape[d];
      const unsigned q = rem / sd;
      const int64_t idx = (int64_t)(rem - q * sd);
      rem = q;
      ox += idx * a.x.st[d];
      om += idx * a.mask.st[d];
      ou += idx * a.up.st[d];
      olp += idx * a.lp.st[d];
      ogx += idx * a.gx.st[d];
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        op[k] += idx * a.p[k].st[d];
        ogp[k] += idx * a.gp[k].st[d];
      }
    }
    T pl[NP > 0 ? NP : 1];
#pragma unroll
    for (int k = 0; k < NP; ++k) pl[k] = reinterpret_cast<const T*>(a.p[k].ptr)[op[k]];
    const T xv = (HASV && a.x.ptr) ? reinterpret_cast<const T*>(a.x.ptr)[ox] : (T)0;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    ElemOut<T> o;
    o.want_dx = a.gx.mode != 0;
    Eval<FAM, T, GRAD>::run(xv, pl, o);
    const T slp = m ? o.lp * scale : (T)0;
    acc[0] += slp;
    if (a.lp.mode == 1) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    if (GRAD) {
      T f = m ? f0 : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      const T gxe = m ? f * o.dx : (T)0;
      acc[1] += gxe;
      if (a.gx.mode == 1) reinterpret_cast<T*>(a.gx.ptr)[ogx] = gxe;
      else if (a.gx.mode == 3) slab[i] = gxe;
#pragma unroll
      for (int k = 0; k < NP; ++k) {
        const T g = m ? f * o.dp[k] : (T)0;
        acc[2 + k] += g;
        if (a.gp[k].mode == 1) reinterpret_cast<T*>(a.gp[k].ptr)[ogp[k]] = g;
        else if (a.gp[k].mode == 3) slab[(size_t)(1 + k) * n + i] = g;
      }
    }
  }
  __shared__ double smem[NRED * 32];
  double red[NRED];
#pragma unroll
  for (int k = 0; k < NRED; ++k) red[k] = (double)acc[k];
  block_sum<NRED>(red, smem);  // ends with a CTA barrier: the slabs are complete and visible
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NRED; ++k) finish_outputs<T>(a, k, red[k]);
  }
  if (GRAD) {
    // ONE copy of the reduction code, looped over the outputs: these kernels run from a cold
    // instruction cache, so a second inlined copy costs more than the loop
#pragma unroll 1
    for (int k = 0; k <= NP; ++k) {
      OutOpnd o = a.gx;
#pragma unroll
      for (int j = 0; j < NP; ++j)
        if (k == j + 1) o = a.gp[j];
      if (o.mode == 3) small_reduce_out<T>(a, o, slab + (size_t)k * n);
    }
  }
}

// host-side launcher for one (family, dtype, grad) combination
template <int FAM, typename T, bool GRAD>
int launch_site(const SiteArgs& a, int kind, cudaStream_t stream) {
  if (kind == kSiteSmall) {
    int threads = (int)((a.n + 31) / 32) * 32;
    if (threads > kSmallThreads) threads = kSmallThreads;
    if (threads < 32) threads = 32;
    site_small_kernel<FAM, T, GRAD><<<1, threads, 0, stream>>>(a);
  } else if (kind == kSiteVec) {
    constexpr int V = VecOf<T>::N;
    constexpr int U = VecUnroll<FAM, T, GRAD>::U;
    const int64_t CV = a.C / V;
    const int TX = 1 << a.tx_log2, TY = 256 / TX;
    // enough CTAs for ~4 waves of resident blocks; each thread then owns >= U vectors per row
    int64_t gx = (CV + (int64_t)TX * U - 1) / ((int64_t)TX * U);
    int64_t gy = (a.R + TY - 1) / TY;
    const int64_t target = (int64_t)kNumSMs * 12;
    if (gx > target) gx = target;
    int64_t gy_cap = target / gx;
    if (gy_cap < 1) gy_cap = 1;
    if (gy > gy_cap) gy = gy_cap;
    if (gy > 65535) gy = 65535;
    dim3 grid((unsigned)gx, (unsigned)gy, 1);
    if (a.mask.ptr || a.up.ptr)
      site_vec_kernel<FAM, T, GRAD, true><<<grid, 256, 0, stream>>>(a);
    else
      site_vec_kernel<FAM, T, GRAD, false><<<grid, 256, 0, stream>>>(a);
  } else {
    int64_t blocks = (a.n + 255) / 256;
    const int64_t target = (int64_t)kNumSMs * 8;
    if (blocks > target) blocks = target;
    if (blocks < 1) blocks = 1;
    site_gen_kernel<FAM, T, GRAD><<<(unsigned)blocks, 256, 0, stream>>>(a);
  }
  count_launch();
  return check_launch();
}

// implemented in site_score_fam*.cu (split so the families compile in parallel)
int dispatch_site_a(int family, int dtype, bool grad, const SiteArgs& a, int kind, cudaStream_t s);
int dispatch_site_b(int family, int dtype, bool grad, const SiteArgs& a, int kind, cudaStream_t s);
int dispatch_site_c(int family, int dtype, bool grad, const SiteArgs& a, int kind, cudaStream_t s);

#define B2_DISPATCH_CASE(FAM)                                                         \
  case FAM:                                                                           \
    if (dtype == B2_F32)                                                              \
      return grad ? launch_site<FAM, float, true>(a, kind, s)                          \
                  : launch_site<FAM, float, false>(a, kind, s);                        \
    else                                                                              \
      return grad ? launch_site<FAM, double, true>(a, kind, s)                         \
                  : launch_site<FAM, double, false>(a, kind, s);

}  // namespace b2
