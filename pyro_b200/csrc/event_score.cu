// event_score.cu -- fused log_prob + score for families with an event dimension:
// Dirichlet, Categorical(logits), MultivariateNormal(scale_tril); and b2_reduce_to.
//
// One sub-warp group of G lanes (G = power of two <= 32, >= event size when that is < 32) owns
// one batch row; event dims are contiguous so the lanes of a group read consecutive addresses.
// Gradients are always written full shape [batch, event...]; batch-broadcast operands are summed
// afterwards by b2_reduce_to (deterministic two-stage tree, no float atomics).
#include <string.h>

#include <stdlib.h>

#include "b2_common.cuh"
#include "b2_math.cuh"

namespace b2 {

struct EvOpnd {
  const void* ptr;
  int64_t st[kMaxD];  // batch strides (elements)
};
struct EvOut {
  void* ptr;
  int64_t st[kMaxD];
};
struct EventArgs {
  int ndim;  // batch dims after coalescing
  int64_t shape[kMaxD];
  int64_t nbatch;
  int K;  // event size
  EvOpnd x, p0, p1, mask, up;
  EvOut lp, gx, gp0, gp1;
  double scale, weight, sum_coeff;
  int flags;
  void* out_sum;
  double* partials;
  unsigned int* ticket;
  int g_log2;  // lanes per row = 1 << g_log2
};

constexpr int kEvIdx32 = 1 << 29;  // EventArgs::flags: one merged batch dim, every operand offset fits 32 bits

template <typename T>
__device__ __forceinline__ T group_sum(T v, int G) {
  for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <typename T>
__device__ __forceinline__ T group_max(T v, int G) {
  for (int o = G >> 1; o > 0; o >>= 1) v = b2_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void batch_offsets(const EventArgs& a, int64_t row, int64_t& ox,
                                              int64_t& op0, int64_t& op1, int64_t& om, int64_t& ou,
                                              int64_t& olp, int64_t& ogx, int64_t& ogp0,
                                              int64_t& ogp1) {
  if (a.ndim <= 1) {
    // the common case after the host merged the batch dims: one multiply per operand, no division
    ox = row * a.x.st[0]; op0 = row * a.p0.st[0]; op1 = row * a.p1.st[0]; om = row * a.mask.st[0];
    ou = row * a.up.st[0]; olp = row * a.lp.st[0]; ogx = row * a.gx.st[0]; ogp0 = row * a.gp0.st[0];
    ogp1 = row * a.gp1.st[0];
    return;
  }
  ox = op0 = op1 = om = ou = olp = ogx = ogp0 = ogp1 = 0;
  int64_t rem = row;
  for (int d = a.ndim - 1; d >= 0; --d) {
    const int64_t q = rem / a.shape[d];
    const int64_t idx = rem - q * a.shape[d];
    rem = q;
    ox += idx * a.x.st[d];
    op0 += idx * a.p0.st[d];
    op1 += idx * a.p1.st[d];
    om += idx * a.mask.st[d];
    ou += idx * a.up.st[d];
    olp += idx * a.lp.st[d];
    ogx += idx * a.gx.st[d];
    ogp0 += idx * a.gp0.st[d];
    ogp1 += idx * a.gp1.st[d];
  }
}

template <typename T>
__device__ __forceinline__ void finish_sum(const EventArgs& a, double tot) {
  if (a.out_sum) {
    T* o = reinterpret_cast<T*>(a.out_sum);
    const double s = a.sum_coeff * tot;
    *o = (a.flags & B2_FLAG_ACCUMULATE_SUM) ? (T)((double)*o + s) : (T)s;
  }
}

// ---- Dirichlet: torch/distributions/dirichlet.py:90-97 -----------------------------------------
//   sum_k xlogy(a_k - 1, x_k) + lgamma(sum a) - sum_k lgamma(a_k)
template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) dirichlet_kernel(const EventArgs a) {
  const int G = 1 << a.g_log2;
  const int lane = threadIdx.x & (G - 1);
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> a.g_log2;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) >> a.g_log2;
  const T* xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* cp = reinterpret_cast<const T*>(a.p0.ptr);
  const int64_t nrows_pad = ((a.nbatch + ngroups - 1) / ngroups) * ngroups;
  T acc = (T)0;
  for (int64_t row = gid; row < nrows_pad; row += ngroups) {
    const bool live = row < a.nbatch;  // keep the whole warp converged for the shuffles
    int64_t ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1;
    batch_offsets(a, live ? row : 0, ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1);
    T s_xlogy = 0, s_conc = 0, s_lg = 0;
    for (int k = lane; k < a.K; k += G) {
      const T c = cp[op0 + k], x = xp[ox + k];
      s_xlogy += (sizeof(T) == 4) ? ((c - (T)1 == (T)0) ? (T)0 : (c - (T)1) * fast_log(x)) : xlogy(c - (T)1, x);
      s_conc += c;
      T lgc, unused;
      lgamma_digamma<T, false>(c, lgc, unused);
      s_lg += lgc;
    }
    s_xlogy = group_sum(s_xlogy, G);
    s_conc = group_sum(s_conc, G);
    s_lg = group_sum(s_lg, G);
    T lgsum, psum;
    lgamma_digamma<T, GRAD>(s_conc, lgsum, psum);
    const T lp = s_xlogy + lgsum - s_lg;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    const T slp = (m && live) ? lp * (T)a.scale : (T)0;
    if (lane == 0 && live) {
      acc += slp;
      if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    }
    if (GRAD && live) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      for (int k = lane; k < a.K; k += G) {
        const T c = cp[op0 + k], x = xp[ox + k];
        if (a.gx.ptr) reinterpret_cast<T*>(a.gx.ptr)[ogx + k] = m ? f * (c - (T)1) / x : (T)0;
        if (a.gp0.ptr) {
          T lgc, psc;
          lgamma_digamma<T, true>(c, lgc, psc);
          reinterpret_cast<T*>(a.gp0.ptr)[ogp0 + k] = m ? f * (b2_log(x) + psum - psc) : (T)0;
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- Categorical(logits): torch/distributions/categorical.py:78 (logits - logsumexp) and
// :151-157 (gather).  value is int64; the gathered index is exact. -------------------------------
template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) categorical_kernel(const EventArgs a) {
  const int G = 1 << a.g_log2;
  const int lane = threadIdx.x & (G - 1);
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> a.g_log2;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) >> a.g_log2;
  const int64_t* vp = reinterpret_cast<const int64_t*>(a.x.ptr);
  const T* lg = reinterpret_cast<const T*>(a.p0.ptr);
  const int64_t nrows_pad = ((a.nbatch + ngroups - 1) / ngroups) * ngroups;
  T acc = (T)0;
  for (int64_t row = gid; row < nrows_pad; row += ngroups) {
    const bool live = row < a.nbatch;
    int64_t ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1;
    batch_offsets(a, live ? row : 0, ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1);
    T mx = -b2_inf<T>();
    for (int k = lane; k < a.K; k += G) mx = b2_max(mx, lg[op0 + k]);
    mx = group_max(mx, G);
    T se = 0;
    for (int k = lane; k < a.K; k += G) se += b2_exp(lg[op0 + k] - mx);
    se = group_sum(se, G);
    const T lse = mx + b2_log(se);
    const int64_t v = vp[ox];
    const bool inb = v >= 0 && v < a.K;
    const T lp = inb ? lg[op0 + v] - lse : b2_nan<T>();
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    const T slp = (m && live) ? lp * (T)a.scale : (T)0;
    if (lane == 0 && live) {
      acc += slp;
      if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    }
    if (GRAD && live && a.gp0.ptr) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      for (int k = lane; k < a.K; k += G) {
        const T sm = b2_exp(lg[op0 + k] - lse);
        reinterpret_cast<T*>(a.gp0.ptr)[ogp0 + k] = m ? f * (((int64_t)k == v ? (T)1 : (T)0) - sm) : (T)0;
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- small event sizes (K <= 32), batch dims merged to one: ONE THREAD PER ROW ----------------------
// A row is K consecutive elements per operand, so a warp covers 32 consecutive rows = one contiguous
// span of memory: every fetched line is fully used (through L1 across the k loop), the K special
// functions of a row are independent work for one thread (ILP without shuffles), and there is no
// per-row integer division; the sub-warp-group kernels above waste most of their lanes at small K.
template <typename T>
B2_HD T xlogy_fast(T c, T x) {
  if (sizeof(T) == 4) return (c == (T)0) ? (T)0 : c * fast_log(x);
  return xlogy(c, x);
}

template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) dirichlet_rowthread_kernel(const EventArgs a) {
  const T* __restrict__ xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* __restrict__ cp = reinterpret_cast<const T*>(a.p0.ptr);
  const int K = a.K;
  T acc = (T)0;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nbatch;
       row += (int64_t)gridDim.x * blockDim.x) {
    const T* x = xp + row * a.x.st[0];
    const T* c = cp + row * a.p0.st[0];
    T s_xlogy = 0, s_conc = 0, s_lg = 0;
    if (a.g_log2 == 1) {
      // rows are 16-byte aligned and K is a multiple of the vector width: one 16-byte load per chunk
      constexpr int V = VecOf<T>::N;
      for (int k = 0; k < K; k += V) {
        const Pack<T> cv = ld_stream(c + k), xv = ld_stream(x + k);
#pragma unroll
        for (int j = 0; j < V; ++j) {
          s_xlogy += xlogy_fast(cv.v[j] - (T)1, xv.v[j]);
          s_conc += cv.v[j];
          T lgc, unused;
          lgamma_digamma<T, false>(cv.v[j], lgc, unused);
          s_lg += lgc;
        }
      }
    } else {
      for (int k = 0; k < K; ++k) {
        const T ck = c[k];
        s_xlogy += xlogy_fast(ck - (T)1, x[k]);
        s_conc += ck;
        T lgc, unused;
        lgamma_digamma<T, false>(ck, lgc, unused);
        s_lg += lgc;
      }
    }
    T lgsum, psum;
    lgamma_digamma<T, GRAD>(s_conc, lgsum, psum);
    const T lp = s_xlogy + lgsum - s_lg;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[row * a.mask.st[0]] != 0 : true;
    const T slp = m ? lp * (T)a.scale : (T)0;
    acc += slp;
    if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[row * a.lp.st[0]] = slp;
    if (GRAD) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[row * a.up.st[0]];
      T* gx = a.gx.ptr ? reinterpret_cast<T*>(a.gx.ptr) + row * a.gx.st[0] : nullptr;
      T* gc = a.gp0.ptr ? reinterpret_cast<T*>(a.gp0.ptr) + row * a.gp0.st[0] : nullptr;
      for (int k = 0; k < K; ++k) {
        const T ck = c[k], xk = x[k];
        if (gx) gx[k] = m ? f * (ck - (T)1) * fast_rcp(xk) : (T)0;
        if (gc) {
          T lgc, psc;
          lgamma_digamma<T, true>(ck, lgc, psc);
          gc[k] = m ? f * (fast_log(xk) + psum - psc) : (T)0;
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) categorical_rowthread_kernel(const EventArgs a) {
  const int64_t* __restrict__ vp = reinterpret_cast<const int64_t*>(a.x.ptr);
  const T* __restrict__ lgp = reinterpret_cast<const T*>(a.p0.ptr);
  const int K = a.K;
  T acc = (T)0;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nbatch;
       row += (int64_t)gridDim.x * blockDim.x) {
    const T* lg = lgp + row * a.p0.st[0];
    const int64_t v = vp[row * a.x.st[0]];  // issued first: overlaps the logits loads
    T mx = -b2_inf<T>();
    T se = 0;
    if (a.g_log2 == 1) {
      // 16-byte loads, online logsumexp over the chunks (one pass over the row)
      constexpr int V = VecOf<T>::N;
      for (int k = 0; k < K; k += V) {
        const Pack<T> lv = ld_keep(lg + k);
        T cm = lv.v[0];
#pragma unroll
        for (int j = 1; j < V; ++j) cm = b2_max(cm, lv.v[j]);
        const T nm = b2_max(mx, cm);
        // no finite logit yet: the running sum (0, or NaN from exp(-inf - -inf)) is dropped, as in the vec kernel
        T sacc = (mx == -b2_inf<T>()) ? (T)0 : se * fast_exp(mx - nm);
#pragma unroll
        for (int j = 0; j < V; ++j) sacc += fast_exp(lv.v[j] - nm);
        se = sacc;
        mx = nm;
      }
    } else {
      for (int k = 0; k < K; ++k) mx = b2_max(mx, lg[k]);
      for (int k = 0; k < K; ++k) se += fast_exp(lg[k] - mx);
    }
    const T lse = mx + fast_log(se);
    const bool inb = v >= 0 && v < K;
    const T lp = inb ? lg[inb ? v : 0] - lse : b2_nan<T>();
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[row * a.mask.st[0]] != 0 : true;
    const T slp = m ? lp * (T)a.scale : (T)0;
    acc += slp;
    if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[row * a.lp.st[0]] = slp;
    if (GRAD && a.gp0.ptr) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[row * a.up.st[0]];
      T* g = reinterpret_cast<T*>(a.gp0.ptr) + row * a.gp0.st[0];
      for (int k = 0; k < K; ++k)
        g[k] = m ? f * (((int64_t)k == v ? (T)1 : (T)0) - fast_exp(lg[k] - lse)) : (T)0;
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- MultivariateNormal(loc, scale_tril): torch/distributions/multivariate_normal.py:256-264,
// _batch_mahalanobis :29-80.   -0.5*(n log 2pi + |L^-1 (x-mu)|^2) - sum log diag L.
// One full warp per row; forward substitution with a warp reduction per pivot.  The residual z (and
// w = L^-T z for the gradients) live in NSLOT registers per lane: NSLOT = 4 covers n <= 128 (round 1),
// NSLOT = 16 / 32 cover n <= 512 / 1024 (round 2: the MVN sizes of BASELINE config 3, H = 512).  The
// per-pivot work is an O(n) dot product read straight from L (L2-resident when the factor is shared by
// the batch), so the kernel is latency-bound, not a tensor-core GEMM; a blocked TRSM on wgmma only
// pays off for thousands of right-hand sides per factor, which no BASELINE config has. ----------
constexpr int kMvnMaxN = 1024;
template <typename T, bool GRAD, int NSLOT = 4>
__global__ void __launch_bounds__(256) mvn_tril_kernel(const EventArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int n = a.K;
  const T* xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* mu = reinterpret_cast<const T*>(a.p0.ptr);
  const T* Lp = reinterpret_cast<const T*>(a.p1.ptr);
  const int64_t nrows_pad = ((a.nbatch + nwarps - 1) / nwarps) * nwarps;
  T acc = (T)0;
  for (int64_t row = wid; row < nrows_pad; row += nwarps) {
    const bool live = row < a.nbatch;
    int64_t ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1;
    batch_offsets(a, live ? row : 0, ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1);
    const T* L = Lp + op1;
    // z = L^-1 (x - mu), element j lives in lane j%32, slot j/32
    T z[NSLOT];
#pragma unroll
    for (int s = 0; s < NSLOT; ++s) z[s] = (T)0;
    T logdet = 0;
    for (int i = 0; i < n; ++i) {
      T part = 0;
#pragma unroll
      for (int s = 0; s < NSLOT; ++s) {
        const int j = s * 32 + lane;
        if (j < i) part += L[(int64_t)i * n + j] * z[s];
      }
      part = warp_sum(part);
      const T lii = L[(int64_t)i * n + i];
      const T zi = ((xp[ox + i] - mu[op0 + i]) - part) / lii;
      logdet += b2_log(lii);
#pragma unroll
      for (int s = 0; s < NSLOT; ++s)
        if (s == (i >> 5) && (i & 31) == lane) z[s] = zi;
    }
    T m2 = 0;
#pragma unroll
    for (int s = 0; s < NSLOT; ++s) m2 += z[s] * z[s];
    m2 = warp_sum(m2);
    const T lp = (T)-0.5 * ((T)n * ((T)2 * Consts<T>::kLogSqrt2Pi) + m2) - logdet;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    const T slp = (m && live) ? lp * (T)a.scale : (T)0;
    if (lane == 0 && live) {
      acc += slp;
      if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    }
    if (GRAD) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      // w = L^-T z  (back substitution):  w_i = (z_i - sum_{j>i} L_ji w_j) / L_ii
      T w[NSLOT];
#pragma unroll
      for (int s = 0; s < NSLOT; ++s) w[s] = (T)0;
      for (int i = n - 1; i >= 0; --i) {
        T part = 0;
#pragma unroll
        for (int s = 0; s < NSLOT; ++s) {
          const int j = s * 32 + lane;
          if (j > i && j < n) part += L[(int64_t)j * n + i] * w[s];
        }
        part = warp_sum(part);
        T zsel = (T)0;
#pragma unroll
        for (int s = 0; s < NSLOT; ++s)
          if (s == (i >> 5)) zsel = z[s];
        const T zi = __shfl_sync(0xffffffffu, zsel, i & 31);
        const T wi = (zi - part) / L[(int64_t)i * n + i];
#pragma unroll
        for (int s = 0; s < NSLOT; ++s)
          if (s == (i >> 5) && (i & 31) == lane) w[s] = wi;
      }
      if (live) {
#pragma unroll
        for (int s = 0; s < NSLOT; ++s) {
          const int j = s * 32 + lane;
          if (j < n) {
            if (a.gx.ptr) reinterpret_cast<T*>(a.gx.ptr)[ogx + j] = m ? -f * w[s] : (T)0;
            if (a.gp0.ptr) reinterpret_cast<T*>(a.gp0.ptr)[ogp0 + j] = m ? f * w[s] : (T)0;
          }
        }
      }
      if (a.gp1.ptr) {
        // dL = f * (tril(w z^T) - diag(1/L_ii)); strictly upper part is zero
        T* gL = reinterpret_cast<T*>(a.gp1.ptr) + ogp1;
        for (int i = 0; i < n; ++i) {
          T wsel = (T)0;
#pragma unroll
          for (int s = 0; s < NSLOT; ++s)
            if (s == (i >> 5)) wsel = w[s];
          const T wi = __shfl_sync(0xffffffffu, wsel, i & 31);
#pragma unroll
          for (int s = 0; s < NSLOT; ++s) {
            const int j = s * 32 + lane;
            if (j < n && live) {
              T g = (T)0;
              if (j < i) g = wi * z[s];
              else if (j == i) g = wi * z[s] - (T)1 / L[(int64_t)i * n + i];
              gL[(int64_t)i * n + j] = m ? f * g : (T)0;
            }
          }
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- MVN, n <= 32: a group of G lanes (G = 2, 4, 8 or 32 >= n) owns a batch row ----------------------------
// Lane j holds ROW j of the factor (Lr[k] = L[j][k]), so forward substitution is a chain of broadcasts:
//   pivot i:  z_i = r_i / L_ii is final on lane i -> one shuffle -> every lane j > i does r_j -= L[j][i] z_i
// i.e. ~35 cycles per pivot (shuffle + FMA) instead of the five dependent shuffle/add steps of a group
// reduction per pivot, which is what a column-owning lane needs (the thread-per-row kernel for n <= 8 walks L with
// 4-byte loads 4*n*n bytes apart across a warp and runs fully unrolled to 8 whatever n is).  Rows are read
// coalesced: G <= 8 as 16-byte (8-byte for G = 2) chunks of consecutive lanes, G = 32 as 32 row-major 128-byte
// lines staged through a padded shared-memory tile and read back transposed.  The gradient pass needs the
// columns as well (w = L^-T z is a broadcast chain for COLUMN owners); they come from the same tile / from L1.
template <typename T, int G>
struct MvnGroupCfg {
  static constexpr int kThreads = (G == 32 && sizeof(T) == 8) ? 128 : 256;   // static shared memory <= 48 KB
  static constexpr int kTile = (G == 32) ? (kThreads / 32) * 32 * 33 : 1;
};

// FULL: n == G (no per-pivot bounds tests, constant address offsets).  IDX32: one merged batch dim whose offsets
// fit 32 bits (one IMAD per operand instead of a 64-bit multiply chain: with G = 2 a warp iteration is 16 rows
// of 36 bytes and the offset arithmetic alone was a third of its instructions).
template <typename T, bool GRAD, int G, bool FULL>
__global__ void __launch_bounds__(MvnGroupCfg<T, G>::kThreads) mvn_group_kernel(const EventArgs a) {
  const int lane = threadIdx.x & (G - 1);
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) / G;
  const int n = FULL ? G : a.K;
  const T* xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* mup = reinterpret_cast<const T*>(a.p0.ptr);
  const T* Lp = reinterpret_cast<const T*>(a.p1.ptr);
  const int64_t nrows_pad = ((a.nbatch + ngroups - 1) / ngroups) * ngroups;
  const bool in = FULL || lane < n;
  const bool idx32 = (a.flags & kEvIdx32) != 0;
  const T scale = (T)a.scale, f0 = (T)(a.weight * a.scale);
  __shared__ T tile[MvnGroupCfg<T, G>::kTile];
  T* tw = tile + ((G == 32) ? (threadIdx.x >> 5) * 32 * 33 : 0);
  // dense rows whose length is the group width are read in 16-byte (8-byte) chunks
  constexpr int V = (G >= 4) ? ((sizeof(T) == 4) ? 4 : 2) : ((sizeof(T) == 4) ? 2 : 1);
  const bool vec_rows = FULL && (G <= 8) && (reinterpret_cast<uintptr_t>(Lp) % 16 == 0) && (a.ndim <= 1) &&
                        (a.p1.st[0] % 4 == 0);
  T acc = (T)0;
  for (int64_t row = gid; row < nrows_pad; row += ngroups) {
    const bool live = row < a.nbatch;
    int64_t ox, op0, op1, om = 0, ou = 0, olp = 0, ogx = 0, ogp0 = 0, ogp1 = 0;
    if (idx32) {
      const int r32 = live ? (int)row : 0;
      ox = r32 * (int)a.x.st[0];
      op0 = r32 * (int)a.p0.st[0];
      op1 = r32 * (int)a.p1.st[0];
      if (a.mask.ptr) om = r32 * (int)a.mask.st[0];
      if (a.lp.ptr) olp = r32 * (int)a.lp.st[0];
      if (GRAD) {
        if (a.up.ptr) ou = r32 * (int)a.up.st[0];
        ogx = r32 * (int)a.gx.st[0];
        ogp0 = r32 * (int)a.gp0.st[0];
        ogp1 = r32 * (int)a.gp1.st[0];
      }
    } else {
      batch_offsets(a, live ? row : 0, ox, op0, op1, om, ou, olp, ogx, ogp0, ogp1);
    }
    const T* L = Lp + op1;
    // Lr[k] = L[lane][k], Lc[r] = L[r][lane]; entries above the diagonal and outside n are never used (forward
    // substitution touches Lr[i] on lanes > i, back substitution Lc[j] on lanes < j), so nothing is masked here
    T Lr[G], Lc[GRAD ? G : 1];
    T dg = (T)1;
    if constexpr (G == 32) {
#pragma unroll
      for (int r = 0; r < G; ++r)
        tw[r * 33 + lane] = (FULL || (r < n && in)) ? __ldcs(L + (FULL ? r * G : r * n) + lane) : (T)0;
      __syncwarp();
#pragma unroll
      for (int k = 0; k < G; ++k) Lr[k] = tw[lane * 33 + k];
      dg = tw[lane * 33 + lane];
      if (GRAD) {
#pragma unroll
        for (int r = 0; r < G; ++r) Lc[GRAD ? r : 0] = tw[r * 33 + lane];
      }
      __syncwarp();
    } else {
      if (vec_rows) {
        using VT = typename VecN<T, V>::type;
#pragma unroll
        for (int c = 0; c < G / V; ++c) {
          const VT v = __ldcs(reinterpret_cast<const VT*>(L + lane * G) + c);
          const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
          for (int j = 0; j < V; ++j) Lr[c * V + j] = e[j];
        }
      } else {
#pragma unroll
        for (int k = 0; k < G; ++k) Lr[k] = (in && (FULL || k < n)) ? L[lane * n + k] : (T)0;
      }
      if (GRAD) {
#pragma unroll
        for (int r = 0; r < G; ++r) Lc[GRAD ? r : 0] = (in && (FULL || r < n)) ? L[r * n + lane] : (T)0;
      }
#pragma unroll
      for (int k = 0; k < G; ++k) dg = (k == lane) ? Lr[k] : dg;
    }
    if (!FULL) dg = in ? dg : (T)1;
    const T idg = (sizeof(T) == 4) ? fast_rcp(dg) : (T)1 / dg;
    T r = in ? xp[ox + lane] - mup[op0 + lane] : (T)0;
#pragma unroll
    for (int i = 0; i < G; ++i) {
      if (FULL || i < n) {  // uniform
        const T zi = __shfl_sync(0xffffffffu, r * idg, i, G);
        r = (lane > i) ? r - Lr[i] * zi : r;
      }
    }
    const T z = r * idg;
    const T m2 = group_sum(in ? z * z : (T)0, G);
    const T logdet = group_sum(in ? ((sizeof(T) == 4) ? fast_log(dg) : b2_log(dg)) : (T)0, G);
    const T lp = (T)-0.5 * ((T)n * ((T)2 * Consts<T>::kLogSqrt2Pi) + m2) - logdet;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[om] != 0 : true;
    const T slp = (m && live) ? lp * scale : (T)0;
    if (lane == 0 && live) {
      acc += slp;
      if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[olp] = slp;
    }
    if (GRAD) {
      T f = m ? f0 : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[ou];
      T sacc = (T)0, w = (T)0;
#pragma unroll
      for (int j = G - 1; j >= 0; --j) {
        if (FULL || j < n) {
          if (lane == j) w = (z - sacc) * idg;
          const T wj = __shfl_sync(0xffffffffu, w, j, G);
          if (lane < j) sacc += Lc[GRAD ? j : 0] * wj;  // Lc[j] on lane i is L[j][i]
        }
      }
      if (live && in) {
        if (a.gx.ptr) reinterpret_cast<T*>(a.gx.ptr)[ogx + lane] = m ? -f * w : (T)0;
        if (a.gp0.ptr) reinterpret_cast<T*>(a.gp0.ptr)[ogp0 + lane] = m ? f * w : (T)0;
      }
      if (a.gp1.ptr) {
        // dL[i][j] = f (w_i z_j - [i == j] / L_ii) for j <= i, 0 above the diagonal; lane j writes column j
        T* gL = reinterpret_cast<T*>(a.gp1.ptr) + ogp1;
#pragma unroll
        for (int i = 0; i < G; ++i) {
          if (FULL || i < n) {
            const T wi = __shfl_sync(0xffffffffu, w, i, G);
            if (live && in) {
              T g = (T)0;
              if (lane < i) g = wi * z;
              else if (lane == i) g = wi * z - idg;
              gL[i * n + lane] = m ? f * g : (T)0;
            }
          }
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- generic strided sum-to ---------------------------------------------------------------------
struct ReduceArgs {
  int nk, nr;                     // kept / reduced dims
  int64_t kshape[kMaxD], rshape[kMaxD];
  int64_t ksrc[kMaxD], kdst[kMaxD], rsrc[kMaxD];
  int64_t nout, nred;
  int splits;
  const void* src;
  void* dst;
  double* partials;  // [nout, splits] when splits > 1
};

template <typename T>
__global__ void __launch_bounds__(256) reduce_to_kernel(const ReduceArgs a) {
  const int64_t o = blockIdx.x;
  const int s = blockIdx.y;
  int64_t rem = o, so = 0, dof = 0;
  for (int d = a.nk - 1; d >= 0; --d) {
    const int64_t q = rem / a.kshape[d];
    const int64_t idx = rem - q * a.kshape[d];
    rem = q;
    so += idx * a.ksrc[d];
    dof += idx * a.kdst[d];
  }
  const int64_t per = (a.nred + a.splits - 1) / a.splits;
  const int64_t lo = (int64_t)s * per;
  int64_t hi = lo + per;
  if (hi > a.nred) hi = a.nred;
  const T* src = reinterpret_cast<const T*>(a.src) + so;
  double acc = 0.0;
  for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    int64_t r = i, off = 0;
    for (int d = a.nr - 1; d >= 0; --d) {
      const int64_t q = r / a.rshape[d];
      off += (r - q * a.rshape[d]) * a.rsrc[d];
      r = q;
    }
    acc += (double)src[off];
  }
  __shared__ double smem[32];
  double red[1] = {acc};
  block_sum<1>(red, smem);
  if (threadIdx.x == 0) {
    if (a.splits == 1) reinterpret_cast<T*>(a.dst)[dof] = (T)red[0];
    else a.partials[o * a.splits + s] = red[0];
  }
}

// Column reduction: the kept dims are the trailing, contiguous ones (dst[C] = sum over R rows of
// src[R, C], row stride C) -- the gradient of a parameter that is broadcast over particles / chains.
// Threads own columns (coalesced), grid.y splits the rows; fixed summation order.  The one-CTA-per-
// output kernel above reads this layout with a 4*C-byte stride between lanes.
template <typename T>
__global__ void __launch_bounds__(256) reduce_cols_kernel(const T* __restrict__ src, T* __restrict__ dst,
                                                          double* __restrict__ partials, int64_t R,
                                                          int64_t C, int splits) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int s = blockIdx.y;
  const int64_t per = (R + splits - 1) / splits;
  const int64_t lo = (int64_t)s * per;
  int64_t hi = lo + per;
  if (hi > R) hi = R;
  double acc = 0.0;
  int64_t r = lo;
  for (; r + 3 < hi; r += 4) {
    const T v0 = src[r * C + c], v1 = src[(r + 1) * C + c], v2 = src[(r + 2) * C + c], v3 = src[(r + 3) * C + c];
    acc += (double)v0;
    acc += (double)v1;
    acc += (double)v2;
    acc += (double)v3;
  }
  for (; r < hi; ++r) acc += (double)src[r * C + c];
  if (splits == 1) dst[c] = (T)acc;
  else partials[(int64_t)s * C + c] = acc;
}

template <typename T>
__global__ void reduce_cols_finish_kernel(const double* __restrict__ partials, T* __restrict__ dst, int64_t C,
                                          int splits) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
  for (int i = 0; i < splits; ++i) s += partials[(int64_t)i * C + c];
  dst[c] = (T)s;
}

template <typename T>
__global__ void reduce_to_finish_kernel(const ReduceArgs a) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= a.nout) return;
  int64_t rem = o, dof = 0;
  for (int d = a.nk - 1; d >= 0; --d) {
    const int64_t q = rem / a.kshape[d];
    dof += (rem - q * a.kshape[d]) * a.kdst[d];
    rem = q;
  }
  double s = 0.0;
  for (int i = 0; i < a.splits; ++i) s += a.partials[o * a.splits + i];
  reinterpret_cast<T*>(a.dst)[dof] = (T)s;
}


// ---- larger event sizes (K a multiple of the vector width, rows 16-byte aligned) ---------------------------
// G = min(32, K/V/4) lanes own a row and each lane takes kChunks = 4 16-byte chunks per step, for two rows
// (row, row + ngroups) at once: 8 independent 16-byte loads in flight per thread, and the per-row overhead --
// the group reductions, the row's own special functions, offsets, the mask -- is spread over >= 16 elements per
// lane.  With one chunk per lane (G = K/V lanes) the kernel is issue-bound, not memory-bound: most of its
// instructions are per-row work amortised over only 4 elements per lane.
constexpr int kChunks = 4;

template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) dirichlet_vec_kernel(const EventArgs a) {
  constexpr int V = VecOf<T>::N;
  constexpr int UR = 1;  // one row per group in flight: 8 chunks (conc + value) already hold 32 registers
  const int G = 1 << a.g_log2;
  const int lane = threadIdx.x & (G - 1);
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> a.g_log2;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) >> a.g_log2;
  const T* xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* cp = reinterpret_cast<const T*>(a.p0.ptr);
  const int KV = a.K / V;
  const int64_t nrows_pad = ((a.nbatch + UR * ngroups - 1) / (UR * ngroups)) * (UR * ngroups);
  const T scale = (T)a.scale, f0 = (T)(a.weight * a.scale);
  T acc = (T)0;
  for (int64_t row0 = gid; row0 < nrows_pad; row0 += UR * ngroups) {
    T s_xlogy[UR], s_conc[UR], s_lg[UR];
    bool live[UR];
    int64_t rows[UR];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      rows[u] = row0 + u * ngroups;
      live[u] = rows[u] < a.nbatch;
      if (!live[u]) rows[u] = 0;
      s_xlogy[u] = s_conc[u] = s_lg[u] = (T)0;
    }
    for (int kv0 = lane; kv0 < KV; kv0 += kChunks * G) {
      Pack<T> cv[UR][kChunks], xv[UR][kChunks];
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        const T* cr = cp + rows[u] * a.p0.st[0];
        const T* xr = xp + rows[u] * a.x.st[0];
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          const int kv = kv0 + c * G;
          if (kv < KV) {
            cv[u][c] = ld_stream(cr + kv * V);
            xv[u][c] = ld_stream(xr + kv * V);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UR; ++u) {
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          if (kv0 + c * G < KV) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
              const T cc = cv[u][c].v[j];
              s_xlogy[u] += xlogy_fast(cc - (T)1, xv[u][c].v[j]);
              s_conc[u] += cc;
              T lgc, unused;
              lgamma_digamma<T, false>(cc, lgc, unused);
              s_lg[u] += lgc;
            }
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      s_xlogy[u] = group_sum(s_xlogy[u], G);
      s_conc[u] = group_sum(s_conc[u], G);
      s_lg[u] = group_sum(s_lg[u], G);
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const int64_t row = rows[u];
      T lgsum, psum;
      lgamma_digamma<T, GRAD>(s_conc[u], lgsum, psum);
      const T lp = s_xlogy[u] + lgsum - s_lg[u];
      const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[row * a.mask.st[0]] != 0 : true;
      const T slp = (m && live[u]) ? lp * scale : (T)0;
      if (lane == 0 && live[u]) {
        acc += slp;
        if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[row * a.lp.st[0]] = slp;
      }
      if (GRAD && live[u]) {
        T f = m ? f0 : (T)0;
        if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[row * a.up.st[0]];
        for (int kv = lane; kv < KV; kv += G) {
          const Pack<T> cv = ld_keep(cp + row * a.p0.st[0] + kv * V);
          const Pack<T> xv = ld_keep(xp + row * a.x.st[0] + kv * V);
          Pack<T> gxv, gcv;
#pragma unroll
          for (int j = 0; j < V; ++j) {
            const T c = cv.v[j], x = xv.v[j];
            gxv.v[j] = m ? f * (c - (T)1) * fast_rcp(x) : (T)0;
            T lgc, psc;
            lgamma_digamma<T, true>(c, lgc, psc);
            gcv.v[j] = m ? f * (fast_log(x) + psum - psc) : (T)0;
          }
          if (a.gx.ptr) st_stream(reinterpret_cast<T*>(a.gx.ptr) + row * a.gx.st[0] + kv * V, gxv);
          if (a.gp0.ptr) st_stream(reinterpret_cast<T*>(a.gp0.ptr) + row * a.gp0.st[0] + kv * V, gcv);
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

template <typename T, bool GRAD>
__global__ void __launch_bounds__(256) categorical_vec_kernel(const EventArgs a) {
  constexpr int V = VecOf<T>::N;
  constexpr int UR = 2;  // rows in flight per lane group
  const int G = 1 << a.g_log2;
  const int lane = threadIdx.x & (G - 1);
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> a.g_log2;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) >> a.g_log2;
  const int64_t* vp = reinterpret_cast<const int64_t*>(a.x.ptr);
  const T* lgp = reinterpret_cast<const T*>(a.p0.ptr);
  const int KV = a.K / V;
  const int64_t nrows_pad = ((a.nbatch + UR * ngroups - 1) / (UR * ngroups)) * (UR * ngroups);
  const T scale = (T)a.scale, f0 = (T)(a.weight * a.scale);
  T acc = (T)0;
  for (int64_t row0 = gid; row0 < nrows_pad; row0 += UR * ngroups) {
    bool live[UR];
    int64_t rows[UR], vidx[UR];
    T mx[UR], se[UR];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      rows[u] = row0 + u * ngroups;
      live[u] = rows[u] < a.nbatch;
      if (!live[u]) rows[u] = 0;
      mx[u] = -b2_inf<T>();
      se[u] = (T)0;
      vidx[u] = vp[rows[u] * a.x.st[0]];  // issued first: overlaps the logits stream
    }
    // online logsumexp, one step = up to kChunks chunks per lane per row: max of the step first, ONE
    // rescale of the running sum, then the exponentials
    for (int kv0 = lane; kv0 < KV; kv0 += kChunks * G) {
      Pack<T> lv[UR][kChunks];
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        const T* lr = lgp + rows[u] * a.p0.st[0];
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          const int kv = kv0 + c * G;
          if (kv < KV) lv[u][c] = ld_keep(lr + kv * V);
        }
      }
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        T cm = -b2_inf<T>();
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          if (kv0 + c * G < KV) {
#pragma unroll
            for (int j = 0; j < V; ++j) cm = b2_max(cm, lv[u][c].v[j]);
          }
        }
        const T nm = b2_max(mx[u], cm);
        T sacc = (mx[u] == -b2_inf<T>()) ? (T)0 : se[u] * fast_exp(mx[u] - nm);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          if (kv0 + c * G < KV) {
#pragma unroll
            for (int j = 0; j < V; ++j) sacc += fast_exp(lv[u][c].v[j] - nm);
          }
        }
        se[u] = sacc;
        mx[u] = nm;
      }
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const T gm = group_max(mx[u], G);
      const T part = (mx[u] == -b2_inf<T>()) ? (T)0 : se[u] * fast_exp(mx[u] - gm);
      se[u] = group_sum(part, G);
      mx[u] = gm;
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const int64_t row = rows[u];
      const T* lg = lgp + row * a.p0.st[0];
      const T lse = mx[u] + fast_log(se[u]);
      const int64_t v = vidx[u];
      const bool inb = v >= 0 && v < a.K;
      const T lp = inb ? lg[inb ? v : 0] - lse : b2_nan<T>();
      const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[row * a.mask.st[0]] != 0 : true;
      const T slp = (m && live[u]) ? lp * scale : (T)0;
      if (lane == 0 && live[u]) {
        acc += slp;
        if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[row * a.lp.st[0]] = slp;
      }
      if (GRAD && live[u] && a.gp0.ptr) {
        T f = m ? f0 : (T)0;
        if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[row * a.up.st[0]];
        for (int kv = lane; kv < KV; kv += G) {
          const Pack<T> lv = ld_keep(lg + kv * V);
          Pack<T> gv;
#pragma unroll
          for (int j = 0; j < V; ++j)
            gv.v[j] = m ? f * (((int64_t)(kv * V + j) == v ? (T)1 : (T)0) - fast_exp(lv.v[j] - lse)) : (T)0;
          st_stream(reinterpret_cast<T*>(a.gp0.ptr) + row * a.gp0.st[0] + kv * V, gv);
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}

// ---- MVN, event size n <= 8: one thread per row ------------------------------------------------------
// The warp-per-row kernel above spends 32 lanes and n warp reductions on a 2x2 .. 8x8 triangular
// solve.  For small n the whole solve fits
// one thread's registers: z = L^-1 (x - mu) by forward substitution, w = L^-T z by back substitution,
// all loops fully unrolled over NMAX with predicates on the runtime n; a warp covers 32 consecutive
// rows, i.e. one contiguous span of each operand.
template <typename T, bool GRAD, int NMAX>
__global__ void __launch_bounds__(256) mvn_rowthread_kernel(const EventArgs a) {
  const T* __restrict__ xp = reinterpret_cast<const T*>(a.x.ptr);
  const T* __restrict__ mup = reinterpret_cast<const T*>(a.p0.ptr);
  const T* __restrict__ Lp = reinterpret_cast<const T*>(a.p1.ptr);
  const int n = a.K;
  T acc = (T)0;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nbatch;
       row += (int64_t)gridDim.x * blockDim.x) {
    const T* x = xp + row * a.x.st[0];
    const T* mu = mup + row * a.p0.st[0];
    const T* L = Lp + row * a.p1.st[0];
    T z[NMAX], inv[NMAX];
    T logdet = 0, m2 = 0;
#pragma unroll
    for (int i = 0; i < NMAX; ++i) {
      z[i] = (T)0;
      inv[i] = (T)0;
      if (i < n) {
        T part = x[i] - mu[i];
#pragma unroll
        for (int j = 0; j < i; ++j) part -= L[i * n + j] * z[j];
        const T lii = L[i * n + i];
        inv[i] = (T)1 / lii;
        z[i] = part * inv[i];
        logdet += (sizeof(T) == 4) ? fast_log(lii) : b2_log(lii);
        m2 += z[i] * z[i];
      }
    }
    const T lp = (T)-0.5 * ((T)n * ((T)2 * Consts<T>::kLogSqrt2Pi) + m2) - logdet;
    const bool m = a.mask.ptr ? reinterpret_cast<const uint8_t*>(a.mask.ptr)[row * a.mask.st[0]] != 0 : true;
    const T slp = m ? lp * (T)a.scale : (T)0;
    acc += slp;
    if (a.lp.ptr) reinterpret_cast<T*>(a.lp.ptr)[row * a.lp.st[0]] = slp;
    if (GRAD) {
      T f = m ? (T)(a.weight * a.scale) : (T)0;
      if (a.up.ptr) f *= reinterpret_cast<const T*>(a.up.ptr)[row * a.up.st[0]];
      T w[NMAX];
#pragma unroll
      for (int i = NMAX - 1; i >= 0; --i) {
        w[i] = (T)0;
        if (i < n) {
          T part = z[i];
#pragma unroll
          for (int j = i + 1; j < NMAX; ++j)
            if (j < n) part -= L[j * n + i] * w[j];
          w[i] = part * inv[i];
        }
      }
      T* gx = a.gx.ptr ? reinterpret_cast<T*>(a.gx.ptr) + row * a.gx.st[0] : nullptr;
      T* gm = a.gp0.ptr ? reinterpret_cast<T*>(a.gp0.ptr) + row * a.gp0.st[0] : nullptr;
      T* gL = a.gp1.ptr ? reinterpret_cast<T*>(a.gp1.ptr) + row * a.gp1.st[0] : nullptr;
#pragma unroll
      for (int i = 0; i < NMAX; ++i) {
        if (i < n) {
          if (gx) gx[i] = m ? -f * w[i] : (T)0;
          if (gm) gm[i] = m ? f * w[i] : (T)0;
          if (gL) {
#pragma unroll
            for (int j = 0; j < NMAX; ++j) {
              if (j < n) {
                T g = (T)0;
                if (j < i) g = w[i] * z[j];
                else if (j == i) g = w[i] * z[j] - inv[i];
                gL[i * n + j] = m ? f * g : (T)0;
              }
            }
          }
        }
      }
    }
  }
  __shared__ double smem[32];
  double red[1] = {(double)acc};
  grid_finish<1>(red, a.partials, a.ticket, smem, [&](int, double tot) { finish_sum<T>(a, tot); });
}


}  // namespace b2

using namespace b2;

extern "C" int b2_event_score(int family, const b2_tensor* value, const b2_tensor* params,
                              int n_params, int event_size, const b2_tensor* mask, double scale,
                              const b2_tensor* upstream, double weight, double sum_coeff,
                              int flags, b2_tensor* out_logprob, void* out_sum,
                              b2_tensor* out_dvalue, b2_tensor* out_dparams, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (!value || !params) return B2_ERR_NULL;
  if (!workspace || workspace_bytes < kReduceWorkspaceBytes) return B2_ERR_WORKSPACE;
  const int want_params = (family == B2_MVN_TRIL) ? 2 : 1;
  if (family != B2_DIRICHLET && family != B2_CATEGORICAL && family != B2_MVN_TRIL)
    return B2_ERR_BAD_FAMILY;
  if (n_params != want_params) return B2_ERR_BAD_SHAPE;
  const int dtype = params[0].dtype;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_BAD_DTYPE;
  if (family == B2_CATEGORICAL) {
    if (value->dtype != B2_I64) return B2_ERR_BAD_DTYPE;
  } else if (value->dtype != dtype) {
    return B2_ERR_BAD_DTYPE;
  }
  if (event_size < 1) return B2_ERR_BAD_SHAPE;
  if (family == B2_MVN_TRIL && event_size > kMvnMaxN) return B2_ERR_TOO_LARGE;
  // `value->shape[:ndim]` is the batch shape shared by every operand; strides are batch strides.
  const int nd = value->ndim;
  if (nd < 0 || nd > B2_MAX_DIMS) return B2_ERR_BAD_SHAPE;

  EventArgs a;
  memset(&a, 0, sizeof(a));
  a.K = event_size;
  a.scale = scale;
  a.weight = weight;
  a.sum_coeff = sum_coeff;
  a.flags = flags;
  a.out_sum = out_sum;
  a.partials = ws_partials(workspace);
  a.ticket = ws_ticket(workspace);
  // drop size-1 batch dims, then merge adjacent dims that every operand walks jointly (contiguous or
  // jointly broadcast): the usual [rows] or [P, rows] batch becomes ONE dim, decoded by a multiply
  int cd = 0;
  int64_t nb = 1;
  int keep[B2_MAX_DIMS];
  for (int d = 0; d < nd; ++d) {
    nb *= value->shape[d];
    if (value->shape[d] != 1) keep[cd++] = d;
  }
  if (cd > kMaxD) return B2_ERR_BAD_SHAPE;
  const b2_tensor* ops[9] = {value, &params[0], n_params > 1 ? &params[1] : nullptr, mask, upstream,
                             out_logprob, out_dvalue, out_dparams ? &out_dparams[0] : nullptr,
                             (out_dparams && n_params > 1) ? &out_dparams[1] : nullptr};
  int64_t shp[B2_MAX_DIMS], ost[9][B2_MAX_DIMS];
  for (int i = 0; i < cd; ++i) {
    shp[i] = value->shape[keep[i]];
    for (int o = 0; o < 9; ++o) ost[o][i] = (ops[o] && ops[o]->ptr) ? ops[o]->stride[keep[i]] : 0;
  }
  for (int d = cd - 2; d >= 0; --d) {
    bool ok = true;
    for (int o = 0; o < 9 && ok; ++o) ok = ost[o][d] == ost[o][d + 1] * shp[d + 1];
    if (!ok) continue;
    shp[d] *= shp[d + 1];
    for (int o = 0; o < 9; ++o) ost[o][d] = ost[o][d + 1];
    for (int e = d + 1; e < cd - 1; ++e) {
      shp[e] = shp[e + 1];
      for (int o = 0; o < 9; ++o) ost[o][e] = ost[o][e + 1];
    }
    --cd;
  }
  a.ndim = cd;
  a.nbatch = nb;
  for (int i = 0; i < cd; ++i) a.shape[i] = shp[i];
  auto fin = [&](EvOpnd& o, int k) {
    if (!ops[k] || !ops[k]->ptr) return;
    o.ptr = ops[k]->ptr;
    for (int i = 0; i < cd; ++i) o.st[i] = ost[k][i];
  };
  auto fout = [&](EvOut& o, int k) {
    if (!ops[k] || !ops[k]->ptr) return;
    o.ptr = ops[k]->ptr;
    for (int i = 0; i < cd; ++i) o.st[i] = ost[k][i];
  };
  fin(a.x, 0);
  fin(a.p0, 1);
  fin(a.p1, 2);
  fin(a.mask, 3);
  fin(a.up, 4);
  fout(a.lp, 5);
  fout(a.gx, 6);
  fout(a.gp0, 7);
  fout(a.gp1, 8);
  if (mask && mask->ptr && mask->dtype != B2_U8) return B2_ERR_BAD_DTYPE;
  const bool grad = a.gx.ptr || a.gp0.ptr || a.gp1.ptr;
  int lg = 0;
  while (lg < 5 && (1 << lg) < event_size) ++lg;
  if (family == B2_MVN_TRIL) lg = 5;
  a.g_log2 = lg;
  const int64_t rows_per_block = 256 >> lg;
  int64_t blocks = (nb + rows_per_block - 1) / rows_per_block;
  const int64_t cap = (int64_t)kNumSMs * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define B2_EV_LAUNCH(KERNEL)                                                        \
  if (dtype == B2_F32) {                                                            \
    if (grad) KERNEL<float, true><<<(unsigned)blocks, 256, 0, s>>>(a);              \
    else KERNEL<float, false><<<(unsigned)blocks, 256, 0, s>>>(a);                  \
  } else {                                                                          \
    if (grad) KERNEL<double, true><<<(unsigned)blocks, 256, 0, s>>>(a);             \
    else KERNEL<double, false><<<(unsigned)blocks, 256, 0, s>>>(a);                 \
  }
  const bool rowthread = cd <= 1 && event_size <= 32 && nb >= 4096 && family != B2_MVN_TRIL;
  // 16-byte path: event size a multiple of the vector width, every row of every float operand 16-byte aligned
  bool vec_rows_ok = event_size > 32 && cd <= 1;
  {
    const int V = (dtype == B2_F32) ? 4 : 2;
    if (event_size % V != 0) vec_rows_ok = false;
    auto al = [&](const void* p, int64_t st) {
      return !p || (reinterpret_cast<uintptr_t>(p) % 16 == 0 && st % V == 0);
    };
    vec_rows_ok = vec_rows_ok && al(a.p0.ptr, a.p0.st[0]) && al(a.gp0.ptr, a.gp0.st[0]);
    if (family == B2_DIRICHLET) vec_rows_ok = vec_rows_ok && al(a.x.ptr, a.x.st[0]) && al(a.gx.ptr, a.gx.st[0]);
  }
  if (family == B2_MVN_TRIL && cd <= 1 && event_size <= 4 && nb >= 1024) {
    // tiny events: one thread per row (no group reductions at all)
    blocks = (nb + 255) / 256;
    if (blocks > cap * 2) blocks = cap * 2;
    if (dtype == B2_F32) {
      if (grad) mvn_rowthread_kernel<float, true, 4><<<(unsigned)blocks, 256, 0, s>>>(a);
      else mvn_rowthread_kernel<float, false, 4><<<(unsigned)blocks, 256, 0, s>>>(a);
    } else {
      if (grad) mvn_rowthread_kernel<double, true, 4><<<(unsigned)blocks, 256, 0, s>>>(a);
      else mvn_rowthread_kernel<double, false, 4><<<(unsigned)blocks, 256, 0, s>>>(a);
    }
  }
  else if (family == B2_MVN_TRIL && event_size <= 32) {
    const int G = event_size <= 2 ? 2 : (event_size <= 4 ? 4 : (event_size <= 8 ? 8 : 32));
    const int threads = (G == 32 && dtype != B2_F32) ? 128 : 256;
    blocks = (nb * G + threads - 1) / threads;
    if (blocks > cap * 2) blocks = cap * 2;
    if (blocks < 1) blocks = 1;
    const bool full = event_size == G;
    {
      int64_t mx = 0;
      for (int o = 0; o < 9; ++o)
        for (int i = 0; i < cd; ++i) { const int64_t v = ost[o][i] < 0 ? -ost[o][i] : ost[o][i]; if (v > mx) mx = v; }
      if (cd <= 1 && (double)nb * (double)(mx > 0 ? mx : 1) + 2.0 * event_size * event_size < 2147483647.0)
        a.flags |= kEvIdx32;
    }
#define B2_MVN_GROUP2(TT, GR, GG)                                                                   \
    if (full) mvn_group_kernel<TT, GR, GG, true><<<(unsigned)blocks, threads, 0, s>>>(a);           \
    else mvn_group_kernel<TT, GR, GG, false><<<(unsigned)blocks, threads, 0, s>>>(a);
#define B2_MVN_GROUP(GG)                                                                          \
    if (dtype == B2_F32) {                                                                          \
      if (grad) { B2_MVN_GROUP2(float, true, GG) } else { B2_MVN_GROUP2(float, false, GG) }         \
    } else {                                                                                        \
      if (grad) { B2_MVN_GROUP2(double, true, GG) } else { B2_MVN_GROUP2(double, false, GG) }       \
    }
    if (G == 2) { B2_MVN_GROUP(2) }
    else if (G == 4) { B2_MVN_GROUP(4) }
    else if (G == 8) { B2_MVN_GROUP(8) }
    else { B2_MVN_GROUP(32) }
#undef B2_MVN_GROUP2
#undef B2_MVN_GROUP
  }
  else if (family != B2_MVN_TRIL && cd <= 1 && !rowthread && vec_rows_ok) {
    // lanes per row: the largest power of two <= K/V/4 (each lane takes 4 chunks per step), at most a warp
    int lgv = 0;
    const int V = (dtype == B2_F32) ? 4 : 2;
    while (lgv < 5 && (2 << lgv) <= event_size / V / 4) ++lgv;
    a.g_log2 = lgv;
    const int64_t rpb = 256 >> lgv;
    const int64_t ur = (family == B2_DIRICHLET) ? 1 : 2;  // rows in flight per lane group
    blocks = (nb + ur * rpb - 1) / (ur * rpb);
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (family == B2_DIRICHLET) { B2_EV_LAUNCH(dirichlet_vec_kernel) }
    else { B2_EV_LAUNCH(categorical_vec_kernel) }
  }
  else if (rowthread) {
    {
      // g_log2 doubles as the "16-byte rows" flag of the row-per-thread kernels
      const int V = (dtype == B2_F32) ? 4 : 2;
      auto al = [&](const void* p, int64_t st) {
        return !p || (reinterpret_cast<uintptr_t>(p) % 16 == 0 && st % V == 0);
      };
      bool v16 = event_size % V == 0 && al(a.p0.ptr, a.p0.st[0]);
      if (family == B2_DIRICHLET) v16 = v16 && al(a.x.ptr, a.x.st[0]);
      a.g_log2 = v16 ? 1 : 0;
    }
    blocks = (nb + 255) / 256;
    if (blocks > cap * 2) blocks = cap * 2;
    if (family == B2_DIRICHLET) { B2_EV_LAUNCH(dirichlet_rowthread_kernel) }
    else { B2_EV_LAUNCH(categorical_rowthread_kernel) }
  }
  else if (family == B2_DIRICHLET) { B2_EV_LAUNCH(dirichlet_kernel) }
  else if (family == B2_CATEGORICAL) { B2_EV_LAUNCH(categorical_kernel) }
  else if (event_size <= 128) { B2_EV_LAUNCH(mvn_tril_kernel) }
  else {
    // n in (128, 1024]: 16 or 32 register slots per lane; few rows per factor -> one warp per CTA slot is fine
#define B2_MVN_BIG(NS)                                                                      \
  if (dtype == B2_F32) {                                                                    \
    if (grad) mvn_tril_kernel<float, true, NS><<<(unsigned)blocks, 256, 0, s>>>(a);         \
    else mvn_tril_kernel<float, false, NS><<<(unsigned)blocks, 256, 0, s>>>(a);             \
  } else {                                                                                  \
    if (grad) mvn_tril_kernel<double, true, NS><<<(unsigned)blocks, 256, 0, s>>>(a);        \
    else mvn_tril_kernel<double, false, NS><<<(unsigned)blocks, 256, 0, s>>>(a);            \
  }
    if (event_size <= 512) { B2_MVN_BIG(16) } else { B2_MVN_BIG(32) }
#undef B2_MVN_BIG
  }
#undef B2_EV_LAUNCH
  count_launch();
  return check_launch();
}

extern "C" int b2_reduce_to(const b2_tensor* src, b2_tensor* dst, void* workspace,
                            size_t workspace_bytes, void* stream) {
  if (!src || !dst || !src->ptr || !dst->ptr) return B2_ERR_NULL;
  if (src->ndim != dst->ndim || src->dtype != dst->dtype) return B2_ERR_BAD_SHAPE;
  if (src->dtype != B2_F32 && src->dtype != B2_F64) return B2_ERR_BAD_DTYPE;
  ReduceArgs a;
  memset(&a, 0, sizeof(a));
  a.nout = 1;
  a.nred = 1;
  for (int d = 0; d < src->ndim; ++d) {
    const int64_t sz = src->shape[d];
    if (sz == 1) continue;
    if (dst->stride[d] == 0) {
      if (a.nr >= kMaxD) return B2_ERR_BAD_SHAPE;
      a.rshape[a.nr] = sz;
      a.rsrc[a.nr] = src->stride[d];
      ++a.nr;
      a.nred *= sz;
    } else {
      if (a.nk >= kMaxD) return B2_ERR_BAD_SHAPE;
      a.kshape[a.nk] = sz;
      a.ksrc[a.nk] = src->stride[d];
      a.kdst[a.nk] = dst->stride[d];
      ++a.nk;
      a.nout *= sz;
    }
  }
  if (a.nout > 0x7fffffffLL) return B2_ERR_TOO_LARGE;
  a.src = src->ptr;
  a.dst = dst->ptr;
  // ---- column reduction: reduced dims lead, kept dims trail, both contiguous -------------------------
  {
    bool cols = a.nk >= 1 && a.nr >= 1 && a.nout >= 256 && a.nout > 0;
    // order in the original tensor: every reduced dim before every kept dim
    bool seen_kept = false;
    for (int d = 0; d < src->ndim && cols; ++d) {
      if (src->shape[d] == 1) continue;
      if (dst->stride[d] == 0) { if (seen_kept) cols = false; }
      else seen_kept = true;
    }
    int64_t expect = 1;
    for (int d = a.nk - 1; d >= 0 && cols; --d) {
      cols = a.ksrc[d] == expect && a.kdst[d] == expect;
      expect *= a.kshape[d];
    }
    for (int d = a.nr - 1; d >= 0 && cols; --d) {
      cols = a.rsrc[d] == expect;
      expect *= a.rshape[d];
    }
    if (cols) {
      const int64_t C = a.nout, R = a.nred;
      const int64_t bx = (C + 255) / 256;
      int64_t sp = ((int64_t)kNumSMs * 8 + bx - 1) / bx;   // enough CTAs for ~8 per SM
      if (sp > R / 16) sp = R / 16;
      if (sp < 1) sp = 1;
      if (sp > 32) sp = 32;
      if (sp > 1 && (!workspace || workspace_bytes < 256 + sizeof(double) * (size_t)C * (size_t)sp)) sp = 1;
      cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
      double* part = workspace ? ws_partials(workspace) : nullptr;
      dim3 grid((unsigned)bx, (unsigned)sp, 1);
      if (src->dtype == B2_F32) {
        reduce_cols_kernel<float><<<grid, 256, 0, st>>>((const float*)a.src, (float*)a.dst, part, R, C, (int)sp);
        if (sp > 1) reduce_cols_finish_kernel<float><<<(unsigned)bx, 256, 0, st>>>(part, (float*)a.dst, C, (int)sp);
      } else {
        reduce_cols_kernel<double><<<grid, 256, 0, st>>>((const double*)a.src, (double*)a.dst, part, R, C, (int)sp);
        if (sp > 1) reduce_cols_finish_kernel<double><<<(unsigned)bx, 256, 0, st>>>(part, (double*)a.dst, C, (int)sp);
      }
      count_launch(sp > 1 ? 2 : 1);
      return check_launch();
    }
  }
  // split the reduced range so that small-output / large-reduction cases still fill the GPU
  int64_t splits = 1;
  const int64_t target_blocks = (int64_t)kNumSMs * 4;
  if (a.nout < target_blocks && a.nred > 4096) {
    splits = target_blocks / (a.nout > 0 ? a.nout : 1);
    const int64_t max_by_work = a.nred / 2048;
    if (splits > max_by_work) splits = max_by_work;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
  }
  if (splits > 1) {
    const size_t need = sizeof(double) * (size_t)a.nout * (size_t)splits;
    if (!workspace || workspace_bytes < 256 + need) splits = 1;
  }
  a.splits = (int)splits;
  a.partials = workspace ? ws_partials(workspace) : nullptr;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a.nout == 0) return B2_OK;
  dim3 grid((unsigned)a.nout, (unsigned)splits, 1);
  if (src->dtype == B2_F32) reduce_to_kernel<float><<<grid, 256, 0, s>>>(a);
  else reduce_to_kernel<double><<<grid, 256, 0, s>>>(a);
  count_launch();
  if (splits > 1) {
    const unsigned fb = (unsigned)((a.nout + 255) / 256);
    if (src->dtype == B2_F32) reduce_to_finish_kernel<float><<<fb, 256, 0, s>>>(a);
    else reduce_to_finish_kernel<double><<<fb, 256, 0, s>>>(a);
    count_launch();
  }
  return check_launch();
}

// ---- b2_elbo_combine: loss = sum_i coeff[i] * term_i over 0-d device scalars ---------------------
namespace b2 {
constexpr int kMaxCombine = 32;
struct CombineArgs {
  const void* ptr[kMaxCombine];
  double coeff[kMaxCombine];
  int n;
};
template <typename T>
__global__ void elbo_combine_kernel(const CombineArgs a, T* out) {
  // one warp; lanes load the terms in parallel, thread 0 adds them in index order (deterministic)
  __shared__ double v[kMaxCombine];
  const int i = threadIdx.x;
  if (i < a.n) v[i] = a.coeff[i] * (double)*reinterpret_cast<const T*>(a.ptr[i]);
  __syncwarp();
  if (i == 0) {
    double s = 0.0;
    for (int k = 0; k < a.n; ++k) s += v[k];
    *out = (T)s;
  }
}
}  // namespace b2

extern "C" int b2_elbo_combine(const void* const* terms, const double* coeffs, int n, int dtype,
                               void* out, void* stream) {
  if (!terms || !coeffs || !out) return B2_ERR_NULL;
  if (n < 0 || n > b2::kMaxCombine) return B2_ERR_TOO_LARGE;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_BAD_DTYPE;
  b2::CombineArgs a;
  a.n = n;
  for (int i = 0; i < n; ++i) {
    if (!terms[i]) return B2_ERR_NULL;
    a.ptr[i] = terms[i];
    a.coeff[i] = coeffs[i];
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == B2_F32)
    b2::elbo_combine_kernel<float><<<1, 32, 0, s>>>(a, reinterpret_cast<float*>(out));
  else
    b2::elbo_combine_kernel<double><<<1, 32, 0, s>>>(a, reinterpret_cast<double*>(out));
  b2::count_launch();
  return b2::check_launch();
}

