// latent.cu -- the "latent sites" block of an SVI step: everything a reparameterised Normal guide site and its
// Normal prior need, in THREE launches per step for ALL such sites instead of ~7 per site.
//
// For a guide site  z ~ Normal(loc, scale)  (scale possibly the positive-constrained image exp(u) of a
// parameter u) whose model site is  z ~ Normal(ploc, pscale)  with gradient-free prior parameters, one SVI
// step of the reference runs (per site): exp (constraint transform, pyro/params/param_store.py:125-156), randn,
// addcmul (torch/distributions/normal.py:82-85), the guide's and the prior's log_prob + sum
// (pyro/poutine/trace_struct.py:264-278), and in the backward pass the two log_prob gradients, the accumulation
// of the two gradients reaching z, the draw's chain rule and the exp's.  Here:
//
//   b2_latent_normal_draw      z = loc + eps*s, s = scale or exp(log_scale); eps from Philox in the kernel;
//                              sum log q(z) (uses log s = u directly when the log-scale is given)
//   b2_latent_normal_prior     sum log Normal(z | ploc, pscale) per job, value only
//   b2_latent_normal_backward  g = gz + pw * d log p(z)/dz ;  d/dloc = g ;  d/dscale = g*eps - c/s, or
//                              d/du = g*eps*s - c ; each reduced to the operand's STORED shape
//
// One CTA per job (a job = one site, <= B2_RSAMPLE_MAX_N elements, <= 6 dims after host-side coalescing is NOT
// required: strides are taken as given), blockIdx.x = job, so the sites of a step share launches.  Reductions
// are in a fixed order (deterministic).
#include <stdint.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "latent.cuh"
#include "nuts_core.cuh"

namespace b2 {

template <typename T>
__global__ void __launch_bounds__(1024) latent_draw_kernel(const LatentArgs a) {
  pdl_enter();
  const LatentJob& j = a.job[blockIdx.x];
  const unsigned long long seed = a.state[0], ctr = a.state[1];
  const bool logs = (j.flags & B2_LATENT_LOG_SCALE) != 0;
  double acc = 0.0;
  for (unsigned i = threadIdx.x; i < j.n; i += blockDim.x) {
    int ol, os, opl, ops;
    unravel(j, i, ol, os, opl, ops);
    Philox rng;
    rng.init(seed, (uint64_t)i, ctr + blockIdx.x);
    const T e = rng.template normal<T>();
    const T loc = reinterpret_cast<const T*>(j.loc)[ol];
    const T sv = reinterpret_cast<const T*>(j.scale)[os];
    const T s = logs ? b2_exp(sv) : sv;
    const T zv = loc + e * s;
    // Normal(loc, s).log_prob(zv) on the ROUNDED zv, torch/distributions/normal.py:87-102; log s = u exactly
    const T d = zv - loc;
    const T lp = -(d * d) / ((T)2 * s * s) - (logs ? sv : b2_log(s)) - Consts<T>::kLogSqrt2Pi;
    reinterpret_cast<T*>(j.z)[i] = zv;
    reinterpret_cast<T*>(j.eps)[i] = e;
    acc += (double)lp;
  }
  __shared__ double smem[32];
  double v[1] = {acc};
  block_sum<1>(v, smem);
  // job k draws what the k-th of n_jobs one-job launches would (counter ctr + k), and the counter advances by
  // n_jobs.  Every thread of a CTA read it before the block_sum barriers; the last CTA to take a ticket (state[2])
  // advances it, so no CTA can read the advanced value
  if (threadIdx.x == 0) {
    *reinterpret_cast<T*>(j.out0) = (T)v[0];
    if (gridDim.x == 1) {
      a.state[1] = ctr + 1ull;
    } else if (atomicAdd(a.state + 2, 1ull) == (unsigned long long)(gridDim.x - 1)) {
      a.state[1] = ctr + gridDim.x;
      a.state[2] = 0ull;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(1024) latent_prior_kernel(const LatentArgs a) {
  const LatentJob& j = a.job[blockIdx.x];
  double acc = 0.0;
  for (unsigned i = threadIdx.x; i < j.n; i += blockDim.x) {
    int ol, os, opl, ops;
    unravel(j, i, ol, os, opl, ops);
    T p[2] = {reinterpret_cast<const T*>(j.ploc)[opl], reinterpret_cast<const T*>(j.pscale)[ops]};
    ElemOut<T> o;
    Eval<kNormal, T, false>::run(reinterpret_cast<const T*>(j.z)[i], p, o);
    acc += (double)o.lp;
  }
  __shared__ double smem[32];
  double v[1] = {acc};
  block_sum<1>(v, smem);
  if (threadIdx.x == 0) *reinterpret_cast<T*>(j.out0) = (T)v[0];
}

// Value-only priors of all jobs AND the assembly of the step's loss in one CTA:
//   *out = sum_j job_coeff[j] * sum log p_j(z_j)  +  sum_t term_coeff[t] * *term[t]
// (the ELBO's other per-site sums -- the draws' log q, the likelihood -- are 0-d device scalars by now).
struct LatentCombine {
  double job_coeff[B2_LATENT_MAX_JOBS];
  const void* term[B2_LATENT_MAX_TERMS];
  double term_coeff[B2_LATENT_MAX_TERMS];
  int n_jobs, n_terms;
  void* out;
};

template <typename T>
__global__ void __launch_bounds__(1024) latent_prior_combine_kernel(const LatentArgs a, const LatentCombine c) {
  pdl_enter();
  __shared__ double smem[32];
  double total = 0.0;
  for (int k = 0; k < c.n_jobs; ++k) {
    const LatentJob& j = a.job[k];
    double acc = 0.0;
    for (unsigned i = threadIdx.x; i < j.n; i += blockDim.x) {
      int ol, os, opl, ops;
      unravel(j, i, ol, os, opl, ops);
      T p[2] = {reinterpret_cast<const T*>(j.ploc)[opl], reinterpret_cast<const T*>(j.pscale)[ops]};
      ElemOut<T> o;
      Eval<kNormal, T, false>::run(reinterpret_cast<const T*>(j.z)[i], p, o);
      acc += (double)o.lp;
    }
    double v[1] = {acc};
    block_sum<1>(v, smem);
    if (threadIdx.x == 0) {
      if (j.out0) *reinterpret_cast<T*>(j.out0) = (T)v[0];
      total += c.job_coeff[k] * v[0];
    }
  }
  if (threadIdx.x == 0) {
    for (int t = 0; t < c.n_terms; ++t) total += c.term_coeff[t] * (double)*reinterpret_cast<const T*>(c.term[t]);
    *reinterpret_cast<T*>(c.out) = (T)total;
  }
}

// Per-element gradients (before the reduction to the stored shapes).
template <typename T>
__device__ __forceinline__ void latent_grad_elem(const LatentJob& j, unsigned i, bool logs, T& gloc, T& gscale) {
  int ol, os, opl, ops;
  unravel(j, i, ol, os, opl, ops);
  const T e = reinterpret_cast<const T*>(j.eps)[i];
  const T sv = reinterpret_cast<const T*>(j.scale)[os];
  const T s = logs ? b2_exp(sv) : sv;
  T g = j.gz ? reinterpret_cast<const T*>(j.gz)[i] : (T)0;
  if (j.ploc) {
    const T pl = reinterpret_cast<const T*>(j.ploc)[opl], ps = reinterpret_cast<const T*>(j.pscale)[ops];
    const T zv = reinterpret_cast<const T*>(j.z)[i];
    g += (T)j.pw * (-(zv - pl) / (ps * ps));
  }
  gloc = g;
  gscale = logs ? g * e * s - (T)j.c : g * e - (T)j.c / s;
}

// out[stored shape] = sum over the broadcast positions; one warp per stored element, fixed order.
template <typename T, int WHICH>
__device__ __forceinline__ void latent_reduce(const LatentJob& j, const int* st, void* outp, bool logs,
                                              bool acc_out) {
  if (!outp) return;
  unsigned cst[kMaxD], m = 1;
  {
    unsigned c = 1;
    for (int d = j.ndim - 1; d >= 0; --d) {
      cst[d] = c;
      c *= j.shape[d];
      if (st[d] != 0) m *= j.shape[d];
    }
  }
  const unsigned q = j.n / m;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  T* out = reinterpret_cast<T*>(outp);
  for (unsigned jj = warp; jj < m; jj += nwarps) {
    unsigned rem = jj, base = 0;
    int off = 0;
    for (int d = j.ndim - 1; d >= 0; --d) {
      if (st[d] == 0) continue;
      const unsigned qq = rem / j.shape[d];
      const unsigned idx = rem - qq * j.shape[d];
      rem = qq;
      base += idx * cst[d];
      off += (int)idx * st[d];
    }
    double s = 0.0;
    for (unsigned t = lane; t < q; t += 32) {
      unsigned r2 = t, flat = base;
      for (int d = j.ndim - 1; d >= 0; --d) {
        if (st[d] != 0) continue;
        const unsigned qq = r2 / j.shape[d];
        flat += (r2 - qq * j.shape[d]) * cst[d];
        r2 = qq;
      }
      T gl, gs;
      latent_grad_elem<T>(j, flat, logs, gl, gs);
      s += (double)(WHICH == 0 ? gl : gs);
    }
    s = warp_sum(s);
    if (lane == 0) out[off] = acc_out ? (T)((double)out[off] + s) : (T)s;
  }
}

// Both reductions in one pass, for a job whose loc and scale broadcast over the same positions
// (kLatentSameReduction, set by the host): each element's d/dloc and d/dscale come from one set of loads and
// go to two sums, and a lane requests the operands of two elements before adding either.  Every output is summed
// over the same positions in the same order as latent_reduce.
template <typename T>
__device__ __forceinline__ void latent_reduce_both(const LatentJob& j, bool logs) {
  unsigned cst[kMaxD], m = 1;
  {
    unsigned c = 1;
    for (int d = j.ndim - 1; d >= 0; --d) {
      cst[d] = c;
      c *= j.shape[d];
      if (j.st_loc[d] != 0) m *= j.shape[d];
    }
  }
  const unsigned q = j.n / m;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  auto flat_of = [&](unsigned t, unsigned base) {
    for (int d = j.ndim - 1; d >= 0; --d) {
      if (j.st_loc[d] != 0) continue;
      const unsigned qq = t / j.shape[d];
      base += (t - qq * j.shape[d]) * cst[d];
      t = qq;
    }
    return base;
  };
  for (unsigned jj = warp; jj < m; jj += nwarps) {
    unsigned rem = jj, base = 0;
    int offl = 0, offs = 0;
    for (int d = j.ndim - 1; d >= 0; --d) {
      if (j.st_loc[d] == 0) continue;
      const unsigned qq = rem / j.shape[d];
      const unsigned idx = rem - qq * j.shape[d];
      rem = qq;
      base += idx * cst[d];
      offl += (int)idx * j.st_loc[d];
      offs += (int)idx * j.st_scale[d];
    }
    double s0 = 0.0, s1 = 0.0;
    for (unsigned t = lane; t < q; t += 64) {
      const bool two = t + 32 < q;
      T gl0, gs0, gl1 = (T)0, gs1 = (T)0;
      latent_grad_elem<T>(j, flat_of(t, base), logs, gl0, gs0);
      if (two) latent_grad_elem<T>(j, flat_of(t + 32, base), logs, gl1, gs1);
      s0 += (double)gl0;
      s1 += (double)gs0;
      if (two) {
        s0 += (double)gl1;
        s1 += (double)gs1;
      }
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    if (lane == 0) {
      if (j.out0) {
        T* out = reinterpret_cast<T*>(j.out0);
        out[offl] = (j.flags & B2_LATENT_ACC_OUT0) ? (T)((double)out[offl] + s0) : (T)s0;
      }
      if (j.out1) {
        T* out = reinterpret_cast<T*>(j.out1);
        out[offs] = (j.flags & B2_LATENT_ACC_OUT1) ? (T)((double)out[offs] + s1) : (T)s1;
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(1024) latent_backward_kernel(const LatentArgs a) {
  pdl_enter();
  const LatentJob& j = a.job[blockIdx.x];
  const bool logs = (j.flags & B2_LATENT_LOG_SCALE) != 0;
  if (j.flags & kLatentSameReduction) {
    latent_reduce_both<T>(j, logs);
    return;
  }
  latent_reduce<T, 0>(j, j.st_loc, j.out0, logs, (j.flags & B2_LATENT_ACC_OUT0) != 0);
  latent_reduce<T, 1>(j, j.st_scale, j.out1, logs, (j.flags & B2_LATENT_ACC_OUT1) != 0);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_latent_normal_draw(const b2_latent_job* jobs, int n_jobs, void* rng_state, void* stream) {
  if (!rng_state) return B2_ERR_NULL;
  LatentArgs a;
  int dtype;
  unsigned nmax;
  const int code = fill_args(a, jobs, n_jobs, dtype, nmax);
  if (code != B2_OK) return code;
  for (int k = 0; k < n_jobs; ++k)
    if (!a.job[k].loc || !a.job[k].scale || !a.job[k].z || !a.job[k].eps || !a.job[k].out0) return B2_ERR_NULL;
  a.state = reinterpret_cast<unsigned long long*>(rng_state);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == B2_F32) launch_pdl(latent_draw_kernel<float>, dim3(n_jobs), dim3(threads_for(nmax)), 0, s, a);
  else launch_pdl(latent_draw_kernel<double>, dim3(n_jobs), dim3(threads_for(nmax)), 0, s, a);
  count_launch();
  return check_launch();
}

extern "C" int b2_latent_normal_prior(const b2_latent_job* jobs, int n_jobs, void* stream) {
  LatentArgs a;
  int dtype;
  unsigned nmax;
  const int code = fill_args(a, jobs, n_jobs, dtype, nmax);
  if (code != B2_OK) return code;
  for (int k = 0; k < n_jobs; ++k)
    if (!a.job[k].ploc || !a.job[k].pscale || !a.job[k].z || !a.job[k].out0) return B2_ERR_NULL;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == B2_F32) latent_prior_kernel<float><<<n_jobs, threads_for(nmax), 0, s>>>(a);
  else latent_prior_kernel<double><<<n_jobs, threads_for(nmax), 0, s>>>(a);
  count_launch();
  return check_launch();
}

extern "C" int b2_latent_normal_prior_combine(const b2_latent_job* jobs, int n_jobs, const double* job_coeffs,
                                              const void* const* terms, const double* term_coeffs, int n_terms,
                                              void* out, void* stream) {
  if (!out || !job_coeffs || (n_terms > 0 && (!terms || !term_coeffs))) return B2_ERR_NULL;
  if (n_terms < 0 || n_terms > B2_LATENT_MAX_TERMS) return B2_ERR_TOO_LARGE;
  LatentArgs a;
  int dtype;
  unsigned nmax;
  const int code = fill_args(a, jobs, n_jobs, dtype, nmax);
  if (code != B2_OK) return code;
  LatentCombine c;
  c.n_jobs = n_jobs;
  c.n_terms = n_terms;
  c.out = out;
  for (int k = 0; k < n_jobs; ++k) {
    if (!a.job[k].ploc || !a.job[k].pscale || !a.job[k].z) return B2_ERR_NULL;
    c.job_coeff[k] = job_coeffs[k];
  }
  for (int t = 0; t < n_terms; ++t) {
    if (!terms[t]) return B2_ERR_NULL;
    c.term[t] = terms[t];
    c.term_coeff[t] = term_coeffs[t];
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == B2_F32) launch_pdl(latent_prior_combine_kernel<float>, dim3(1), dim3(threads_for(nmax)), 0, s, a, c);
  else launch_pdl(latent_prior_combine_kernel<double>, dim3(1), dim3(threads_for(nmax)), 0, s, a, c);
  count_launch();
  return check_launch();
}

extern "C" int b2_latent_normal_backward(const b2_latent_job* jobs, int n_jobs, void* stream) {
  LatentArgs a;
  int dtype;
  unsigned nmax;
  const int code = fill_args(a, jobs, n_jobs, dtype, nmax);
  if (code != B2_OK) return code;
  for (int k = 0; k < n_jobs; ++k) {
    if (!a.job[k].scale || !a.job[k].eps) return B2_ERR_NULL;
    if ((a.job[k].ploc != nullptr) != (a.job[k].pscale != nullptr)) return B2_ERR_NULL;
    if (a.job[k].ploc && !a.job[k].z) return B2_ERR_NULL;
    a.job[k].flags &= ~kLatentSameReduction;
    if (latent_same_reduction(a.job[k])) a.job[k].flags |= kLatentSameReduction;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == B2_F32) launch_pdl(latent_backward_kernel<float>, dim3(n_jobs), dim3(threads_for(nmax)), 0, s, a);
  else launch_pdl(latent_backward_kernel<double>, dim3(n_jobs), dim3(threads_for(nmax)), 0, s, a);
  count_launch();
  return check_launch();
}
