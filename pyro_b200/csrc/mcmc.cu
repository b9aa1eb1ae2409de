// mcmc.cu -- HMC/NUTS kernels.
//   * leapfrog halves over [C, D] chain-major state (pyro/ops/integrator.py:45-65)
//   * native potentials U, dU/dz for C chains in one launch (pyro/infer/mcmc/util.py:275-286)
//   * nuts_small_kernel: whole NUTS transitions, one thread per chain, for small latent dims
#include <string.h>

#include "b2_common.cuh"
#include "nuts_core.cuh"

namespace b2 {

// ---- leapfrog halves ------------------------------------------------------------------------------
// kick_drift:  r <- r - (eps/2) g ;  z <- z + eps * minv * r        (integrator.py:52-59)
template <typename T>
__global__ void __launch_bounds__(256) kick_drift_kernel(T* __restrict__ z, T* __restrict__ r,
                                                         const T* __restrict__ g,
                                                         const T* __restrict__ eps,
                                                         const T* __restrict__ minv,
                                                         int64_t minv_cs,
                                                         const uint8_t* __restrict__ active,
                                                         int64_t C, int64_t D) {
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    if (active && !active[c]) continue;
    const T e = eps[c];
    const T* mi = minv + c * minv_cs;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    // 4 independent elements per trip: all loads are issued before the first store
    for (; d + 3 * stride < D; d += 4 * stride) {
      T rv[4], gv[4], zv[4], mv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t i = c * D + d + u * stride;
        rv[u] = r[i]; gv[u] = g[i]; zv[u] = z[i]; mv[u] = mi[d + u * stride];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t i = c * D + d + u * stride;
        const T rn = rv[u] + (T)0.5 * e * (-gv[u]);
        r[i] = rn;
        z[i] = zv[u] + e * (mv[u] * rn);
      }
    }
    for (; d < D; d += stride) {
      const int64_t i = c * D + d;
      const T rn = r[i] + (T)0.5 * e * (-g[i]);
      r[i] = rn;
      z[i] = z[i] + e * (mi[d] * rn);
    }
  }
}

// kick:  r <- r - (eps/2) g ;  ke[c] = 0.5 * sum_d minv * r * r     (integrator.py:62-63, hmc.py:152-156)
// grid = (bx, C): partial sums go to partials[c * bx + blockIdx.x]; finished by ke_finish_kernel.
template <typename T>
__global__ void __launch_bounds__(256) kick_kernel(T* __restrict__ r, const T* __restrict__ g,
                                                   const T* __restrict__ eps,
                                                   const T* __restrict__ minv, int64_t minv_cs,
                                                   const uint8_t* __restrict__ active,
                                                   double* __restrict__ partials, int64_t C,
                                                   int64_t D) {
  __shared__ double smem[32];
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    double acc = 0.0;
    if (!(active && !active[c])) {
      const T e = eps[c];
      const T* mi = minv + c * minv_cs;
      const int64_t stride = (int64_t)gridDim.x * blockDim.x;
      int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
      double accf = 0.0;
      for (; d + 3 * stride < D; d += 4 * stride) {
        T t4 = (T)0;
        T rv[4], gv[4], mv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int64_t i = c * D + d + u * stride;
          rv[u] = r[i]; gv[u] = g[i]; mv[u] = mi[d + u * stride];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const T rn = rv[u] + (T)0.5 * e * (-gv[u]);
          r[c * D + d + u * stride] = rn;
          t4 += mv[u] * rn * rn;
        }
        accf += (double)t4;
      }
      for (; d < D; d += stride) {
        const int64_t i = c * D + d;
        const T rn = r[i] + (T)0.5 * e * (-g[i]);
        r[i] = rn;
        accf += (double)(mi[d] * rn * rn);
      }
      acc = accf;
    }
    double red[1] = {acc};
    block_sum<1>(red, smem);
    if (threadIdx.x == 0 && partials) partials[c * gridDim.x + blockIdx.x] = red[0];
  }
}

template <typename T>
__global__ void ke_finish_kernel(const double* __restrict__ partials, int nb,
                                 const uint8_t* __restrict__ active, T* __restrict__ ke,
                                 int64_t C) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (active && !active[c]) return;
  double s = 0.0;
  for (int i = 0; i < nb; ++i) s += partials[c * nb + i];
  ke[c] = (T)(0.5 * s);
}

// ---- native potentials over [C, D] ------------------------------------------------------------------
// HierNormal: grid = (bx, C). Each CTA strides over j, writes grad_eta elementwise, and reduces
// (U_part, sum_res, sum_res_eta); a finish kernel assembles U, dU/dmu, dU/dt per chain.
template <typename T>
__global__ void __launch_bounds__(256) hier_normal_kernel(const T* __restrict__ z,
                                                          const T* __restrict__ y,
                                                          const T* __restrict__ sigma,
                                                          T* __restrict__ grad,
                                                          const uint8_t* __restrict__ active,
                                                          double* __restrict__ partials,
                                                          int64_t C, int64_t J) {
  __shared__ double smem[3 * 32];
  const int64_t D = J + 2;
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    double acc[3] = {0.0, 0.0, 0.0};
    if (!(active && !active[c])) {
      const T* zc = z + c * D;
      const T mu = zc[0];
      const T tau = b2_exp(zc[1]);
      const int64_t stride = (int64_t)gridDim.x * blockDim.x;
      int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
      double a0 = 0, a1 = 0, a2 = 0;  // fp32 within a trip of 4, fp64 across trips
      for (; j + 3 * stride < J; j += 4 * stride) {
        T t0 = 0, t1 = 0, t2 = 0;
        T ev[4], sv[4], yv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ev[u] = zc[2 + j + u * stride];
          sv[u] = __ldg(sigma + j + u * stride);
          yv[u] = __ldg(y + j + u * stride);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const T d = yv[u] - mu - tau * ev[u];
          const T isg = fast_rcp(sv[u]);
          const T res = d * isg * isg;
          grad[c * D + 2 + j + u * stride] = ev[u] - tau * res;
          t0 += (T)0.5 * ev[u] * ev[u] + (T)0.5 * d * res + fast_log(sv[u]);
          t1 += res;
          t2 += res * ev[u];
        }
        a0 += (double)t0; a1 += (double)t1; a2 += (double)t2;
      }
      for (; j < J; j += stride) {
        const T eta = zc[2 + j];
        const T sg = __ldg(sigma + j);
        const T d = __ldg(y + j) - mu - tau * eta;
        const T isg = fast_rcp(sg);
        const T res = d * isg * isg;
        grad[c * D + 2 + j] = eta - tau * res;
        a0 += (double)((T)0.5 * eta * eta + (T)0.5 * d * res + fast_log(sg));
        a1 += (double)res;
        a2 += (double)(res * eta);
      }
      acc[0] = a0; acc[1] = a1; acc[2] = a2;
    }
    block_sum<3>(acc, smem);
    if (threadIdx.x == 0) {
      double* p = partials + (c * gridDim.x + blockIdx.x) * 3;
      p[0] = acc[0]; p[1] = acc[1]; p[2] = acc[2];
    }
  }
}

template <typename T>
__global__ void hier_normal_finish_kernel(const T* __restrict__ z,
                                          const double* __restrict__ partials, int nb,
                                          const uint8_t* __restrict__ active, T* __restrict__ U,
                                          T* __restrict__ grad, int64_t C, int64_t J, double s_mu,
                                          double s_tau) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (active && !active[c]) return;
  const int64_t D = J + 2;
  double a0 = 0, a1 = 0, a2 = 0;
  for (int i = 0; i < nb; ++i) {
    const double* p = partials + (c * nb + i) * 3;
    a0 += p[0]; a1 += p[1]; a2 += p[2];
  }
  const double mu = (double)z[c * D], t = (double)z[c * D + 1];
  const double tau = exp(t);
  const double u = tau / s_tau, u2 = u * u;
  const double c0 = 0.91893853320467274178;  // log sqrt(2 pi)
  double Uv = 0.5 * mu * mu / (s_mu * s_mu) + log(s_mu) + c0;
  Uv += 1.14472988584940017414 + log(s_tau) - 0.69314718055994530942 + log1p(u2) - t;
  Uv += a0 + 2.0 * c0 * (double)J;
  U[c] = (T)Uv;
  grad[c * D] = (T)(mu / (s_mu * s_mu) - a1);
  grad[c * D + 1] = (T)(2.0 * u2 / (1.0 + u2) - 1.0 - tau * a2);
}

// Logistic: grid = (bx, C); CTA strides over data rows; D <= 64 gradient components reduced
// through shared memory.  beta is staged in shared memory.
constexpr int kLogisticMaxD = 64;
template <typename T>
__global__ void __launch_bounds__(256) logistic_kernel(const T* __restrict__ z,
                                                       const T* __restrict__ X,
                                                       const T* __restrict__ y,
                                                       const uint8_t* __restrict__ active,
                                                       double* __restrict__ partials, int64_t C,
                                                       int64_t N, int D) {
  __shared__ T beta[kLogisticMaxD];
  __shared__ double smem[32];
  __shared__ double gacc[kLogisticMaxD + 1];
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    const bool on = !(active && !active[c]);
    __syncthreads();
    if (threadIdx.x < D) beta[threadIdx.x] = z[c * D + threadIdx.x];
    if (threadIdx.x <= D) gacc[threadIdx.x] = 0.0;
    __syncthreads();
    T gl[kLogisticMaxD];
    double ul = 0.0;
#pragma unroll
    for (int d = 0; d < kLogisticMaxD; ++d) gl[d] = 0;
    if (on) {
      for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N;
           n += (int64_t)gridDim.x * blockDim.x) {
        T l = 0;
        for (int d = 0; d < D; ++d) l += X[n * D + d] * beta[d];
        T sp, sg;
        softplus_sigmoid(l, sp, sg);
        const T yn = y[n];
        ul -= (double)(yn * l - sp);
        const T rr = sg - yn;
#pragma unroll
        for (int d = 0; d < kLogisticMaxD; ++d)
          if (d < D) gl[d] += rr * X[n * D + d];
      }
    }
    // reduce: one component at a time (D is small)
    {
      double red[1] = {ul};
      block_sum<1>(red, smem);
      if (threadIdx.x == 0) gacc[D] = red[0];
    }
#pragma unroll
    for (int d = 0; d < kLogisticMaxD; ++d) {
      if (d < D) {
        double red[1] = {(double)gl[d]};
        block_sum<1>(red, smem);
        if (threadIdx.x == 0) gacc[d] = red[0];
      }
    }
    __syncthreads();
    if (threadIdx.x <= D)
      partials[(c * gridDim.x + blockIdx.x) * (kLogisticMaxD + 1) + threadIdx.x] = gacc[threadIdx.x];
  }
}

template <typename T>
__global__ void logistic_finish_kernel(const T* __restrict__ z,
                                       const double* __restrict__ partials, int nb,
                                       const uint8_t* __restrict__ active, T* __restrict__ U,
                                       T* __restrict__ grad, int64_t C, int D, double s) {
  const int64_t c = blockIdx.x;
  if (c >= C) return;
  if (active && !active[c]) return;
  const int d = threadIdx.x;
  if (d > D) return;
  double a = 0.0;
  for (int i = 0; i < nb; ++i) a += partials[(c * nb + i) * (kLogisticMaxD + 1) + d];
  if (d < D) {
    grad[c * D + d] = (T)(a + (double)z[c * D + d] / (s * s));
  } else {
    double prior = 0.0;
    for (int k = 0; k < D; ++k) {
      const double zk = (double)z[c * D + k];
      prior += 0.5 * zk * zk / (s * s) + log(s) + 0.91893853320467274178;
    }
    U[c] = (T)(a + prior);
  }
}

// ---- whole-transition NUTS, one thread per chain -----------------------------------------------------
template <typename T, typename Model, int MAXD>
__global__ void nuts_small_kernel(Model model, int D, T* __restrict__ z, T* __restrict__ U,
                                  T* __restrict__ grad, const T* __restrict__ step_size,
                                  const T* __restrict__ minv, int64_t C, int num_transitions,
                                  int max_depth, T max_delta, uint64_t seed,
                                  uint64_t* __restrict__ rng_counter, T* __restrict__ samples,
                                  T* __restrict__ accept_out, int32_t* __restrict__ depth_out,
                                  int32_t* __restrict__ div_out, int32_t* __restrict__ steps_out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  T zl[MAXD], gl[MAXD], sm[MAXD];
  for (int d = 0; d < D; ++d) {
    zl[d] = z[c * D + d];
    gl[d] = grad[c * D + d];
    sm[d] = b2_sqrt(minv[c * D + d]);
  }
  T Ul = U[c];
  const T eps = step_size[c];
  Philox rng;
  rng.init(seed, (uint64_t)c, rng_counter ? rng_counter[c] : 0);
  for (int t = 0; t < num_transitions; ++t) {
    NutsStats st;
    nuts_transition<T, Model, MAXD>(model, D, zl, gl, Ul, eps, sm, max_depth, max_delta, rng, st);
    const int64_t o = (int64_t)t * C + c;
    if (samples)
      for (int d = 0; d < D; ++d) samples[o * D + d] = zl[d];
    if (accept_out) accept_out[o] = (T)st.accept_prob;
    if (depth_out) depth_out[o] = st.depth;
    if (div_out) div_out[o] = st.diverging;
    if (steps_out) steps_out[o] = st.num_steps;
  }
  for (int d = 0; d < D; ++d) {
    z[c * D + d] = zl[d];
    grad[c * D + d] = gl[d];
  }
  U[c] = Ul;
  if (rng_counter) rng_counter[c] = rng.counter() + 1;
}

inline unsigned bx_for(int64_t D, int64_t C) {
  // CTAs along the data axis per chain: enough to fill the machine, few enough to keep the
  // second-stage reduction short
  // each thread owns >= 4 elements per chain row; ~2 waves of resident CTAs over all chains
  int64_t bx = (D + 256 * 4 - 1) / (256 * 4);
  const int64_t cap = ((int64_t)kNumSMs * 16 + C - 1) / (C > 0 ? C : 1);
  if (bx > cap) bx = cap;
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  return (unsigned)bx;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_leapfrog_half_kick_drift(void* z, void* r, const void* g, const void* eps,
                                           const void* minv, int64_t minv_chain_stride,
                                           const uint8_t* active, int64_t C, int64_t D, int dtype,
                                           void* stream) {
  if (!z || !r || !g || !eps || !minv) return B2_ERR_NULL;
  if (C <= 0 || D <= 0) return B2_OK;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid(bx_for(D, C), (unsigned)(C > 65535 ? 65535 : C), 1);
  if (dtype == B2_F32)
    kick_drift_kernel<float><<<grid, 256, 0, s>>>((float*)z, (float*)r, (const float*)g,
                                                  (const float*)eps, (const float*)minv,
                                                  minv_chain_stride, active, C, D);
  else if (dtype == B2_F64)
    kick_drift_kernel<double><<<grid, 256, 0, s>>>((double*)z, (double*)r, (const double*)g,
                                                   (const double*)eps, (const double*)minv,
                                                   minv_chain_stride, active, C, D);
  else
    return B2_ERR_BAD_DTYPE;
  count_launch();
  return check_launch();
}

extern "C" size_t b2_mcmc_workspace(int64_t C) {
  // partials: C chains x up to 64 CTAs x (kLogisticMaxD + 1) doubles
  return (size_t)(C > 0 ? C : 1) * 64 * (kLogisticMaxD + 1) * sizeof(double);
}

extern "C" int b2_leapfrog_half_kick(void* r, const void* g, const void* eps, const void* minv,
                                     int64_t minv_chain_stride, const uint8_t* active, void* ke,
                                     int64_t C, int64_t D, int dtype, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  if (!r || !g || !eps || !minv) return B2_ERR_NULL;
  if (C <= 0 || D <= 0) return B2_OK;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned bx = bx_for(D, C);
  if (C > 65535) return B2_ERR_TOO_LARGE;
  double* partials = nullptr;
  if (ke) {
    if (!workspace || workspace_bytes < (size_t)C * bx * sizeof(double)) return B2_ERR_WORKSPACE;
    partials = reinterpret_cast<double*>(workspace);
  }
  dim3 grid(bx, (unsigned)C, 1);
  if (dtype == B2_F32) {
    kick_kernel<float><<<grid, 256, 0, s>>>((float*)r, (const float*)g, (const float*)eps,
                                            (const float*)minv, minv_chain_stride, active,
                                            partials, C, D);
    if (ke) ke_finish_kernel<float><<<(unsigned)((C + 127) / 128), 128, 0, s>>>(partials, (int)bx, active, (float*)ke, C);
  } else if (dtype == B2_F64) {
    kick_kernel<double><<<grid, 256, 0, s>>>((double*)r, (const double*)g, (const double*)eps,
                                             (const double*)minv, minv_chain_stride, active,
                                             partials, C, D);
    if (ke) ke_finish_kernel<double><<<(unsigned)((C + 127) / 128), 128, 0, s>>>(partials, (int)bx, active, (double*)ke, C);
  } else {
    return B2_ERR_BAD_DTYPE;
  }
  count_launch(ke ? 2 : 1);
  return check_launch();
}

extern "C" size_t b2_potential_workspace(const b2_model* model, int64_t C) {
  (void)model;
  return b2_mcmc_workspace(C);
}

extern "C" int b2_potential_grad(const b2_model* model, const void* z, void* U, void* grad,
                                 int64_t C, const uint8_t* active, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (!model || !z || !U || !grad || !model->data0 || !model->data1) return B2_ERR_NULL;
  if (C <= 0) return B2_OK;
  if (C > 65535) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_mcmc_workspace(C)) return B2_ERR_WORKSPACE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  double* partials = reinterpret_cast<double*>(workspace);
  const int dt = model->dtype;
  if (dt != B2_F32 && dt != B2_F64) return B2_ERR_BAD_DTYPE;
  if (model->model == B2_MODEL_HIER_NORMAL) {
    const int64_t J = model->J;
    if (model->D != J + 2) return B2_ERR_BAD_SHAPE;
    const unsigned bx = bx_for(J, C);
    dim3 grid(bx, (unsigned)C, 1);
    const unsigned fb = (unsigned)((C + 127) / 128);
    if (dt == B2_F32) {
      hier_normal_kernel<float><<<grid, 256, 0, s>>>((const float*)z, (const float*)model->data0,
                                                     (const float*)model->data1, (float*)grad,
                                                     active, partials, C, J);
      hier_normal_finish_kernel<float><<<fb, 128, 0, s>>>((const float*)z, partials, (int)bx, active,
                                                          (float*)U, (float*)grad, C, J,
                                                          model->hyper[0], model->hyper[1]);
    } else {
      hier_normal_kernel<double><<<grid, 256, 0, s>>>((const double*)z, (const double*)model->data0,
                                                      (const double*)model->data1, (double*)grad,
                                                      active, partials, C, J);
      hier_normal_finish_kernel<double><<<fb, 128, 0, s>>>((const double*)z, partials, (int)bx,
                                                           active, (double*)U, (double*)grad, C, J,
                                                           model->hyper[0], model->hyper[1]);
    }
    count_launch(2);
    return check_launch();
  }
  if (model->model == B2_MODEL_LOGISTIC) {
    const int D = (int)model->D;
    if (D < 1 || D > kLogisticMaxD) return B2_ERR_TOO_LARGE;
    const unsigned bx = bx_for(model->J, C);
    dim3 grid(bx, (unsigned)C, 1);
    if (dt == B2_F32) {
      logistic_kernel<float><<<grid, 256, 0, s>>>((const float*)z, (const float*)model->data0,
                                                  (const float*)model->data1, active, partials, C,
                                                  model->J, D);
      logistic_finish_kernel<float><<<(unsigned)C, 128, 0, s>>>((const float*)z, partials, (int)bx,
                                                                active, (float*)U, (float*)grad, C,
                                                                D, model->hyper[0]);
    } else {
      logistic_kernel<double><<<grid, 256, 0, s>>>((const double*)z, (const double*)model->data0,
                                                   (const double*)model->data1, active, partials, C,
                                                   model->J, D);
      logistic_finish_kernel<double><<<(unsigned)C, 128, 0, s>>>((const double*)z, partials, (int)bx,
                                                                 active, (double*)U, (double*)grad,
                                                                 C, D, model->hyper[0]);
    }
    count_launch(2);
    return check_launch();
  }
  return B2_ERR_BAD_FAMILY;
}

namespace {
template <typename T, int MAXD>
int launch_nuts_small(const b2_model* model, void* z, void* U, void* grad, const void* step_size,
                      const void* minv, int64_t C, int num_transitions, int max_tree_depth,
                      double max_delta, uint64_t seed, uint64_t* rng_counter, void* samples,
                      void* accept, int32_t* depth, int32_t* div, int32_t* steps, cudaStream_t s) {
  const int threads = 32;  // one warp per CTA: chains are independent, spread them over SMs
  const unsigned blocks = (unsigned)((C + threads - 1) / threads);
  const int D = (int)model->D;
  if (model->model == B2_MODEL_HIER_NORMAL) {
    HierNormalModel<T> m{(const T*)model->data0, (const T*)model->data1, model->J,
                         (T)model->hyper[0], (T)model->hyper[1]};
    nuts_small_kernel<T, HierNormalModel<T>, MAXD><<<blocks, threads, 0, s>>>(
        m, D, (T*)z, (T*)U, (T*)grad, (const T*)step_size, (const T*)minv, C, num_transitions,
        max_tree_depth, (T)max_delta, seed, rng_counter, (T*)samples, (T*)accept, depth, div, steps);
  } else if (model->model == B2_MODEL_LOGISTIC) {
    LogisticModel<T> m{(const T*)model->data0, (const T*)model->data1, model->J, D,
                       (T)model->hyper[0]};
    nuts_small_kernel<T, LogisticModel<T>, MAXD><<<blocks, threads, 0, s>>>(
        m, D, (T*)z, (T*)U, (T*)grad, (const T*)step_size, (const T*)minv, C, num_transitions,
        max_tree_depth, (T)max_delta, seed, rng_counter, (T*)samples, (T*)accept, depth, div, steps);
  } else {
    return B2_ERR_BAD_FAMILY;
  }
  count_launch();
  return check_launch();
}
}  // namespace

extern "C" int b2_nuts_small(const b2_model* model, void* z, void* U, void* grad,
                             const void* step_size, const void* minv, int64_t C,
                             int num_transitions, int max_tree_depth, double max_delta_energy,
                             uint64_t seed, uint64_t* rng_counter, void* samples_out,
                             void* accept_prob_out, int32_t* depth_out, int32_t* diverging_out,
                             int32_t* num_steps_out, void* stream) {
  if (!model || !z || !U || !grad || !step_size || !minv) return B2_ERR_NULL;
  if (C <= 0 || num_transitions <= 0) return B2_OK;
  if (max_tree_depth < 1 || max_tree_depth > kNutsMaxDepth) return B2_ERR_BAD_SHAPE;
  if (model->D < 1 || model->D > B2_NUTS_SMALL_MAX_D) return B2_ERR_TOO_LARGE;
  if (model->model == B2_MODEL_HIER_NORMAL && model->D != model->J + 2) return B2_ERR_BAD_SHAPE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define B2_NUTS_ARGS                                                                         \
  model, z, U, grad, step_size, minv, C, num_transitions, max_tree_depth, max_delta_energy, \
      seed, rng_counter, samples_out, accept_prob_out, depth_out, diverging_out, num_steps_out, s
  if (model->dtype == B2_F32) {
    if (model->D <= 16) return launch_nuts_small<float, 16>(B2_NUTS_ARGS);
    return launch_nuts_small<float, 64>(B2_NUTS_ARGS);
  } else if (model->dtype == B2_F64) {
    if (model->D <= 16) return launch_nuts_small<double, 16>(B2_NUTS_ARGS);
    return launch_nuts_small<double, 64>(B2_NUTS_ARGS);
  }
#undef B2_NUTS_ARGS
  return B2_ERR_BAD_DTYPE;
}

namespace b2 {

// ---- lockstep NUTS: per-leaf vector bookkeeping in ONE pass over [C, D] ---------------------------
// After a leapfrog (kick_drift, potential, kick) and the per-chain scalar decisions, every active
// chain must (nuts.py:197-248, 285-342 restated iteratively, see nuts_core.cuh):
//   ru = r * sqrt(minv)                       whitened momentum of the new leaf
//   rsub += ru                                running momentum sum of the subtree
//   if take[c]: zs = z, gs = g                progressive multinomial proposal
//   even leaf:  rck[slot] = ru, sck[slot] = rsub            (checkpoint)
//   odd leaf:   for each of the nblk blocks ending here, the two U-turn dot products
//               a_first = <rck[k], rho>, a_last = <ru, rho>, rho = (rsub - sck[k] + rck[k]) - (rck[k] + ru)/2
// grid = (bx, C); dot partials go to partials[(c * bx + blockIdx.x) * 2*nblk + ...], finished by
// nuts_dots_finish_kernel into dots[c * 2*nblk + ...].
constexpr int kNutsMaxBlocks = 12;
template <typename T>
__global__ void __launch_bounds__(256) nuts_leaf_vector_kernel(
    const T* __restrict__ z, const T* __restrict__ r, const T* __restrict__ g, const T* __restrict__ minv,
    int64_t minv_cs, const uint8_t* __restrict__ active, const uint8_t* __restrict__ take,
    T* __restrict__ rsub, T* __restrict__ zs, T* __restrict__ gs, T* __restrict__ rck, T* __restrict__ sck,
    int64_t ck_stride /* = C*D */, int store_slot /* >= 0: even leaf */, int idx_max, int nblk,
    double* __restrict__ partials, int64_t C, int64_t D) {
  __shared__ double smem[2 * kNutsMaxBlocks * 32];
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    double acc[2 * kNutsMaxBlocks];
#pragma unroll
    for (int k = 0; k < 2 * kNutsMaxBlocks; ++k) acc[k] = 0.0;
    const bool on = active[c] != 0;
    if (on) {
      const bool tk = take[c] != 0;
      const T* mi = minv + c * minv_cs;
      for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < D;
           d += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = c * D + d;
        const T ru = r[i] * b2_sqrt(mi[d]);
        const T rs = rsub[i] + ru;
        rsub[i] = rs;
        if (tk) {
          zs[i] = z[i];
          gs[i] = g[i];
        }
        if (store_slot >= 0) {
          rck[(int64_t)store_slot * ck_stride + i] = ru;
          sck[(int64_t)store_slot * ck_stride + i] = rs;
        } else {
          for (int j = 0; j < nblk; ++j) {
            const int64_t o = (int64_t)(idx_max - j) * ck_stride + i;
            const T rk = rck[o];
            const T rho = (rs - sck[o] + rk) - (T)0.5 * (rk + ru);
            acc[2 * j] += (double)(rk * rho);
            acc[2 * j + 1] += (double)(ru * rho);
          }
        }
      }
    }
    if (nblk > 0) {
      // block reduce the 2*nblk sums
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      for (int k = 0; k < 2 * nblk; ++k) {
        const double w = warp_sum(acc[k]);
        if (lane == 0) smem[k * 32 + warp] = w;
      }
      __syncthreads();
      if (warp == 0) {
        for (int k = 0; k < 2 * nblk; ++k) {
          double w = (lane < (int)(blockDim.x >> 5)) ? smem[k * 32 + lane] : 0.0;
          w = warp_sum(w);
          if (lane == 0) partials[(c * gridDim.x + blockIdx.x) * 2 * nblk + k] = w;
        }
      }
      __syncthreads();
    }
  }
}

template <typename T>
__global__ void nuts_dots_finish_kernel(const double* __restrict__ partials, int nb, int nvals,
                                        T* __restrict__ dots, int64_t C) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * nvals) return;
  const int64_t c = i / nvals;
  const int k = (int)(i - c * nvals);
  double s = 0.0;
  for (int b = 0; b < nb; ++b) s += partials[(c * nb + b) * nvals + k];
  dots[i] = (T)s;
}


// ---- lockstep NUTS, hierarchical-Normal model class: ONE pass per leaf ------------------------------
// The generic lockstep leaf costs five launches that move ~65 B per chain-element (kick_drift,
// potential, kick, leaf_vector + finish) plus ~20 [C]-sized torch ops.  For the model class of
// BASELINE configs 1/4 the latent vector is [mu, log tau | eta_1..J] and, given the two global
// coordinates, dU/d eta_j is local:  g_j = eta_j - tau * (y_j - mu - tau*eta_j) / sigma_j^2.
// So one kernel can take the whole velocity-Verlet step (pyro/ops/integrator.py:45-65) for the
// local coordinates WITHOUT a stored gradient vector -- the old gradient is recomputed from the old
// (mu, tau), the new one from the drifted (mu', tau') that every thread derives from six scalars --
// and, in the same pass, everything the tree needs from the new leaf (nuts.py:197-248,285-342
// restated iteratively, see nuts_core.cuh): whitened momentum, running sum, checkpoint store or
// the U-turn dot products, and the proposal copy of the PREVIOUS leaf (its value is read here
// anyway).  Traffic: read eta, r, minv, rsub (+ y, sigma from L2), write eta, r, rsub, plus the
// checkpoint row(s): ~40 B per chain-element.  A warp-per-chain finish kernel then assembles U,
// the two global gradients, finishes the global coordinates' kick, and runs the per-chain scalar
// logic of the tree (energy, divergence, multinomial draw with Philox, U-turn flags).
struct LeafHierArgs {
  void *zL, *rL, *zR, *rR;              // [C, D] the two ends of the trajectory; dir[c] picks the one that grows
  const uint8_t* dir;                   // [C] 1 = the right end grows
  void *gscL, *gscR;                    // [C, 2] global-coordinate gradients at the two ends
  void *rsub, *zs, *rck, *sck;          // [C, D] / [slots, C, D]
  const void *minv, *y, *sigma;         // [C, D] (chain stride minv_cs), [J], [J]
  const void* eps;                      // [C] signed step
  void* gsc_s;                          // [C, 2] global-coordinate gradients at the proposal
  void *U, *Us, *logw_sub, *sum_accept, *num_prop;  // [C]
  const void* energy0;                  // [C]
  uint8_t *done, *diverged, *take;      // [C]
  int32_t* nleaf;                       // [C] leapfrogs taken (nullable)
  uint64_t* rng_counter;                // [C]
  double* partials;
  int64_t C, J, minv_cs, ck_stride;
  uint64_t seed;
  double s_mu, s_tau, max_delta;
  int leaf, store_slot, idx_max, nblk, nb;
};

constexpr int kLeafHierBase = 4;  // a0 (U part), a1 (sum res), a2 (sum res*eta), ke

// NBMAX: compile-time bound on the U-turn blocks checked at this leaf (0 = even leaf; 2 covers 75%
// of the odd leaves; kNutsMaxBlocks the rest) -- keeps the dot accumulators in registers without
// paying 24 of them on every leaf.
template <typename T, int NBMAX>
__global__ void __launch_bounds__(256) nuts_leaf_hier_kernel(const LeafHierArgs a) {
  __shared__ double smem[(kLeafHierBase + 2 * kNutsMaxBlocks) * 8];
  const int64_t J = a.J, D = J + 2;
  const int NV = kLeafHierBase + 2 * a.nblk;
  const T* __restrict__ y = reinterpret_cast<const T*>(a.y);
  const T* __restrict__ sigma = reinterpret_cast<const T*>(a.sigma);
  for (int64_t c = blockIdx.y; c < a.C; c += gridDim.y) {
    if (a.done[c]) continue;  // uniform over the CTA
    const bool right = a.dir[c] != 0;
    T* __restrict__ zc = reinterpret_cast<T*>(right ? a.zR : a.zL) + c * D;
    T* __restrict__ rc = reinterpret_cast<T*>(right ? a.rR : a.rL) + c * D;
    T* __restrict__ rs = reinterpret_cast<T*>(a.rsub) + c * D;
    T* __restrict__ zsc = reinterpret_cast<T*>(a.zs) + c * D;
    const T* __restrict__ mi = reinterpret_cast<const T*>(a.minv) + c * a.minv_cs;
    const T* gsc = reinterpret_cast<const T*>(right ? a.gscR : a.gscL) + c * 2;
    const bool tk = a.take[c] != 0;  // the previous leaf was drawn as the proposal
    const bool first = a.leaf == 0;  // the subtree's momentum sum starts at zero: nothing to read
    const T e = reinterpret_cast<const T*>(a.eps)[c];
    const T he = (T)0.5 * e;
    // global coordinates: every thread repeats the (cheap) scalar update; the finish kernel stores it
    const T mu = zc[0], lt = zc[1];
    const T mu2 = mu + e * mi[0] * (rc[0] - he * gsc[0]);
    const T lt2 = lt + e * mi[1] * (rc[1] - he * gsc[1]);
    const T tau = b2_exp(lt), tau2 = b2_exp(lt2);
    // the four energy/gradient sums in fp64; the U-turn dot products in T per thread (each thread
    // owns ~100 elements of a chain) and fp64 from the warp reduction on -- all in registers
    double acc[kLeafHierBase];
    T dacc[NBMAX > 0 ? 2 * NBMAX : 1];
#pragma unroll
    for (int k = 0; k < kLeafHierBase; ++k) acc[k] = 0.0;
#pragma unroll
    for (int k = 0; k < (NBMAX > 0 ? 2 * NBMAX : 1); ++k) dacc[k] = (T)0;
    T* ck_r = reinterpret_cast<T*>(a.rck);
    T* ck_s = reinterpret_cast<T*>(a.sck);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    constexpr int UN = 2;  // elements in flight per thread (4 raises the register count and lowers occupancy)
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    auto elem = [&](int64_t jj, T eta, T rj, T mv, T rsv, T yv, T sv) {
      const T isg = fast_rcp(sv);
      const T isg2 = isg * isg;
      const T g0 = eta - tau * ((yv - mu - tau * eta) * isg2);     // dU/d eta_j at z
      const T rh = rj - he * g0;                                    // half kick
      const T eta2 = eta + e * mv * rh;                             // drift
      const T d2 = yv - mu2 - tau2 * eta2;
      const T res2 = d2 * isg2;
      const T r2 = rh - he * (eta2 - tau2 * res2);                  // half kick with the new gradient
      if (tk) zsc[2 + jj] = eta;
      zc[2 + jj] = eta2;
      rc[2 + jj] = r2;
      const T ru = r2 * b2_sqrt(mv);
      const T rsn = rsv + ru;
      rs[2 + jj] = rsn;
      T t[kLeafHierBase];
      t[0] = (T)0.5 * eta2 * eta2 + (T)0.5 * d2 * res2 + fast_log(sv);
      t[1] = res2;
      t[2] = res2 * eta2;
      t[3] = mv * r2 * r2;
#pragma unroll
      for (int k = 0; k < kLeafHierBase; ++k) acc[k] += (double)t[k];
      const int64_t i = c * D + 2 + jj;
      if (NBMAX == 0) {
        ck_r[(int64_t)a.store_slot * a.ck_stride + i] = ru;
        ck_s[(int64_t)a.store_slot * a.ck_stride + i] = rsn;
      } else {
#pragma unroll
        for (int b = 0; b < NBMAX; ++b) {
          if (b < a.nblk) {
            const int64_t o = (int64_t)(a.idx_max - b) * a.ck_stride + i;
            const T rk = ck_r[o];
            const T rho = (rsn - ck_s[o] + rk) - (T)0.5 * (rk + ru);
            dacc[2 * b] += rk * rho;
            dacc[2 * b + 1] += ru * rho;
          }
        }
      }
    };
    for (; j + (UN - 1) * stride < J; j += UN * stride) {
      T ev[UN], rv[UN], mv[UN], sv[UN], yv[UN], gv[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const int64_t jj = j + u * stride;
        ev[u] = zc[2 + jj];
        rv[u] = rc[2 + jj];
        mv[u] = mi[2 + jj];
        sv[u] = first ? (T)0 : rs[2 + jj];
        yv[u] = __ldg(y + jj);
        gv[u] = __ldg(sigma + jj);
      }
#pragma unroll
      for (int u = 0; u < UN; ++u) elem(j + u * stride, ev[u], rv[u], mv[u], sv[u], yv[u], gv[u]);
    }
    for (; j < J; j += stride)
      elem(j, zc[2 + j], rc[2 + j], mi[2 + j], first ? (T)0 : rs[2 + j], __ldg(y + j), __ldg(sigma + j));
    // CTA reduction of the NV sums (fixed order), one partial row per (chain, CTA)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kLeafHierBase; ++k) {
      const double w = warp_sum(acc[k]);
      if (lane == 0) smem[k * 8 + warp] = w;
    }
#pragma unroll
    for (int k = 0; k < 2 * NBMAX; ++k) {
      if (k < 2 * a.nblk) {
        const double w = warp_sum((double)dacc[k]);
        if (lane == 0) smem[(kLeafHierBase + k) * 8 + warp] = w;
      }
    }
    __syncthreads();
    if (warp == 0) {
      for (int k = 0; k < NV; ++k) {
        double w = (lane < 8) ? smem[k * 8 + lane] : 0.0;
        w = warp_sum(w);
        if (lane == 0) a.partials[((size_t)c * gridDim.x + blockIdx.x) * NV + k] = w;
      }
    }
    __syncthreads();
  }
}

B2_HD double logaddexp_d(double x, double y) {
  const double m = x > y ? x : y;
  if (m == -INFINITY) return -INFINITY;
  return m + log(exp(x - m) + exp(y - m));
}

// one warp per chain: sum the CTA partials, finish the global coordinates, run the scalar tree logic
template <typename T>
__global__ void __launch_bounds__(128) nuts_leaf_hier_finish_kernel(const LeafHierArgs a) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= a.C) return;
  if (a.done[c]) return;
  const int NV = kLeafHierBase + 2 * a.nblk;
  double v[kLeafHierBase + 2 * kNutsMaxBlocks];
  for (int k = 0; k < NV; ++k) {
    double s = 0.0;
    for (int b = lane; b < a.nb; b += 32) s += a.partials[((size_t)c * a.nb + b) * NV + k];
    v[k] = warp_sum(s);
  }
  if (lane != 0) return;
  const int64_t J = a.J, D = J + 2;
  const bool right = a.dir[c] != 0;
  T* zc = reinterpret_cast<T*>(right ? a.zR : a.zL) + c * D;
  T* rc = reinterpret_cast<T*>(right ? a.rR : a.rL) + c * D;
  T* rs = reinterpret_cast<T*>(a.rsub) + c * D;
  T* zsc = reinterpret_cast<T*>(a.zs) + c * D;
  const T* mi = reinterpret_cast<const T*>(a.minv) + c * a.minv_cs;
  T* gsc = reinterpret_cast<T*>(right ? a.gscR : a.gscL) + c * 2;
  const bool tk = a.take[c] != 0;
  const T e = reinterpret_cast<const T*>(a.eps)[c];
  const T he = (T)0.5 * e;
  // global coordinates (same arithmetic, in T, as the vector kernel used)
  const T mu = zc[0], lt = zc[1];
  const T rh0 = rc[0] - he * gsc[0], rh1 = rc[1] - he * gsc[1];
  const T mu2 = mu + e * mi[0] * rh0;
  const T lt2 = lt + e * mi[1] * rh1;
  // potential and global gradients at the new point (as hier_normal_finish_kernel)
  const double mud = (double)mu2, t = (double)lt2;
  const double tau = exp(t);
  const double u = tau / a.s_tau, u2 = u * u;
  const double c0 = 0.91893853320467274178;  // log sqrt(2 pi)
  double Uv = 0.5 * mud * mud / (a.s_mu * a.s_mu) + log(a.s_mu) + c0;
  Uv += 1.14472988584940017414 + log(a.s_tau) - 0.69314718055994530942 + log1p(u2) - t;
  Uv += v[0] + 2.0 * c0 * (double)J;
  const T g0 = (T)(mud / (a.s_mu * a.s_mu) - v[1]);
  const T g1 = (T)(2.0 * u2 / (1.0 + u2) - 1.0 - tau * v[2]);
  const T r0 = rh0 - he * g0, r1 = rh1 - he * g1;
  if (tk) {
    zsc[0] = mu;
    zsc[1] = lt;
  }
  zc[0] = mu2; zc[1] = lt2;
  rc[0] = r0; rc[1] = r1;
  gsc[0] = g0; gsc[1] = g1;
  const double ke = 0.5 * (v[3] + (double)(mi[0] * r0 * r0) + (double)(mi[1] * r1 * r1));
  // tree vectors of the two global coordinates
  bool turn = false;
  {
    const T ru[2] = {r0 * b2_sqrt(mi[0]), r1 * b2_sqrt(mi[1])};
    T rsn[2];
    for (int d = 0; d < 2; ++d) {
      rsn[d] = (a.leaf == 0 ? (T)0 : rs[d]) + ru[d];
      rs[d] = rsn[d];
    }
    T* ck_r = reinterpret_cast<T*>(a.rck);
    T* ck_s = reinterpret_cast<T*>(a.sck);
    if (a.store_slot >= 0) {
      for (int d = 0; d < 2; ++d) {
        ck_r[(int64_t)a.store_slot * a.ck_stride + c * D + d] = ru[d];
        ck_s[(int64_t)a.store_slot * a.ck_stride + c * D + d] = rsn[d];
      }
    } else {
      for (int b = 0; b < a.nblk; ++b) {
        double d0 = v[kLeafHierBase + 2 * b], d1 = v[kLeafHierBase + 2 * b + 1];
        for (int d = 0; d < 2; ++d) {
          const int64_t o = (int64_t)(a.idx_max - b) * a.ck_stride + c * D + d;
          const T rk = ck_r[o];
          const T rho = (rsn[d] - ck_s[o] + rk) - (T)0.5 * (rk + ru[d]);
          d0 += (double)(rk * rho);
          d1 += (double)(ru[d] * rho);
        }
        // the comparison happens in T, like the torch glue of the generic path ((T)dots <= 0)
        turn = turn || ((T)d0 <= (T)0) || ((T)d1 <= (T)0);
      }
    }
  }
  // ---- scalar tree logic (nuts.py:197-248 for one new leaf) ----------------------------------------
  T* Uarr = reinterpret_cast<T*>(a.U);
  const T Unew = (T)Uv;
  Uarr[c] = Unew;
  T energy = Unew + (T)ke;
  if (energy != energy) energy = b2_inf<T>();
  const T delta = energy - reinterpret_cast<const T*>(a.energy0)[c];
  const bool div_now = delta > (T)a.max_delta;
  T accp = b2_exp(-delta);
  accp = accp > (T)1 ? (T)1 : accp;
  reinterpret_cast<T*>(a.sum_accept)[c] += accp;
  reinterpret_cast<T*>(a.num_prop)[c] += (T)1;
  if (a.nleaf) a.nleaf[c] += 1;
  const T w_leaf = -delta;
  T* lws = reinterpret_cast<T*>(a.logw_sub);
  bool take;
  T nw;
  if (a.leaf == 0) {
    nw = w_leaf;
    take = true;
  } else {
    nw = (T)logaddexp_d((double)lws[c], (double)w_leaf);
    Philox rng;
    rng.init(a.seed, (uint64_t)c, a.rng_counter[c]);
    const T un = rng.uniform<T>();
    a.rng_counter[c] = rng.counter() + 1;
    take = un < b2_exp(w_leaf - nw);
  }
  lws[c] = nw;
  if (take) {
    reinterpret_cast<T*>(a.Us)[c] = Unew;
    T* gs = reinterpret_cast<T*>(a.gsc_s) + c * 2;
    gs[0] = g0;
    gs[1] = g1;
  }
  a.take[c] = take ? 1 : 0;
  if (div_now) a.diverged[c] = 1;
  if (div_now || (turn && !div_now)) a.done[c] = 1;
}


// ---- top-level merge of a finished subtree (nuts.py:285-342 at the root of the doubling loop) --------
// For every chain still active:  rsum += rsub ;  rho = rsum - (ruL + ruR)/2 ;  the two U-turn dot
// products <ruL, rho>, <ruR, rho> of the whole tree, ru = r * sqrt(minv) at the two ends.  One pass over
// [C, D] (28 B per chain-element) instead of ~8 elementwise/reduction launches.
template <typename T>
__global__ void __launch_bounds__(256) nuts_tree_merge_kernel(
    const T* __restrict__ rL, const T* __restrict__ rR, const T* __restrict__ minv, int64_t minv_cs,
    T* __restrict__ rsum, const T* __restrict__ rsub, const uint8_t* __restrict__ done,
    double* __restrict__ partials, int64_t C, int64_t D) {
  __shared__ double smem[2 * 32];
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    double acc[2] = {0.0, 0.0};
    if (!done[c]) {
      const T* mi = minv + c * minv_cs;
      T a0 = 0, a1 = 0;
      for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < D;
           d += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = c * D + d;
        const T sq = b2_sqrt(mi[d]);
        const T ul = rL[i] * sq, ur = rR[i] * sq;
        const T rs = rsum[i] + rsub[i];
        rsum[i] = rs;
        const T rho = rs - (T)0.5 * (ul + ur);
        a0 += ul * rho;
        a1 += ur * rho;
      }
      acc[0] = (double)a0;
      acc[1] = (double)a1;
    }
    block_sum<2>(acc, smem);
    if (threadIdx.x == 0) {
      partials[(c * gridDim.x + blockIdx.x) * 2] = acc[0];
      partials[(c * gridDim.x + blockIdx.x) * 2 + 1] = acc[1];
    }
  }
}


// dst[c, :] = src[c, :] for the chains with mask[c] != 0 (proposal hand-over at the root of the tree:
// only the accepted rows move, 8 B per moved element, instead of a full-size torch.where)
template <typename T>
__global__ void __launch_bounds__(256) rows_copy_masked_kernel(T* __restrict__ dst, const T* __restrict__ src,
                                                               const uint8_t* __restrict__ mask, int64_t C,
                                                               int64_t D) {
  for (int64_t c = blockIdx.y; c < C; c += gridDim.y) {
    if (!mask[c]) continue;
    for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < D; d += (int64_t)gridDim.x * blockDim.x)
      dst[c * D + d] = src[c * D + d];
  }
}

}  // namespace b2
extern "C" int b2_nuts_leaf_vector(const void* z, const void* r, const void* g, const void* minv,
                                   int64_t minv_chain_stride, const uint8_t* active,
                                   const uint8_t* take, void* rsub, void* zs, void* gs, void* rck,
                                   void* sck, int store_slot, int idx_max, int nblk, void* dots,
                                   int64_t C, int64_t D, int dtype, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  using namespace b2;
  if (!z || !r || !g || !minv || !active || !take || !rsub || !zs || !gs || !rck || !sck) return B2_ERR_NULL;
  if (C <= 0 || D <= 0) return B2_OK;
  if (C > 65535) return B2_ERR_TOO_LARGE;
  if (nblk < 0 || nblk > kNutsMaxBlocks) return B2_ERR_BAD_SHAPE;
  if (nblk > 0 && !dots) return B2_ERR_NULL;
  const unsigned bx = bx_for(D, C);
  if (nblk > 0 && (!workspace || workspace_bytes < (size_t)C * bx * 2 * nblk * sizeof(double)))
    return B2_ERR_WORKSPACE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  double* partials = reinterpret_cast<double*>(workspace);
  dim3 grid(bx, (unsigned)C, 1);
  const int64_t cks = C * D;
  if (dtype == B2_F32) {
    nuts_leaf_vector_kernel<float><<<grid, 256, 0, s>>>(
        (const float*)z, (const float*)r, (const float*)g, (const float*)minv, minv_chain_stride, active,
        take, (float*)rsub, (float*)zs, (float*)gs, (float*)rck, (float*)sck, cks, store_slot, idx_max,
        nblk, partials, C, D);
    if (nblk > 0)
      nuts_dots_finish_kernel<float><<<(unsigned)((C * 2 * nblk + 127) / 128), 128, 0, s>>>(
          partials, (int)bx, 2 * nblk, (float*)dots, C);
  } else if (dtype == B2_F64) {
    nuts_leaf_vector_kernel<double><<<grid, 256, 0, s>>>(
        (const double*)z, (const double*)r, (const double*)g, (const double*)minv, minv_chain_stride,
        active, take, (double*)rsub, (double*)zs, (double*)gs, (double*)rck, (double*)sck, cks,
        store_slot, idx_max, nblk, partials, C, D);
    if (nblk > 0)
      nuts_dots_finish_kernel<double><<<(unsigned)((C * 2 * nblk + 127) / 128), 128, 0, s>>>(
          partials, (int)bx, 2 * nblk, (double*)dots, C);
  } else {
    return B2_ERR_BAD_DTYPE;
  }
  count_launch(nblk > 0 ? 2 : 1);
  return check_launch();
}

extern "C" size_t b2_nuts_leaf_hier_workspace(int64_t C, int64_t J) {
  return (size_t)C * b2::bx_for(J, C) * (b2::kLeafHierBase + 2 * b2::kNutsMaxBlocks) * sizeof(double);
}

extern "C" int b2_nuts_leaf_hier(const b2_model* model, const b2_nuts_lockstep* st, int leaf,
                                 int store_slot, int idx_max, int nblk, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  using namespace b2;
  if (!model || !st) return B2_ERR_NULL;
  if (model->model != B2_MODEL_HIER_NORMAL) return B2_ERR_BAD_FAMILY;
  if (model->dtype != B2_F32 && model->dtype != B2_F64) return B2_ERR_BAD_DTYPE;
  if (!st->zL || !st->rL || !st->zR || !st->rR || !st->dir || !st->gscL || !st->gscR || !st->rsub ||
      !st->zs || !st->rck || !st->sck || !st->minv || !st->eps ||
      !st->gsc_s || !st->U || !st->Us || !st->energy0 || !st->logw_sub ||
      !st->sum_accept || !st->num_prop || !st->done || !st->diverged || !st->take || !st->rng_counter)
    return B2_ERR_NULL;
  const int64_t C = st->C, J = model->J;
  if (C <= 0 || J <= 0) return B2_OK;
  if (C > 65535) return B2_ERR_TOO_LARGE;
  if (nblk < 0 || nblk > kNutsMaxBlocks) return B2_ERR_BAD_SHAPE;
  if (!workspace || workspace_bytes < b2_nuts_leaf_hier_workspace(C, J)) return B2_ERR_WORKSPACE;
  LeafHierArgs a;
  a.zL = st->zL; a.rL = st->rL; a.zR = st->zR; a.rR = st->rR; a.dir = st->dir;
  a.gscL = st->gscL; a.gscR = st->gscR;
  a.rsub = st->rsub; a.zs = st->zs; a.rck = st->rck; a.sck = st->sck;
  a.minv = st->minv; a.y = model->data0; a.sigma = model->data1; a.eps = st->eps;
  a.gsc_s = st->gsc_s; a.U = st->U; a.Us = st->Us; a.energy0 = st->energy0;
  a.logw_sub = st->logw_sub; a.sum_accept = st->sum_accept; a.num_prop = st->num_prop;
  a.done = st->done; a.diverged = st->diverged; a.take = st->take; a.nleaf = st->num_leapfrogs;
  a.rng_counter = st->rng_counter;
  a.partials = reinterpret_cast<double*>(workspace);
  a.C = C; a.J = J; a.minv_cs = st->minv_chain_stride; a.ck_stride = C * (J + 2);
  a.seed = st->seed; a.s_mu = model->hyper[0]; a.s_tau = model->hyper[1];
  a.max_delta = st->max_delta_energy;
  a.leaf = leaf; a.store_slot = store_slot; a.idx_max = idx_max; a.nblk = nblk;
  const unsigned bx = bx_for(J, C);
  a.nb = (int)bx;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid(bx, (unsigned)C, 1);
  const unsigned fin_blocks = (unsigned)((C * 32 + 127) / 128);
  if ((store_slot >= 0) != (nblk == 0)) return B2_ERR_BAD_SHAPE;  // even leaf <=> no blocks end here
  if (model->dtype == B2_F32) {
    if (nblk == 0) nuts_leaf_hier_kernel<float, 0><<<grid, 256, 0, s>>>(a);
    else if (nblk <= 2) nuts_leaf_hier_kernel<float, 2><<<grid, 256, 0, s>>>(a);
    else if (nblk <= 4) nuts_leaf_hier_kernel<float, 4><<<grid, 256, 0, s>>>(a);
    else nuts_leaf_hier_kernel<float, kNutsMaxBlocks><<<grid, 256, 0, s>>>(a);
    nuts_leaf_hier_finish_kernel<float><<<fin_blocks, 128, 0, s>>>(a);
  } else {
    if (nblk == 0) nuts_leaf_hier_kernel<double, 0><<<grid, 256, 0, s>>>(a);
    else if (nblk <= 2) nuts_leaf_hier_kernel<double, 2><<<grid, 256, 0, s>>>(a);
    else if (nblk <= 4) nuts_leaf_hier_kernel<double, 4><<<grid, 256, 0, s>>>(a);
    else nuts_leaf_hier_kernel<double, kNutsMaxBlocks><<<grid, 256, 0, s>>>(a);
    nuts_leaf_hier_finish_kernel<double><<<fin_blocks, 128, 0, s>>>(a);
  }
  count_launch(2);
  return check_launch();
}

extern "C" int b2_nuts_tree_merge(const void* rL, const void* rR, const void* minv,
                                  int64_t minv_chain_stride, void* rsum, const void* rsub,
                                  const uint8_t* done, void* dots, int64_t C, int64_t D, int dtype,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b2;
  if (!rL || !rR || !minv || !rsum || !rsub || !done || !dots) return B2_ERR_NULL;
  if (C <= 0 || D <= 0) return B2_OK;
  if (C > 65535) return B2_ERR_TOO_LARGE;
  const unsigned bx = bx_for(D, C);
  if (!workspace || workspace_bytes < (size_t)C * bx * 2 * sizeof(double)) return B2_ERR_WORKSPACE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  double* partials = reinterpret_cast<double*>(workspace);
  dim3 grid(bx, (unsigned)C, 1);
  if (dtype == B2_F32) {
    nuts_tree_merge_kernel<float><<<grid, 256, 0, s>>>((const float*)rL, (const float*)rR, (const float*)minv,
                                                        minv_chain_stride, (float*)rsum, (const float*)rsub,
                                                        done, partials, C, D);
    nuts_dots_finish_kernel<float><<<(unsigned)((C * 2 + 127) / 128), 128, 0, s>>>(partials, (int)bx, 2,
                                                                                     (float*)dots, C);
  } else if (dtype == B2_F64) {
    nuts_tree_merge_kernel<double><<<grid, 256, 0, s>>>((const double*)rL, (const double*)rR,
                                                         (const double*)minv, minv_chain_stride,
                                                         (double*)rsum, (const double*)rsub, done, partials, C, D);
    nuts_dots_finish_kernel<double><<<(unsigned)((C * 2 + 127) / 128), 128, 0, s>>>(partials, (int)bx, 2,
                                                                                      (double*)dots, C);
  } else {
    return B2_ERR_BAD_DTYPE;
  }
  count_launch(2);
  return check_launch();
}

extern "C" int b2_rows_copy_masked(void* dst, const void* src, const uint8_t* mask, int64_t C, int64_t D,
                                   int dtype, void* stream) {
  using namespace b2;
  if (!dst || !src || !mask) return B2_ERR_NULL;
  if (C <= 0 || D <= 0) return B2_OK;
  if (C > 65535) return B2_ERR_TOO_LARGE;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid(bx_for(D, C), (unsigned)C, 1);
  if (dtype == B2_F32)
    rows_copy_masked_kernel<float><<<grid, 256, 0, s>>>((float*)dst, (const float*)src, mask, C, D);
  else if (dtype == B2_F64)
    rows_copy_masked_kernel<double><<<grid, 256, 0, s>>>((double*)dst, (const double*)src, mask, C, D);
  else
    return B2_ERR_BAD_DTYPE;
  count_launch();
  return check_launch();
}

