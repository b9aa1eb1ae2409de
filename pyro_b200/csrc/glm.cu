// glm.cu -- fused Bayesian-logistic-regression likelihood term for P particles (BASELINE config 2).
//
// One pass over X[N,D] and y[N] yields, for every particle p:
//   sum_p = SUM_n  y_n * l_pn - softplus(l_pn),      l_pn = <X[n,:], W[p,:]> + b[p]
//   dW[p,:] = weight * SUM_n (y_n - sigmoid(l_pn)) X[n,:],   db[p] = weight * SUM_n (y_n - sigmoid(l_pn))
// so X and y are read from HBM exactly once for the value AND the gradient (132 MB at
// N=1e6, D=32), instead of materialising the [P,N] logits / log_prob / grad tensors that the
// reference chain (matmul -> Bernoulli.log_prob -> sum -> backward) writes and re-reads.
//
// fp32 SIMT kernel (D in {4, 8, 16}; at D = 32: N < 8192 rows, B2_FLAG_GLM_FP32, and operands the wgmma
// kernel of glm_tc.cu cannot load; every other D in 1..128 takes the wgmma kernel of glm_flat_tc.cu).
// glm_finish_kernel below, launched by launch_glm_finish (glm_host.cuh), is the second launch of every GLM likelihood
// call: Bernoulli, softmax (b2_glm_categorical_logits), Poisson (b2_glm_poisson_log_rate), Normal (b2_glm_normal_loc)
// and Binomial (b2_glm_binomial_logits).  SIMT kernel: CTA = 256 threads = 4 row groups x 64
// particles.  Each thread keeps W[p,:] and its dW[p,:] accumulator in registers; X tiles are staged through shared memory
// with cp.async double buffering and read back as warp-wide broadcasts (every lane of a warp has a
// different particle but the same row, so an LDS.128 serves 4 FMAs x 2 uses for all 32 lanes).
// FLOPs = 4*N*D*P; at P=64, D=32 the FMA pipe, not HBM, bounds this kernel (see DESIGN.md).
#include <cuda_pipeline.h>

#include "b2_common.cuh"
#include "b2_math.cuh"
#include "glm_host.cuh"
#include "latent.cuh"

namespace b2 {

constexpr int kGlmTileRows = 64;     // rows per shared-memory tile
constexpr int kGlmParticles = 64;    // particles per CTA (blockIdx.y slabs of 64)
constexpr int kGlmRowGroups = 4;     // 256 / 64

template <int D>
__global__ void __launch_bounds__(256) glm_bernoulli_kernel(const float* __restrict__ X,
                                                            const float* __restrict__ y,
                                                            const float* __restrict__ W,
                                                            const float* __restrict__ b, int64_t N,
                                                            int P, float* __restrict__ partials) {
  // partials layout: [gridDim.x][P][D + 2]  (dW..., db, sum)
  __shared__ __align__(16) float xs[2][kGlmTileRows * D];
  __shared__ float ys[2][kGlmTileRows];
  const int tid = threadIdx.x;
  const int pl = tid & (kGlmParticles - 1);
  const int rg = tid >> 6;
  const int p = blockIdx.y * kGlmParticles + pl;
  const bool pon = p < P;

  float w[D], dw[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    w[d] = pon ? W[(int64_t)p * D + d] : 0.f;
    dw[d] = 0.f;
  }
  const float bias = (pon && b) ? b[p] : 0.f;
  float db = 0.f, sum = 0.f;

  const int64_t ntiles = (N + kGlmTileRows - 1) / kGlmTileRows;
  constexpr int kVecPerTile = kGlmTileRows * D / 4;

  auto stage = [&](int buf, int64_t tile) {
    const int64_t row0 = tile * kGlmTileRows;
    const int64_t rows = (N - row0 < kGlmTileRows) ? (N - row0) : kGlmTileRows;
    const float4* src = reinterpret_cast<const float4*>(X + row0 * D);
    float4* dst = reinterpret_cast<float4*>(xs[buf]);
    const int nvec = (int)(rows * D / 4);
    for (int i = tid; i < kVecPerTile; i += 256) {
      if (i < nvec) __pipeline_memcpy_async(dst + i, src + i, 16);
      else dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < kGlmTileRows) {
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
    const int64_t row0 = tile * kGlmTileRows;
    const int rows = (int)((N - row0 < kGlmTileRows) ? (N - row0) : kGlmTileRows);
    const float* xt = xs[buf];
#pragma unroll 2
    for (int r = rg; r < rows; r += kGlmRowGroups) {
      const float4* xr = reinterpret_cast<const float4*>(xt + r * D);
      float xv[D];
#pragma unroll
      for (int q = 0; q < D / 4; ++q) {
        const float4 v = xr[q];
        xv[4 * q + 0] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w;
      }
      // four independent partial dot products: a single accumulator is a chain of D dependent
      // FMAs (4 cycles each), which 4 resident warps per scheduler cannot hide
      float l0 = bias, l1 = 0.f, l2 = 0.f, l3 = 0.f;
#pragma unroll
      for (int d = 0; d < D; d += 4) {
        l0 = fmaf(xv[d + 0], w[d + 0], l0);
        l1 = fmaf(xv[d + 1], w[d + 1], l1);
        l2 = fmaf(xv[d + 2], w[d + 2], l2);
        l3 = fmaf(xv[d + 3], w[d + 3], l3);
      }
      const float l = (l0 + l1) + (l2 + l3);
      const float yn = ys[buf][r];
      // softplus / sigmoid sharing one exp (fast intrinsics: ex2.approx / lg2.approx / rcp)
      const float e = __expf(-fabsf(l));
      const float inv = __frcp_rn(1.f + e);
      const float sp = fmaxf(l, 0.f) + __logf(1.f + e);
      const float sg = (l >= 0.f) ? inv : e * inv;
      sum += yn * l - sp;
      const float g = yn - sg;
      db += g;
#pragma unroll
      for (int d = 0; d < D; ++d) dw[d] = fmaf(g, xv[d], dw[d]);
    }
    __syncthreads();
    buf ^= 1;
  }
  __pipeline_wait_prior(0);

  // reduce the 4 row groups through shared memory (reuse xs[0]: 64*D floats >= 3*64*(D+2)? no: use a loop)
  __syncthreads();
  float* red = xs[0];  // capacity kGlmTileRows*D = 64*D floats; we need 64 floats per pass
  float* out = partials + ((int64_t)blockIdx.x * P + p) * (D + 2);
#pragma unroll
  for (int d = 0; d < D + 2; ++d) {
    const float v = (d < D) ? dw[d < D ? d : 0] : (d == D ? db : sum);
    // stage groups 1..3, group 0 adds them in a fixed order
    if (rg > 0) red[(rg - 1) * kGlmParticles + pl] = v;
    __syncthreads();
    if (rg == 0 && pon) {
      out[d] = ((v + red[pl]) + red[kGlmParticles + pl]) + red[2 * kGlmParticles + pl];
    }
    __syncthreads();
  }
}

// Loss assembly in the finish (b2_glm_bernoulli_logits_elbo): the value-only Normal priors of the step's latent
// sites and the other 0-d terms of the ELBO, so that the likelihood call also writes the step's loss
//   *out = SUM_j job_coeff[j] * SUM log Normal(z_j | prior_j)  +  SUM_t term_coeff[t] * *term[t]
// with the arithmetic of latent_prior_combine_kernel (latent.cu), bit for bit: that kernel's CTA of nwarps warps
// is replayed by nwarps warps per job here (warp w adds the elements w*32 + lane + k*nwarps*32 in fp64, then the
// same shuffle tree), and the last warp to arrive sums the nwarps per-warp values of each job with the shuffle
// tree of block_sum and adds the jobs, then the terms, in order, in fp64.  A null term is this call's own total.
struct GlmElbo {
  LatentJob job[B2_LATENT_MAX_JOBS];   // z (fp32, contiguous), ploc / pscale with their strides
  double job_coeff[B2_LATENT_MAX_JOBS];
  const float* term[B2_LATENT_MAX_TERMS];
  double term_coeff[B2_LATENT_MAX_TERMS];
  int n_jobs, n_terms, nwarps;
  double* warp_sums;                   // [n_jobs][32]
  float* out;
};

// second stage: fixed-order sum over the CTAs' partials [nblocks][P][K (D + 1) + 1] (per class dW[0..D-1]
// and db, then the particle's lp sum; K = 1 but for softmax); applies weight / scale.  (The Poisson and Binomial
// kernels have already folded their data terms into the lp partials.)  sigma (Normal only, else null; sigma[p * sigma_stride] for particle p) turns the sufficient
// statistics of the Normal tile kernel into the lp sum and gradients: the lp slot holds S = SUM (y - l)^2 and
// dW / db hold SUM (y - l) [x | 1]; the warp of sum_p[p] also writes out_dsigma[p] (nullable), n is N.
// One WARP per entry of the [P, K (D + 1) + 1] table: lanes stride over the CTAs (L2-resident partials),
// then a shuffle tree (a thread-per-entry loop is a chain of ~300 dependent loads).  The 8 warps of a CTA
// take 8 adjacent entries, whose partials are one 32-byte sector per CTA: the CTA first copies that
// [nblocks][8] slice to shared memory, every thread's loads issued at once, so the sum of a warp's lane reads
// no global memory (read directly, a warp's lanes would touch one sector per CTA for 4 useful bytes each).
// With E, E->n_jobs * E->nwarps more warps score the priors, and the ticket counts them too.
constexpr int kFinishThreads = 256;
constexpr int kFinishEntries = kFinishThreads / 32;      // entries (warps) per CTA
constexpr int kFinishMaxBlocks = 2 * kNumSMs;             // nblocks <= glm_grid_x, glm_tc_grid_x
constexpr int kFinishLoads = (kFinishMaxBlocks * kFinishEntries + kFinishThreads - 1) / kFinishThreads;
constexpr int kFinishPitch = kFinishEntries + 1;         // odd row pitch: the lanes of a warp hit 32 banks

__device__ __forceinline__ void glm_finish_body(const float* __restrict__ partials, int nblocks, int P, int K, int D,
                                                double scale, double weight, float* __restrict__ sum_p,
                                                float* __restrict__ out_dW, float* __restrict__ out_db,
                                                double sum_coeff, int flags, float* __restrict__ out_total,
                                                unsigned int* __restrict__ ticket,
                                                const float* __restrict__ sigma, int sigma_stride, int64_t n,
                                                float* __restrict__ out_dsigma, const GlmElbo* E) {
  pdl_enter();
  const int S = K * (D + 1) + 1;
  const int total = P * S;
  const int n_prior = E ? E->n_jobs * E->nwarps : 0;
  const int e0 = blockIdx.x * kFinishEntries;
  const int e = e0 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  __shared__ float tile[kFinishMaxBlocks * kFinishPitch];
  if (e0 < total) {
    const int ncol = total - e0 < kFinishEntries ? total - e0 : kFinishEntries;
    float v[kFinishLoads];
#pragma unroll
    for (int k = 0; k < kFinishLoads; ++k) {
      const int i = threadIdx.x + k * kFinishThreads, bl = i / kFinishEntries, c = i % kFinishEntries;
      v[k] = (bl < nblocks && c < ncol) ? partials[(int64_t)bl * total + e0 + c] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < kFinishLoads; ++k) {
      const int i = threadIdx.x + k * kFinishThreads, bl = i / kFinishEntries, c = i % kFinishEntries;
      if (bl < nblocks) tile[bl * kFinishPitch + c] = v[k];
    }
    __syncthreads();
  }
  if (e >= total + n_prior) return;
  unsigned int t = 0;
  if (e >= total) {
    const int k = (e - total) / E->nwarps, w = (e - total) - k * E->nwarps;
    const LatentJob& j = E->job[k];
    double acc = 0.0;
    for (unsigned i = (unsigned)(w * 32 + lane); i < j.n; i += (unsigned)(E->nwarps * 32)) {
      int ol, os, opl, ops;
      unravel(j, i, ol, os, opl, ops);
      float p[2] = {reinterpret_cast<const float*>(j.ploc)[opl], reinterpret_cast<const float*>(j.pscale)[ops]};
      ElemOut<float> o;
      Eval<kNormal, float, false>::run(reinterpret_cast<const float*>(j.z)[i], p, o);
      acc += (double)o.lp;
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      E->warp_sums[k * 32 + w] = acc;
      __threadfence();
      t = atomicAdd(ticket, 1u);
    }
  } else {
    double s = 0.0;
    for (int bl = lane; bl < nblocks; bl += 32) s += (double)tile[bl * kFinishPitch + (e - e0)];
    s = warp_sum(s);
    const int p = e / S, r = e - p * S;
    if (r < K * (D + 1)) {
      const int k = r / (D + 1), c = r - k * (D + 1);
      if (lane == 0) {
        if (sigma) {                           // Normal: SUM r x / sigma^2
          const double sg = (double)sigma[(int64_t)p * sigma_stride];
          s *= 1.0 / (sg * sg);
        }
        if (c < D) {
          if (out_dW) out_dW[((int64_t)p * K + k) * D + c] = (float)(weight * scale * s);
        } else if (out_db) {
          out_db[(int64_t)p * K + k] = (float)(weight * scale * s);
        }
      }
      return;
    }
    if (sigma) {
      // Normal: s is S = SUM (y - l)^2; lp sum = -S / (2 sigma^2) - n (log sigma + log(2 pi) / 2) and
      // d/dsigma = S / sigma^3 - n / sigma, all in fp64
      const double sg = (double)sigma[(int64_t)p * sigma_stride], S = s, nn = (double)n;
      s = -S / (2.0 * sg * sg) - nn * (log(sg) + 0.91893853320467274178);
      if (lane == 0 && out_dsigma) out_dsigma[p] = (float)(weight * scale * (S / (sg * sg * sg) - nn / sg));
    }
    // per-particle sum; the LAST of the P warps (and prior warps) to get here also totals them (fixed order),
    // with the ELBO coefficient -- a ticket instead of a third launch
    if (lane == 0) {
      sum_p[p] = (float)(scale * s);
      if (out_total) {
        __threadfence();
        t = atomicAdd(ticket, 1u);
      }
    }
    if (!out_total) return;
  }
  t = __shfl_sync(0xffffffffu, t, 0);
  if (t != (unsigned)(P + n_prior - 1)) return;
  __threadfence();
  // every value the rest adds is requested before the first add, not one job or term after another
  double acc = 0.0;
  for (int q = lane; q < P; q += 32) acc += (double)__ldcg(sum_p + q);
  static_assert(B2_LATENT_MAX_TERMS <= 32, "one term per lane");
  double ws[B2_LATENT_MAX_JOBS];
  float tv = 0.f;   // lane q holds term q; a term that is out_total itself reads as own below
  if (E) {
#pragma unroll
    for (int k = 0; k < B2_LATENT_MAX_JOBS; ++k)
      ws[k] = (k < E->n_jobs && lane < E->nwarps) ? __ldcg(E->warp_sums + k * 32 + lane) : 0.0;
    if (lane < E->n_terms && E->term[lane] && E->term[lane] != out_total) tv = __ldcg(E->term[lane]);
  }
  acc = warp_sum(acc);
  float own = 0.f;
  if (lane == 0) {
    const double v = sum_coeff * acc;
    own = (flags & B2_FLAG_ACCUMULATE_SUM) ? (float)((double)*out_total + v) : (float)v;
    *out_total = own;
    *ticket = 0u;
  }
  if (!E) return;
  double loss = 0.0;
#pragma unroll
  for (int k = 0; k < B2_LATENT_MAX_JOBS; ++k) {
    if (k >= E->n_jobs) break;
    loss += E->job_coeff[k] * warp_sum(ws[k]);
  }
  for (int q = 0; q < E->n_terms; ++q) {
    const float t = __shfl_sync(0xffffffffu, tv, q);
    if (lane == 0) loss += E->term_coeff[q] * (double)(E->term[q] && E->term[q] != out_total ? t : own);
  }
  if (lane == 0) *E->out = (float)loss;
}

__global__ void __launch_bounds__(kFinishThreads) glm_finish_kernel(const float* __restrict__ partials, int nblocks, int P,
                                                         int K, int D, double scale, double weight,
                                                         float* __restrict__ sum_p, float* __restrict__ out_dW,
                                                         float* __restrict__ out_db, double sum_coeff, int flags,
                                                         float* __restrict__ out_total,
                                                         unsigned int* __restrict__ ticket,
                                                         const float* __restrict__ sigma, int sigma_stride,
                                                         int64_t n, float* __restrict__ out_dsigma) {
  glm_finish_body(partials, nblocks, P, K, D, scale, weight, sum_p, out_dW, out_db, sum_coeff, flags, out_total,
                  ticket, sigma, sigma_stride, n, out_dsigma, nullptr);
}

__global__ void __launch_bounds__(kFinishThreads) glm_finish_elbo_kernel(const float* __restrict__ partials, int nblocks, int P,
                                                              int K, int D, double scale, double weight,
                                                              float* __restrict__ sum_p, float* __restrict__ out_dW,
                                                              float* __restrict__ out_db, double sum_coeff,
                                                              int flags, float* __restrict__ out_total,
                                                              unsigned int* __restrict__ ticket, const GlmElbo E) {
  glm_finish_body(partials, nblocks, P, K, D, scale, weight, sum_p, out_dW, out_db, sum_coeff, flags, out_total,
                  ticket, nullptr, 0, 0, nullptr, &E);
}

// The per-particle sums go to out_sum_p, or without one to the [P] row of the workspace after the partials.
static float* glm_sum_p(const float* partials, float* out_sum_p, int gx, int total) {
  return out_sum_p ? out_sum_p : const_cast<float*>(partials) + (size_t)gx * total;
}

void launch_glm_finish(const float* partials, unsigned int* ticket, int gx, int P, int K, int D, double scale,
                       double weight, double sum_coeff, int flags, float* out_sum_p, float* out_total,
                       float* out_dW, float* out_db, cudaStream_t s, const float* sigma,
                       int sigma_stride, int64_t n, float* out_dsigma) {
  const int total = P * (K * (D + 1) + 1);
  launch_pdl(glm_finish_kernel, dim3((total + kFinishEntries - 1) / kFinishEntries), dim3(kFinishThreads), 0, s,
             partials, gx, P, K, D, scale, weight, glm_sum_p(partials, out_sum_p, gx, total), out_dW, out_db,
             sum_coeff, flags, out_total, ticket, sigma, sigma_stride, n, out_dsigma);
}

inline int glm_grid_x(int64_t N) {
  const int64_t ntiles = (N + kGlmTileRows - 1) / kGlmTileRows;
  int64_t gx = (int64_t)kNumSMs * 2;  // two 256-thread CTAs per SM (register-limited)
  if (gx > ntiles) gx = ntiles;
  if (gx < 1) gx = 1;
  return (int)gx;
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_elbo_workspace(void) { return (size_t)B2_LATENT_MAX_JOBS * 32 * sizeof(double); }

extern "C" size_t b2_glm_workspace(int64_t N, int D, int P) {
  // [ticket, 256 B] + CTA partials + one [P] row for the per-particle sums
  return 256 + ((size_t)glm_grid_x(N) * (size_t)P * (size_t)(D + 2) + (size_t)P) * sizeof(float);
}

static int glm_bernoulli(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                         double scale, double weight, double sum_coeff, int flags, float* out_sum_p,
                         float* out_total, float* out_dW, float* out_db, void* workspace, size_t workspace_bytes,
                         cudaStream_t s, const GlmElbo* E, GlmGroups grp = {}) {
  if (!X || !y || !W) return B2_ERR_NULL;
  if (N <= 0 || P <= 0) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0) return B2_ERR_BAD_SHAPE;
  // with a group effect the contraction is D + G columns wide (W, dW, partials)
  const int Da = D + grp.cols();
  if (D < 1 || Da > 128) return B2_ERR_BAD_SHAPE;
  if (grp.idx && (grp.G < 1 || reinterpret_cast<uintptr_t>(grp.idx) % 16 != 0)) return B2_ERR_BAD_SHAPE;
  // D in {4, 8, 16, 32} keep their kernels; every other D, and every D with a group effect, takes the wgmma
  // kernel of glm_flat_tc.cu, which has no fp32 SIMT counterpart and loads y by 16-byte bulk copies with 32-bit
  // row counts
  const bool flat = grp.idx || !(D == 4 || D == 8 || D == 16 || D == 32);
  if (flat && (flags & B2_FLAG_GLM_FP32)) return B2_ERR_BAD_SHAPE;
  if (flat && reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (flat && N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  if (!workspace || workspace_bytes < b2_glm_workspace(N, Da, P)) return B2_ERR_WORKSPACE;
  // below 8 Ki rows the single-pass TF32 gradient contraction has not averaged its operand rounding
  // (2^-12 relative per term) below the fp32 tolerance yet: those sizes take the exact fp32 SIMT kernel
  // unless the tensor-core kernel is asked for explicitly (B2_FLAG_GLM_3XTF32).  The TMA loads need a
  // 16-byte aligned y and 32-bit row coordinates; other operands take the SIMT kernel as well.
  const bool use_tc = (D == 32) && !(flags & B2_FLAG_GLM_FP32) && reinterpret_cast<uintptr_t>(y) % 16 == 0 &&
                      N < ((int64_t)1 << 31) && (N >= 8192 || (flags & B2_FLAG_GLM_3XTF32));
  const int gx = (use_tc || flat) ? glm_tc_grid_x(N) : glm_grid_x(N);
  dim3 grid((unsigned)gx, (unsigned)((P + kGlmParticles - 1) / kGlmParticles), 1);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
  float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
  if (flat || use_tc) {
    const bool split_x = glm_split_x(flags, N);
    const int rc = flat ? launch_glm_flat_tc(X, y, W, b, N, D, P, partials, gx, split_x, s, grp)
                        : launch_glm_tc(X, y, W, b, N, P, partials, gx, split_x, s);
    if (rc != 0) return rc;
  } else
  switch (D) {
    case 4: glm_bernoulli_kernel<4><<<grid, 256, 0, s>>>(X, y, W, b, N, P, partials); break;
    case 8: glm_bernoulli_kernel<8><<<grid, 256, 0, s>>>(X, y, W, b, N, P, partials); break;
    case 16: glm_bernoulli_kernel<16><<<grid, 256, 0, s>>>(X, y, W, b, N, P, partials); break;
    case 32: glm_bernoulli_kernel<32><<<grid, 256, 0, s>>>(X, y, W, b, N, P, partials); break;
    default: return B2_ERR_BAD_SHAPE;
  }
  if (E) {
    const int total = P * (D + 2);
    launch_pdl(glm_finish_elbo_kernel, dim3((total + E->n_jobs * E->nwarps + kFinishEntries - 1) / kFinishEntries),
               dim3(kFinishThreads), 0, s, partials, gx,
               P, 1, D, scale, weight, glm_sum_p(partials, out_sum_p, gx, total), out_dW, out_db, sum_coeff, flags,
               out_total, ticket, *E);
  } else {
    launch_glm_finish(partials, ticket, gx, P, 1, Da, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW,
                      out_db, s);
  }
  count_launch(2);
  return check_launch();
}

int b2::glm_bernoulli_logits(const float* X, const float* y, const float* W, const float* b, int64_t N, int D, int P,
                             double scale, double weight, double sum_coeff, int flags, float* out_sum_p,
                             float* out_total, float* out_dW, float* out_db, void* workspace, size_t workspace_bytes,
                             cudaStream_t s, GlmGroups grp) {
  return glm_bernoulli(X, y, W, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW, out_db,
                       workspace, workspace_bytes, s, nullptr, grp);
}

extern "C" int b2_glm_bernoulli_logits(const float* X, const float* y, const float* W,
                                       const float* b, int64_t N, int D, int P, double scale,
                                       double weight, double sum_coeff, int flags,
                                       float* out_sum_p, float* out_total, float* out_dW,
                                       float* out_db, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  return glm_bernoulli(X, y, W, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW, out_db,
                       workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), nullptr);
}

extern "C" int b2_glm_bernoulli_logits_elbo(const float* X, const float* y, const float* W,
                                            const float* b, int64_t N, int D, int P, double scale,
                                            double weight, double sum_coeff, int flags,
                                            float* out_sum_p, float* out_total, float* out_dW,
                                            float* out_db, void* workspace, size_t workspace_bytes,
                                            const b2_latent_job* jobs, int n_jobs, const double* job_coeffs,
                                            const void* const* terms, const double* term_coeffs, int n_terms,
                                            void* loss, void* warp_sums, size_t warp_sums_bytes, void* stream) {
  if (!out_total || !loss || !job_coeffs || (n_terms > 0 && (!terms || !term_coeffs))) return B2_ERR_NULL;
  if (n_terms < 0 || n_terms > B2_LATENT_MAX_TERMS) return B2_ERR_TOO_LARGE;
  if (!warp_sums || warp_sums_bytes < b2_glm_elbo_workspace()) return B2_ERR_WORKSPACE;
  LatentArgs a;
  int dtype;
  unsigned nmax;
  const int code = fill_args(a, jobs, n_jobs, dtype, nmax);
  if (code != B2_OK) return code;
  if (dtype != B2_F32) return B2_ERR_BAD_DTYPE;
  GlmElbo E;
  for (int k = 0; k < n_jobs; ++k) {
    if (!a.job[k].ploc || !a.job[k].pscale || !a.job[k].z) return B2_ERR_NULL;
    E.job[k] = a.job[k];
    E.job_coeff[k] = job_coeffs[k];
  }
  for (int t = 0; t < n_terms; ++t) {
    E.term[t] = static_cast<const float*>(terms[t]);   // null: this call's own total
    E.term_coeff[t] = term_coeffs[t];
  }
  E.n_jobs = n_jobs;
  E.n_terms = n_terms;
  E.nwarps = threads_for(nmax) / 32;
  E.warp_sums = static_cast<double*>(warp_sums);
  E.out = static_cast<float*>(loss);
  return glm_bernoulli(X, y, W, b, N, D, P, scale, weight, sum_coeff, flags, out_sum_p, out_total, out_dW, out_db,
                       workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream), &E);
}
