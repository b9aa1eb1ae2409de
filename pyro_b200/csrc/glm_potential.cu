// glm_potential.cu -- HMC / NUTS potential energy of Bayesian logistic, softmax, Poisson, Binomial and linear
// regression for C chains.
//
//   U[c]    = -( SUM_n log p(y_n | logits_cn) + SUM log Normal(w; 0, s_w) + SUM log Normal(b; 0, s_b) )
//   grad[c] = dU / dz[c]                                           (in z's layout)
//
// The likelihood and its gradient come from the fused GLM likelihood entry points (b2_glm_bernoulli_logits,
// b2_glm_categorical_logits, b2_glm_poisson_log_rate, b2_glm_normal_loc, b2_glm_binomial_logits: a tile kernel and
// glm_finish_kernel each) with their particle axis set to the chains, so X is read once per evaluation for every
// chain together.  Each entry point checks its own arguments, then glm_potential_run makes the one fixed launch
// sequence, with no host sync (CUDA graph capturable):
//   1. glm_potential_pack_kernel    z's weight / bias columns -> the contiguous [C, K*D] / [C, K] operands
//                                   (z's rows also hold the other site, so their stride is not the kernels')
//   2. the likelihood call          weight = -1: dW, db are d(-loglik)/dW, d(-loglik)/db; sum_p = loglik
//   3. glm_potential_finish_kernel  adds the Normal prior value and gradient, one warp per chain, fp64
//                                   accumulation in a fixed order, and writes U and grad
// The GLM kernels always run with every logit fp32-exact (B2_FLAG_GLM_3XTF32; the Normal kernels always split X),
// so the sampler targets the posterior of the data as given, not of X rounded to TF32.
// With a noise scale (linear regression) the pack also writes each chain's sigma_c = exp(z[c, s_off]) (or the
// constant), and the finish adds sigma's prior and the Jacobian of sigma = e^t in fp64.  Binomial regression passes
// the trial counts to its likelihood call as a fixed operand.  b2_glm_scaled_potential runs the same sequence for a
// latent weight scale (w ~ Normal(0, tau * lam)), with glm_scaled_potential_finish_kernel as step 3, and
// b2_glm_group_potential for a varying intercept alpha[g] by group and up to three varying slopes beta_k[g] on
// columns of X: glm_group_potential_pack_kernel writes [w | alpha | beta_1 ..] as each chain's weight row, the
// likelihood runs on [X | onehot(g) | x_{c_1} onehot(g) ..] (glm_flat_tc.cuh GROUPS), and
// glm_group_potential_finish_kernel is step 3.
#include <math.h>

#include "b2_common.cuh"
#include "glm_host.cuh"

namespace b2 {

// sig (linear regression only, else null): sig[c] = exp(z[c, s_off]) for a latent noise scale (z holds its log),
// the constant s_const when s_off < 0.  A group effect's weight rows are glm_group_potential_pack_kernel's.
__global__ void __launch_bounds__(256) glm_potential_pack_kernel(const float* __restrict__ z, int64_t C,
                                                                 int64_t Dz, int64_t w_off, int64_t b_off,
                                                                 int KD, int Kb, float* __restrict__ Wp,
                                                                 float* __restrict__ bp, int64_t s_off,
                                                                 float s_const, float* __restrict__ sig) {
  const int64_t per = KD + Kb;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (sig != nullptr && i < C) sig[i] = s_off >= 0 ? expf(z[i * Dz + s_off]) : s_const;
  if (i >= C * per) return;
  const int64_t c = i / per;
  const int64_t j = i - c * per;
  if (j < KD) Wp[c * KD + j] = z[c * Dz + w_off + j];
  else bp[c * Kb + (j - KD)] = z[c * Dz + b_off + (j - KD)];
}

// glm_potential_pack_kernel for a group effect: each chain's weight row is [w | alpha | beta_1 .. beta_S], KD =
// D + G (1 + S) wide.  Block 0 is alpha, block k slope k; each is z's columns, or s * eta for a non-centred block
// (s its scale: exp of its z column, or its constant).
__global__ void __launch_bounds__(256) glm_group_potential_pack_kernel(const float* __restrict__ z, int64_t C,
                                                                       int64_t Dz, int64_t w_off, int64_t b_off,
                                                                       int KD, int Kb, float* __restrict__ Wp,
                                                                       float* __restrict__ bp, int64_t s_off,
                                                                       float s_const, float* __restrict__ sig,
                                                                       b2_glm_group_effect ge) {
  const int64_t per = KD + Kb;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (sig != nullptr && i < C) sig[i] = s_off >= 0 ? expf(z[i * Dz + s_off]) : s_const;
  if (i >= C * per) return;
  const int64_t c = i / per;
  const int64_t j = i - c * per;
  const int D = KD - ge.G * (1 + ge.S);
  if (j < D) {
    Wp[c * KD + j] = z[c * Dz + w_off + j];
  } else if (j < KD) {
    const int k = (int)(j - D) / ge.G, a = (int)(j - D) - k * ge.G;   // block k, group a
    int64_t off = ge.a_off, so = ge.s_off;
    int nc = ge.noncentred;
    double sc = ge.s_const;
#pragma unroll
    for (int m = 0; m < 3; ++m)                // selected, not indexed: the parameter struct stays in param space
      if (k == m + 1) {
        off = ge.slope[m].b_off;
        so = ge.slope[m].s_off;
        nc = ge.slope[m].noncentred;
        sc = ge.slope[m].s_const;
      }
    float v = z[c * Dz + off + a];
    if (nc) v *= so >= 0 ? expf(z[c * Dz + so]) : (float)sc;
    Wp[c * KD + j] = v;
  } else {
    bp[c * Kb + (j - KD)] = z[c * Dz + b_off + (j - KD)];
  }
}

constexpr double kHalfLog2Pi = 0.91893853320467274178;

// log p(v) and d log p / dv of a positive scale v under prior code `prior` (B2_SIGMA_*): HalfNormal(p0),
// HalfCauchy(p0), Exponential(p0) or LogNormal(p0, p1).  The priors of a noise scale and of a weight scale.
__device__ __forceinline__ void positive_prior(int prior, double p0, double p1, double v, double& lp, double& dlp) {
  constexpr double kLog2 = 0.69314718055994531, kLogPi = 1.14472988584940017;
  if (prior == B2_SIGMA_HALFNORMAL) {             // p0 = scale
    lp = kLog2 - log(p0) - kHalfLog2Pi - v * v / (2.0 * p0 * p0);
    dlp = -v / (p0 * p0);
  } else if (prior == B2_SIGMA_HALFCAUCHY) {      // p0 = scale
    lp = kLog2 - kLogPi - log(p0) - log1p(v * v / (p0 * p0));
    dlp = -2.0 * v / (p0 * p0 + v * v);
  } else if (prior == B2_SIGMA_EXPONENTIAL) {     // p0 = rate
    lp = log(p0) - p0 * v;
    dlp = -p0;
  } else {                                        // B2_SIGMA_LOGNORMAL: p0 = loc, p1 = scale
    const double lv = log(v), q = (lv - p0) / p1;
    lp = -lv - log(p1) - kHalfLog2Pi - 0.5 * q * q;
    dlp = -1.0 / v - q / (p1 * v);
  }
}

// a latent positive scale v = e^t under prior (prior, p0, p1): U += -log p(v) - t (the Jacobian of v = e^t), and
// dU/dt = h - v (d log p / dv)(v) - 1, h being the derivative of the rest of U with respect to t
__device__ __forceinline__ double latent_scale_terms(int prior, double p0, double p1, double t, double h, double& u) {
  const double v = exp(t);
  double lp, dlp;
  positive_prior(prior, p0, p1, v, lp, dlp);
  u += -lp - t;
  return h - v * dlp - 1.0;
}

// a latent noise scale v = e^t, t = z[c, s_off]: U += -log p(v) - t (the Jacobian of v = e^t), and
// dU/dt = v (dU/dv) - 1 with dU/dv = dsig (the likelihood's, already negated) - d log p(v) / dv
__device__ __forceinline__ void add_latent_sigma_terms(const float* zc, float* gc, int64_t s_off, const float* sig,
                                                       const float* dsig, int64_t c, int s_prior, double sp0,
                                                       double sp1, double& u) {
  const double t = (double)zc[s_off], v = (double)sig[c];
  double lp, dlp;
  positive_prior(s_prior, sp0, sp1, v, lp, dlp);
  u += -lp - t;
  gc[s_off] = (float)(v * ((double)dsig[c] - dlp) - 1.0);
}

__global__ void __launch_bounds__(256) glm_potential_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const double iw = 1.0 / (s_w * s_w);
  const double ib = Kb ? 1.0 / (s_b * s_b) : 0.0;
  const float* zc = z + c * Dz;
  float* gc = grad + c * Dz;
  double qw = 0.0, qb = 0.0;  // SUM w^2 / s_w^2, SUM b^2 / s_b^2
  for (int j = lane; j < KD; j += 32) {
    const double v = (double)zc[w_off + j];
    qw += v * v * iw;
    gc[w_off + j] = (float)((double)dW[c * KD + j] + v * iw);
  }
  for (int j = lane; j < Kb; j += 32) {
    const double v = (double)zc[b_off + j];
    qb += v * v * ib;
    gc[b_off + j] = (float)((double)db[c * Kb + j] + v * ib);
  }
  qw = warp_sum(qw);
  qb = warp_sum(qb);
  if (lane == 0) {
    double u = -(double)sum_p[c] + 0.5 * qw + (double)KD * (log(s_w) + kHalfLog2Pi);
    if (Kb) u += 0.5 * qb + (double)Kb * (log(s_b) + kHalfLog2Pi);
    if (sig != nullptr && s_off >= 0) add_latent_sigma_terms(zc, gc, s_off, sig, dsig, c, s_prior, sp0, sp1, u);
    U[c] = (float)u;
  }
}

// glm_potential_finish_kernel with a latent weight scale: one warp per chain, fp64, lane-strided over the KD
// coefficients and then the shuffle tree, so every result is in a fixed order.  Per coefficient j, with
// s_j = tau lam_j and a_j = 1 - w_j^2 / s_j^2:
//   U += w_j^2 / (2 s_j^2) + log s_j + log(2 pi) / 2           dU/dw_j = dW_j + w_j / s_j^2
//   U += -log p(lam_j) - l_j                                   dU/dl_j = a_j - lam_j (d log p / d lam)(lam_j) - 1
// and once per chain U += -log p(tau) - t, dU/dt = SUM_j a_j - tau (d log p / d tau)(tau) - 1.  The bias prior and
// the noise scale's terms are those of glm_potential_finish_kernel.
__global__ void __launch_bounds__(256) glm_scaled_potential_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_b,
    const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1, b2_glm_weight_scale ws) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const double ib = Kb ? 1.0 / (s_b * s_b) : 0.0;
  const float* zc = z + c * Dz;
  float* gc = grad + c * Dz;
  const double t = ws.tau_off >= 0 ? (double)zc[ws.tau_off] : 0.0;
  double uw = 0.0, asum = 0.0, qb = 0.0;  // the weight and lam terms of U, SUM a_j, SUM b^2 / s_b^2
  for (int j = lane; j < KD; j += 32) {
    const double v = (double)zc[w_off + j];
    const double l = ws.lam_off >= 0 ? (double)zc[ws.lam_off + j] : 0.0;
    const double ls = t + l;               // log s_j
    const double is2 = exp(-2.0 * ls);     // 1 / s_j^2
    const double q = v * v * is2;
    uw += 0.5 * q + ls + kHalfLog2Pi;
    gc[w_off + j] = (float)((double)dW[c * KD + j] + v * is2);
    const double a = 1.0 - q;
    asum += a;
    if (ws.lam_off >= 0) gc[ws.lam_off + j] = (float)latent_scale_terms(ws.lam_prior, ws.lam_p0, ws.lam_p1, l, a, uw);
  }
  for (int j = lane; j < Kb; j += 32) {
    const double v = (double)zc[b_off + j];
    qb += v * v * ib;
    gc[b_off + j] = (float)((double)db[c * Kb + j] + v * ib);
  }
  uw = warp_sum(uw);
  asum = warp_sum(asum);
  qb = warp_sum(qb);
  if (lane == 0) {
    double u = -(double)sum_p[c] + uw;
    if (Kb) u += 0.5 * qb + (double)Kb * (log(s_b) + kHalfLog2Pi);
    if (sig != nullptr && s_off >= 0) add_latent_sigma_terms(zc, gc, s_off, sig, dsig, c, s_prior, sp0, sp1, u);
    if (ws.tau_off >= 0) gc[ws.tau_off] = (float)latent_scale_terms(ws.tau_prior, ws.tau_p0, ws.tau_p1, t, asum, u);
    U[c] = (float)u;
  }
}

// glm_potential_finish_kernel with a group effect alpha (ge.G values after w in each chain's [w | alpha | beta_1 ..]
// row of dW, KD = D + G (1 + S) wide): one warp per chain, fp64, lane-strided over the coefficients and then the
// shuffle tree, so every result is in a fixed order.  With s = s_a (= e^t when latent) and dW_g = d(-loglik)/d alpha_g:
//   centred      U += alpha_g^2 / (2 s^2) + log s + log(2 pi) / 2    dU/dalpha_g = dW_g + alpha_g / s^2
//                dU/dt = SUM_g (1 - alpha_g^2 / s^2) - s (d log p / ds)(s) - 1
//   non-centred  U += eta_g^2 / 2 + log(2 pi) / 2                    dU/deta_g = s dW_g + eta_g
//                dU/dt = s SUM_g eta_g dW_g - s (d log p / ds)(s) - 1
// and for a latent s once per chain U += -log p(s) - t.  The weight and bias priors and the noise scale's terms
// are those of glm_potential_finish_kernel.  Each slope block k (beta_k or e_k, scale s_k) then adds the same terms
// with its own dW columns and scale, after every term of the intercept-only potential, in the order of k.
__global__ void __launch_bounds__(256) glm_group_potential_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1, b2_glm_group_effect ge) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const int D = KD - ge.G * (1 + ge.S);
  const double iw = 1.0 / (s_w * s_w);
  const double ib = Kb ? 1.0 / (s_b * s_b) : 0.0;
  const float* zc = z + c * Dz;
  float* gc = grad + c * Dz;
  const float* dWc = dW + c * KD;
  const double t = ge.s_off >= 0 ? (double)zc[ge.s_off] : 0.0;
  const double sa = ge.s_off >= 0 ? exp(t) : ge.s_const, isa2 = 1.0 / (sa * sa);
  double qw = 0.0, qb = 0.0, ua = 0.0, h = 0.0;  // SUM w^2 / s_w^2, SUM b^2 / s_b^2, the alpha terms of U, dU/dt
  for (int j = lane; j < D; j += 32) {
    const double v = (double)zc[w_off + j];
    qw += v * v * iw;
    gc[w_off + j] = (float)((double)dWc[j] + v * iw);
  }
  for (int j = lane; j < ge.G; j += 32) {
    const double v = (double)zc[ge.a_off + j], g = (double)dWc[D + j];
    if (ge.noncentred) {
      ua += 0.5 * v * v + kHalfLog2Pi;
      h += sa * v * g;
      gc[ge.a_off + j] = (float)(sa * g + v);
    } else {
      const double q = v * v * isa2;
      ua += 0.5 * q + kHalfLog2Pi;
      h += 1.0 - q;
      gc[ge.a_off + j] = (float)(g + v * isa2);
    }
  }
  for (int j = lane; j < Kb; j += 32) {
    const double v = (double)zc[b_off + j];
    qb += v * v * ib;
    gc[b_off + j] = (float)((double)db[c * Kb + j] + v * ib);
  }
  qw = warp_sum(qw);
  qb = warp_sum(qb);
  ua = warp_sum(ua);
  h = warp_sum(h);
  double u = 0.0;
  if (lane == 0) {
    u = -(double)sum_p[c] + 0.5 * qw + (double)D * (log(s_w) + kHalfLog2Pi) + ua;
    if (!ge.noncentred) u += (double)ge.G * log(sa);
    if (Kb) u += 0.5 * qb + (double)Kb * (log(s_b) + kHalfLog2Pi);
    if (sig != nullptr && s_off >= 0) add_latent_sigma_terms(zc, gc, s_off, sig, dsig, c, s_prior, sp0, sp1, u);
    if (ge.s_off >= 0) gc[ge.s_off] = (float)latent_scale_terms(ge.s_prior, ge.sp0, ge.sp1, t, h, u);
  }
  for (int k = 0; k < ge.S; ++k) {
    const b2_glm_group_slope& sl = ge.slope[k];
    const float* dWk = dWc + D + (k + 1) * ge.G;
    const double tk = sl.s_off >= 0 ? (double)zc[sl.s_off] : 0.0;
    const double sk = sl.s_off >= 0 ? exp(tk) : sl.s_const, isk2 = 1.0 / (sk * sk);
    double ub = 0.0, hb = 0.0;                 // the block's terms of U, dU/dt_k
    for (int j = lane; j < ge.G; j += 32) {
      const double v = (double)zc[sl.b_off + j], g = (double)dWk[j];
      if (sl.noncentred) {
        ub += 0.5 * v * v + kHalfLog2Pi;
        hb += sk * v * g;
        gc[sl.b_off + j] = (float)(sk * g + v);
      } else {
        const double q = v * v * isk2;
        ub += 0.5 * q + kHalfLog2Pi;
        hb += 1.0 - q;
        gc[sl.b_off + j] = (float)(g + v * isk2);
      }
    }
    ub = warp_sum(ub);
    hb = warp_sum(hb);
    if (lane == 0) {
      u += ub;
      if (!sl.noncentred) u += (double)ge.G * log(sk);
      if (sl.s_off >= 0) gc[sl.s_off] = (float)latent_scale_terms(sl.s_prior, sl.sp0, sl.sp1, tk, hb, u);
    }
  }
  if (lane == 0) U[c] = (float)u;
}

// workspace areas, each 256-byte aligned: [likelihood workspace of lik_bytes][Wp][bp][dW][db][sum_p], then with a
// noise scale [sig][dsig]
struct GlmPotentialLayout {
  size_t wp, bp, dw, db, sum_p, sig, dsig, total;
};

inline size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }

inline GlmPotentialLayout glm_potential_layout(size_t lik_bytes, int64_t KD, int K, int64_t C, bool with_sigma) {
  GlmPotentialLayout L;
  const size_t kd = (size_t)KD, c = (size_t)C;
  size_t off = round256(lik_bytes);
  L.wp = off; off += round256(c * kd * sizeof(float));
  L.bp = off; off += round256(c * K * sizeof(float));
  L.dw = off; off += round256(c * kd * sizeof(float));
  L.db = off; off += round256(c * K * sizeof(float));
  L.sum_p = off; off += round256(c * sizeof(float));
  L.sig = L.dsig = 0;
  if (with_sigma) {
    L.sig = off; off += round256(c * sizeof(float));
    L.dsig = off; off += round256(c * sizeof(float));
  }
  L.total = off;
  return L;
}

// The noise scale of linear regression: latent when s_off >= 0 (z[c, s_off] holds its log; prior s_prior with
// parameters sp0, sp1), else the constant s_const.
struct PotentialSigma {
  int64_t s_off;
  float s_const;
  int s_prior;
  double sp0, sp1;
};

// One potential evaluation after the entry point's own checks: pack -> likelihood -> potential finish.
// lik(Wp, bp, sig, dsig, sum_p, dW, db, ws, ws_bytes) makes the likelihood call on the chains' packed operands
// with weight -1, writing sum_p, dW, db (and dsig) into the layout's areas, and returns its B2 code.  sg is
// null without a noise scale; wsc is null for a constant weight scale s_w, else the latent weight scale, finished
// by glm_scaled_potential_finish_kernel.  ge is null without a group effect, else KD counts its G columns and
// glm_group_potential_finish_kernel finishes.
template <class Likelihood>
int glm_potential_run(size_t lik_bytes, const float* z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD,
                      int K, int has_bias, double s_w, double s_b, const PotentialSigma* sg,
                      const b2_glm_weight_scale* wsc, const b2_glm_group_effect* ge, float* U, float* grad,
                      void* workspace, size_t workspace_bytes, cudaStream_t s, Likelihood lik) {
  const GlmPotentialLayout L = glm_potential_layout(lik_bytes, KD, K, C, sg != nullptr);
  if (!workspace || workspace_bytes < L.total) return B2_ERR_WORKSPACE;
  const int Kb = has_bias ? K : 0;
  char* ws = reinterpret_cast<char*>(workspace);
  float* Wp = reinterpret_cast<float*>(ws + L.wp);
  float* bp = has_bias ? reinterpret_cast<float*>(ws + L.bp) : nullptr;
  float* dW = reinterpret_cast<float*>(ws + L.dw);
  float* db = has_bias ? reinterpret_cast<float*>(ws + L.db) : nullptr;
  float* sum_p = reinterpret_cast<float*>(ws + L.sum_p);
  float* sig = sg ? reinterpret_cast<float*>(ws + L.sig) : nullptr;
  float* dsig = sg ? reinterpret_cast<float*>(ws + L.dsig) : nullptr;
  const int64_t s_off = sg ? sg->s_off : -1;

  const int64_t npack = C * (KD + Kb);
  if (ge != nullptr)
    glm_group_potential_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(
        z, C, Dz, w_off, b_off, KD, Kb, Wp, bp, s_off, sg ? sg->s_const : 0.f, sig, *ge);
  else
    glm_potential_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(z, C, Dz, w_off, b_off, KD, Kb, Wp, bp,
                                                                               s_off, sg ? sg->s_const : 0.f, sig);
  count_launch(1);
  int rc = check_launch();
  if (rc != 0) return rc;
  rc = lik(Wp, bp, sig, dsig, sum_p, dW, db, ws, L.wp);
  if (rc != 0) return rc;
  const unsigned grid = (unsigned)((C * 32 + 255) / 256);
  if (ge != nullptr)
    glm_group_potential_finish_kernel<<<grid, 256, 0, s>>>(z, C, Dz, w_off, b_off, KD, Kb, s_w, s_b, sum_p, dW, db, U,
                                                           grad, sig, dsig, s_off, sg ? sg->s_prior : 0,
                                                           sg ? sg->sp0 : 0.0, sg ? sg->sp1 : 0.0, *ge);
  else if (wsc == nullptr)
    glm_potential_finish_kernel<<<grid, 256, 0, s>>>(z, C, Dz, w_off, b_off, KD, Kb, s_w, s_b, sum_p, dW, db, U, grad,
                                                     sig, dsig, s_off, sg ? sg->s_prior : 0, sg ? sg->sp0 : 0.0,
                                                     sg ? sg->sp1 : 0.0);
  else
    glm_scaled_potential_finish_kernel<<<grid, 256, 0, s>>>(z, C, Dz, w_off, b_off, KD, Kb, s_b, sum_p, dW, db, U,
                                                            grad, sig, dsig, s_off, sg ? sg->s_prior : 0,
                                                            sg ? sg->sp0 : 0.0, sg ? sg->sp1 : 0.0, *wsc);
  count_launch(1);
  return check_launch();
}

// Scope of the likelihood kernels (K == 1 except for softmax); the kind codes of b2_glm_scaled_potential
inline bool glm_potential_in_scope(int kind, int64_t N, int D, int K, int64_t C) {
  if (N < 1 || C < 1 || C >= ((int64_t)1 << 31)) return false;
  if (kind == B2_GLM_BERNOULLI) return K == 1 && (D == 4 || D == 8 || D == 16 || D == 32);
  if (kind == B2_GLM_CATEGORICAL) return D == 32 && K >= 2 && K <= 16;
  if (kind == B2_GLM_POISSON || kind == B2_GLM_NORMAL || kind == B2_GLM_BINOMIAL)
    return K == 1 && D >= 1 && D <= 128;
  return false;
}

// the kinds b2_glm_potential takes (Normal and Binomial regression have their own entry points)
inline bool glm_plain_kind(int kind) {
  return kind == B2_GLM_BERNOULLI || kind == B2_GLM_CATEGORICAL || kind == B2_GLM_POISSON;
}

// the likelihood workspace of an in-scope kind
inline size_t glm_potential_lik_bytes(int kind, int64_t N, int D, int K, int64_t C) {
  switch (kind) {
    case B2_GLM_BERNOULLI: return b2_glm_workspace(N, D, (int)C);
    case B2_GLM_POISSON: return b2_glm_poisson_workspace(N, D, (int)C);
    case B2_GLM_NORMAL: return b2_glm_normal_workspace(N, D, (int)C);
    case B2_GLM_BINOMIAL: return b2_glm_binomial_workspace(N, D, (int)C);
    default: return b2_glm_categorical_workspace(N, D, K, (int)C);
  }
}

// The likelihood call of glm_potential_run for every kind: weight = -1, so dW, db (and dsig) are derivatives of
// -loglik; every logit fp32-exact (B2_FLAG_GLM_3XTF32; the Normal kernels always split X).  The noise scale `sig`
// and its gradient `dsig` (null for a constant noise scale) are Normal regression's, trials Binomial's; grp the
// group effect of every kind but Categorical (Wp and dW then D + G wide).
inline int glm_potential_likelihood(int kind, const float* X, const void* y, const float* trials, int trials_per_row,
                                    int64_t N, int D, int K, int64_t C, const float* Wp, const float* bp,
                                    const float* sig, float* dsig, float* sum_p, float* dW, float* db, void* ws,
                                    size_t ws_bytes, void* stream, GlmGroups grp = {}) {
  const float* yf = static_cast<const float*>(y);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  switch (kind) {
    case B2_GLM_BERNOULLI:
      return glm_bernoulli_logits(X, yf, Wp, bp, N, D, (int)C, 1.0, -1.0, 1.0, B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW,
                                  db, ws, ws_bytes, s, grp);
    case B2_GLM_POISSON:
      return glm_poisson_log_rate(X, yf, Wp, bp, N, D, (int)C, 1.0, -1.0, 1.0, B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW,
                                  db, ws, ws_bytes, s, grp);
    case B2_GLM_NORMAL:
      return glm_normal_loc(X, yf, Wp, bp, sig, 1, N, D, (int)C, 1.0, -1.0, 1.0, 0, sum_p, nullptr, dW, db, dsig, ws,
                            ws_bytes, s, grp);
    case B2_GLM_BINOMIAL:
      return glm_binomial_logits(X, yf, trials, trials_per_row, Wp, bp, N, D, (int)C, 1.0, -1.0, 1.0,
                                 B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws, ws_bytes, s, grp);
    default:
      return b2_glm_categorical_logits(X, static_cast<const int64_t*>(y), Wp, bp, N, D, K, (int)C, 1.0, -1.0, 1.0,
                                       B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws, ws_bytes, stream);
  }
}

inline bool positive_prior_ok(int prior, double p0, double p1) {
  return prior == B2_SIGMA_LOGNORMAL ? p1 > 0.0 && fabs(p0) < INFINITY
                                     : prior >= B2_SIGMA_HALFNORMAL && prior <= B2_SIGMA_EXPONENTIAL && p0 > 0.0;
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_potential_workspace(int kind, int64_t N, int D, int K, int64_t C) {
  if (!glm_plain_kind(kind) || !glm_potential_in_scope(kind, N, D, K, C)) return 256;
  return glm_potential_layout(glm_potential_lik_bytes(kind, N, D, K, C), (int64_t)K * D, K, C, false).total;
}

extern "C" int b2_glm_potential(int kind, const float* X, const void* y, int64_t N, int D, int K, int has_bias,
                                const float* z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, double s_w,
                                double s_b, float* U, float* grad, void* workspace, size_t workspace_bytes,
                                void* stream) {
  if (!X || !y || !z || !U || !grad) return B2_ERR_NULL;
  if (!glm_plain_kind(kind) || !glm_potential_in_scope(kind, N, D, K, C)) return B2_ERR_BAD_SHAPE;
  const int KD = K * D, Kb = has_bias ? K : 0;
  // z's row is exactly the weight block and the bias block, neither overlapping nor out of the row
  if (Dz != (int64_t)KD + Kb || w_off < 0 || w_off + KD > Dz) return B2_ERR_BAD_SHAPE;
  if (has_bias && (b_off < 0 || b_off + Kb > Dz || (b_off < w_off + KD && w_off < b_off + Kb)))
    return B2_ERR_BAD_SHAPE;
  if (!(s_w > 0.0) || (has_bias && !(s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  return glm_potential_run(
      glm_potential_lik_bytes(kind, N, D, K, C), z, C, Dz, w_off, b_off, KD, K, has_bias, s_w, s_b, nullptr, nullptr,
      nullptr, U, grad, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream),
      [&](const float* Wp, const float* bp, const float*, float*, float* sum_p, float* dW, float* db, void* ws,
          size_t ws_bytes) {
        return glm_potential_likelihood(kind, X, y, nullptr, 0, N, D, K, C, Wp, bp, nullptr, nullptr, sum_p, dW, db,
                                        ws, ws_bytes, stream);
      });
}

// ---- linear regression: Normal(X @ w + b, sigma), sigma constant or latent with a positive-support prior ----
extern "C" size_t b2_glm_normal_potential_workspace(int64_t N, int D, int64_t C) {
  if (N < 1 || D < 1 || D > 128 || C < 1 || C >= ((int64_t)1 << 31)) return 256;
  return glm_potential_layout(b2_glm_normal_workspace(N, D, (int)C), D, 1, C, true).total;
}

extern "C" int b2_glm_normal_potential(const float* X, const float* y, int64_t N, int D, int has_bias,
                                       const float* z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off,
                                       int64_t s_off, double s_w, double s_b, int s_prior, double sp0, double sp1,
                                       double sigma, float* U, float* grad, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  if (!X || !y || !z || !U || !grad) return B2_ERR_NULL;
  if (N < 1 || D < 1 || D > 128 || C < 1 || C >= ((int64_t)1 << 31)) return B2_ERR_BAD_SHAPE;
  const int Kb = has_bias ? 1 : 0, Ks = s_off >= 0 ? 1 : 0;
  // z's row is exactly the weight block, the bias and log sigma, none overlapping another or out of the row
  if (Dz != (int64_t)D + Kb + Ks || w_off < 0 || w_off + D > Dz) return B2_ERR_BAD_SHAPE;
  if (has_bias && (b_off < 0 || b_off >= Dz || (b_off >= w_off && b_off < w_off + D))) return B2_ERR_BAD_SHAPE;
  if (Ks && (s_off >= Dz || (s_off >= w_off && s_off < w_off + D) || (has_bias && s_off == b_off)))
    return B2_ERR_BAD_SHAPE;
  if (!(s_w > 0.0) || (has_bias && !(s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  if (Ks) {
    if (!positive_prior_ok(s_prior, sp0, sp1)) return B2_ERR_BAD_SHAPE;
  } else if (!(sigma > 0.0) || !((float)sigma > 0.f)) {
    return B2_ERR_BAD_SHAPE;
  }
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  const PotentialSigma sg = {Ks ? s_off : (int64_t)-1, (float)sigma, s_prior, sp0, sp1};
  return glm_potential_run(
      b2_glm_normal_workspace(N, D, (int)C), z, C, Dz, w_off, b_off, D, 1, has_bias, s_w, s_b, &sg, nullptr, nullptr,
      U, grad, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream),
      [&](const float* Wp, const float* bp, const float* sig, float* dsig, float* sum_p, float* dW, float* db,
          void* ws, size_t ws_bytes) {
        return glm_potential_likelihood(B2_GLM_NORMAL, X, y, nullptr, 0, N, D, 1, C, Wp, bp, sig, Ks ? dsig : nullptr,
                                        sum_p, dW, db, ws, ws_bytes, stream);
      });
}

// ---- Binomial regression: Binomial(m, logits = X @ w + b), m one count for every row or one per row ------------
extern "C" size_t b2_glm_binomial_potential_workspace(int64_t N, int D, int64_t C) {
  if (N < 1 || D < 1 || D > 128 || C < 1 || C >= ((int64_t)1 << 31)) return 256;
  return glm_potential_layout(b2_glm_binomial_workspace(N, D, (int)C), D, 1, C, false).total;
}

extern "C" int b2_glm_binomial_potential(const float* X, const float* y, const float* trials, int trials_per_row,
                                         int64_t N, int D, int has_bias, const float* z, int64_t C, int64_t Dz,
                                         int64_t w_off, int64_t b_off, double s_w, double s_b, float* U,
                                         float* grad, void* workspace, size_t workspace_bytes, void* stream) {
  if (!X || !y || !trials || !z || !U || !grad) return B2_ERR_NULL;
  if (N < 1 || D < 1 || D > 128 || C < 1 || C >= ((int64_t)1 << 31)) return B2_ERR_BAD_SHAPE;
  if (trials_per_row != 0 && trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  const int Kb = has_bias ? 1 : 0;
  // z's row is exactly the weight block and the bias, neither overlapping the other or out of the row
  if (Dz != (int64_t)D + Kb || w_off < 0 || w_off + D > Dz) return B2_ERR_BAD_SHAPE;
  if (has_bias && (b_off < 0 || b_off >= Dz || (b_off >= w_off && b_off < w_off + D))) return B2_ERR_BAD_SHAPE;
  if (!(s_w > 0.0) || (has_bias && !(s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0) return B2_ERR_BAD_SHAPE;
  return glm_potential_run(
      b2_glm_binomial_workspace(N, D, (int)C), z, C, Dz, w_off, b_off, D, 1, has_bias, s_w, s_b, nullptr, nullptr,
      nullptr, U, grad, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream),
      [&](const float* Wp, const float* bp, const float*, float*, float* sum_p, float* dW, float* db, void* ws,
          size_t ws_bytes) {
        return glm_potential_likelihood(B2_GLM_BINOMIAL, X, y, trials, trials_per_row, N, D, 1, C, Wp, bp, nullptr,
                                        nullptr, sum_p, dW, db, ws, ws_bytes, stream);
      });
}

// ---- any kind with a latent weight scale: w ~ Normal(0, tau * lam) -------------------------------------------
extern "C" size_t b2_glm_scaled_potential_workspace(int kind, int64_t N, int D, int K, int64_t C) {
  if (!glm_potential_in_scope(kind, N, D, K, C)) return 256;
  return glm_potential_layout(glm_potential_lik_bytes(kind, N, D, K, C), (int64_t)K * D, K, C,
                              kind == B2_GLM_NORMAL).total;
}

extern "C" int b2_glm_scaled_potential(int kind, const float* X, const void* y, const float* trials,
                                       int trials_per_row, int64_t N, int D, int K, int has_bias, const float* z,
                                       int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int64_t s_off, double s_b,
                                       int s_prior, double sp0, double sp1, double sigma,
                                       const b2_glm_weight_scale* scale, float* U, float* grad, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  if (!X || !y || !z || !U || !grad || !scale) return B2_ERR_NULL;
  if (kind == B2_GLM_BINOMIAL && !trials) return B2_ERR_NULL;
  if (!glm_potential_in_scope(kind, N, D, K, C)) return B2_ERR_BAD_SHAPE;
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  const b2_glm_weight_scale sc = *scale;
  const bool normal = kind == B2_GLM_NORMAL, has_tau = sc.tau_off >= 0, has_lam = sc.lam_off >= 0;
  if (!has_tau && !has_lam) return B2_ERR_BAD_SHAPE;    // a constant weight scale is b2_glm_potential's
  if (!normal && s_off >= 0) return B2_ERR_BAD_SHAPE;   // only linear regression has a noise scale
  const int64_t KD = (int64_t)K * D;
  // z's row is exactly w, b, log sigma, log tau and log lam: each block inside the row, no two overlapping, and
  // their widths summing to Dz
  const int64_t off[5] = {w_off, has_bias ? b_off : -1, s_off, sc.tau_off, sc.lam_off};
  const int64_t len[5] = {KD, has_bias ? K : 0, s_off >= 0 ? 1 : 0, has_tau ? 1 : 0, has_lam ? KD : 0};
  int64_t width = 0;
  for (int i = 0; i < 5; ++i) {
    if (len[i] == 0) continue;
    if (off[i] < 0 || off[i] > Dz - len[i]) return B2_ERR_BAD_SHAPE;
    for (int j = 0; j < i; ++j)
      if (len[j] && off[i] < off[j] + len[j] && off[j] < off[i] + len[i]) return B2_ERR_BAD_SHAPE;
    width += len[i];
  }
  if (width != Dz) return B2_ERR_BAD_SHAPE;
  if (has_bias && !(s_b > 0.0)) return B2_ERR_BAD_SHAPE;
  if (has_tau && !positive_prior_ok(sc.tau_prior, sc.tau_p0, sc.tau_p1)) return B2_ERR_BAD_SHAPE;
  if (has_lam && !positive_prior_ok(sc.lam_prior, sc.lam_p0, sc.lam_p1)) return B2_ERR_BAD_SHAPE;
  if (normal && s_off >= 0 && !positive_prior_ok(s_prior, sp0, sp1)) return B2_ERR_BAD_SHAPE;
  if (normal && s_off < 0 && (!(sigma > 0.0) || !((float)sigma > 0.f))) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row != 0 && trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  const PotentialSigma sg = {s_off >= 0 ? s_off : (int64_t)-1, (float)sigma, s_prior, sp0, sp1};
  const bool latent_sigma = normal && s_off >= 0;
  return glm_potential_run(
      glm_potential_lik_bytes(kind, N, D, K, C), z, C, Dz, w_off, b_off, (int)KD, K, has_bias, 1.0, s_b,
      normal ? &sg : nullptr, &sc, nullptr, U, grad, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream),
      [&](const float* Wp, const float* bp, const float* sig, float* dsig, float* sum_p, float* dW, float* db,
          void* ws, size_t ws_bytes) {
        return glm_potential_likelihood(kind, X, y, trials, trials_per_row, N, D, K, C, Wp, bp, sig,
                                        latent_sigma ? dsig : nullptr, sum_p, dW, db, ws, ws_bytes, stream);
      });
}

// ---- a varying intercept by group: alpha[g], centred or non-centred, with a constant or latent scale s_a, and up to
// three varying slopes beta_k[g] X[n, c_k] with scales of the same forms ------------------------------------------
// Scope: kinds Bernoulli, Poisson, Normal and Binomial, 1 <= G and D + G (1 + S) <= 128 (G here: the group columns).
inline bool glm_group_in_scope(int kind, int64_t N, int D, int G, int64_t C) {
  if (kind != B2_GLM_BERNOULLI && kind != B2_GLM_POISSON && kind != B2_GLM_NORMAL && kind != B2_GLM_BINOMIAL)
    return false;
  return N >= 1 && C >= 1 && C < ((int64_t)1 << 31) && D >= 1 && G >= 1 && D + G <= 128;
}

extern "C" size_t b2_glm_group_potential_workspace(int kind, int64_t N, int D, int G, int64_t C) {
  if (!glm_group_in_scope(kind, N, D, G, C)) return 256;
  return glm_potential_layout(glm_potential_lik_bytes(kind, N, D + G, 1, C), D + G, 1, C, kind == B2_GLM_NORMAL).total;
}

extern "C" int b2_glm_group_potential(int kind, const float* X, const void* y, const float* trials,
                                      int trials_per_row, int64_t N, int D, int has_bias, const float* z, int64_t C,
                                      int64_t Dz, int64_t w_off, int64_t b_off, int64_t s_off, double s_w,
                                      double s_b, int s_prior, double sp0, double sp1, double sigma,
                                      const b2_glm_group_effect* ge, float* U, float* grad, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  if (!X || !y || !z || !U || !grad || !ge || !ge->groups) return B2_ERR_NULL;
  if (kind == B2_GLM_BINOMIAL && !trials) return B2_ERR_NULL;
  const b2_glm_group_effect g = *ge;
  if (g.S < 0 || g.S > 3 || g.G < 1 || g.G > 128) return B2_ERR_BAD_SHAPE;
  const int Da = D + g.G * (1 + g.S);
  if (!glm_group_in_scope(kind, N, D, g.G * (1 + g.S), C)) return B2_ERR_BAD_SHAPE;
  if (N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  const bool normal = kind == B2_GLM_NORMAL;
  if (!normal && s_off >= 0) return B2_ERR_BAD_SHAPE;   // only linear regression has a noise scale
  if (g.noncentred != 0 && g.noncentred != 1) return B2_ERR_BAD_SHAPE;
  for (int k = 0; k < g.S; ++k) {
    const b2_glm_group_slope& sl = g.slope[k];
    if (sl.col < 0 || sl.col >= D || (sl.noncentred != 0 && sl.noncentred != 1)) return B2_ERR_BAD_SHAPE;
    for (int j = 0; j < k; ++j)
      if (g.slope[j].col == sl.col) return B2_ERR_BAD_SHAPE;
    if (sl.s_off >= 0 && !positive_prior_ok(sl.s_prior, sl.sp0, sl.sp1)) return B2_ERR_BAD_SHAPE;
    if (sl.s_off < 0 && (!(sl.s_const > 0.0) || !((float)sl.s_const > 0.f))) return B2_ERR_BAD_SHAPE;
  }
  // z's row is exactly w, b, log sigma, alpha (or eta), log s_a and each slope's beta_k (or e_k) and log s_k: each
  // block inside the row, no two overlapping, and their widths summing to Dz
  int64_t off[11] = {w_off, has_bias ? b_off : -1, s_off, g.a_off, g.s_off};
  int64_t len[11] = {D, has_bias ? 1 : 0, s_off >= 0 ? 1 : 0, g.G, g.s_off >= 0 ? 1 : 0};
  const int nblk = 5 + 2 * g.S;
  for (int k = 0; k < g.S; ++k) {
    off[5 + 2 * k] = g.slope[k].b_off;
    len[5 + 2 * k] = g.G;
    off[6 + 2 * k] = g.slope[k].s_off;
    len[6 + 2 * k] = g.slope[k].s_off >= 0 ? 1 : 0;
  }
  int64_t width = 0;
  for (int i = 0; i < nblk; ++i) {
    if (len[i] == 0) continue;
    if (off[i] < 0 || off[i] > Dz - len[i]) return B2_ERR_BAD_SHAPE;
    for (int j = 0; j < i; ++j)
      if (len[j] && off[i] < off[j] + len[j] && off[j] < off[i] + len[i]) return B2_ERR_BAD_SHAPE;
    width += len[i];
  }
  if (width != Dz) return B2_ERR_BAD_SHAPE;
  if (!(s_w > 0.0) || (has_bias && !(s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  if (g.s_off >= 0 && !positive_prior_ok(g.s_prior, g.sp0, g.sp1)) return B2_ERR_BAD_SHAPE;
  if (g.s_off < 0 && (!(g.s_const > 0.0) || !((float)g.s_const > 0.f))) return B2_ERR_BAD_SHAPE;
  if (normal && s_off >= 0 && !positive_prior_ok(s_prior, sp0, sp1)) return B2_ERR_BAD_SHAPE;
  if (normal && s_off < 0 && (!(sigma > 0.0) || !((float)sigma > 0.f))) return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row != 0 && trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  if (reinterpret_cast<uintptr_t>(X) % 16 != 0 || reinterpret_cast<uintptr_t>(y) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(g.groups) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  if (kind == B2_GLM_BINOMIAL && trials_per_row && reinterpret_cast<uintptr_t>(trials) % 16 != 0)
    return B2_ERR_BAD_SHAPE;
  const PotentialSigma sg = {s_off >= 0 ? s_off : (int64_t)-1, (float)sigma, s_prior, sp0, sp1};
  const bool latent_sigma = normal && s_off >= 0;
  GlmGroups grp;
  grp.idx = g.groups;
  grp.G = g.G;
  grp.S = g.S;
  for (int k = 0; k < g.S; ++k) grp.col[k] = g.slope[k].col;
  return glm_potential_run(
      glm_potential_lik_bytes(kind, N, Da, 1, C), z, C, Dz, w_off, b_off, Da, 1, has_bias, s_w, s_b,
      normal ? &sg : nullptr, nullptr, &g, U, grad, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream),
      [&](const float* Wp, const float* bp, const float* sig, float* dsig, float* sum_p, float* dW, float* db,
          void* ws, size_t ws_bytes) {
        return glm_potential_likelihood(kind, X, y, trials, trials_per_row, N, D, 1, C, Wp, bp, sig,
                                        latent_sigma ? dsig : nullptr, sum_p, dW, db, ws, ws_bytes, stream, grp);
      });
}
