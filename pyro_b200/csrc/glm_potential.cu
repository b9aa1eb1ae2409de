// glm_potential.cu -- HMC / NUTS potential energy of Bayesian logistic, softmax, Poisson, Binomial and linear
// regression for C chains: b2_glm_potential on one b2_glm_regression.
//
//   U[c]    = -( SUM_n log p(y_n | logits_cn) + log p(w) + log p(b) [+ log p(sigma)] [+ group effect] ) + Jacobians
//   grad[c] = dU / dz[c]                                           (in z's layout)
//
// The likelihood and its gradient come from the fused GLM likelihood calls (glm_bernoulli_logits,
// b2_glm_categorical_logits, glm_poisson_log_rate, glm_normal_loc, glm_binomial_logits: a tile kernel and
// glm_finish_kernel each) with their particle axis set to the chains, so X is read once per evaluation for every
// chain together.  b2_glm_potential checks every argument, then makes the one fixed launch sequence, with no host
// sync (CUDA graph capturable):
//   1. glm_potential_pack_kernel    z's weight / bias columns -> the contiguous [C, KD] / [C, K] operands
//                                   (z's rows also hold the other sites, so their stride is not the kernels')
//   2. the likelihood call          weight = -1: dW, db are d(-loglik)/dW, d(-loglik)/db; sum_p = loglik
//   3. glm_potential_finish_kernel  adds the priors' values and gradients, one warp per chain, fp64 accumulation
//                                   in a fixed order, and writes U and grad
// The GLM kernels always run with every logit fp32-exact (B2_FLAG_GLM_3XTF32; the Normal kernels always split X),
// so the sampler targets the posterior of the data as given, not of X rounded to TF32.
// With a noise scale (linear regression) the pack also writes each chain's sigma_c = exp(z[c, s_off]) (or the
// constant), and the finish adds sigma's prior and the Jacobian of sigma = e^t in fp64.  Binomial regression passes
// the trial counts to its likelihood call as a fixed operand.  A latent weight scale (w ~ Normal(0, tau * lam))
// changes only the finish's weight terms.  A group effect, a varying intercept alpha[g] and up to three varying
// slopes beta_k[g] on columns of X, makes each chain's packed weight row [w | alpha | beta_1 ..], and the likelihood
// runs on [X | onehot(g) | x_{c_1} onehot(g) ..] (glm_flat_tc.cuh GROUPS) when those D + G (1 + S) columns fit in
// 128.  Past that (rows sorted by group) the group effect is gathered (glm_flat_tc.cuh GATHER,
// glm_group_gather_tc.cu): the pack writes the group-major tables T_k [1 + S][G][cp] and zeroes the group-gradient
// table, the likelihood runs D wide and leaves the run sums of each group, and the finish adds the runs that cross
// the warpgroups' ranges (gather_fixup) before the same prior terms.
#include <math.h>

#include "b2_common.cuh"
#include "glm_host.cuh"

namespace b2 {

// Each chain's weight row [w | alpha | beta_1 .. beta_S], KD = D + G (1 + S) wide with a group effect (GROUP; else
// KD = K*D and ge is not read).  Group block 0 is alpha, block k slope k; each is z's columns, or s * eta for a
// non-centred block (s its scale: exp of its z column, or its constant).  sig (linear regression only, else null):
// sig[c] = exp(z[c, s_off]) for a latent noise scale (z holds its log), the constant s_const when s_off < 0.
template <bool GROUP>
__global__ void __launch_bounds__(256) glm_potential_pack_kernel(const float* __restrict__ z, int64_t C, int64_t Dz,
                                                                 int64_t w_off, int64_t b_off, int KD, int Kb,
                                                                 float* __restrict__ Wp, float* __restrict__ bp,
                                                                 int64_t s_off, float s_const,
                                                                 float* __restrict__ sig, b2_glm_group_effect ge) {
  const int64_t per = KD + Kb;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (sig != nullptr && i < C) sig[i] = s_off >= 0 ? expf(z[i * Dz + s_off]) : s_const;
  if (i >= C * per) return;
  const int64_t c = i / per;
  const int64_t j = i - c * per;
  const int D = GROUP ? KD - ge.G * (1 + ge.S) : KD;
  if (j < D) {
    Wp[c * KD + j] = z[c * Dz + w_off + j];
  } else if (GROUP && j < KD) {
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

// The gathered route: Wp / bp / sig as glm_potential_pack_kernel<false> (KD = D), then tab[k][a][c] (c < cp) the
// value of group a in block k for chain c (0 for c >= C), and gsum zeroed
__global__ void __launch_bounds__(256) glm_potential_gather_pack_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int D, int Kb,
    float* __restrict__ Wp, float* __restrict__ bp, int64_t s_off, float s_const, float* __restrict__ sig,
    b2_glm_group_effect ge, int cp, float* __restrict__ tab, float* __restrict__ gsum) {
  const int64_t per = D + Kb, nw = C * per;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (sig != nullptr && i < C) sig[i] = s_off >= 0 ? expf(z[i * Dz + s_off]) : s_const;
  if (i < nw) {
    const int64_t c = i / per, j = i - c * per;
    if (j < D) Wp[c * D + j] = z[c * Dz + w_off + j];
    else bp[c * Kb + (j - D)] = z[c * Dz + b_off + (j - D)];
    return;
  }
  const int64_t e = i - nw;
  if (e >= (int64_t)(1 + ge.S) * ge.G * cp) return;
  const int64_t kg = e / cp, c = e - kg * cp;
  const int k = (int)(kg / ge.G), a = (int)(kg - (int64_t)k * ge.G);
  int64_t off = ge.a_off, so = ge.s_off;
  int nc = ge.noncentred;
  double sc = ge.s_const;
#pragma unroll
  for (int m = 0; m < 3; ++m)
    if (k == m + 1) {
      off = ge.slope[m].b_off;
      so = ge.slope[m].s_off;
      nc = ge.slope[m].noncentred;
      sc = ge.slope[m].s_const;
    }
  float v = 0.f;
  if (c < C) {
    v = z[c * Dz + off + a];
    if (nc) v *= so >= 0 ? expf(z[c * Dz + so]) : (float)sc;
  }
  tab[e] = v;
  gsum[e] = 0.f;
}

constexpr double kHalfLog2Pi = 0.91893853320467274178;

// log p(v) and d log p / dv of a positive scale v under prior code `prior` (B2_SIGMA_*): HalfNormal(p0),
// HalfCauchy(p0), Exponential(p0) or LogNormal(p0, p1).  The priors of a noise scale, a weight scale and a group
// effect's scale.
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

// One block of a group effect (the intercept, described as a slope, or a slope): its G values v_g at z columns
// b.b_off (alpha_g or beta_k,g when centred, e_g when non-centred) with the scale s = e^t, t = z[c, b.s_off] (or the
// constant b.s_const), and dWb[g] = d(-loglik)/d(the block's coefficient of group g):
//   centred      U += v_g^2 / (2 s^2) + log s + log(2 pi) / 2    dU/dv_g = dWb_g + v_g / s^2
//                dU/dt = SUM_g (1 - v_g^2 / s^2) - s (d log p / ds)(s) - 1
//   non-centred  U += v_g^2 / 2 + log(2 pi) / 2                  dU/dv_g = s dWb_g + v_g
//                dU/dt = s SUM_g v_g dWb_g - s (d log p / ds)(s) - 1
// and for a latent s once per chain U += -log p(s) - t.  Lane-strided over the G values, then the shuffle tree:
// writes dU/dv_g and returns, in every lane, t, s and the warp's sums u (the block's terms of U but G log s) and h
// (dU/dt before the prior's terms).
struct GroupBlockSums {
  double t, s, u, h;
};

// GATHER: dWb[j * stride] is the run sum of group j, d loglik / dv scaled by fac to d(-loglik)/dv; bad: NaN instead
template <bool GATHER = false>
__device__ __forceinline__ GroupBlockSums group_block_sums(const b2_glm_group_slope& b, int G, const float* zc,
                                                           float* gc, const float* dWb, int lane,
                                                           int64_t stride = 1, double fac = 1.0, bool bad = false) {
  GroupBlockSums r;
  r.t = b.s_off >= 0 ? (double)zc[b.s_off] : 0.0;
  r.s = b.s_off >= 0 ? exp(r.t) : b.s_const;
  const double is2 = 1.0 / (r.s * r.s);
  double u = 0.0, h = 0.0;
  for (int j = lane; j < G; j += 32) {
    const double v = (double)zc[b.b_off + j],
                 g = GATHER ? (bad ? __longlong_as_double(0x7ff8000000000000ll) : fac * (double)dWb[j * stride])
                            : (double)dWb[j];
    if (b.noncentred) {
      u += 0.5 * v * v + kHalfLog2Pi;
      h += r.s * v * g;
      gc[b.b_off + j] = (float)(r.s * g + v);
    } else {
      const double q = v * v * is2;
      u += 0.5 * q + kHalfLog2Pi;
      h += 1.0 - q;
      gc[b.b_off + j] = (float)(g + v * is2);
    }
  }
  r.u = warp_sum(u);
  r.h = warp_sum(h);
  return r;
}

// lane 0: a group block's terms of U, G log s for a centred one last
__device__ __forceinline__ void add_group_block_u(const b2_glm_group_slope& b, int G, const GroupBlockSums& r,
                                                  double& u) {
  u += r.u;
  if (!b.noncentred) u += (double)G * log(r.s);
}

// One warp per chain, fp64, lane-strided over each block of coefficients and then the shuffle tree, so every result
// is in a fixed order.  The weight prior over the D = KD - G (1 + S) coefficients of w is the constant-scale
//   U += SUM_j w_j^2 / (2 s_w^2) + D (log s_w + log(2 pi) / 2)    dU/dw_j = dW_j + w_j / s_w^2
// or, with a latent weight scale (LATENT: ws), per coefficient j, with s_j = tau lam_j and a_j = 1 - w_j^2 / s_j^2:
//   U += w_j^2 / (2 s_j^2) + log s_j + log(2 pi) / 2           dU/dw_j = dW_j + w_j / s_j^2
//   U += -log p(lam_j) - l_j                                   dU/dl_j = a_j - lam_j (d log p / d lam)(lam_j) - 1
// and once per chain U += -log p(tau) - t, dU/dt = SUM_j a_j - tau (d log p / d tau)(tau) - 1.  Then come the bias
// prior, the noise scale's terms and, with a group effect (GROUP: ge), its blocks: the intercept block's U terms
// before the bias prior and its latent scale's after the noise scale's, then each slope block, in the order of k.
// LATENT and GROUP are template flags, so each configuration runs only its own code.  GATHER (with GROUP): the
// gathered route, KD = D, the group blocks' d loglik from gather_fixup's table times -1 (-1 / sigma_c^2 for linear
// regression, as glm_finish_kernel scales dW), and U NaN for a bad index or a descending pair.
template <bool LATENT, bool GROUP, bool GATHER = false>
__device__ __forceinline__ void glm_potential_finish(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1, const b2_glm_weight_scale& ws, const b2_glm_group_effect& ge,
    const GlmGatherFinish& gf) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const int D = GROUP && !GATHER ? KD - ge.G * (1 + ge.S) : KD;
  bool bad = false;
  double gfac = 1.0;
  if constexpr (GATHER) {
    bad = gather_fixup(gf, ge.G, ge.S, c, lane);
    const double sg = sig != nullptr ? (double)sig[c] : 1.0;
    gfac = sig != nullptr ? -1.0 / (sg * sg) : -1.0;
  }
  const double ib = Kb ? 1.0 / (s_b * s_b) : 0.0;
  const float* zc = z + c * Dz;
  float* gc = grad + c * Dz;
  const float* dWc = dW + c * KD;
  const double t = LATENT && ws.tau_off >= 0 ? (double)zc[ws.tau_off] : 0.0;
  const b2_glm_group_slope icpt = {ge.a_off, ge.s_off, 0, ge.noncentred, ge.s_prior, ge.s_const, ge.sp0, ge.sp1};
  GroupBlockSums a = {};
  if (GATHER) a = group_block_sums<true>(icpt, ge.G, zc, gc, gf.gsum + c, lane, gf.cp, gfac, bad);
  else if (GROUP) a = group_block_sums(icpt, ge.G, zc, gc, dWc + D, lane);
  // uw: SUM w^2 / s_w^2 for a constant weight scale, the weight and lam terms of U for a latent one; asum: SUM a_j;
  // qb: SUM b^2 / s_b^2
  double uw = 0.0, asum = 0.0, qb = 0.0;
  if (LATENT) {
    for (int j = lane; j < D; j += 32) {
      const double v = (double)zc[w_off + j];
      const double l = ws.lam_off >= 0 ? (double)zc[ws.lam_off + j] : 0.0;
      const double ls = t + l;               // log s_j
      const double is2 = exp(-2.0 * ls);     // 1 / s_j^2
      const double q = v * v * is2;
      uw += 0.5 * q + ls + kHalfLog2Pi;
      gc[w_off + j] = (float)((double)dWc[j] + v * is2);
      const double a = 1.0 - q;
      asum += a;
      if (ws.lam_off >= 0)
        gc[ws.lam_off + j] = (float)latent_scale_terms(ws.lam_prior, ws.lam_p0, ws.lam_p1, l, a, uw);
    }
  } else {
    const double iw = 1.0 / (s_w * s_w);
    for (int j = lane; j < D; j += 32) {
      const double v = (double)zc[w_off + j];
      uw += v * v * iw;
      gc[w_off + j] = (float)((double)dWc[j] + v * iw);
    }
  }
  for (int j = lane; j < Kb; j += 32) {
    const double v = (double)zc[b_off + j];
    qb += v * v * ib;
    gc[b_off + j] = (float)((double)db[c * Kb + j] + v * ib);
  }
  uw = warp_sum(uw);
  if (LATENT) asum = warp_sum(asum);
  qb = warp_sum(qb);
  double u = 0.0;
  if (lane == 0) {
    u = LATENT ? -(double)sum_p[c] + uw : -(double)sum_p[c] + 0.5 * uw + (double)D * (log(s_w) + kHalfLog2Pi);
    if (GROUP) add_group_block_u(icpt, ge.G, a, u);
    if (Kb) u += 0.5 * qb + (double)Kb * (log(s_b) + kHalfLog2Pi);
    if (sig != nullptr && s_off >= 0) add_latent_sigma_terms(zc, gc, s_off, sig, dsig, c, s_prior, sp0, sp1, u);
    if (LATENT && ws.tau_off >= 0)
      gc[ws.tau_off] = (float)latent_scale_terms(ws.tau_prior, ws.tau_p0, ws.tau_p1, t, asum, u);
    if (GROUP && ge.s_off >= 0) gc[ge.s_off] = (float)latent_scale_terms(ge.s_prior, ge.sp0, ge.sp1, a.t, a.h, u);
  }
  for (int k = 0; GROUP && k < ge.S; ++k) {
    const b2_glm_group_slope& sl = ge.slope[k];
    const GroupBlockSums b =
        GATHER ? group_block_sums<true>(sl, ge.G, zc, gc, gf.gsum + (int64_t)(k + 1) * ge.G * gf.cp + c, lane, gf.cp,
                                        gfac, bad)
               : group_block_sums(sl, ge.G, zc, gc, dWc + D + (k + 1) * ge.G, lane);
    if (lane == 0) {
      add_group_block_u(sl, ge.G, b, u);
      if (sl.s_off >= 0) gc[sl.s_off] = (float)latent_scale_terms(sl.s_prior, sl.sp0, sl.sp1, b.t, b.h, u);
    }
  }
  if (lane == 0) U[c] = GATHER && bad ? __int_as_float(0x7fc00000) : (float)u;
}

template <bool LATENT, bool GROUP>
__global__ void __launch_bounds__(256) glm_potential_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int KD, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1, b2_glm_weight_scale ws, b2_glm_group_effect ge) {
  glm_potential_finish<LATENT, GROUP>(z, C, Dz, w_off, b_off, KD, Kb, s_w, s_b, sum_p, dW, db, U, grad, sig, dsig,
                                      s_off, s_prior, sp0, sp1, ws, ge, {});
}

__global__ void __launch_bounds__(256) glm_potential_gather_finish_kernel(
    const float* __restrict__ z, int64_t C, int64_t Dz, int64_t w_off, int64_t b_off, int D, int Kb, double s_w,
    double s_b, const float* __restrict__ sum_p, const float* __restrict__ dW, const float* __restrict__ db,
    float* __restrict__ U, float* __restrict__ grad, const float* __restrict__ sig, const float* __restrict__ dsig,
    int64_t s_off, int s_prior, double sp0, double sp1, b2_glm_group_effect ge, GlmGatherFinish gf) {
  const b2_glm_weight_scale no_scale = {-1, -1, 0, 0, 0.0, 0.0, 0.0, 0.0};
  glm_potential_finish<false, true, true>(z, C, Dz, w_off, b_off, D, Kb, s_w, s_b, sum_p, dW, db, U, grad, sig, dsig,
                                          s_off, s_prior, sp0, sp1, no_scale, ge, gf);
}

// the group columns of the likelihood's contraction, G (1 + S); 0 without a group effect
inline int glm_group_cols(const b2_glm_regression& m) { return m.group ? m.group->G * (1 + m.group->S) : 0; }

// a group effect past the contraction's 128 columns: the gathered route
inline bool glm_gathered(const b2_glm_regression& m) { return m.group && m.D + glm_group_cols(m) > 128; }

// The kinds and widths the likelihood kernels take (K == 1 except for softmax).  With a group effect: every kind
// but softmax, 1 <= D <= 128, 1 <= G <= 65536, a constant weight scale, and past D + G (1 + S) = 128 columns only
// with the caller's promise that the rows are sorted by group, and not for Binomial regression (the gathered
// route has no Binomial kernel).
inline bool glm_regression_in_scope(const b2_glm_regression& m, int64_t C) {
  if (m.N < 1 || C < 1 || C >= ((int64_t)1 << 31)) return false;
  if (m.group) {
    const b2_glm_group_effect& g = *m.group;
    if (m.scale || g.S < 0 || g.S > 3 || g.G < 1 || g.G > 65536 || (g.sorted != 0 && g.sorted != 1)) return false;
    return (m.kind == B2_GLM_BERNOULLI || m.kind == B2_GLM_POISSON || m.kind == B2_GLM_NORMAL ||
            m.kind == B2_GLM_BINOMIAL) &&
           m.K == 1 && m.D >= 1 && m.D <= 128 &&
           (m.D + glm_group_cols(m) <= 128 || (g.sorted == 1 && m.kind != B2_GLM_BINOMIAL));
  }
  if (m.kind == B2_GLM_BERNOULLI) return m.K == 1 && (m.D == 4 || m.D == 8 || m.D == 16 || m.D == 32);
  if (m.kind == B2_GLM_CATEGORICAL) return m.D == 32 && m.K >= 2 && m.K <= 16;
  if (m.kind == B2_GLM_POISSON || m.kind == B2_GLM_NORMAL || m.kind == B2_GLM_BINOMIAL)
    return m.K == 1 && m.D >= 1 && m.D <= 128;
  return false;
}

// workspace areas, each 256-byte aligned: [likelihood workspace][Wp][bp][dW][db][sum_p], then for linear
// regression [sig][dsig], then for the gathered route [tab][gsum][slots][status] (none grows with N past the
// likelihood's CTA partials)
struct GlmPotentialLayout {
  size_t wp, bp, dw, db, sum_p, sig, dsig, tab, gsum, slots, status, total;
  int cp, Q;
};

inline size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }

// the layout of an in-scope regression
inline GlmPotentialLayout glm_potential_layout(const b2_glm_regression& m, int64_t C) {
  const bool gathered = glm_gathered(m);
  const int Da = gathered ? m.D : m.D + glm_group_cols(m);
  size_t lik_bytes;
  if (gathered) lik_bytes = glm_row_workspace(m.N, m.D, (int)C);
  else switch (m.kind) {
    case B2_GLM_BERNOULLI: lik_bytes = b2_glm_workspace(m.N, Da, (int)C); break;
    case B2_GLM_POISSON: lik_bytes = b2_glm_poisson_workspace(m.N, Da, (int)C); break;
    case B2_GLM_NORMAL: lik_bytes = b2_glm_normal_workspace(m.N, Da, (int)C); break;
    case B2_GLM_BINOMIAL: lik_bytes = b2_glm_binomial_workspace(m.N, Da, (int)C); break;
    default: lik_bytes = b2_glm_categorical_workspace(m.N, Da, m.K, (int)C);
  }
  GlmPotentialLayout L;
  const size_t kd = (size_t)Da * m.K, k = (size_t)m.K, c = (size_t)C;
  size_t off = round256(lik_bytes);
  L.wp = off; off += round256(c * kd * sizeof(float));
  L.bp = off; off += round256(c * k * sizeof(float));
  L.dw = off; off += round256(c * kd * sizeof(float));
  L.db = off; off += round256(c * k * sizeof(float));
  L.sum_p = off; off += round256(c * sizeof(float));
  L.sig = L.dsig = 0;
  if (m.kind == B2_GLM_NORMAL) {
    L.sig = off; off += round256(c * sizeof(float));
    L.dsig = off; off += round256(c * sizeof(float));
  }
  L.tab = L.gsum = L.slots = L.status = 0;
  L.cp = L.Q = 0;
  if (gathered) {
    L.cp = (int)((C + 63) / 64 * 64);
    L.Q = glm_gather_ranges(m.N, m.D);
    const size_t table = (size_t)(1 + m.group->S) * m.group->G * L.cp * sizeof(float);
    L.tab = off; off += round256(table);
    L.gsum = off; off += round256(table);
    L.slots = off; off += round256((size_t)L.Q * 2 * 4 * L.cp * sizeof(float));
    L.status = off; off += round256((size_t)L.Q * sizeof(int));
  }
  L.total = off;
  return L;
}

// The likelihood call for every kind: weight = -1, so dW, db (and dsig) are derivatives of -loglik; every logit
// fp32-exact (B2_FLAG_GLM_3XTF32; the Normal kernels always split X).  The noise scale `sig` and its gradient `dsig`
// (null for a constant noise scale) are Normal regression's, trials Binomial's; grp the group effect of every kind
// but Categorical (Wp and dW then D + G (1 + S) wide).
inline int glm_potential_likelihood(const b2_glm_regression& m, int64_t C, const float* Wp, const float* bp,
                                    const float* sig, float* dsig, float* sum_p, float* dW, float* db, void* ws,
                                    size_t ws_bytes, void* stream, GlmGroups grp) {
  const float* yf = static_cast<const float*>(m.y);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  switch (m.kind) {
    case B2_GLM_BERNOULLI:
      return glm_bernoulli_logits(m.X, yf, Wp, bp, m.N, m.D, (int)C, 1.0, -1.0, 1.0, B2_FLAG_GLM_3XTF32, sum_p,
                                  nullptr, dW, db, ws, ws_bytes, s, grp);
    case B2_GLM_POISSON:
      return glm_poisson_log_rate(m.X, yf, Wp, bp, m.N, m.D, (int)C, 1.0, -1.0, 1.0, B2_FLAG_GLM_3XTF32, sum_p,
                                  nullptr, dW, db, ws, ws_bytes, s, grp);
    case B2_GLM_NORMAL:
      return glm_normal_loc(m.X, yf, Wp, bp, sig, 1, m.N, m.D, (int)C, 1.0, -1.0, 1.0, 0, sum_p, nullptr, dW, db,
                            dsig, ws, ws_bytes, s, grp);
    case B2_GLM_BINOMIAL:
      return glm_binomial_logits(m.X, yf, m.trials, m.trials_per_row, Wp, bp, m.N, m.D, (int)C, 1.0, -1.0, 1.0,
                                 B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws, ws_bytes, s, grp);
    default:
      return b2_glm_categorical_logits(m.X, static_cast<const int64_t*>(m.y), Wp, bp, m.N, m.D, m.K, (int)C, 1.0,
                                       -1.0, 1.0, B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws, ws_bytes, stream);
  }
}

inline bool positive_prior_ok(int prior, double p0, double p1) {
  return prior == B2_SIGMA_LOGNORMAL ? p1 > 0.0 && fabs(p0) < INFINITY
                                     : prior >= B2_SIGMA_HALFNORMAL && prior <= B2_SIGMA_EXPONENTIAL && p0 > 0.0;
}

// a scale latent at z column s_off with a valid prior, or else the constant s_const, positive in fp32 too
inline bool positive_scale_ok(int64_t s_off, int prior, double p0, double p1, double s_const) {
  return s_off >= 0 ? positive_prior_ok(prior, p0, p1) : s_const > 0.0 && (float)s_const > 0.f;
}

inline bool misaligned(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; }

// Every check of b2_glm_potential that needs no workspace: 0, or the B2 code of the first one that fails.
inline int glm_potential_check(const b2_glm_regression* mp, const float* z, int64_t C, int64_t Dz, const float* U,
                               const float* grad) {
  if (!mp || !mp->X || !mp->y || !z || !U || !grad) return B2_ERR_NULL;
  const b2_glm_regression& m = *mp;
  if ((m.kind == B2_GLM_BINOMIAL && !m.trials) || (m.group && !m.group->groups)) return B2_ERR_NULL;
  if (!glm_regression_in_scope(m, C)) return B2_ERR_BAD_SHAPE;
  // the others leave N to their likelihood call, whose SIMT Bernoulli kernel takes any N
  if ((m.scale || m.group) && m.N >= ((int64_t)1 << 31)) return B2_ERR_TOO_LARGE;
  const bool normal = m.kind == B2_GLM_NORMAL, binomial = m.kind == B2_GLM_BINOMIAL;
  if (!normal && m.s_off >= 0) return B2_ERR_BAD_SHAPE;   // only linear regression has a noise scale
  if (normal && !positive_scale_ok(m.s_off, m.s_prior, m.sp0, m.sp1, m.sigma)) return B2_ERR_BAD_SHAPE;
  if (binomial && m.trials_per_row != 0 && m.trials_per_row != 1) return B2_ERR_BAD_SHAPE;
  if ((!m.scale && !(m.s_w > 0.0)) || (m.has_bias && !(m.s_b > 0.0))) return B2_ERR_BAD_SHAPE;
  // z's row is exactly w, b, log sigma, log tau, log lam, alpha (or eta), log s_a and each slope's beta_k (or e_k)
  // and log s_k: each present block inside the row, no two overlapping, and their widths summing to Dz
  const int64_t KD = (int64_t)m.K * m.D;
  int64_t off[13] = {m.w_off, m.b_off, m.s_off}, len[13] = {KD, m.has_bias ? m.K : 0, m.s_off >= 0 ? 1 : 0};
  int nblk = 3;
  if (const b2_glm_weight_scale* sc = m.scale) {
    if (sc->tau_off < 0 && sc->lam_off < 0) return B2_ERR_BAD_SHAPE;   // a constant weight scale is s_w
    if (sc->tau_off >= 0 && !positive_prior_ok(sc->tau_prior, sc->tau_p0, sc->tau_p1)) return B2_ERR_BAD_SHAPE;
    if (sc->lam_off >= 0 && !positive_prior_ok(sc->lam_prior, sc->lam_p0, sc->lam_p1)) return B2_ERR_BAD_SHAPE;
    off[nblk] = sc->tau_off, len[nblk++] = sc->tau_off >= 0 ? 1 : 0;
    off[nblk] = sc->lam_off, len[nblk++] = sc->lam_off >= 0 ? KD : 0;
  }
  if (const b2_glm_group_effect* g = m.group) {
    const b2_glm_group_slope icpt = {g->a_off, g->s_off, 0, g->noncentred, g->s_prior, g->s_const, g->sp0, g->sp1};
    for (int k = -1; k < g->S; ++k) {        // the intercept, then each slope
      const b2_glm_group_slope& b = k < 0 ? icpt : g->slope[k];
      if (b.noncentred != 0 && b.noncentred != 1) return B2_ERR_BAD_SHAPE;
      if (!positive_scale_ok(b.s_off, b.s_prior, b.sp0, b.sp1, b.s_const)) return B2_ERR_BAD_SHAPE;
      if (k >= 0 && (b.col < 0 || b.col >= m.D)) return B2_ERR_BAD_SHAPE;
      for (int j = 0; j < k; ++j)
        if (g->slope[j].col == b.col) return B2_ERR_BAD_SHAPE;
      off[nblk] = b.b_off, len[nblk++] = g->G;
      off[nblk] = b.s_off, len[nblk++] = b.s_off >= 0 ? 1 : 0;
    }
    if (misaligned(g->groups)) return B2_ERR_BAD_SHAPE;
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
  // Bernoulli, softmax and Poisson with a constant weight scale and no group effect leave X and y to their
  // likelihood call (the SIMT Bernoulli kernel needs neither aligned)
  if ((m.scale || m.group || normal || binomial) && (misaligned(m.X) || misaligned(m.y))) return B2_ERR_BAD_SHAPE;
  if (binomial && m.trials_per_row && misaligned(m.trials)) return B2_ERR_BAD_SHAPE;
  return 0;
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_glm_potential_workspace(const b2_glm_regression* m, int64_t C) {
  if (!m || !glm_regression_in_scope(*m, C)) return 256;
  return glm_potential_layout(*m, C).total;
}

extern "C" int b2_glm_potential(const b2_glm_regression* mp, const float* z, int64_t C, int64_t Dz, float* U,
                                float* grad, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = glm_potential_check(mp, z, C, Dz, U, grad);
  if (rc != 0) return rc;
  const b2_glm_regression& m = *mp;
  const GlmPotentialLayout L = glm_potential_layout(m, C);
  if (!workspace || workspace_bytes < L.total) return B2_ERR_WORKSPACE;
  const bool normal = m.kind == B2_GLM_NORMAL, gathered = glm_gathered(m);
  const int KD = m.K * m.D + (gathered ? 0 : glm_group_cols(m)), Kb = m.has_bias ? m.K : 0;
  char* ws = reinterpret_cast<char*>(workspace);
  float* Wp = reinterpret_cast<float*>(ws + L.wp);
  float* bp = m.has_bias ? reinterpret_cast<float*>(ws + L.bp) : nullptr;
  float* dW = reinterpret_cast<float*>(ws + L.dw);
  float* db = m.has_bias ? reinterpret_cast<float*>(ws + L.db) : nullptr;
  float* sum_p = reinterpret_cast<float*>(ws + L.sum_p);
  float* sig = normal ? reinterpret_cast<float*>(ws + L.sig) : nullptr;
  float* dsig = normal && m.s_off >= 0 ? reinterpret_cast<float*>(ws + L.dsig) : nullptr;
  const b2_glm_weight_scale no_scale = {-1, -1, 0, 0, 0.0, 0.0, 0.0, 0.0};
  const b2_glm_group_effect no_group = {};
  const b2_glm_group_effect& ge = m.group ? *m.group : no_group;
  GlmGroups grp;
  if (m.group) {
    grp.idx = ge.groups;
    grp.G = ge.G;
    grp.S = ge.S;
    for (int k = 0; k < ge.S; ++k) grp.col[k] = ge.slope[k].col;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  if (gathered) {
    GlmGather ga;
    ga.idx = ge.groups;
    ga.G = ge.G;
    ga.S = ge.S;
    for (int k = 0; k < ge.S; ++k) ga.col[k] = ge.slope[k].col;
    ga.cp = L.cp;
    float* tab = reinterpret_cast<float*>(ws + L.tab);
    ga.tab = tab;
    ga.gsum = reinterpret_cast<float*>(ws + L.gsum);
    ga.slots = reinterpret_cast<float*>(ws + L.slots);
    ga.status = reinterpret_cast<int*>(ws + L.status);
    const int64_t npack = C * (KD + Kb) + (int64_t)(1 + ge.S) * ge.G * L.cp;
    glm_potential_gather_pack_kernel<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(
        z, C, Dz, m.w_off, m.b_off, KD, Kb, Wp, bp, m.s_off, (float)m.sigma, sig, ge, L.cp, tab, ga.gsum);
    count_launch(1);
    rc = check_launch();
    if (rc != 0) return rc;
    // the flags and noise-scale arguments of the kind's own likelihood call (glm_potential_likelihood)
    rc = glm_gather_likelihood(m.kind, m.X, static_cast<const float*>(m.y), Wp, bp, sig, 1, dsig, m.N, m.D, (int)C,
                               1.0, -1.0, 1.0, normal ? 0 : B2_FLAG_GLM_3XTF32, sum_p, nullptr, dW, db, ws, s, ga);
    if (rc != 0) return rc;
    const GlmGatherFinish gf = {ga.gsum, ga.slots, ga.status, ge.groups, L.cp, L.Q, m.N};
    glm_potential_gather_finish_kernel<<<(unsigned)((C * 32 + 255) / 256), 256, 0, s>>>(
        z, C, Dz, m.w_off, m.b_off, KD, Kb, m.s_w, m.s_b, sum_p, dW, db, U, grad, sig, dsig, m.s_off, m.s_prior, m.sp0,
        m.sp1, ge, gf);
    count_launch(1);
    return check_launch();
  }

  const int64_t npack = C * (KD + Kb);
  const auto pack = m.group ? glm_potential_pack_kernel<true> : glm_potential_pack_kernel<false>;
  pack<<<(unsigned)((npack + 255) / 256), 256, 0, s>>>(z, C, Dz, m.w_off, m.b_off, KD, Kb, Wp, bp, m.s_off,
                                                       (float)m.sigma, sig, ge);
  count_launch(1);
  rc = check_launch();
  if (rc != 0) return rc;
  rc = glm_potential_likelihood(m, C, Wp, bp, sig, dsig, sum_p, dW, db, ws, L.wp, stream, grp);
  if (rc != 0) return rc;
  const auto finish = m.group   ? glm_potential_finish_kernel<false, true>
                      : m.scale ? glm_potential_finish_kernel<true, false>
                                : glm_potential_finish_kernel<false, false>;
  finish<<<(unsigned)((C * 32 + 255) / 256), 256, 0, s>>>(
      z, C, Dz, m.w_off, m.b_off, KD, Kb, m.s_w, m.s_b, sum_p, dW, db, U, grad, sig, dsig, m.s_off, m.s_prior, m.sp0,
      m.sp1, m.scale ? *m.scale : no_scale, ge);
  count_launch(1);
  return check_launch();
}
