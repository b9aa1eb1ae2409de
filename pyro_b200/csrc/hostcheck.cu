// hostcheck.cu -- TEST INFRASTRUCTURE ONLY.  Builds the __host__ __device__ element functors
// of b2_math.cuh (and the NUTS tree logic of nuts_core.cuh) for the CPU so tests can pin the
// arithmetic against the oracle without a GPU.  It is a separate shared object
// (libpyro_b200_hostcheck.so); nothing in the product path loads it.
#include <stdint.h>

#include "b2_math.cuh"

using namespace b2;

namespace {
template <typename T>
int eval_t(int family, int grad, int64_t n, const T* x, const T* const* p, T* lp, T* dx,
           T* const* dp) {
  for (int64_t i = 0; i < n; ++i) {
    ElemOut<T> o;
    T pl[4] = {p[0] ? p[0][i] : (T)0, p[1] ? p[1][i] : (T)0, p[2] ? p[2][i] : (T)0,
               p[3] ? p[3][i] : (T)0};
    const T xv = x ? x[i] : (T)0;
#define B2H_CASE(F)                                   \
  case F:                                             \
    if (grad) Eval<F, T, true>::run(xv, pl, o);       \
    else Eval<F, T, false>::run(xv, pl, o);           \
    break;
    switch (family) {
      B2H_CASE(kNormal)
      B2H_CASE(kBernoulliLogits)
      B2H_CASE(kGamma)
      B2H_CASE(kBeta)
      B2H_CASE(kPoisson)
      B2H_CASE(kCauchy)
      B2H_CASE(kHalfCauchy)
      B2H_CASE(kExponential)
      B2H_CASE(kLogNormal)
      B2H_CASE(kHalfNormal)
      B2H_CASE(kBernoulliProbs)
      B2H_CASE(kUniform)
      B2H_CASE(kKLNormalNormal)
      B2H_CASE(kKLGammaGamma)
      B2H_CASE(kNormalRsample)
      B2H_CASE(kNormalRsampleBwd)
      B2H_CASE(kBinomialLogits)
      B2H_CASE(kBinomialProbs)
      default:
        return -3;
    }
#undef B2H_CASE
    lp[i] = o.lp;
    if (grad) {
      if (dx) dx[i] = o.dx;
      for (int k = 0; k < 4; ++k)
        if (dp[k]) dp[k][i] = o.dp[k];
    }
  }
  return 0;
}
}  // namespace

extern "C" int b2h_eval_f32(int family, int grad, int64_t n, const float* x, const float* const* p,
                            float* lp, float* dx, float* const* dp) {
  return eval_t<float>(family, grad, n, x, p, lp, dx, dp);
}
extern "C" int b2h_eval_f64(int family, int grad, int64_t n, const double* x,
                            const double* const* p, double* lp, double* dx, double* const* dp) {
  return eval_t<double>(family, grad, n, x, p, lp, dx, dp);
}
extern "C" double b2h_digamma(double x) { return digamma<double>(x); }
extern "C" float b2h_digammaf(float x) { return digamma<float>(x); }
extern "C" double b2h_trigamma(double x) { return trigamma<double>(x); }

// ---- Gamma sampler + implicit-reparameterisation gradient on the host ---------------------------------
#include "gamma_sample.cuh"
extern "C" double b2h_standard_gamma_grad(double a, double x) { return standard_gamma_grad<double>(a, x); }
extern "C" float b2h_standard_gamma_gradf(float a, float x) { return standard_gamma_grad<float>(a, x); }
extern "C" void b2h_standard_gamma_sample(uint64_t seed, int64_t n, double a, double* out) {
  for (int64_t i = 0; i < n; ++i) {
    Philox r;
    r.init(seed, (uint64_t)i, 0);
    out[i] = standard_gamma_sample<double>(a, r);
  }
}
extern "C" void b2h_standard_gamma_samplef(uint64_t seed, int64_t n, float a, float* out) {
  for (int64_t i = 0; i < n; ++i) {
    Philox r;
    r.init(seed, (uint64_t)i, 0);
    out[i] = standard_gamma_sample<float>(a, r);
  }
}

// ---- NUTS core on the host (same code path as nuts_small_kernel, one chain at a time) ----------
#include "nuts_core.cuh"

namespace {
template <typename Model>
int run_nuts_host(const Model& model, int D, int64_t C, double* z, double* U, double* g,
                  const double* eps, const double* minv, int T, int max_depth, double max_delta,
                  uint64_t seed, double* samples, double* acc, int32_t* depth, int32_t* div,
                  int32_t* steps) {
  if (D > 64) return -8;
  for (int64_t c = 0; c < C; ++c) {
    double zl[64], gl[64], sm[64];
    for (int d = 0; d < D; ++d) {
      zl[d] = z[c * D + d];
      gl[d] = g[c * D + d];
      sm[d] = sqrt(minv[c * D + d]);
    }
    double Ul = U[c];
    Philox rng;
    rng.init(seed, (uint64_t)c, 0);
    for (int t = 0; t < T; ++t) {
      NutsStats st;
      nuts_transition<double, Model, 64>(model, D, zl, gl, Ul, eps[c], sm, max_depth, max_delta, rng, st);
      const int64_t o = (int64_t)t * C + c;
      if (samples) for (int d = 0; d < D; ++d) samples[o * D + d] = zl[d];
      if (acc) acc[o] = st.accept_prob;
      if (depth) depth[o] = st.depth;
      if (div) div[o] = st.diverging;
      if (steps) steps[o] = st.num_steps;
    }
    for (int d = 0; d < D; ++d) { z[c * D + d] = zl[d]; g[c * D + d] = gl[d]; }
    U[c] = Ul;
  }
  return 0;
}
}  // namespace

extern "C" double b2h_potential_hier_normal(const double* y, const double* sigma, int64_t J,
                                            double s_mu, double s_tau, const double* z, double* g) {
  HierNormalModel<double> m{y, sigma, J, s_mu, s_tau};
  return m.value_and_grad(z, g);
}
extern "C" double b2h_potential_logistic(const double* X, const double* y, int64_t N, int D,
                                         double s, const double* z, double* g) {
  LogisticModel<double> m{X, y, N, D, s};
  return m.value_and_grad(z, g);
}
extern "C" int b2h_nuts_hier_normal(const double* y, const double* sigma, int64_t J, double s_mu,
                                    double s_tau, int64_t C, double* z, double* U, double* g,
                                    const double* eps, const double* minv, int T, int max_depth,
                                    double max_delta, uint64_t seed, double* samples, double* acc,
                                    int32_t* depth, int32_t* div, int32_t* steps) {
  HierNormalModel<double> m{y, sigma, J, s_mu, s_tau};
  return run_nuts_host(m, (int)(J + 2), C, z, U, g, eps, minv, T, max_depth, max_delta, seed,
                       samples, acc, depth, div, steps);
}
extern "C" int b2h_nuts_logistic(const double* X, const double* y, int64_t N, int D, double s,
                                 int64_t C, double* z, double* U, double* g, const double* eps,
                                 const double* minv, int T, int max_depth, double max_delta,
                                 uint64_t seed, double* samples, double* acc, int32_t* depth,
                                 int32_t* div, int32_t* steps) {
  LogisticModel<double> m{X, y, N, D, s};
  return run_nuts_host(m, D, C, z, U, g, eps, minv, T, max_depth, max_delta, seed, samples, acc,
                       depth, div, steps);
}
extern "C" void b2h_philox(uint64_t seed, uint64_t stream, uint64_t counter, int n, uint32_t* out) {
  Philox r;
  r.init(seed, stream, counter);
  for (int i = 0; i < n; ++i) out[i] = r.next_u32();
}

#include "latent.cuh"
// 1 when b2_latent_normal_backward reduces the job's d/dloc and d/dscale in one pass, 0 when in two, or the
// B2_ERR code with which it rejects the job
extern "C" int b2h_latent_same_reduction(const b2_latent_job* job) {
  LatentJob j;
  const int code = fill_job(j, *job, job->dtype);
  if (code != B2_OK) return code;
  return latent_same_reduction(j) ? 1 : 0;
}
