// b2_math.cuh -- per-element densities and their partial derivatives.
//
// Everything here is __host__ __device__ so the SAME code is exercised on the CPU by the
// test-only host harness (hostcheck.cu, used by tests/ to pin the arithmetic against the
// oracle before any GPU time is spent) and on the device by the fused kernels.
//
// The formulas restate torch.distributions (the arithmetic reference Pyro delegates to through
// pyro/distributions/torch.py:23-257); operation order follows the cited torch source so fp32
// results agree with the reference to rounding.  SURVEY.md Appendix A lists the originals.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#else
#define B2_HD inline
#endif

namespace b2 {

template <typename T>
struct Consts;
template <>
struct Consts<float> {
  static constexpr float kLogSqrt2Pi = 0.91893853320467274178f;  // log(sqrt(2*pi))
  static constexpr float kLogPi = 1.14472988584940017414f;
  static constexpr float kLog2 = 0.69314718055994530942f;
  static constexpr float kHalfLog2OverPi = -0.22579135264472743236f;  // 0.5*log(2/pi)
  static constexpr float kPi = 3.14159265358979323846f;
};
template <>
struct Consts<double> {
  static constexpr double kLogSqrt2Pi = 0.91893853320467274178;
  static constexpr double kLogPi = 1.14472988584940017414;
  static constexpr double kLog2 = 0.69314718055994530942;
  static constexpr double kHalfLog2OverPi = -0.22579135264472743236;
  static constexpr double kPi = 3.14159265358979323846;
};

// ---- thin overload set so templates pick the right libm / CUDA math entry ------------------
B2_HD float b2_log(float x) { return logf(x); }
B2_HD double b2_log(double x) { return log(x); }
B2_HD float b2_exp(float x) { return expf(x); }
B2_HD double b2_exp(double x) { return exp(x); }
B2_HD float b2_log1p(float x) { return log1pf(x); }
B2_HD double b2_log1p(double x) { return log1p(x); }
B2_HD float b2_sqrt(float x) { return sqrtf(x); }
B2_HD double b2_sqrt(double x) { return sqrt(x); }
B2_HD float b2_lgamma(float x) { return lgammaf(x); }
B2_HD double b2_lgamma(double x) { return lgamma(x); }
B2_HD float b2_abs(float x) { return fabsf(x); }
B2_HD double b2_abs(double x) { return fabs(x); }
B2_HD float b2_floor(float x) { return floorf(x); }
B2_HD double b2_floor(double x) { return floor(x); }
B2_HD float b2_tan(float x) { return tanf(x); }
B2_HD double b2_tan(double x) { return tan(x); }
B2_HD float b2_max(float a, float b) { return fmaxf(a, b); }
B2_HD double b2_max(double a, double b) { return fmax(a, b); }
B2_HD float b2_min(float a, float b) { return fminf(a, b); }
B2_HD double b2_min(double a, double b) { return fmin(a, b); }

template <typename T>
B2_HD T b2_inf() {
  return (T)INFINITY;
}
template <typename T>
B2_HD T b2_nan() {
  return (T)NAN;
}

// xlogy(x, y) = x*log(y) with 0 where x == 0 (and NaN propagation from y), as
// torch.xlogy (used by gamma.py:94-95, dirichlet.py:93, poisson.py:79).
template <typename T>
B2_HD T xlogy(T x, T y) {
  if (y != y) return y;
  if (x == (T)0) return (T)0;
  return x * b2_log(y);
}

// digamma(x).  Positive arguments: upward recurrence to x >= 6 (fp32) / 12 (fp64) followed by the asymptotic
// expansion  psi(x) ~ ln x - 1/(2x) - sum_k B_2k / (2k x^2k).  Non-positive arguments use the
// reflection formula; poles return -inf at 0 (torch convention) and NaN at negative integers.
template <typename T>
B2_HD T digamma(T x) {
  if (x != x) return x;
  T reflect = (T)0;
  if (x <= (T)0) {
    if (x == (T)0) return -b2_inf<T>();
    if (x == b2_floor(x)) return b2_nan<T>();
    // psi(1-x) - psi(x) = pi / tan(pi x)
    T frac = x - b2_floor(x);
    reflect = -Consts<T>::kPi / b2_tan(Consts<T>::kPi * frac);
    x = (T)1 - x;
  }
  T acc = (T)0;
  const T shift = sizeof(T) == 8 ? (T)12 : (T)6;  // series error ~ x^-16
  while (x < shift) {
    acc -= (T)1 / x;
    x += (T)1;
  }
  const T inv = (T)1 / x;
  const T inv2 = inv * inv;
  // Bernoulli-number coefficients B_2k/(2k): 1/12, -1/120, 1/252, -1/240, 1/132, -691/32760, 1/12
  T series = inv2 * ((T)(1.0 / 12.0) -
             inv2 * ((T)(1.0 / 120.0) -
             inv2 * ((T)(1.0 / 252.0) -
             inv2 * ((T)(1.0 / 240.0) -
             inv2 * ((T)(1.0 / 132.0) -
             inv2 * ((T)(691.0 / 32760.0) - inv2 * (T)(1.0 / 12.0)))))));
  return acc + b2_log(x) - (T)0.5 * inv - series + reflect;
}

// ---- fp32 device fast paths -------------------------------------------------------------------
// On the device, fp32 kernels use the SFU approximations (MUFU.EX2 / LG2 / RCP: ~2 ulp) instead
// of the libm-accurate expf / log1pf / IEEE division, whose ~50 instructions per element made the
// HBM-bound kernels issue-bound.  Absolute error of each result stays below 4e-7, inside the stated fp32 tolerance
// |d| <= 1e-5 * max(1, |lp|).  fp64 and the host build keep the accurate functions.
B2_HD float fast_exp(float x) {
#ifdef __CUDA_ARCH__
  return __expf(x);
#else
  return expf(x);
#endif
}
B2_HD double fast_exp(double x) { return exp(x); }
B2_HD float fast_log(float x) {
#ifdef __CUDA_ARCH__
  return __logf(x);
#else
  return logf(x);
#endif
}
B2_HD double fast_log(double x) { return log(x); }
// log(x) for x known to be a NORMAL positive number (>= 2^-126): bare MUFU.LG2 + FMUL.  __logf spends four
// more instructions per call on rescuing denormal arguments.
B2_HD float fast_log_normal(float x) {
#ifdef __CUDA_ARCH__
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r * 0.69314718055994530942f;
#else
  return logf(x);
#endif
}
B2_HD double fast_log_normal(double x) { return log(x); }
B2_HD float fast_rcp(float x) {
#ifdef __CUDA_ARCH__
  float r;  // MUFU.RCP (1 ulp); __frcp_rn would add a Newton step and a denormal slow path
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return 1.0f / x;
#endif
}
B2_HD double fast_rcp(double x) { return 1.0 / x; }
// log(1 + e) for e in [0, 1]
B2_HD float fast_log1p_unit(float e) {
#ifdef __CUDA_ARCH__
  return __logf(1.0f + e);
#else
  return log1pf(e);
#endif
}
B2_HD double fast_log1p_unit(double e) { return log1p(e); }

// lgamma(x), digamma(x) (and trigamma(x)) for fp32, x > 0: ONE upward shift by 4 when x < 4, then the
// Stirling / asymptotic series at x >= 4 (truncation below 7e-8 there).  The shift is closed form:
//   p = x(x+3),  (x)(x+1)(x+2)(x+3) = p(p+2),   sum_{i<4} 1/(x+i) = (2x+3)(2p+2) / (p(p+2))
// so lgamma + digamma cost two logs and two reciprocals in total (libm's lgammaf alone is ~100
// instructions and made the Gamma/Beta/Poisson kernels issue-bound; a per-unit shift loop to x >= 8
// costs more instructions than the closed form).  Absolute error ~1e-6 for lgamma, relative ~1e-6 for digamma / trigamma: inside the fp32
// tolerance.  Non-positive arguments (never produced by valid parameters) take the accurate route.
// The accurate route is OUT OF LINE on purpose: inlined into the 16-element unrolled loop bodies of the vector
// kernels it made them 6-18 k instructions (Beta: 259 KB of SASS, far beyond the instruction cache) although it
// never executes for valid parameters.
#if defined(__CUDACC__)
#define B2_COLD static __host__ __device__ __noinline__
#else
#define B2_COLD static __attribute__((noinline))
#endif
B2_COLD void lgamma_polygamma_slow(float x, int want, float* out) {
  out[0] = lgammaf(x);
  if (want & 1) out[1] = digamma<float>(x);
  if (want & 2) out[2] = x - x == 0.f ? 1.f / (x * x) : x;  // invalid concentration: inf / NaN
}
template <bool WANT_PSI, bool WANT_TRI>
B2_HD void lgamma_polygamma_f32(float x, float& lg, float& psi, float& tri) {
  // the fast route is evaluated unconditionally (garbage, but no trap, for arguments outside its domain) and
  // overwritten by the accurate one afterwards: the rare branch then only skips a call instead of fencing the
  // whole series, which lets the compiler interleave the elements of an unrolled loop
  const bool slow = !(x > 1e-30f) || x > 1e30f;
  const float xin = x;
  const bool shift = x < 4.f;
  const float p = x * (x + 3.f);
  const float prod = shift ? p * (p + 2.f) : 1.f;   // in [6e-30, 840]: a normal number
  float acc2 = 0.f;
  if (WANT_TRI) {
    if (shift) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float r = fast_rcp(x + (float)i);
        acc2 += r * r;
      }
    }
  }
  const float x0 = x;
  x = shift ? x + 4.f : x;
  const float lx = fast_log_normal(x);
  float inv, acc = 0.f;
  if (WANT_PSI) {
    // 1/x and 1/prod from ONE reciprocal (x*prod stays inside [2e-29, 1e30])
    const float r = fast_rcp(x * prod);
    inv = r * prod;
    acc = shift ? -(2.f * x0 + 3.f) * (2.f * p + 2.f) * (r * x) : 0.f;
  } else {
    inv = fast_rcp(x);
  }
  const float inv2 = inv * inv;
  // Stirling: (x - 1/2) ln x - x + ln sqrt(2 pi) + 1/(12x) - 1/(360 x^3) + 1/(1260 x^5)
  lg = (x - 0.5f) * lx - x + 0.91893853320467274178f +
       inv * (0.083333333333333333f - inv2 * (0.0027777777777777778f - inv2 * 0.00079365079365079365f)) -
       fast_log_normal(prod);
  if (WANT_PSI) {
    // psi(x) ~ ln x - 1/(2x) - 1/(12x^2) + 1/(120x^4) - 1/(252x^6)
    psi = acc + lx - 0.5f * inv -
          inv2 * (0.083333333333333333f - inv2 * (0.0083333333333333333f - inv2 * 0.0039682539682539683f));
  }
  if (WANT_TRI) {
    // psi'(x) ~ 1/x + 1/(2x^2) + 1/(6x^3) - 1/(30x^5) + 1/(42x^7)
    tri = acc2 + inv + 0.5f * inv2 +
          inv * inv2 * (0.16666666666666667f - inv2 * (0.033333333333333333f - inv2 * 0.023809523809523810f));
  }
  if (slow) {
    float out[3];
    lgamma_polygamma_slow(xin, (WANT_PSI ? 1 : 0) | (WANT_TRI ? 2 : 0), out);
    lg = out[0];
    if (WANT_PSI) psi = out[1];
    if (WANT_TRI) tri = out[2];
  }
}

B2_COLD void lbeta_terms_slow(float c1, float c0, bool want_psi, float* out) {
  float lg[3], ps[3] = {0.f, 0.f, 0.f}, t;
  const float xs[3] = {c1 + c0, c1, c0};
  for (int i = 0; i < 3; ++i) {
    if (want_psi) lgamma_polygamma_f32<true, false>(xs[i], lg[i], ps[i], t);
    else lgamma_polygamma_f32<false, false>(xs[i], lg[i], ps[i], t);
  }
  out[0] = lg[0] - (lg[1] + lg[2]);
  out[1] = ps[0];
  out[2] = ps[1];
  out[3] = ps[2];
}

// log B-function pieces for Beta(c1, c0) in fp32: lsum = lgamma(c1 + c0) - lgamma(c1) - lgamma(c0) and, with
// WANT_PSI, the three digammas -- evaluated TOGETHER so that the special-function unit is used 5 times instead
// of 9 (value) / 12 (gradients): every reciprocal the three Stirling series and the three shift terms need comes
// out of ONE MUFU.RCP of their product (recovered with prefix/suffix multiplications on the FMA pipe), and the
// three shift products enter through one logarithm of their ratio.  Same series, same accuracy as three calls of
// lgamma_polygamma_f32 (absolute ~1e-6).  Outside 1e-6 < c < 1e9 the per-argument route above is taken.
template <bool WANT_PSI>
B2_HD void lbeta_terms_f32(float c1, float c0, float& lsum, float& psi_s, float& psi_1, float& psi_0) {
  const float cs = c1 + c0;
  const bool fast = (c1 > 1e-6f) && (c0 > 1e-6f) && (cs < 1e9f);
  if (!fast) {
    float out[4];
    lbeta_terms_slow(c1, c0, WANT_PSI, out);
    lsum = out[0];
    if (WANT_PSI) {
      psi_s = out[1];
      psi_1 = out[2];
      psi_0 = out[3];
    }
    return;
  }
  const float xs[3] = {cs, c1, c0};
  float xp[3], pr[3], pp[3];
  bool sh[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    sh[i] = xs[i] < 4.f;
    pp[i] = xs[i] * (xs[i] + 3.f);
    pr[i] = sh[i] ? pp[i] * (pp[i] + 2.f) : 1.f;
    xp[i] = sh[i] ? xs[i] + 4.f : xs[i];
  }
  float inv[3], ipr[3] = {0.f, 0.f, 0.f}, ratio;
  if (WANT_PSI) {
    // six reciprocals from one: factors xp[0..2], pr[1], pr[2], pr[0]
    const float f0 = xp[0], f1 = xp[1], f2 = xp[2], f3 = pr[1], f4 = pr[2], f5 = pr[0];
    const float p1 = f0 * f1, p2 = p1 * f2, p3 = p2 * f3, p4 = p3 * f4;
    const float r = fast_rcp(p4 * f5);
    const float s4 = f4 * f5, s3 = f3 * s4, s2 = f2 * s3, s1 = f1 * s2;
    inv[0] = r * s1;
    inv[1] = r * f0 * s2;
    inv[2] = r * p1 * s3;
    ipr[1] = r * p2 * s4;
    ipr[2] = r * p3 * f5;
    ipr[0] = r * p4;
    ratio = pr[0] * ipr[1] * ipr[2];
  } else {
    const float d = pr[1] * pr[2];
    const float p1 = xp[0] * xp[1], s2 = xp[2] * d;
    const float r = fast_rcp(p1 * s2);
    const float rs = r * s2, rp = r * p1;
    inv[0] = rs * xp[1];
    inv[1] = rs * xp[0];
    inv[2] = rp * d;
    ratio = pr[0] * (rp * xp[2]);
  }
  float L[3], st[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    L[i] = fast_log_normal(xp[i]);
    const float i2 = inv[i] * inv[i];
    st[i] = (xp[i] - 0.5f) * L[i] - xp[i] +
            inv[i] * (0.083333333333333333f - i2 * (0.0027777777777777778f - i2 * 0.00079365079365079365f));
    if (WANT_PSI) {
      const float a = sh[i] ? -(2.f * xs[i] + 3.f) * (2.f * pp[i] + 2.f) * ipr[i] : 0.f;
      const float ps = a + L[i] - 0.5f * inv[i] -
                       i2 * (0.083333333333333333f - i2 * (0.0083333333333333333f - i2 * 0.0039682539682539683f));
      if (i == 0) psi_s = ps;
      if (i == 1) psi_1 = ps;
      if (i == 2) psi_0 = ps;
    }
  }
  // lgamma_i = st_i + ln sqrt(2 pi) - ln prod_i
  lsum = (st[0] - (st[1] + st[2])) - 0.91893853320467274178f - fast_log_normal(ratio);
}

template <bool WANT_PSI>
B2_HD void lgamma_digamma_f32(float x, float& lg, float& psi) {
  float tri;
  lgamma_polygamma_f32<WANT_PSI, false>(x, lg, psi, tri);
}
template <typename T, bool WANT_PSI>
B2_HD void lgamma_digamma(T x, T& lg, T& psi) {
  if (sizeof(T) == 4) {
    float l, p = 0.f;
    lgamma_digamma_f32<WANT_PSI>((float)x, l, p);
    lg = (T)l;
    psi = (T)p;
  } else {
    lg = b2_lgamma(x);
    if (WANT_PSI) psi = digamma(x);
  }
}

// softplus(l) = log(1 + exp(l)) and sigmoid(l), sharing one exp.
template <typename T>
B2_HD void softplus_sigmoid(T l, T& sp, T& sg) {
  const T e = fast_exp(-b2_abs(l));  // in (0, 1]
  const T inv = fast_rcp((T)1 + e);
  sp = b2_max(l, (T)0) + fast_log1p_unit(e);
  sg = (l >= (T)0) ? inv : e * inv;
}

// Result of one element: log density and partials w.r.t. value and up to four parameters.
template <typename T>
struct ElemOut {
  T lp, dx, dp[4];
  // set by the kernel before Eval::run: false when nobody reads dx (observed sites) -- families whose value
  // derivative costs extra special-function work skip it (dx is then 0)
  bool want_dx = true;
};

enum : int {
  kNormal = 0,
  kBernoulliLogits = 1,
  kGamma = 2,
  kBeta = 3,
  kPoisson = 4,
  kCauchy = 5,
  kHalfCauchy = 6,
  kExponential = 7,
  kLogNormal = 8,
  kHalfNormal = 9,
  kBernoulliProbs = 10,
  kUniform = 11,
  kKLNormalNormal = 12,
  kKLGammaGamma = 13,
  kNormalRsample = 14,     // reparameterised draw + its own log density (guide sites)
  kNormalRsampleBwd = 15,  // chain rule of that draw back to (loc, scale)
  kBinomialLogits = 16,
  kBinomialProbs = 17,
  kNumElementwise = 18
};

template <int FAM>
struct FamilyTraits;
#define B2_TRAITS(F, NP, HASV) \
  template <>                  \
  struct FamilyTraits<F> {     \
    static constexpr int kNumParams = NP; \
    static constexpr bool kHasValue = HASV; \
  };
B2_TRAITS(kNormal, 2, true)
B2_TRAITS(kBernoulliLogits, 1, true)
B2_TRAITS(kGamma, 2, true)
B2_TRAITS(kBeta, 2, true)
B2_TRAITS(kPoisson, 1, true)
B2_TRAITS(kCauchy, 2, true)
B2_TRAITS(kHalfCauchy, 1, true)
B2_TRAITS(kExponential, 1, true)
B2_TRAITS(kLogNormal, 2, true)
B2_TRAITS(kHalfNormal, 1, true)
B2_TRAITS(kBernoulliProbs, 1, true)
B2_TRAITS(kUniform, 2, true)
B2_TRAITS(kKLNormalNormal, 4, false)
B2_TRAITS(kKLGammaGamma, 4, false)
B2_TRAITS(kNormalRsample, 2, true)
B2_TRAITS(kNormalRsampleBwd, 3, true)
B2_TRAITS(kBinomialLogits, 2, true)
B2_TRAITS(kBinomialProbs, 2, true)
#undef B2_TRAITS

// eval<FAM, T, GRAD>(x, p, out): p[k] are the parameters in the order pyro_b200.h documents.
// With GRAD == false only out.lp is defined.
template <int FAM, typename T, bool GRAD>
struct Eval;

// Normal(loc, scale): torch/distributions/normal.py:87-102
//   -((x - loc)^2) / (2 var) - log(scale) - log(sqrt(2 pi)),  var = scale^2
template <typename T, bool GRAD>
struct Eval<kNormal, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T loc = p[0], scale = p[1];
    const T d = x - loc;
    if (sizeof(T) == 4) {
      // fp32: one reciprocal + one SFU log instead of two IEEE divisions and logf
      const T inv_s = fast_rcp(scale);
      const T u = d * inv_s;
      o.lp = (T)-0.5 * u * u - fast_log(scale) - Consts<T>::kLogSqrt2Pi;
      if (GRAD) {
        const T dloc = u * inv_s;
        o.dx = -dloc;
        o.dp[0] = dloc;
        o.dp[1] = (u * u - (T)1) * inv_s;
      }
    } else {
      const T var = scale * scale;
      o.lp = -(d * d) / ((T)2 * var) - b2_log(scale) - Consts<T>::kLogSqrt2Pi;
      if (GRAD) {
        const T dloc = d / var;
        o.dx = -dloc;
        o.dp[0] = dloc;
        o.dp[1] = (d * d / var - (T)1) / scale;
      }
    }
  }
};

// Bernoulli(logits): torch/distributions/bernoulli.py:121-125 = -BCE_with_logits(l, x)
//   = x*l - softplus(l)
template <typename T, bool GRAD>
struct Eval<kBernoulliLogits, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T l = p[0];
    T sp, sg;
    softplus_sigmoid(l, sp, sg);
    o.lp = x * l - sp;
    if (GRAD) {
      o.dx = l;
      o.dp[0] = x - sg;
    }
  }
};

// Bernoulli(probs): logits = log(p) - log1p(-p) with p clamped to [eps, 1-eps]
// (torch/distributions/utils.py probs_to_logits + clamp_probs), then as above.
template <typename T>
B2_HD T b2_eps();
template <>
B2_HD float b2_eps<float>() { return 1.1920928955078125e-07f; }
template <>
B2_HD double b2_eps<double>() { return 2.220446049250313e-16; }

template <typename T, bool GRAD>
struct Eval<kBernoulliProbs, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T eps = b2_eps<T>();
    const T pr = p[0];
    const bool clamped = (pr < eps) || (pr > (T)1 - eps);
    const T pc = b2_min(b2_max(pr, eps), (T)1 - eps);
    const T l = b2_log(pc) - b2_log1p(-pc);
    T sp, sg;
    softplus_sigmoid(l, sp, sg);
    o.lp = x * l - sp;
    if (GRAD) {
      o.dx = l;
      // d l / d p = 1/(p (1-p)); zero gradient where the clamp is active
      o.dp[0] = clamped ? (T)0 : (x - sg) / (pc * ((T)1 - pc));
    }
  }
};

// Gamma(concentration a, rate b): torch/distributions/gamma.py:89-98
//   xlogy(a, b) + xlogy(a - 1, x) - b*x - lgamma(a)
template <typename T, bool GRAD>
struct Eval<kGamma, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T a = p[0], b = p[1];
    T lga, psia;
    lgamma_digamma<T, GRAD>(a, lga, psia);
    if (sizeof(T) == 4) {
      const T lb = fast_log(b), lx = fast_log(x);
      // xlogy semantics: a zero coefficient contributes 0 even when the log is -inf
      o.lp = ((a == (T)0) ? (T)0 : a * lb) + ((a == (T)1) ? (T)0 : (a - (T)1) * lx) - b * x - lga;
      if (GRAD) {
        o.dx = o.want_dx ? (a - (T)1) * fast_rcp(x) - b : (T)0;
        o.dp[0] = lb + lx - psia;
        o.dp[1] = a * fast_rcp(b) - x;
      }
    } else {
      o.lp = xlogy(a, b) + xlogy(a - (T)1, x) - b * x - lga;
      if (GRAD) {
        o.dx = (a - (T)1) / x - b;
        o.dp[0] = b2_log(b) + b2_log(x) - psia;
        o.dp[1] = a / b - x;
      }
    }
  }
};

// Beta(c1, c0): torch/distributions/beta.py:87-91 -> Dirichlet([c1, c0]).log_prob([x, 1-x])
// dirichlet.py:90-97:  xlogy(c1-1, x) + xlogy(c0-1, 1-x) + lgamma(c1+c0) - lgamma(c1) - lgamma(c0)
template <typename T, bool GRAD>
struct Eval<kBeta, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T c1 = p[0], c0 = p[1];
    const T omx = (T)1 - x;
    if (sizeof(T) == 4) {
      float lsum, psum = 0.f, ps1 = 0.f, ps0 = 0.f;
      lbeta_terms_f32<GRAD>((float)c1, (float)c0, lsum, psum, ps1, ps0);
      const T lx = fast_log(x), l1 = fast_log(omx);
      // xlogy semantics: a zero coefficient contributes 0 even when the log is -inf
      o.lp = (((c1 == (T)1) ? (T)0 : (c1 - (T)1) * lx) + ((c0 == (T)1) ? (T)0 : (c0 - (T)1) * l1)) + (T)lsum;
      if (GRAD) {
        o.dx = o.want_dx ? (c1 - (T)1) * fast_rcp(x) - (c0 - (T)1) * fast_rcp(omx) : (T)0;
        o.dp[0] = lx + (T)(psum - ps1);
        o.dp[1] = l1 + (T)(psum - ps0);
      }
      return;
    }
    T lgs, psum, lg1, ps1, lg0, ps0;
    lgamma_digamma<T, GRAD>(c1 + c0, lgs, psum);
    lgamma_digamma<T, GRAD>(c1, lg1, ps1);
    lgamma_digamma<T, GRAD>(c0, lg0, ps0);
    o.lp = (xlogy(c1 - (T)1, x) + xlogy(c0 - (T)1, omx)) + lgs - (lg1 + lg0);
    if (GRAD) {
      o.dx = (c1 - (T)1) / x - (c0 - (T)1) / omx;
      o.dp[0] = b2_log(x) + psum - ps1;
      o.dp[1] = b2_log(omx) + psum - ps0;
    }
  }
};

// Value-only terms.  Some densities carry a term that depends on the value alone (Poisson's
// lgamma(x + 1)); when the value is shared by many rows of parameters -- observations scored
// against [particles, ...] rates -- the vector kernel evaluates it once per column and reuses it
// for every row.  ValueAux<FAM, T, GRAD>::kHas marks such families; make(x) computes the term,
// Eval::run_aux consumes it.
template <int FAM, typename T, bool GRAD>
struct ValueAux {
  static constexpr bool kHas = false;
  struct type {};
  static B2_HD type make(T) { return type{}; }
};

// log(k!) and digamma(k + 1) for k = 0..63, correctly rounded: Poisson observations are small counts, and a
// cached 512-byte gather replaces the two logarithms, the reciprocal and ~25 FMA-pipe instructions of the
// series per element (the Poisson kernel is otherwise issue-bound).
#if defined(__CUDACC__)
static __device__ const float kLogFactorialF32[64] = {0.0f, 0.0f, 0.693147181f, 1.79175947f, 3.17805383f, 4.78749174f, 6.57925121f, 8.52516136f, 10.6046029f, 12.8018275f, 15.1044126f, 17.5023078f, 19.9872145f, 22.5521639f, 25.1912212f, 27.8992714f, 30.6718601f, 33.5050735f, 36.3954452f, 39.3398842f, 42.3356165f, 45.3801389f, 48.4711814f, 51.6066756f, 54.7847294f, 58.0036052f, 61.2617018f, 64.5575386f, 67.8897431f, 71.257039f, 74.6582363f, 78.0922236f, 81.5579595f, 85.054467f, 88.5808275f, 92.1361756f, 95.7196945f, 99.3306125f, 102.968199f, 106.63176f, 110.32064f, 114.034212f, 117.771881f, 121.533082f, 125.317271f, 129.123934f, 132.952575f, 136.802723f, 140.673924f, 144.565744f, 148.477767f, 152.409593f, 156.360836f, 160.331128f, 164.320112f, 168.327445f, 172.352797f, 176.395848f, 180.456291f, 184.533829f, 188.628173f, 192.739047f, 196.866182f, 201.009316f};
static __device__ const float kDigammaIntF32[64] = {-0.577215665f, 0.422784335f, 0.922784335f, 1.25611767f, 1.50611767f, 1.70611767f, 1.87278434f, 2.01564148f, 2.14064148f, 2.25175259f, 2.35175259f, 2.44266168f, 2.52599501f, 2.60291809f, 2.67434666f, 2.74101333f, 2.80351333f, 2.86233686f, 2.91789241f, 2.97052399f, 3.02052399f, 3.06814304f, 3.11359759f, 3.15707585f, 3.19874251f, 3.23874251f, 3.27720405f, 3.31424109f, 3.34995537f, 3.38443813f, 3.41777147f, 3.45002953f, 3.48127953f, 3.51158256f, 3.54099433f, 3.56956575f, 3.59734353f, 3.62437056f, 3.65068635f, 3.67632737f, 3.70132737f, 3.72571762f, 3.74952714f, 3.77278296f, 3.79551023f, 3.81773245f, 3.83947158f, 3.86074818f, 3.88158151f, 3.90198967f, 3.92198967f, 3.94159752f, 3.96082829f, 3.97969621f, 3.99821473f, 4.01639655f, 4.03425369f, 4.05179755f, 4.06903893f, 4.08598808f, 4.10265475f, 4.11904819f, 4.13517722f, 4.15105024f};
// log(k!) for k = 0..63 in fp64, for the data terms of the GLM kernels (glm_tc_common.cuh): summed over millions of
// rows, the rounding of an fp32 entry repeats on every row with that count and no longer averages out.
static __device__ const double kLogFactorialF64[64] = {0.0, 0.0, 0.693147180559945, 1.7917594692280554, 3.178053830347945, 4.787491742782047, 6.579251212010102, 8.525161361065415, 10.604602902745249, 12.801827480081467, 15.104412573075514, 17.502307845873887, 19.987214495661885, 22.55216385312342, 25.191221182738683, 27.89927138384089, 30.671860106080672, 33.50507345013689, 36.39544520803305, 39.339884187199495, 42.335616460753485, 45.38013889847691, 48.47118135183522, 51.60667556776438, 54.78472939811232, 58.00360522298052, 61.26170176100201, 64.55753862700634, 67.88974313718153, 71.257038967168, 74.65823634883017, 78.0922235533153, 81.55795945611503, 85.05446701758152, 88.58082754219768, 92.1361756036871, 95.7196945421432, 99.33061245478743, 102.96819861451381, 106.63176026064346, 110.32063971475738, 114.03421178146169, 117.77188139974507, 121.53308151543864, 125.3172711493569, 129.12393363912722, 132.95257503561632, 136.80272263732635, 140.67392364823425, 144.5657439463449, 148.47776695177305, 152.40959258449732, 156.3608363030788, 160.3311282166309, 164.32011226319514, 168.32744544842765, 172.35279713916282, 176.39584840699737, 180.45629141754375, 184.53382886144948, 188.62817342367163, 192.7390472878449, 196.86618167288998, 201.00931639928152};
// log(v!) = lgamma(v + 1) in fp64: the table for integer v < 64, Stirling's series from 64 on (the first omitted
// term, 1/(1680 x^7), is below 2e-16 there), CUDA's lgamma for every other v (fractional, negative, huge, NaN).
__device__ __forceinline__ double log_factorial_f64(float v) {
  const int k = __float2int_rz(v);
  if ((unsigned)k < 64u && (float)k == v) return __ldg(&kLogFactorialF64[k]);
  const double x = (double)v + 1.0;
  if (v >= 64.f && v < 1e15f) {
    // 1/x only scales the correction terms (below 1.3e-3 here): a rounded fp32 reciprocal is exact enough
    const double inv = (double)__frcp_rn((float)x), inv2 = inv * inv;
    return (x - 0.5) * log(x) - x + 0.91893853320467274178 +
           inv * (1.0 / 12.0 - inv2 * (1.0 / 360.0 - inv2 * (1.0 / 1260.0)));
  }
  return lgamma(x);
}
#endif

// Poisson(rate): torch/distributions/poisson.py:75-79   xlogy(x, rate) - rate - lgamma(x + 1)
template <typename T, bool GRAD>
struct ValueAux<kPoisson, T, GRAD> {
  static constexpr bool kHas = true;
  struct type {
    T lgx, psx;
  };
  static B2_HD type make(T x) {
    type a;
#ifdef __CUDA_ARCH__
    if (sizeof(T) == 4) {
      const int k = __float2int_rz((float)x);
      if ((unsigned)k < 64u && (float)k == (float)x) {
        a.lgx = (T)__ldg(&kLogFactorialF32[k]);
        a.psx = GRAD ? (T)__ldg(&kDigammaIntF32[k]) : (T)0;
        return a;
      }
    }
#endif
    lgamma_digamma<T, GRAD>(x + (T)1, a.lgx, a.psx);
    return a;
  }
};

template <typename T, bool GRAD>
struct Eval<kPoisson, T, GRAD> {
  using Aux = typename ValueAux<kPoisson, T, GRAD>::type;
  static B2_HD void run_aux(T x, const Aux& ax, const T* p, ElemOut<T>& o) {
    const T rate = p[0];
    if (sizeof(T) == 4) {
      const T lr = fast_log(rate);
      o.lp = ((x == (T)0) ? (T)0 : x * lr) - rate - ax.lgx;
      if (GRAD) {
        o.dx = lr - ax.psx;
        o.dp[0] = x * fast_rcp(rate) - (T)1;
      }
    } else {
      o.lp = xlogy(x, rate) - rate - ax.lgx;
      if (GRAD) {
        o.dx = b2_log(rate) - ax.psx;
        o.dp[0] = x / rate - (T)1;
      }
    }
  }
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    run_aux(x, ValueAux<kPoisson, T, GRAD>::make(x), p, o);
  }
};

// Binomial(total_count n, logits l): pyro/distributions/torch.py:83-101 with log_binomial (pyro/ops/special.py:93-108)
// at tol = 0
//   k*l - n*(max(l, 0) + log1p(e^-|l|)) + lgamma(n + 1) - lgamma(k + 1) - lgamma(n - k + 1)
// The reference evaluates log_binomial under torch.no_grad, so autograd of it gives d/dl = k - n*sigmoid(l),
// d/dn = -softplus(l) and d/dk = l: the lgamma terms carry no gradient, and these are the gradients here too.
// lgamma(v + 1) of an integer count below 64 comes from the table of the Poisson family.
template <typename T>
B2_HD T lfact(T v) {
  return ValueAux<kPoisson, T, false>::make(v).lgx;
}
template <typename T, bool GRAD>
B2_HD void binomial_logits_run(T x, T n, T l, ElemOut<T>& o) {
  T sp, sg;
  softplus_sigmoid(l, sp, sg);
  o.lp = x * l - n * sp + (lfact(n) - lfact(x) - lfact(n - x));
  if (GRAD) {
    o.dx = l;
    o.dp[0] = -sp;
    o.dp[1] = x - n * sg;
  }
}

template <typename T, bool GRAD>
struct Eval<kBinomialLogits, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) { binomial_logits_run<T, GRAD>(x, p[0], p[1], o); }
};

// Binomial(total_count n, probs): logits = log(p) - log1p(-p) with p clamped to [eps, 1-eps] (torch's
// probs_to_logits, as for kBernoulliProbs), then as above; zero probs gradient where the clamp is active
template <typename T, bool GRAD>
struct Eval<kBinomialProbs, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T eps = b2_eps<T>();
    const T pr = p[1];
    const bool clamped = (pr < eps) || (pr > (T)1 - eps);
    const T pc = b2_min(b2_max(pr, eps), (T)1 - eps);
    const T l = b2_log(pc) - b2_log1p(-pc);
    binomial_logits_run<T, GRAD>(x, p[0], l, o);
    if (GRAD) o.dp[1] = clamped ? (T)0 : o.dp[1] / (pc * ((T)1 - pc));
  }
};

// Cauchy(loc, scale): torch/distributions/cauchy.py:81-88
//   -log(pi) - log(scale) - log1p(((x - loc)/scale)^2)
template <typename T, bool GRAD>
struct Eval<kCauchy, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T loc = p[0], scale = p[1];
    if (sizeof(T) == 4) {
      const T inv_s = fast_rcp(scale);
      const T u = (x - loc) * inv_s;
      const T q = (T)1 + u * u;
      o.lp = -Consts<T>::kLogPi - fast_log(scale) - fast_log(q);
      if (GRAD) {
        const T inv_q = fast_rcp(q);
        const T w = (T)2 * u * inv_q * inv_s;
        o.dx = -w;
        o.dp[0] = w;
        o.dp[1] = ((T)1 - (T)2 * inv_q) * inv_s;   // (-1 + 2u^2/(1+u^2)) / s
      }
    } else {
      const T u = (x - loc) / scale;
      const T u2 = u * u;
      o.lp = -Consts<T>::kLogPi - b2_log(scale) - b2_log1p(u2);
      if (GRAD) {
        const T w = (T)2 * u / (((T)1 + u2) * scale);  // d log1p(u^2) / d x
        o.dx = -w;
        o.dp[0] = w;
        o.dp[1] = (-(T)1 + (T)2 * u2 / ((T)1 + u2)) / scale;
      }
    }
  }
};

// HalfCauchy(scale): torch/distributions/half_cauchy.py:73-81
//   Cauchy(0, scale).log_prob(x) + log 2, -inf where x < 0
template <typename T, bool GRAD>
struct Eval<kHalfCauchy, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T scale = p[0];
    const bool out = x < (T)0;
    if (sizeof(T) == 4) {
      const T inv_s = fast_rcp(scale);
      const T u = x * inv_s;
      const T q = (T)1 + u * u;
      const T lp = (-Consts<T>::kLogPi - fast_log(scale) - fast_log(q)) + Consts<T>::kLog2;
      o.lp = out ? -b2_inf<T>() : lp;
      if (GRAD) {
        const T inv_q = fast_rcp(q);
        o.dx = out ? (T)0 : -(T)2 * u * inv_q * inv_s;
        o.dp[0] = out ? (T)0 : ((T)1 - (T)2 * inv_q) * inv_s;
      }
    } else {
      const T u = x / scale;
      const T u2 = u * u;
      const T lp = (-Consts<T>::kLogPi - b2_log(scale) - b2_log1p(u2)) + Consts<T>::kLog2;
      o.lp = out ? -b2_inf<T>() : lp;
      if (GRAD) {
        const T w = (T)2 * u / (((T)1 + u2) * scale);
        o.dx = out ? (T)0 : -w;
        o.dp[0] = out ? (T)0 : (-(T)1 + (T)2 * u2 / ((T)1 + u2)) / scale;
      }
    }
  }
};

// Exponential(rate): rate.log() - rate * x
template <typename T, bool GRAD>
struct Eval<kExponential, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T rate = p[0];
    if (sizeof(T) == 4) {
      o.lp = fast_log(rate) - rate * x;
      if (GRAD) {
        o.dx = -rate;
        o.dp[0] = fast_rcp(rate) - x;
      }
      return;
    }
    o.lp = b2_log(rate) - rate * x;
    if (GRAD) {
      o.dx = -rate;
      o.dp[0] = (T)1 / rate - x;
    }
  }
};

// LogNormal(loc, scale) = TransformedDistribution(Normal, ExpTransform):
//   Normal.log_prob(log x) - log x
template <typename T, bool GRAD>
struct Eval<kLogNormal, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T loc = p[0], scale = p[1];
    if (sizeof(T) == 4) {
      // fp32: SFU log / reciprocal as in the Normal kernel (the IEEE divisions and logf of the generic route
      // below are ~60 instructions per element)
      const T lx = fast_log(x);
      const T d = lx - loc;
      const T inv_s = fast_rcp(scale);
      const T u = d * inv_s;
      o.lp = ((T)-0.5 * u * u - fast_log(scale) - Consts<T>::kLogSqrt2Pi) - lx;
      if (GRAD) {
        const T dloc = u * inv_s;
        o.dx = o.want_dx ? (-dloc - (T)1) * fast_rcp(x) : (T)0;
        o.dp[0] = dloc;
        o.dp[1] = (u * u - (T)1) * inv_s;
      }
      return;
    }
    const T lx = b2_log(x);
    const T var = scale * scale;
    const T d = lx - loc;
    o.lp = (-(d * d) / ((T)2 * var) - b2_log(scale) - Consts<T>::kLogSqrt2Pi) - lx;
    if (GRAD) {
      const T dloc = d / var;
      o.dx = (-dloc - (T)1) / x;
      o.dp[0] = dloc;
      o.dp[1] = (d * d / var - (T)1) / scale;
    }
  }
};

// HalfNormal(scale): Normal(0, scale).log_prob(x) + log 2, -inf where x < 0
template <typename T, bool GRAD>
struct Eval<kHalfNormal, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T scale = p[0];
    const bool out = x < (T)0;
    if (sizeof(T) == 4) {
      const T inv_s = fast_rcp(scale);
      const T u = x * inv_s;
      const T lpf = ((T)-0.5 * u * u - fast_log(scale) - Consts<T>::kLogSqrt2Pi) + Consts<T>::kLog2;
      o.lp = out ? -b2_inf<T>() : lpf;
      if (GRAD) {
        o.dx = out ? (T)0 : -u * inv_s;
        o.dp[0] = out ? (T)0 : (u * u - (T)1) * inv_s;
      }
      return;
    }
    const T var = scale * scale;
    const T lp = (-(x * x) / ((T)2 * var) - b2_log(scale) - Consts<T>::kLogSqrt2Pi) +
                 Consts<T>::kLog2;
    o.lp = out ? -b2_inf<T>() : lp;
    if (GRAD) {
      o.dx = out ? (T)0 : -x / var;
      o.dp[0] = out ? (T)0 : (x * x / var - (T)1) / scale;
    }
  }
};

// Uniform(low, high): torch/distributions/uniform.py  log(lb*ub) - log(high - low)
template <typename T, bool GRAD>
struct Eval<kUniform, T, GRAD> {
  static B2_HD void run(T x, const T* p, ElemOut<T>& o) {
    const T low = p[0], high = p[1];
    const bool in = (low <= x) && (x < high);
    const T w = high - low;
    o.lp = in ? -b2_log(w) : -b2_inf<T>();
    if (GRAD) {
      o.dx = (T)0;
      o.dp[0] = in ? (T)1 / w : (T)0;
      o.dp[1] = in ? -(T)1 / w : (T)0;
    }
  }
};

// KL(Normal p || Normal q): torch/distributions/kl.py:468-471
//   var_ratio = (sp/sq)^2 ; t1 = ((mp - mq)/sq)^2 ; 0.5*(var_ratio + t1 - 1 - log var_ratio)
// "lp" carries the KL value; params = (loc_p, scale_p, loc_q, scale_q).
template <typename T, bool GRAD>
struct Eval<kKLNormalNormal, T, GRAD> {
  static B2_HD void run(T, const T* p, ElemOut<T>& o) {
    const T mp = p[0], sp = p[1], mq = p[2], sq = p[3];
    const T ratio = sp / sq;
    const T var_ratio = ratio * ratio;
    const T dm = (mp - mq) / sq;
    const T t1 = dm * dm;
    o.lp = (T)0.5 * (var_ratio + t1 - (T)1 - b2_log(var_ratio));
    if (GRAD) {
      o.dx = (T)0;
      o.dp[0] = dm / sq;
      o.dp[1] = sp / (sq * sq) - (T)1 / sp;
      o.dp[2] = -dm / sq;
      o.dp[3] = (-var_ratio - t1 + (T)1) / sq;
    }
  }
};

// KL(Gamma p || Gamma q): torch/distributions/kl.py:301-306
//   t1 = aq*log(bp/bq); t2 = lgamma(aq) - lgamma(ap); t3 = (ap-aq)*digamma(ap); t4 = (bq-bp)*ap/bp
// params = (conc_p, rate_p, conc_q, rate_q).  d/d ap needs trigamma.
template <typename T>
B2_HD T trigamma(T x) {
  // positive arguments only (concentrations); recurrence to x >= 6 then asymptotic series
  T acc = (T)0;
  const T shift = sizeof(T) == 8 ? (T)16 : (T)6;
  while (x < shift) {
    acc += (T)1 / (x * x);
    x += (T)1;
  }
  const T inv = (T)1 / x;
  const T inv2 = inv * inv;
  // 1/x + 1/(2x^2) + sum B_2k / x^(2k+1): 1/6, -1/30, 1/42, -1/30, 5/66
  return acc + inv + (T)0.5 * inv2 +
         inv * inv2 * ((T)(1.0 / 6.0) -
         inv2 * ((T)(1.0 / 30.0) -
         inv2 * ((T)(1.0 / 42.0) - inv2 * ((T)(1.0 / 30.0) - inv2 * (T)(5.0 / 66.0)))));
}

template <typename T, bool GRAD>
struct Eval<kKLGammaGamma, T, GRAD> {
  static B2_HD void run(T, const T* p, ElemOut<T>& o) {
    const T ap = p[0], bp = p[1], aq = p[2], bq = p[3];
    if (sizeof(T) == 4) {
      // fp32: shared shift-and-Stirling evaluation of lgamma / digamma / trigamma, SFU log and
      // reciprocal (the libdevice routes made this kernel issue-bound, like Gamma / Beta)
      float lga, psia, tria = 0.f, lgq, psiq = 0.f, unused;
      lgamma_polygamma_f32<true, GRAD>((float)ap, lga, psia, tria);
      lgamma_polygamma_f32<GRAD, false>((float)aq, lgq, psiq, unused);
      const T lratio = fast_log(bp) - fast_log(bq);
      const T inv_bp = fast_rcp(bp);
      o.lp = aq * lratio + ((T)lgq - (T)lga) + (ap - aq) * (T)psia + (bq - bp) * (ap * inv_bp);
      if (GRAD) {
        o.dx = (T)0;
        o.dp[0] = (ap - aq) * (T)tria + (bq - bp) * inv_bp;
        o.dp[1] = (aq - ap * bq * inv_bp) * inv_bp;
        o.dp[2] = lratio + (T)psiq - (T)psia;
        o.dp[3] = ap * inv_bp - aq * fast_rcp(bq);
      }
      return;
    }
    const T t1 = aq * b2_log(bp / bq);
    const T t2 = b2_lgamma(aq) - b2_lgamma(ap);
    const T psi = digamma(ap);
    const T t3 = (ap - aq) * psi;
    const T t4 = (bq - bp) * (ap / bp);
    o.lp = t1 + t2 + t3 + t4;
    if (GRAD) {
      o.dx = (T)0;
      o.dp[0] = (ap - aq) * trigamma(ap) + (bq - bp) / bp;  // -psi + psi cancel
      o.dp[1] = aq / bp - ap * bq / (bp * bp);
      o.dp[2] = b2_log(bp / bq) + digamma(aq) - psi;
      o.dp[3] = -aq / bq + ap / bp;
    }
  }
};

// Reparameterised Normal draw fused with its own score (guide sites; SURVEY.md 8(f) row 1).
//   value = eps ~ N(0,1);  params = (loc, scale)
//   z   = loc + eps*scale                 torch/distributions/normal.py:82-85   -> "dx" slot
//   lp  = Normal(loc, scale).log_prob(z)  normal.py:87-102, evaluated on the ROUNDED z exactly as a
//         separate log_prob(z) call would
// The kernel is launched with scale = weight = 1 so the dx slot holds z itself.
template <typename T, bool GRAD>
struct Eval<kNormalRsample, T, GRAD> {
  static B2_HD void run(T eps, const T* p, ElemOut<T>& o) {
    const T z = p[0] + eps * p[1];
    ElemOut<T> n;
    Eval<kNormal, T, false>::run(z, p, n);
    o.lp = n.lp;
    if (GRAD) {
      o.dx = z;
      o.dp[0] = (T)0;
      o.dp[1] = (T)0;
    }
  }
};

// Backward of the fused draw.  value = gz (gradient reaching z from its consumers, already
// weighted); params = (eps, scale, c) with c the coefficient on d(sum log q)/d(.) -- the total
// derivative of log q(z(loc, scale)) is 0 w.r.t. loc and -1/scale w.r.t. scale, so
//   d/dloc   = gz                      -> dp[0] (reduced to loc's stored shape by the kernel)
//   d/dscale = gz*eps - c/scale        -> dp[1]
template <typename T, bool GRAD>
struct Eval<kNormalRsampleBwd, T, GRAD> {
  static B2_HD void run(T gz, const T* p, ElemOut<T>& o) {
    o.lp = (T)0;
    if (GRAD) {
      o.dx = (T)0;
      o.dp[0] = gz;
      o.dp[1] = gz * p[0] - p[2] / p[1];
      o.dp[2] = (T)0;
    }
  }
};

}  // namespace b2
