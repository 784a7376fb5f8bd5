// Per-element arithmetic of the ZINB / NB negative log-likelihood and its gradient.
//
// Restates dca/loss.py:72-156 (reference formulas; every epsilon kept where it is representable
// in fp32) and the closed-form derivatives TF autodiff produces for them (SURVEY.md A.4),
// re-arranged so that fp32 does not cancel catastrophically and so that ONE reciprocal serves
// the whole element.  With  te = theta+eps,  den = te+mu,  q = mu/den,  r = te/den = 1-q:
//   log(1+mu/te) = -log r =: L1            (series in q for q < 1/16, else lg2)
//   t2 (loss.py:88) = (theta+y) L1 + y (log te - log(mu+eps)) = theta L1 - y log((mu+eps)/den)
//   zero_nb (loss.py:136) = r^theta = exp(-theta L1)
//   d/dmu * mu      = theta (mu + eps - y)/den * mu/(mu+eps)   (nb; the second factor is the eps of log(mu+eps): 1 - 5e-4
//                     at mu = 2e-7, i.e. MeanAct's floor times a small size factor)   |  w theta q          (zero)
//   d/dtheta        = [L1 - q] + y/den - (psi(y+te)-psi(te))  (nb)   |  w [L1 - q]   (zero)
//   lgamma(te)-lgamma(y+te) = -sum_{k<y} log(te+k),  psi(te)-psi(y+te) = -sum_{k<y} 1/(te+k)
//     (integer y <= 16: product recurrence; otherwise shifted Stirling / asymptotic digamma)
//
// The same source compiles for the host (PreciseOps: libm) -- exported as dca_zinb_elem_host so
// the formulas are unit-tested against the oracle without a GPU -- and for the device
// (FastOps: MUFU rcp / lg2 / ex2 approximations, ~1 ulp each).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace dca {
namespace zmath {

#define DCA_HD __host__ __device__ __forceinline__

constexpr float kEps = 1e-10f;            // dca/loss.py:65
constexpr float kHalfLog2Pi = 0.918938533204672742f;
constexpr float kLn2 = 0.693147180559945f;
constexpr float kLog2e = 1.442695040888963f;
constexpr int kLogFactN = 64;             // table of log(k!) for k < 64 (shared memory on the device)

struct PreciseOps {
  static DCA_HD float rcp(float x) { return 1.0f / x; }
  static DCA_HD float lg2(float x) { return log2f(x); }
  static DCA_HD float ex2(float x) { return exp2f(x); }
};

#ifdef __CUDACC__
struct FastOps {   // device only: one MUFU instruction each
  static __device__ __forceinline__ float rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
  static __device__ __forceinline__ float lg2(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
  static __device__ __forceinline__ float ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
};
#endif

// log(k!) table filler (host: static table; device: copied into shared memory by the kernel)
inline void fill_log_fact(float* t) {
  double acc = 0.0;
  t[0] = 0.f;
  for (int k = 1; k < kLogFactN; ++k) { acc += log((double)k); t[k] = (float)acc; }
}

// lgamma(x) - [(x-0.5)log x - x + 0.5 log 2pi]  for x >= 8
template <class Ops>
DCA_HD float stirling_corr(float x) {
  const float r = Ops::rcp(x), r2 = r * r;
  return r * (0.0833333333f + r2 * (-0.00277777778f + r2 * 0.000793650794f));
}
// psi(x) - log(x) for x >= 8
template <class Ops>
DCA_HD float digamma_corr(float x) {
  const float r = Ops::rcp(x), r2 = r * r;
  return -0.5f * r - r2 * (0.0833333333f - r2 * (0.00833333333f - r2 * 0.00396825397f));
}

// log prod_{k<n}(x+k) and sum_{k<n} 1/(x+k): factors are multiplied four at a time (the product of four
// factors <= (1e4+16)^4 cannot overflow), one lg2 + one rcp per group:
//   1/t0+1/t1+1/t2+1/t3 = ((t0+t1) t2 t3 + t0 t1 (t2+t3)) / (t0 t1 t2 t3)
template <class Ops>
DCA_HD void rising_log_and_recsum(float x, int n, float& logprod, float& recsum) {
  float lg = 0.f, rs = 0.f;
  int k = 0;
  for (; k + 4 <= n; k += 4) {
    const float t0 = x + (float)k, t1 = t0 + 1.0f, t2 = t0 + 2.0f, t3 = t0 + 3.0f;
    const float a = t0 * t1, b = t2 * t3, P = a * b;
    lg += Ops::lg2(P);
    rs = fmaf(fmaf(t0 + t1, b, a * (t2 + t3)), Ops::rcp(P), rs);
  }
  const int rem = n - k;
  if (rem > 0) {
    const float t0 = x + (float)k, t1 = t0 + 1.0f, t2 = t0 + 2.0f;
    float P = t0, num = 1.0f;
    if (rem >= 2) { num = t0 + t1; P = t0 * t1; }
    if (rem == 3) { num = fmaf(num, t2, P); P *= t2; }
    lg += Ops::lg2(P);
    rs = fmaf(num, Ops::rcp(P), rs);
  }
  logprod = lg * kLn2;
  recsum = rs;
}

// lgamma(y+1), y >= 0   (only the loss VALUE needs it; it has no gradient)
template <class Ops>
DCA_HD float lgamma_1p(float y, const float* lf_table) {
  if (y < (float)kLogFactN - 0.5f && y == rintf(y)) return lf_table[(int)y];
  float x = y + 1.0f, shift = 0.f;
  if (x < 8.f) { float s; rising_log_and_recsum<Ops>(x, 8, shift, s); x += 8.f; }
  return (x - 0.5f) * (kLn2 * Ops::lg2(x)) - x + kHalfLog2Pi + stirling_corr<Ops>(x) - shift;
}

// lg = lgamma(th+y) - lgamma(th),  dg = psi(th+y) - psi(th);   th > 0, y >= 0
template <class Ops>
DCA_HD void lgam_digam_diff(float th, float y, float& lg, float& dg) {
  if (y <= 16.f && y == rintf(y)) { rising_log_and_recsum<Ops>(th, (int)y, lg, dg); return; }
  float a = th, b = th + y, sh_lg = 0.f, sh_dg = 0.f;
  if (a < 8.f) { float lp, rs; rising_log_and_recsum<Ops>(a, 8, lp, rs); sh_lg += lp; sh_dg += rs; a += 8.f; }
  if (b < 8.f) { float lp, rs; rising_log_and_recsum<Ops>(b, 8, lp, rs); sh_lg -= lp; sh_dg -= rs; b += 8.f; }
  // log(b/a) = log1p((b-a)/a): series when the ratio is close to one
  const float u = (b - a) * Ops::rcp(a);
  float lr;
  if (fabsf(u) < 0.125f) {
    float p = fmaf(u, -0.1f, 0.111111111f);
    p = fmaf(u, p, -0.125f); p = fmaf(u, p, 0.142857143f); p = fmaf(u, p, -0.166666667f);
    p = fmaf(u, p, 0.2f); p = fmaf(u, p, -0.25f); p = fmaf(u, p, 0.333333333f); p = fmaf(u, p, -0.5f);
    lr = fmaf(u * u, p, u);
  } else {
    lr = kLn2 * Ops::lg2(1.0f + u);
  }
  lg = (a - 0.5f) * lr + (b - a) * (kLn2 * Ops::lg2(b) - 1.0f) + stirling_corr<Ops>(b) - stirling_corr<Ops>(a) + sh_lg;
  dg = lr + digamma_corr<Ops>(b) - digamma_corr<Ops>(a) + sh_dg;
}

struct Elem {
  float loss;   // element NLL (+ ridge*pi^2)
  float gm;     // dL/d zm   (mean pre-activation), clip mask applied, NOT yet / N
  float gd;     // COND_DISP: dL/d zd ; else raw dL/dtheta
  float gp;     // dL/d zp
};

// Quantities shared by both branches of loss.py:138
struct Shared { float mu, th, te, rden, q, L1, f; };

template <class Ops>
DCA_HD Shared shared_terms(float m, float sf, float th) {
  Shared s;
  s.mu = m * sf;                                            // dca/layers.py:85
  s.th = fminf(th, 1e6f);                                   // dca/loss.py:85
  s.te = s.th + kEps;                                       // dca/loss.py:87
  s.rden = Ops::rcp(s.te + s.mu);
  s.q = s.mu * s.rden;
  if (s.q < 0.0625f) {                                      // -log(1-q) = q + q^2/2 + q^3/3 + ... (q^9/9 < 2e-11 q)
    const float q = s.q;
    float p = fmaf(q, 0.125f, 0.142857143f);
    p = fmaf(q, p, 0.166666667f); p = fmaf(q, p, 0.2f); p = fmaf(q, p, 0.25f);
    p = fmaf(q, p, 0.333333333f); p = fmaf(q, p, 0.5f);
    s.f = q * q * p;                                        // L1 - q
    s.L1 = q + s.f;
  } else {
    s.L1 = -kLn2 * Ops::lg2(s.te * s.rden);                 // log(1 + mu/(theta+eps))   loss.py:88
    s.f = s.L1 - s.q;
  }
  return s;
}

// 1 - exp(-d) = sigmoid(zd) when d = softplus(zd)
template <class Ops>
DCA_HD float one_minus_exp_neg(float d) {
  if (d < 0.03125f) {                         // d - d^2/2 + d^3/6 - d^4/24; next term d^5/120 < 1e-8 d
    float p = fmaf(d, 0.0416666667f, -0.166666667f);
    p = fmaf(d, p, 0.5f);
    return d - d * d * p;
  }
  return 1.0f - Ops::ex2(-d * kLog2e);
}

// Chain rule through the output activations + ridge, shared by both branches.
template <class Ops, bool HAS_PI, bool COND_DISP>
DCA_HD void finish_elem(Elem& o, float dth, float dpi, float m, float th, float pi, float ridge) {
  const bool m_pass = (m > 1e-5f) && (m < 1e6f);           // clip_by_value gradient mask (network.py:38)
  o.gm = m_pass ? o.gm : 0.f;
  if (COND_DISP) {
    const bool d_pass = (th > 1e-4f) && (th < 1e4f);       // DispAct clip mask (network.py:39)
    o.gd = d_pass ? dth * one_minus_exp_neg<Ops>(th) : 0.f;
  } else {
    o.gd = dth;
  }
  if (HAS_PI) {
    if (ridge != 0.f) {                                    // loss.py:139-140 (uniform branch; ridge defaults to 0)
      o.loss = fmaf(ridge * pi, pi, o.loss);
      dpi = fmaf(2.0f * ridge, pi, dpi);
    }
    o.gp = dpi * (pi * (1.0f - pi));
  } else {
    o.gp = 0.f;
  }
}

// zero branch of loss.py:138 (y < 1e-8), ZINB models only
template <class Ops, bool COND_DISP>
DCA_HD Elem zinb_elem_zero(float m, float sf, float th, float pi, float ridge) {
  const Shared s = shared_terms<Ops>(m, sf, th);
  Elem o;
  const float z = Ops::ex2(-s.th * s.L1 * kLog2e);         // pow(theta/(theta+mu+eps), theta)  loss.py:136
  const float omp = 1.0f - pi;
  const float D = pi + omp * z + kEps;                     // loss.py:137
  const float rD = Ops::rcp(D);
  o.loss = -kLn2 * Ops::lg2(D);
  const float w = omp * z * rD;
  o.gm = w * s.th * s.q;
  finish_elem<Ops, true, COND_DISP>(o, w * s.f /* -w*(log r + 1 - r) */, (z - 1.0f) * rD, m, th, pi, ridge);
  return o;
}

// NB branch of loss.py:87-88,130 (all elements of NB models; y >= 1e-8 for ZINB models)
template <class Ops, bool HAS_PI, bool COND_DISP>
DCA_HD Elem zinb_elem_nb(float y, float m, float sf, float th, float pi, float ridge, const float* lf_table) {
  const Shared s = shared_terms<Ops>(m, sf, th);
  Elem o;
  float lg, dg, dpi = 0.f;
  lgam_digam_diff<Ops>(s.te, y, lg, dg);
  float nb = lgamma_1p<Ops>(y, lf_table) - lg + s.th * s.L1 - y * (kLn2 * Ops::lg2((s.mu + kEps) * s.rden));
  if (nb != nb) nb = INFINITY;                             // _nan2inf  loss.py:105
  o.gm = s.th * (s.mu + kEps - y) * s.rden * (s.mu * Ops::rcp(s.mu + kEps));
  if (HAS_PI) {
    const float qq = 1.0f - pi + kEps;
    nb -= kLn2 * Ops::lg2(qq);                             // loss.py:130
    dpi = Ops::rcp(qq);
  }
  o.loss = nb;
  finish_elem<Ops, HAS_PI, COND_DISP>(o, s.f + y * s.rden - dg, dpi, m, th, pi, ridge);
  return o;
}

// ------------------------------------------------------------------------------------ packed (f32x2) formulation
// The element-wise chains below are written over float2 (two genes of a thread): the two chains are independent, so
// they interleave in the FMA pipe; MUFU, min/max and selects stay scalar.  sm_90 has no paired fp32 FMA, so device
// and host evaluate the same component-wise expressions (fmaf) and the formulas are unit-tested without a GPU
// (dca_zinb_elem_host, variant 0x200).
DCA_HD float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
DCA_HD float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
DCA_HD float2 add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
DCA_HD float2 splat(float v) { return make_float2(v, v); }
DCA_HD float2 neg2(float2 a) { return make_float2(-a.x, -a.y); }

// Raw (un-chained, un-scaled) derivatives of one element: what the two branches of loss.py:138 hand to the shared
// finishing step  dzm = gmu * [m-clip mask] / N,  dzd = dth * sigmoid(zd) * [d-clip mask] / N,  dzp = dpi * pi (1-pi) / N.
struct Raw2 { float2 lgD, gmu, dth, dpi; };

// zero branch (y < 1e-8) of two ZINB elements: loss = -ln2 * lgD,  gmu = dL/dmu * mu,  dth = dL/dtheta,  dpi = dL/dpi
// (the formulas of zinb_elem_zero without control flow: both sides of the series / MUFU choice are evaluated and
// selected, so the independent chains of a thread's elements interleave).  mu = m * sf is computed by the caller (the
// NB items need it too).
// TH_BOUNDED: the caller knows theta <= 1e6 (the kernels check the row's theta range once per thread), so the
// min(theta, 1e6) of loss.py:85,134 is the identity and is skipped.
template <class Ops, bool TH_BOUNDED = false>
DCA_HD Raw2 zinb_zero_pair(float2 mu, float2 th_in, float2 pi) {
  const float2 th = TH_BOUNDED ? th_in : make_float2(fminf(th_in.x, 1e6f), fminf(th_in.y, 1e6f));   // loss.py:85,134
  const float2 te = add2(th, splat(kEps));
  const float2 den = add2(te, mu);
  const float2 rden = make_float2(Ops::rcp(den.x), Ops::rcp(den.y));
  const float2 q = mul2(mu, rden);
  float2 p = fma2(q, splat(0.125f), splat(0.142857143f));
  p = fma2(q, p, splat(0.166666667f)); p = fma2(q, p, splat(0.2f)); p = fma2(q, p, splat(0.25f));
  p = fma2(q, p, splat(0.333333333f)); p = fma2(q, p, splat(0.5f));
  const float2 f_ser = mul2(mul2(q, q), p), L1_ser = add2(q, f_ser);
  const float2 r = mul2(te, rden);
  const float2 lg = make_float2(Ops::lg2(r.x), Ops::lg2(r.y));
  const float2 L1_log = mul2(lg, splat(-kLn2)), f_log = fma2(lg, splat(-kLn2), neg2(q));
  const bool s0 = q.x < 0.0625f, s1 = q.y < 0.0625f;
  const float2 L1 = make_float2(s0 ? L1_ser.x : L1_log.x, s1 ? L1_ser.y : L1_log.y);
  const float2 f = make_float2(s0 ? f_ser.x : f_log.x, s1 ? f_ser.y : f_log.y);
  const float2 e = mul2(mul2(th, splat(-kLog2e)), L1);
  const float2 z = make_float2(Ops::ex2(e.x), Ops::ex2(e.y));                           // loss.py:136
  const float2 omp = fma2(pi, splat(-1.0f), splat(1.0f));
  const float2 D = add2(fma2(omp, z, pi), splat(kEps));                                // loss.py:137
  const float2 rD = make_float2(Ops::rcp(D.x), Ops::rcp(D.y));
  Raw2 o;
  o.lgD = make_float2(Ops::lg2(D.x), Ops::lg2(D.y));
  const float2 w = mul2(mul2(omp, z), rD);
  o.gmu = mul2(mul2(w, th), q);
  o.dth = mul2(w, f);
  o.dpi = mul2(add2(z, splat(-1.0f)), rD);
  return o;
}

// Finishing factors of two elements (chain rule through MeanAct / DispAct / sigmoid, clip masks, 1/N):
//   dzm = gmu * fm,  dzd = dth * fd,  dzp = dpi * fp
struct Fin2 { float2 fm, fd, fp; };
template <class Ops, bool COND_DISP>
DCA_HD Fin2 finish_factors_pair(float2 m, float2 th_in, float2 pi, float inv_n) {
  Fin2 o;
  o.fm = make_float2(((m.x > 1e-5f) && (m.x < 1e6f)) ? inv_n : 0.f,                     // network.py:38 clip mask
                     ((m.y > 1e-5f) && (m.y < 1e6f)) ? inv_n : 0.f);
  if (COND_DISP) {                                                                     // 1 - exp(-d) = sigmoid(zd)
    float2 pp = fma2(th_in, splat(0.0416666667f), splat(-0.166666667f));
    pp = fma2(th_in, pp, splat(0.5f));
    const float2 ser = fma2(neg2(mul2(th_in, th_in)), pp, th_in);
    const float2 a = mul2(th_in, splat(-kLog2e));
    const float2 ex = fma2(make_float2(Ops::ex2(a.x), Ops::ex2(a.y)), splat(-1.0f), splat(1.0f));
    const float2 ome = make_float2(th_in.x < 0.03125f ? ser.x : ex.x, th_in.y < 0.03125f ? ser.y : ex.y);
    const float2 sc = mul2(ome, splat(inv_n));
    o.fd = make_float2(((th_in.x > 1e-4f) && (th_in.x < 1e4f)) ? sc.x : 0.f,           // network.py:39 clip mask
                       ((th_in.y > 1e-4f) && (th_in.y < 1e4f)) ? sc.y : 0.f);
  } else {
    o.fd = splat(1.0f);                                   // raw dL/dtheta: summed per gene, chained by theta_grad_finish
  }
  const float2 omp = fma2(pi, splat(-1.0f), splat(1.0f));
  o.fp = mul2(mul2(pi, omp), splat(inv_n));
  return o;
}

// One group of up to four factors of the rising product prod_{k<n}(x+k), starting at x0 = x + k0 with nrem = n - k0 >= 1
// factors left: accumulates lg2 of the group product and the sum of reciprocals, WITHOUT control flow (absent factors
// are replaced by 1; d/dx of the product by the product rule):  sum 1/t = P'/P.
template <class Ops>
DCA_HD void rising_group_masked(float x0, float nrem, float& lg2acc, float& rs) {
  const bool h1 = nrem > 1.5f, h2 = nrem > 2.5f, h3 = nrem > 3.5f;
  const float f1 = h1 ? x0 + 1.0f : 1.0f, f2 = h2 ? x0 + 2.0f : 1.0f, f3 = h3 ? x0 + 3.0f : 1.0f;
  const float a = x0 * f1, ap = f1 + (h1 ? x0 : 0.f);
  const float b = f2 * f3, bp = (h2 ? f3 : 0.f) + (h3 ? f2 : 0.f);
  const float P = a * b;
  lg2acc += Ops::lg2(P);
  rs = fmaf(fmaf(ap, b, a * bp), Ops::rcp(P), rs);
}

// The same factors when every activation of the pair is known to lie strictly inside its clip range and theta >= 1/32
// (checked once per thread and row with min / max over its four genes, warp-uniform branch): no masks, no series.
template <class Ops, bool COND_DISP>
DCA_HD Fin2 finish_factors_pair_plain(float2 th_in, float2 pi, float inv_n) {
  Fin2 o;
  o.fm = splat(inv_n);
  if (COND_DISP) {
    const float2 a = mul2(th_in, splat(-kLog2e));
    o.fd = fma2(make_float2(Ops::ex2(a.x), Ops::ex2(a.y)), splat(-inv_n), splat(inv_n));   // (1 - exp(-d)) / N
  } else {
    o.fd = splat(1.0f);
  }
  const float2 omp = fma2(pi, splat(-1.0f), splat(1.0f));
  o.fp = mul2(mul2(pi, omp), splat(inv_n));
  return o;
}

// NB branch (y >= 1e-8) of one ZINB element from mu = m * sf: element NLL and the raw derivatives of struct Raw2
// (no clip masks, no activation chain, no ridge: the element's owner applies finish_factors_pair).  Straight-line for
// integer counts <= 4 (the bulk of a scRNA-seq matrix); counts 5..16 loop over further masked groups, anything else
// (large or non-integer) takes the shifted-Stirling path of lgam_digam_diff.
struct Raw1 { float loss, gmu, dth, dpi; };
template <class Ops>
DCA_HD Raw1 zinb_nb_raw(float y, float mu, float th_in, float pi, const float* lf_table) {
  const float th = fminf(th_in, 1e6f);                                                 // loss.py:85
  const float te = th + kEps;
  const float rden = Ops::rcp(te + mu);
  const float q = mu * rden;
  float p = fmaf(q, 0.125f, 0.142857143f);
  p = fmaf(q, p, 0.166666667f); p = fmaf(q, p, 0.2f); p = fmaf(q, p, 0.25f);
  p = fmaf(q, p, 0.333333333f); p = fmaf(q, p, 0.5f);
  const float f_ser = q * q * p;
  const float lgr = Ops::lg2(te * rden);
  const bool small_q = q < 0.0625f;
  const float L1 = small_q ? q + f_ser : -kLn2 * lgr;                                  // log(1 + mu/(theta+eps))  loss.py:88
  const float f = small_q ? f_ser : fmaf(-kLn2, lgr, -q);                              // L1 - q
  float lg, dg;
  if (y <= 16.f && y == rintf(y)) {
    float l2 = 0.f, rs = 0.f, x = te, n = y;
    rising_group_masked<Ops>(x, n, l2, rs);
    while (n > 4.5f) { x += 4.0f; n -= 4.0f; rising_group_masked<Ops>(x, n, l2, rs); }
    lg = l2 * kLn2; dg = rs;
  } else {
    lgam_digam_diff<Ops>(te, y, lg, dg);
  }
  const float mue = mu + kEps;
  float nb = lgamma_1p<Ops>(y, lf_table) - lg + th * L1 - y * (kLn2 * Ops::lg2(mue * rden));
  if (nb != nb) nb = INFINITY;                             // _nan2inf  loss.py:105
  const float qq = 1.0f - pi + kEps;
  Raw1 o;
  o.loss = nb - kLn2 * Ops::lg2(qq);                       // loss.py:130
  o.gmu = th * (mue - y) * rden * (mu * Ops::rcp(mue));    // exact: the eps of log(mu + eps) kept (see the header note)
  o.dth = f + y * rden - dg;
  o.dpi = Ops::rcp(qq);
  return o;
}

// y: raw count; m: MeanAct output (before *sf); sf: size factor; th: DispAct output or per-gene
// theta; pi: sigmoid output; lf_table: log(k!) for k < kLogFactN.
template <class Ops, bool HAS_PI, bool COND_DISP>
DCA_HD Elem zinb_elem(float y, float m, float sf, float th, float pi, float ridge, const float* lf_table) {
  if (HAS_PI && y < 1e-8f) return zinb_elem_zero<Ops, COND_DISP>(m, sf, th, pi, ridge);   // loss.py:138
  return zinb_elem_nb<Ops, HAS_PI, COND_DISP>(y, m, sf, th, pi, ridge, lf_table);
}

// forward-only value
template <class Ops, bool HAS_PI>
DCA_HD float zinb_elem_loss(float y, float m, float sf, float th, float pi, float ridge, const float* lf_table) {
  const Shared s = shared_terms<Ops>(m, sf, th);
  float l;
  if (HAS_PI && y < 1e-8f) {
    const float z = Ops::ex2(-s.th * s.L1 * kLog2e);
    l = -kLn2 * Ops::lg2(pi + (1.0f - pi) * z + kEps);
  } else {
    float lg, dg;
    lgam_digam_diff<Ops>(s.te, y, lg, dg);
    l = lgamma_1p<Ops>(y, lf_table) - lg + s.th * s.L1 - y * (kLn2 * Ops::lg2((s.mu + kEps) * s.rden));
    if (l != l) l = INFINITY;
    if (HAS_PI) l -= kLn2 * Ops::lg2(1.0f - pi + kEps);
  }
  if (HAS_PI) l = fmaf(ridge * pi, pi, l);
  return l;
}

}  // namespace zmath
}  // namespace dca
