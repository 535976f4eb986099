/* TEST INFRASTRUCTURE ONLY — serial float64 references of the recursive filters that the device runs as chunked scans
 * (tests/test_scan_precision.py):
 *   SVF sections of the parametric EQ    src/dsp/SVF.cpp:139-245 (processBlock / processBlock6dB)
 *   the send chain's Filter::eval          src/dsp/Filter.cpp:23-68 (6 / 12 / 24 dB; LP, BP, HP)
 *   JUCE's resampler low pass              juce_ResamplingAudioSource.cpp:210-275 (already double in JUCE)
 * Each recurrence is written once per precision with the same equations in the same order, starting from the float32
 * coefficients the oracle computes (recalc_oracle.c::oc_svf_make, chain_oracle.c::oc_filter_init).  Run in float, the
 * runs must reproduce the oracle bit for bit (the self-check of the test file); run in double they are the reference.
 * The oracle source is included so that its static coefficient functions are the ones used here.  Compiled with
 * oracle/chain_oracle.c and oracle/partconv_oracle.c, -ffp-contract=off as the oracle is.
 */
#include "../../oracle/recalc_oracle.c"

/* chain_oracle.c */
typedef struct sf_filter_c {
  int slope, mode;
  float g, k, k2, a1, a2, a3, a12, a22, a32;
  float ic1, ic2, ic3, ic4, state;
} sf_filter_c;
void oc_filter_init(sf_filter_c* f, int slope, int mode, float srate, float freq, float q);
float oc_filter_eval(sf_filter_c* f, float sample);

/* ---- SVF sections ---- */
/* c[8] = g, r2, a1, a2, a3, cl, cb, ch ; returns the mode the section runs as (Off / unknown -> PK) */
int sf_svf_coeffs(int mode, float freq, float q, float gain, float srate, float* c) {
  oc_eq_band b = {mode, freq, q, gain};
  oc_svf f;
  oc_svf_make(&f, srate, &b);
  c[0] = f.g; c[1] = f.r2; c[2] = f.a1; c[3] = f.a2; c[4] = f.a3; c[5] = f.cl; c[6] = f.cb; c[7] = f.ch;
  return f.mode;
}

#define SF_SVF_RUN(T, NAME)                                                                                  \
  void NAME(int mode, const float* c, const T* x, T* y, size_t n) {                                       \
    const T g = c[0], r2 = c[1], a1 = c[2], a2 = c[3], a3 = c[4], cl = c[5], cb = c[6], ch = c[7];        \
    T s1 = 0, s2 = 0;                                                                                      \
    if (mode == OC_HP6 || mode == OC_LP6) {                                                                \
      for (size_t i = 0; i < n; ++i) {                                                                     \
        const T sample = x[i];                                                                             \
        const T delta = g * (sample - s1);                                                                 \
        s1 += delta;                                                                                       \
        y[i] = mode == OC_LP6 ? s1 : sample - s1;                                                          \
      }                                                                                                    \
      return;                                                                                              \
    }                                                                                                      \
    for (size_t i = 0; i < n; ++i) {                                                                       \
      const T sample = x[i];                                                                               \
      const T v3 = sample - s2;                                                                            \
      const T v1 = a1 * s1 + a2 * v3;                                                                      \
      const T v2 = s2 + a2 * s1 + a3 * v3;                                                                 \
      s1 = (T)2 * v1 - s1;                                                                                 \
      s2 = (T)2 * v2 - s2;                                                                                 \
      y[i] = cl * v2 + cb * v1 + ch * (sample - r2 * v1 - v2);                                             \
    }                                                                                                      \
  }
SF_SVF_RUN(double, sf_svf_run64)
SF_SVF_RUN(float, sf_svf_run32)

/* the oracle's own section, in place (self-check) */
void sf_svf_oracle(int mode, float freq, float q, float gain, float srate, float* buf, size_t n) {
  oc_eq_band b = {mode, freq, q, gain};
  oc_svf f;
  oc_svf_make(&f, srate, &b);
  oc_svf_run(&f, buf, n);
}

/* ---- Filter (the send chain's low / high cut) ---- */
/* c[9] = g, k, k2, a1, a2, a3, a12, a22, a32 of Filter::init with the processor's q */
void sf_filter_coeffs(int slope, int mode, float srate, float freq, float* c) {
  sf_filter_c f;
  oc_filter_init(&f, slope, mode, srate, freq, slope == 2 ? 0.0765f : 0.2929f);
  c[0] = f.g; c[1] = f.k; c[2] = f.k2; c[3] = f.a1; c[4] = f.a2; c[5] = f.a3; c[6] = f.a12; c[7] = f.a22; c[8] = f.a32;
}

/* st[5] = ic1, ic2, ic3, ic4, state carried in and out, so that a stream of calls and slope switches keep them */
#define SF_FILTER_RUN(T, NAME)                                                                               \
  void NAME(int slope, int mode, const float* c, T* st, const T* x, T* y, size_t n) {                     \
    const T g = c[0], k = c[1], k2 = c[2], a1 = c[3], a2 = c[4], a3 = c[5], a12 = c[6], a22 = c[7], a32 = c[8]; \
    for (size_t i = 0; i < n; ++i) {                                                                       \
      const T sample = x[i];                                                                               \
      if (slope == 0) {                                                                                    \
        const T delta = g * (sample - st[4]);                                                              \
        st[4] += delta;                                                                                    \
        y[i] = mode == 0 ? st[4] : sample - st[4];                                                         \
        continue;                                                                                          \
      }                                                                                                    \
      T v3 = sample - st[1];                                                                               \
      T v1 = a1 * st[0] + a2 * v3;                                                                         \
      T v2 = st[1] + a2 * st[0] + a3 * v3;                                                                 \
      st[0] = (T)2 * v1 - st[0];                                                                           \
      st[1] = (T)2 * v2 - st[1];                                                                           \
      T out = mode == 0 ? v2 : (mode == 1 ? v1 : sample - k * v1 - v2);                                   \
      if (slope == 2) {                                                                                    \
        v3 = out - st[3];                                                                                  \
        v1 = a12 * st[2] + a22 * v3;                                                                       \
        v2 = st[3] + a22 * st[2] + a32 * v3;                                                               \
        st[2] = (T)2 * v1 - st[2];                                                                         \
        st[3] = (T)2 * v2 - st[3];                                                                         \
        out = mode == 0 ? v2 : (mode == 1 ? v1 : out - k2 * v1 - v2);                                      \
      }                                                                                                    \
      y[i] = out;                                                                                          \
    }                                                                                                      \
  }
SF_FILTER_RUN(double, sf_filter_run64)
SF_FILTER_RUN(float, sf_filter_run32)

/* the oracle's own filter from a zero state (self-check) */
void sf_filter_oracle(int slope, int mode, float srate, float freq, const float* x, float* y, size_t n) {
  sf_filter_c f;
  oc_filter_init(&f, slope, mode, srate, freq, slope == 2 ? 0.0765f : 0.2929f);
  for (size_t i = 0; i < n; ++i) y[i] = oc_filter_eval(&f, x[i]);
}

/* ---- JUCE resampler low pass ---- */
/* createLowPass for `ratio` input samples per output sample, then applyFilter over x (n samples, zero state);
 * flush != 0: JUCE_INTEL's flush of |y| <= 1e-8 to zero */
void sf_rs_lowpass64(double ratio, const double* x, double* y, size_t n, int flush) {
  const double prop = ratio > 1.0 ? 0.5 / ratio : 0.5 * ratio;
  const double nn = 1.0 / tan(oc_pi * (prop > 0.001 ? prop : 0.001));
  const double n2 = nn * nn;
  const double c1 = 1.0 / (1.0 + oc_sqrt2 * nn + n2);
  const double c[6] = {c1, c1 * 2.0f, c1, 1.0, c1 * 2.0 * (1.0 - n2), c1 * (1.0 - oc_sqrt2 * nn + n2)};
  double x1 = 0, x2 = 0, y1 = 0, y2 = 0;
  for (size_t i = 0; i < n; ++i) {
    double out = c[0] * x[i] + c[1] * x1 + c[2] * x2 - c[4] * y1 - c[5] * y2;
    if (flush && !(out < -1.0e-8 || out > 1.0e-8)) out = 0;
    x2 = x1; x1 = x[i];
    y2 = y1; y1 = out;
    y[i] = out;
  }
}

/* sum over the first n samples of |h| of the low pass's recursive part 1 / (1 + c4 z^-1 + c5 z^-2): the gain by which
 * a per-sample perturbation (the flush) can grow on its way through the filter */
double sf_rs_feedback_l1(double ratio, size_t n) {
  const double prop = ratio > 1.0 ? 0.5 / ratio : 0.5 * ratio;
  const double nn = 1.0 / tan(oc_pi * (prop > 0.001 ? prop : 0.001));
  const double n2 = nn * nn;
  const double c1 = 1.0 / (1.0 + oc_sqrt2 * nn + n2);
  const double c4 = c1 * 2.0 * (1.0 - n2), c5 = c1 * (1.0 - oc_sqrt2 * nn + n2);
  double y1 = 0, y2 = 0, s = 0;
  for (size_t i = 0; i < n; ++i) {
    const double out = (i == 0 ? 1.0 : 0.0) - c4 * y1 - c5 * y2;
    y2 = y1; y1 = out;
    s += fabs(out);
  }
  return s;
}
