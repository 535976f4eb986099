/* TEST INFRASTRUCTURE ONLY — CPU restatement of the whole of Impulse::recalcImpulse (src/dsp/Impulse.cpp:299-360), the
 * oracle of b200conv_ir_recalc / b200conv_init_*_recalc: chain_oracle.c::oc_ir_shape's steps plus resampling to the
 * project rate (:362-389) and stretch (:391-434) — JUCE's ResamplingAudioSource (juce_ResamplingAudioSource.cpp:92-275)
 * run serially as JUCE runs it: position accumulated sample by sample, low pass in double with the x86 flush of
 * |y| <= 1e-8 — the parametric EQ (:503-537, SVF sections of src/dsp/SVF.cpp, float) and the decay table built from
 * bands (:562-591 with SVF::getMagnitude).  Pinned by the reference compiled into oracle/_ref/librefimpulse.so
 * (tests/test_ir_recalc.py).  Built with partconv_oracle.c and chain_oracle.c into oracle/librecalc.so
 * (oracle/recalc.mk); nothing in the product may link this file.
 */
#include <math.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <complex.h>

/* chain_oracle.c: auto gain, reverse, trim, gain, decay EQ, clip, envelope */
size_t oc_ir_shape(float** ch, int C, size_t n, int autogain, int reverse, float trim_left, float trim_right, float gain,
                   const double* lut, double srate, int clip, float attack, float decay);

typedef struct oc_eq_band { int mode; float freq, q, gain; } oc_eq_band;          /* SVF::EQBand, SVF.h:28-33 */
typedef struct oc_svf { int mode; float srate, g, r2, a1, a2, a3, cl, cb, ch; } oc_svf;
enum { OC_LP, OC_BP, OC_HP, OC_LS, OC_HS, OC_PK, OC_BS, OC_HP6, OC_LP6, OC_OFF };   /* SVF::Mode, SVF.h:9-20 */
static const float oc_pi_f = 3.14159265358979323846f;
static const double oc_pi = 3.14159265358979323846, oc_sqrt2 = 1.41421356237309504880;   /* MathConstants<double> */

static void oc_svf_setup(oc_svf* f, float freq, float q, float resfactor) {          /* SVF.cpp:4-16 */
  f->g = tanf(oc_pi_f * fminf(freq / f->srate, 0.49f));
  f->r2 = (1.0f / q) * resfactor;
  f->a1 = 1.0f / (1.0f + f->g * (f->g + f->r2));
  f->a2 = f->g * f->a1;
  f->a3 = f->g * f->a2;
}

/* the if / else chain of Impulse.cpp:511-519: Off and unknown modes become a peak band */
static void oc_svf_make(oc_svf* f, float srate, const oc_eq_band* b) {
  memset(f, 0, sizeof(*f));
  f->srate = srate;
  f->cl = 1.0f;
  switch (b->mode) {
    case OC_LP: f->mode = OC_LP; oc_svf_setup(f, b->freq, b->q, 1.f); f->cl = 1.f; f->cb = 0.f; f->ch = 0.f; break;
    case OC_BP: f->mode = OC_BP; oc_svf_setup(f, b->freq, b->q, 1.f); f->cl = 0.f; f->cb = 1.f / b->q; f->ch = 0.f; break;
    case OC_HP: f->mode = OC_HP; oc_svf_setup(f, b->freq, b->q, 1.f); f->cl = 0.f; f->cb = 0.f; f->ch = 1.f; break;
    case OC_LS:
      f->mode = OC_LS; oc_svf_setup(f, b->freq * powf(b->gain, -0.25f), b->q, 1.f);
      f->cl = b->gain; f->cb = f->r2 * sqrtf(b->gain); f->ch = 1.f; break;
    case OC_HS:
      f->mode = OC_HS; oc_svf_setup(f, b->freq * powf(b->gain, 0.25f), b->q, 1.f);
      f->cl = 1.f; f->cb = f->r2 * sqrtf(b->gain); f->ch = b->gain; break;
    case OC_BS: f->mode = OC_BS; oc_svf_setup(f, b->freq, b->q, 1.f); f->cl = 1.f; f->cb = 0.f; f->ch = 1.f; break;
    case OC_HP6:
    case OC_LP6:
      f->mode = b->mode;
      f->g = tanf(oc_pi_f * fminf(b->freq / srate, 0.49f));
      f->g = f->g / (1.0f + f->g);
      break;
    default:
      f->mode = OC_PK; oc_svf_setup(f, b->freq, b->q, b->gain < 1.f ? 7.5f : 1.f);
      f->cl = 1.f; f->cb = f->r2 * b->gain; f->ch = 1.f;
  }
}

/* SVF::processBlock / processBlock6dB with constant coefficients from a zero state (SVF.cpp:139-245), in place */
static void oc_svf_run(const oc_svf* f, float* buf, size_t n) {
  float s1 = 0.0f, s2 = 0.0f;
  if (f->mode == OC_HP6 || f->mode == OC_LP6) {
    for (size_t i = 0; i < n; ++i) {
      float sample = buf[i];
      float delta = f->g * (sample - s1);
      s1 += delta;
      buf[i] = f->mode == OC_LP6 ? s1 : sample - s1;
    }
    return;
  }
  for (size_t i = 0; i < n; ++i) {
    float sample = buf[i];
    float v3 = sample - s2;
    float v1 = f->a1 * s1 + f->a2 * v3;
    float v2 = s2 + f->a2 * s1 + f->a3 * v3;
    s1 = 2.0f * v1 - s1;
    s2 = 2.0f * v2 - s2;
    buf[i] = f->cl * v2 + f->cb * v1 + f->ch * (sample - f->r2 * v1 - v2);
  }
}

static float oc_svf_magnitude(const oc_svf* f, float freq) {                         /* SVF.cpp:253-284 */
  const float lim = 0.49f * f->srate;
  if (lim < freq) freq = lim;
  if (f->mode == OC_LP6 || f->mode == OC_HP6) {
    float omega = 2.0f * oc_pi_f * freq / f->srate;
    float a = f->g, b = 1.0f - a, c = cosf(omega);
    float denom = 1.0f + b * b - 2.0f * b * c;
    if (denom < 1e-12f) denom = 1e-12f;
    float num = f->mode == OC_LP6 ? a * a : 2.0f - 2.0f * c;
    return sqrtf(num / denom);
  }
  float g_eval = tanf(oc_pi_f * fminf(freq / f->srate, 0.49f));
  float gn = g_eval / f->g;
  float complex denom = CMPLXF(gn * gn - 1.0f, gn * f->r2);
  /* -cl * (1, 0) + cb * (0, gn) + ch * (gn^2, 0), component by component as std::complex<float> evaluates it */
  float nre = ((-f->cl * 1.0f) + (f->cb * 0.0f)) + (f->ch * (gn * gn));
  float nim = ((-f->cl * 0.0f) + (f->cb * gn)) + (f->ch * 0.0f);
  float complex h = CMPLXF(nre, nim) / denom;
  return cabsf(h);
}

static float oc_clampf(float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); }

/* Impulse::applyDecayEQ's table (Impulse.cpp:562-591): 2049 per-bin decay factors per STFT block */
void oc_decay_lut(const oc_eq_band* bands, int nb, double srate, float decay_rate, double* lut) {
  const int size = 4096 / 2 + 1;
  const float max_gain = 24.f;                                                   /* EQ_MAX_GAIN, Globals.h:36 */
  oc_svf eq[16];
  for (int i = 0; i < nb && i < 16; ++i) oc_svf_make(&eq[i], (float)srate, &bands[i]);
  double decay_per_s = 1.0 - (double)0.9f, grow_per_s = 1.0 + (double)2.f;     /* EQ_MAX_DECAY_RATE_NEG / _POS */
  double ln_decay = log(pow(decay_per_s, (4096 / srate) * (double)decay_rate));
  double ln_grow = log(pow(grow_per_s, (4096 / srate) * (double)decay_rate));
  for (int i = 0; i < size; ++i) {
    float freq = (float)i / (float)(size - 1) * (float)srate * 0.5f;
    freq = oc_clampf(freq, 20.f, 20000.f);
    float mag = 1.f;
    for (int k = 0; k < nb && k < 16; ++k) mag *= oc_svf_magnitude(&eq[k], freq);
    float db = 20.0f * log10f(mag);
    float norm = oc_clampf((max_gain - db) / (2.f * max_gain), 0.f, 1.f);
    norm = (norm * 2.f - 1.f) * -1.f;
    double d = 1.0;
    if (norm > 0.f) d = exp(norm * ln_grow);
    else if (norm < 0.f) d = exp(-norm * ln_decay);
    lut[i] = d;
  }
}

/* ResamplingAudioSource::applyFilter (:251-275): st = x1, x2, y1, y2 */
static double oc_rs_filter(const double* c, double in, double* st) {
  double out = c[0] * in + c[1] * st[0] + c[2] * st[1] - c[4] * st[2] - c[5] * st[3];
  if (!(out < -1.0e-8 || out > 1.0e-8)) out = 0;                                 /* JUCE_INTEL */
  st[1] = st[0]; st[0] = in;
  st[3] = st[2]; st[2] = out;
  return out;
}

/* one ResamplingAudioSource run: in (ns taps, zeros after) -> out (M taps), `ratio` input samples per output sample */
static void oc_resample(const float* in, size_t ns, double ratio, size_t M, float* out) {
  const double prop = ratio > 1.0 ? 0.5 / ratio : 0.5 * ratio;                  /* createLowPass (:210-243) */
  const double nn = 1.0 / tan(oc_pi * (prop > 0.001 ? prop : 0.001));
  const double n2 = nn * nn;
  const double c1 = 1.0 / (1.0 + oc_sqrt2 * nn + n2);
  const double c[6] = {c1, c1 * 2.0f, c1, 1.0, c1 * 2.0 * (1.0 - n2), c1 * (1.0 - oc_sqrt2 * nn + n2)};
  double st[4] = {0, 0, 0, 0};
  const float* src = in;
  size_t nsrc = ns;
  float* stream = NULL;
  if (ratio > 1.0001) {                                                          /* down-sampling: filter first */
    nsrc = (size_t)((double)M * ratio) + 8;
    stream = (float*)malloc(nsrc * sizeof(float));
    for (size_t i = 0; i < nsrc; ++i) stream[i] = (float)oc_rs_filter(c, (double)(i < ns ? in[i] : 0.0f), st);
    src = stream;
  }
  double sub = 0.0;                                                              /* subSampleOffset (:155-177) */
  size_t pos = 0;
  for (size_t m = 0; m < M; ++m) {
    const float a = pos < nsrc ? src[pos] : 0.0f, b = pos + 1 < nsrc ? src[pos + 1] : 0.0f;
    const float alpha = (float)sub;
    out[m] = a + alpha * (b - a);
    sub += ratio;
    while (sub >= 1.0) { ++pos; sub -= 1.0; }
  }
  if (ratio < 0.9999)                                                            /* up-sampling: filter after */
    for (size_t m = 0; m < M; ++m) out[m] = (float)oc_rs_filter(c, (double)out[m], st);
  free(stream);
}

/* lengths of Impulse.cpp:364-409: after resampling (*n1, ratio *rs or 0) and after stretch (*n2, ratio *sr or 0) */
static void oc_recalc_lengths(size_t n, double ir_srate, double srate, float stretch, size_t* n1, double* rs, size_t* n2, double* sr) {
  *n1 = n; *rs = 0.0;
  if (n > 0 && !(fabs(ir_srate - srate) < 1e-6)) {
    *rs = ir_srate / srate;
    *n1 = (size_t)(int)ceil((int)n / *rs);
  }
  *n2 = *n1; *sr = 0.0;
  if (stretch != 0.f && *n1 > 0) {
    double stretchsrate = pow(2, stretch) * srate;
    if (!(fabs(stretchsrate - srate) < 1e-6 || stretchsrate < 1.0 || srate < 1.0)) {
      *sr = srate / stretchsrate;
      *n2 = (size_t)(int)ceil((int)*n1 * stretchsrate / srate);
    }
  }
}

size_t oc_ir_recalc_len(size_t n, double ir_srate, double srate, float stretch, float trim_left, float trim_right) {
  size_t n1, n2;
  double rs, sr;
  oc_recalc_lengths(n, ir_srate, srate, stretch, &n1, &rs, &n2, &sr);
  size_t start = (size_t)(trim_left * (float)n2), end = n2 - (size_t)(trim_right * (float)n2);
  if (n2 == 0 || start >= end || start >= n2 || end > n2) return 0;
  return end - start;
}

/* raw[c]: C channels {LL, RR[, LR, RL]} of n taps; out[c] gets min(result, out_cap) taps; returns the result's length */
size_t oc_ir_recalc(const float* const* raw, int C, size_t n, double ir_srate, double srate, float stretch, int autogain,
                    int reverse, float trim_left, float trim_right, float gain, int n_param, const oc_eq_band* param_eq,
                    int n_decay, const oc_eq_band* decay_eq, float decay_rate, int clip, float attack, float decay,
                    float* const* out, size_t out_cap) {
  size_t n1, n2;
  double rs, sr;
  oc_recalc_lengths(n, ir_srate, srate, stretch, &n1, &rs, &n2, &sr);
  if (n == 0 || C < 2 || C > 8) return 0;
  size_t cap = n > n1 ? n : n1;
  if (n2 > cap) cap = n2;
  float* ch[8];
  float* tmp = (float*)malloc(cap * sizeof(float));
  for (int c = 0; c < C; ++c) {
    ch[c] = (float*)malloc(cap * sizeof(float));
    memcpy(ch[c], raw[c], n * sizeof(float));
  }
  /* auto gain (:315-324) and reverse (:326-334) */
  oc_ir_shape(ch, C, n, autogain, reverse, 0.f, 0.f, 1.0f, NULL, srate, 0, 0.f, 0.f);
  size_t len = n;
  if (rs != 0.0) {                                                               /* resampleIRToProjectRate */
    for (int c = 0; c < C; ++c) {
      oc_resample(ch[c], len, rs, n1, tmp);
      for (size_t i = 0; i < n1; ++i) tmp[i] *= (float)rs;
      memcpy(ch[c], tmp, n1 * sizeof(float));
    }
    len = n1;
  }
  if (sr != 0.0) {                                                               /* applyStretch */
    for (int c = 0; c < C; ++c) {
      oc_resample(ch[c], len, sr, n2, tmp);
      memcpy(ch[c], tmp, n2 * sizeof(float));
    }
    len = n2;
  }
  size_t m = 0;
  size_t start = (size_t)(trim_left * (float)len), end = len - (size_t)(trim_right * (float)len);
  if (!(start >= end || start >= len || end > len)) {
    m = end - start;
    for (int c = 0; c < C; ++c) {                                                /* applyTrim, applyGain */
      memmove(ch[c], ch[c] + start, m * sizeof(float));
      for (size_t i = 0; i < m; ++i) ch[c][i] *= gain;
    }
    for (int b = 0; b < n_param; ++b) {                                          /* applyParamEQ */
      oc_svf f;
      oc_svf_make(&f, (float)srate, &param_eq[b]);
      for (int c = 0; c < C; ++c) oc_svf_run(&f, ch[c], m);
    }
    double lut[2049];
    if (n_decay > 0) oc_decay_lut(decay_eq, n_decay, srate, decay_rate, lut);
    /* decay EQ, clip, envelope (trim and gain already applied: identity here) */
    m = oc_ir_shape(ch, C, m, 0, 0, 0.f, 0.f, 1.0f, n_decay > 0 ? lut : NULL, srate, clip, attack, decay);
    for (int c = 0; c < C; ++c) memcpy(out[c], ch[c], (m < out_cap ? m : out_cap) * sizeof(float));
  }
  for (int c = 0; c < C; ++c) free(ch[c]);
  free(tmp);
  return m;
}
