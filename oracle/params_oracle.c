/* TEST INFRASTRUCTURE ONLY — the oracle of b200conv_chain_update: the parameter changes of processBlock on top of the
 * restatements of chain_oracle.c (send / wet chain) and hotswap_oracle.c (warmer, warm-up, crossfade, swap):
 *
 *   onSlider   Filter::setSlope + Filter::init of the four cut filters, no reset          src/PluginProcessor.cpp:837-848
 *              (setSlope: src/dsp/Filter.h:38 ; init: src/dsp/Filter.cpp:3-21)
 *   per block  cut on / off (> 20 Hz, < 20 kHz), predelay, width, dry / wet, tsenabled   :1151-1188, :1643, :1647
 *   delay line D = (int)(2.0f * srate) at prepareToPlay, D = 2 * predelay + clear() + delaypos = 0 when a block's
 *              predelay exceeds D                                                        :640, :1184-1188
 *
 * oc_chain_set / oc_hs_set_params (oc_hs_set names the IR sets of hotswap_oracle.c) take effect at the next
 * oc_chain_send / oc_hs_process call, as a parameter change takes effect at the top of the next processBlock.  The filter re-init is pinned bit for bit against the reference's own
 * Filter.cpp (tests/test_chain_params.py).  Nothing in the product may link this file.
 */
#include "hotswap_oracle.c"

/* Filter::setSlope + Filter::init without reset: coefficients change, ic1..ic4 and state carry on.  Like the
 * reference, the 12 / 24 dB coefficients are left as they were when the slope is 6 dB. */
static void filter_reinit(oc_filter* f, int slope, float srate, float freq, float q) {
  const float q2 = 0.6173f;
  f->slope = slope;
  f->g = oc_filter_coeff(freq, srate);
  f->k = 2 - 2 * q;
  f->k2 = 2 - 2 * q2;
  if (slope == 0) {
    f->g = f->g / (1.0f + f->g);
  } else {
    f->a1 = 1.0f / (1.0f + f->g * (f->g + f->k));
    f->a2 = f->g * f->a1;
    f->a3 = f->g * f->a2;
    f->a12 = 1.0f / (1.0f + f->g * (f->g + f->k2));
    f->a22 = f->g * f->a12;
    f->a32 = f->g * f->a22;
  }
}

void oc_filter_set(void* f, int slope, float srate, float freq, float q) { filter_reinit((oc_filter*)f, slope, srate, freq, q); }

/* delayBuffer.setSize(2, predelay * 2) ; clear() ; delaypos = 0 when predelay > D (:1184-1188) */
static void chain_set_predelay(oc_chain* c, int predelay) {
  if (predelay > c->delay_size) {
    c->delay_size = predelay * 2;
    for (int ch = 0; ch < 2; ++ch) {
      free(c->delay[ch]);
      c->delay[ch] = (float*)calloc((size_t)c->delay_size, sizeof(float));
    }
    c->delaypos = 0;
  }
  c->predelay = predelay;
}

void oc_chain_set(void* p, float lowcut_hz, int lowcut_slope, float highcut_hz, int highcut_slope, int predelay,
                  float width, float drygain, float wetgain) {
  oc_chain* c = (oc_chain*)p;
  c->lowcut_on = lowcut_hz > 20.0f;                               /* :1643 */
  c->highcut_on = highcut_hz < 20000.0f;                          /* :1647 */
  for (int ch = 0; ch < 2; ++ch) {                                /* :837-848 */
    filter_reinit(&c->lc[ch], lowcut_slope, c->srate, lowcut_hz, q_for(lowcut_slope));
    filter_reinit(&c->hc[ch], highcut_slope, c->srate, highcut_hz, q_for(highcut_slope));
  }
  chain_set_predelay(c, predelay);
  c->width = width; c->drygain = drygain; c->wetgain = wetgain;
}

/* the chain as prepareToPlay leaves it: D = (int)(2.0f * srate), grown by the first block if the predelay is longer */
void* oc_chain_create_ref(float srate, float lowcut_hz, int lowcut_slope, float highcut_hz, int highcut_slope,
                          int predelay, float width, float drygain, float wetgain) {
  oc_chain* c = (oc_chain*)oc_chain_create(srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, 0,
                                           (int)(2.0f * srate), width, drygain, wetgain);
  chain_set_predelay(c, predelay);
  return c;
}

int oc_chain_delay_size(const void* p) { return ((const oc_chain*)p)->delay_size; }

/* the hot-swap restatement on that delay line */
void* oc_hs_create_ref(double srate, float lowcut_hz, int lowcut_slope, float highcut_hz, int highcut_slope,
                       int predelay, float width, float drygain, float wetgain, int true_stereo) {
  oc_hotswap* h = (oc_hotswap*)oc_hs_create(srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, 0, width,
                                            drygain, wetgain, true_stereo);
  oc_chain_destroy(h->chain);
  h->chain = (oc_chain*)oc_chain_create_ref((float)srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope,
                                            predelay, width, drygain, wetgain);
  return h;
}

void oc_hs_set_params(void* p, float lowcut_hz, int lowcut_slope, float highcut_hz, int highcut_slope, int predelay,
                      float width, float drygain, float wetgain, int true_stereo) {
  oc_hotswap* h = (oc_hotswap*)p;
  oc_chain_set(h->chain, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, predelay, width, drygain, wetgain);
  h->true_stereo = true_stereo;
}

int oc_hs_delay_size(const void* p) { return ((const oc_hotswap*)p)->chain->delay_size; }
