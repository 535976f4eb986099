/* TEST INFRASTRUCTURE ONLY — CPU restatement of the IR hot swap of REEVRAudioProcessor::processBlock, the oracle of
 * b200conv_chain_swap + b200conv_chain_process, one host callback per oc_hs_process call:
 *
 *   send    dry * ysend ; low cut ; high cut                                src/PluginProcessor.cpp:1639-1653
 *   warmer  ring of W = (int)ceil(srate) / 4 send samples per channel       :610, :1655-1668
 *   warm-up numBlocks = W / host_block blocks from (warmwritepos + 1) % W through FRESH filters into the LL / RR
 *           convolvers of the load set (force2Chans)                       :1694-1756
 *   delay   predelay ring                                                   :1766-1790
 *   conv    live set on the delayed send; during the fade the load set's LL / RR on the UNDELAYED send  :1793-1806
 *   fade    alpha = clamp(1 - xfade / xfadelen, 0, 1) per sample, swap at the end of the callback where xfade <= 0
 *                                                                           :1808-1830
 *   wet     0 + load LL / RR, + live LL / RR, + live RL / LR ; * yrev ; width ; dry / wet mix   :1832-1876
 *
 * with the two deviations DESIGN §5 states: in the callback in which the swap completes, the new live set's LR / RL
 * (stale buffers in the reference) count as zero; the fade counts the samples a call processes (the reference counts
 * samplesPerBlock per callback), and a call longer than W leaves the last W send samples in the warmer.
 *
 * The parts are pinned to the compiled reference elsewhere: the filters (chain_oracle.c, against src/dsp/Filter.cpp)
 * and the two-stage convolvers (partconv_oracle.c, against libs/FFTConvolver).  PluginProcessor.cpp itself cannot be
 * compiled without JUCE's GUI modules, so this state machine is a restatement of those lines, not a build of them.
 * Nothing in the product may link this file.
 */
#include "chain_oracle.c"
#include "partconv_oracle.c"

typedef struct {
  int C;                                  /* 2 (LL, RR) or 4 (LL, RR, LR, RL) */
  oc_twostage* cv[4];
} oc_hs_set;

typedef struct {
  oc_chain* chain;                        /* filters, predelay ring, width / gains */
  int true_stereo;
  int W, warmwritepos;
  float* warmer[2];
  oc_hs_set live, load;
  int host_block;
  int state;                              /* 0 idle, 1 ready (warm-up at the next callback), 2 fading */
  int xfade, xfadelen;
  int swapped;                            /* the last callback completed a swap */
} oc_hotswap;

static void set_free(oc_hs_set* s) {
  for (int c = 0; c < 4; ++c) { oc_twostage_destroy(s->cv[c]); s->cv[c] = NULL; }
  s->C = 0;
}

static int set_load(oc_hs_set* s, int C, size_t head, size_t tail, const float* const* irs, size_t n) {
  set_free(s);
  s->C = C;
  for (int c = 0; c < C; ++c) {
    s->cv[c] = oc_twostage_create();
    if (!oc_twostage_init(s->cv[c], head, tail, irs[c], n)) return 0;
  }
  return 1;
}

void* oc_hs_create(double srate, float lowcut_hz, int lowcut_slope, float highcut_hz, int highcut_slope, int predelay,
                   float width, float drygain, float wetgain, int true_stereo) {
  oc_hotswap* h = (oc_hotswap*)calloc(1, sizeof(oc_hotswap));
  h->chain = (oc_chain*)oc_chain_create((float)srate, lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, predelay,
                                        1 << 20, width, drygain, wetgain);
  h->true_stereo = true_stereo;
  h->W = (int)ceil(srate) / 4;                                              /* :610 */
  for (int ch = 0; ch < 2; ++ch) h->warmer[ch] = (float*)calloc((size_t)h->W, sizeof(float));
  return h;
}

void oc_hs_destroy(void* p) {
  oc_hotswap* h = (oc_hotswap*)p;
  set_free(&h->live); set_free(&h->load);
  oc_chain_destroy(h->chain);
  free(h->warmer[0]); free(h->warmer[1]); free(h);
}

/* the live IR set (what b200conv_init_twostage + b200conv_chain_configure give the live handle) */
int oc_hs_set_live(void* p, int C, size_t head, size_t tail, const float* const* irs, size_t n) {
  return set_load(&((oc_hotswap*)p)->live, C, head, tail, irs, n);
}

/* loadConvolver->loadImpulse + loadState = kReady (:1689-1690); host_block = samplesPerBlock (convolver->size) */
int oc_hs_arm(void* p, int C, size_t head, size_t tail, const float* const* irs, size_t n, int host_block) {
  oc_hotswap* h = (oc_hotswap*)p;
  if (!set_load(&h->load, C, head, tail, irs, n)) return 0;
  h->host_block = host_block;
  h->state = 1;
  return 1;
}

int oc_hs_state(const void* p) { return ((const oc_hotswap*)p)->state; }
int oc_hs_swapped(const void* p) { return ((const oc_hotswap*)p)->swapped; }

static float clampf(float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); }

void oc_hs_process(void* p, const float* dryL, const float* dryR, const float* ysend, const float* yrev, float* outL,
                   float* outR, size_t len) {
  oc_hotswap* h = (oc_hotswap*)p;
  oc_chain* c = h->chain;
  const int n = (int)len;
  const float* dry[2] = {dryL, dryR};
  float* send[2]; float* delayed[2]; float* wet[2]; float* ylive[4]; float* yload[2];
  for (int ch = 0; ch < 2; ++ch) {
    send[ch] = (float*)malloc(len * sizeof(float)); delayed[ch] = (float*)malloc(len * sizeof(float));
    wet[ch] = (float*)calloc(len, sizeof(float)); yload[ch] = (float*)malloc(len * sizeof(float));
  }
  for (int k = 0; k < 4; ++k) ylive[k] = (float*)malloc(len * sizeof(float));
  h->swapped = 0;

  for (int ch = 0; ch < 2; ++ch)                                            /* :1640-1653 */
    for (int i = 0; i < n; ++i) {
      float v = dry[ch][i] * ysend[i];
      if (c->lowcut_on) v = oc_filter_eval(&c->lc[ch], v);
      if (c->highcut_on) v = oc_filter_eval(&c->hc[ch], v);
      send[ch][i] = v;
    }
  for (int ch = 0; ch < 2; ++ch)                                            /* :1657-1668, any call length */
    for (int i = 0; i < n; ++i) h->warmer[ch][(h->warmwritepos + i) % h->W] = send[ch][i];
  h->warmwritepos = (int)(((long long)h->warmwritepos + n) % h->W);

  if (h->state == 1) {                                                      /* :1695-1756 */
    const int size = h->host_block, W = h->W;
    const int numBlocks = W / size;
    int start = (h->warmwritepos + 1) % W;
    oc_filter lc[2], hc[2];
    float* chunk[2] = {(float*)malloc((size_t)size * sizeof(float)), (float*)malloc((size_t)size * sizeof(float))};
    float* scratch = (float*)malloc((size_t)size * sizeof(float));
    for (int ch = 0; ch < 2; ++ch) {
      lc[ch] = c->lc[ch]; oc_filter_reset(&lc[ch], 0.0f);
      hc[ch] = c->hc[ch]; oc_filter_reset(&hc[ch], 0.0f);
    }
    for (int b = 0; b < numBlocks; ++b) {
      for (int ch = 0; ch < 2; ++ch)
        for (int s = 0; s < size; ++s) chunk[ch][s] = h->warmer[ch][(start + s) % W];
      for (int s = 0; s < size; ++s)
        for (int ch = 0; ch < 2; ++ch) {
          float v = chunk[ch][s];
          if (c->lowcut_on) v = oc_filter_eval(&lc[ch], v);
          if (c->highcut_on) v = oc_filter_eval(&hc[ch], v);
          chunk[ch][s] = v;
        }
      for (int ch = 0; ch < 2; ++ch) oc_twostage_process(h->load.cv[ch], chunk[ch], scratch, (size_t)size);
      start = (start + size) % W;
    }
    free(chunk[0]); free(chunk[1]); free(scratch);
    h->state = 2;
    h->xfade = (int)ceil((double)c->srate * 50 / 1000.0);
    h->xfadelen = h->xfade;
  }

  {                                                                         /* :1767-1790 */
    const int delaySize = c->delay_size;
    for (int ch = 0; ch < 2; ++ch)
      for (int i = 0; i < n; ++i) c->delay[ch][(c->delaypos + i) % delaySize] = send[ch][i];
    const int readpos = (c->delaypos + delaySize - c->predelay) % delaySize;
    for (int ch = 0; ch < 2; ++ch)
      for (int i = 0; i < n; ++i) delayed[ch][i] = c->delay[ch][(readpos + i) % delaySize];
    c->delaypos = (c->delaypos + n) % delaySize;
  }
  for (int k = 0; k < h->live.C; ++k) oc_twostage_process(h->live.cv[k], delayed[k & 1], ylive[k], len);

  int live_ts = h->live.C == 4 && h->true_stereo;
  if (h->state == 2) {                                                      /* :1800-1830 */
    for (int ch = 0; ch < 2; ++ch) oc_twostage_process(h->load.cv[ch], send[ch], yload[ch], len);
    for (int i = 0; i < n; ++i) {
      const float alpha = clampf(1.f - (float)h->xfade / (float)h->xfadelen, 0.f, 1.f);
      ylive[0][i] *= 1.f - alpha;
      ylive[1][i] *= 1.f - alpha;
      yload[0][i] *= alpha;
      yload[1][i] *= alpha;
      if (live_ts) { ylive[2][i] *= 1.f - alpha; ylive[3][i] *= 1.f - alpha; }
      h->xfade--;
    }
    if (h->xfade <= 0) {
      /* std::swap(loadConvolver, convolver): the wet sum below reads the OLD set first, then the new one, whose
       * LR / RL were not written in this callback (zero here, DESIGN §5) */
      for (int i = 0; i < n; ++i) { wet[0][i] += ylive[0][i]; wet[1][i] += ylive[1][i]; }
      for (int i = 0; i < n; ++i) { wet[0][i] += yload[0][i]; wet[1][i] += yload[1][i]; }
      oc_hs_set t = h->live; h->live = h->load; h->load = t;
      h->state = 0;
      h->swapped = 1;
    } else {
      for (int i = 0; i < n; ++i) { wet[0][i] += yload[0][i]; wet[1][i] += yload[1][i]; }       /* :1828-1829 */
    }
  }
  if (!h->swapped) {                                                        /* :1833-1838 */
    for (int i = 0; i < n; ++i) { wet[0][i] += ylive[0][i]; wet[1][i] += ylive[1][i]; }
    if (live_ts)
      for (int i = 0; i < n; ++i) { wet[0][i] += ylive[3][i]; wet[1][i] += ylive[2][i]; }
  }
  oc_chain_wet(c, dryL, dryR, wet[0], wet[1], NULL, NULL, yrev, outL, outR, len);   /* :1840-1876 */

  for (int ch = 0; ch < 2; ++ch) { free(send[ch]); free(delayed[ch]); free(wet[ch]); free(yload[ch]); }
  for (int k = 0; k < 4; ++k) free(ylive[k]);
}
