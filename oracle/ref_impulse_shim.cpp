// TEST INFRASTRUCTURE ONLY — C entry point into the UNMODIFIED Impulse::recalcImpulse of the reference
// (src/dsp/Impulse.cpp:299-360), compiled with SVF.cpp, AudioFFT.cpp and the JUCE modules into
// oracle/_ref/librefimpulse.so (oracle/recalc.mk).  Pins recalc_oracle.c::oc_ir_recalc.
#include "JuceHeader.h"
#include "Impulse.h"

#include <algorithm>
#include <cstring>

namespace BinaryData { const char* Hall_Quad_flac = ""; const int Hall_Quad_flacSize = 0; }   // load() is never called

extern "C" {

// raw[c] / out[c]: C = 2 ({LL, RR}) or 4 ({LL, RR, LR, RL}) channels; bands as (mode, freq, q, gain) quadruples.
// Auto gain and clip are always on in recalcImpulse.  Returns the output length (out[c] must have room for out_cap taps; longer outputs are cut to out_cap).
size_t ref_impulse_recalc(const float* const* raw, int C, size_t n, double ir_srate, double srate, float stretch,
                          int reverse, float trim_left, float trim_right, float gain,
                          int n_param, const float* param_eq, int n_decay, const float* decay_eq, float decay_rate,
                          float attack, float decay, float* const* out, size_t out_cap) {
  Impulse imp;
  imp.prepare(srate);
  imp.irsrate = ir_srate;
  imp.isQuad = C == 4;
  imp.numChans = C;
  std::vector<float>* raws[4] = {&imp.rawBufferLL, &imp.rawBufferRR, &imp.rawBufferLR, &imp.rawBufferRL};
  std::vector<float>* bufs[4] = {&imp.bufferLL, &imp.bufferRR, &imp.bufferLR, &imp.bufferRL};
  for (int c = 0; c < C; ++c) {
    raws[c]->assign(raw[c], raw[c] + n);
    // the display-only peak loop (Impulse.cpp:339-345) reads numSamples = raw length taps of the resampled buffers
    bufs[c]->reserve(n);
  }
  imp.stretch = stretch;
  imp.reverse = reverse != 0;
  imp.trimLeft = trim_left;
  imp.trimRight = trim_right;
  imp.gain = gain;
  auto bands = [](int nb, const float* b) {
    std::vector<SVF::EQBand> v;
    for (int i = 0; i < nb; ++i) v.push_back({(SVF::Mode)(int)b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]});
    return v;
  };
  imp.paramEQ = bands(n_param, param_eq);
  imp.decayEQ = bands(n_decay, decay_eq);
  imp.decayRate = decay_rate;
  imp.attack = attack;
  imp.decay = decay;
  imp.recalcImpulse();
  const size_t m = imp.bufferLL.size();
  for (int c = 0; c < C; ++c) std::memcpy(out[c], bufs[c]->data(), std::min(m, out_cap) * sizeof(float));
  return m;
}

}  // extern "C"
