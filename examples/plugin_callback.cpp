// plugin_callback.cpp — what REEV-R's reverb section looks like with the whole chain on the device:
// loader thread: raw IR -> b200conv_init_twostage_shaped (shaping + partition spectra on the GPU, one upload);
// audio thread:  one b200conv_chain_process per callback (dry L/R + the two envelopes in, final mix out) instead of
//                src/PluginProcessor.cpp:1639-1653 (send + filters), :1766-1790 (predelay), :1793 (4 convolvers),
//                :1832-1876 (mixdown, reverb envelope, width, dry/wet); knob moves (an automated dry/wet ramp and
//                low-cut sweep here) go in with b200conv_chain_update before the callback's process call, as
//                onSlider / the per-block parameter reads do (:1151-1233), without resetting filters or predelay.
// The second half cross-checks the wet path against four drop-in convolver objects mixed on the host the reference's way.
//
//   g++ -O2 -std=c++17 -I include examples/plugin_callback.cpp -L reevr_b200 -l:libb200conv.so \
//       -Wl,-rpath,$PWD/reevr_b200 -o plugin_callback && ./plugin_callback
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "TwoStageFFTConvolver.h"

static std::vector<float> noise_decay(size_t n, unsigned seed)
{
  std::vector<float> h(n);
  unsigned s = seed;
  for (size_t i = 0; i < n; ++i)
  {
    s = s * 1664525u + 1013904223u;
    h[i] = ((static_cast<float>(s >> 8) / 8388608.0f) - 1.0f) * std::exp(-6.9f * static_cast<float>(i) / static_cast<float>(n));
  }
  return h;
}

int main()
{
  const double srate = 48000.0;
  const size_t hostBlock = 128, callbacks = 300, n = hostBlock * callbacks;
  const size_t taps = 60000;
  std::vector<std::vector<float>> raw = { noise_decay(taps, 1), noise_decay(taps, 2), noise_decay(taps, 3), noise_decay(taps, 4) };
  std::vector<float> L(n), R(n), ysend(n), yrev(n);
  for (size_t i = 0; i < n; ++i)
  {
    L[i] = 0.3f * std::sin(0.011f * i);
    R[i] = 0.3f * std::cos(0.017f * i);
    ysend[i] = 0.5f + 0.5f * std::fabs(std::sin(1e-3f * i));
    yrev[i] = 0.25f + 0.75f * std::fabs(std::cos(7e-4f * i));
  }

  // ---- device chain ---------------------------------------------------------------------------------------
  b200conv_config cfg = {};
  cfg.n_channels = 4; cfg.shard_count = 1;
  b200conv_t* h = b200conv_create(&cfg);
  b200conv_ir_shape_params sp = {};
  sp.autogain = 1; sp.gain = 30.0f; sp.clip = 1; sp.attack = 0.0f; sp.decay = 0.2f; sp.srate = srate;    // no decay EQ here
  const float* rawp[4] = { raw[0].data(), raw[1].data(), raw[2].data(), raw[3].data() };
  const size_t head = 128, tail = 8192;                         // StereoConvolver::prepare(128)
  if (b200conv_init_twostage_shaped(h, head, tail, rawp, taps, &sp) != B200CONV_OK)
  {
    std::printf("init failed: %s\n", b200conv_last_error(h));
    return 2;
  }
  b200conv_chain_config cc = {};
  cc.srate = srate; cc.lowcut_hz = 150.0f; cc.lowcut_slope = 1; cc.highcut_hz = 7000.0f; cc.highcut_slope = 2;
  cc.predelay = 960; cc.width = 0.7f; cc.drygain = 0.8f; cc.wetgain = 0.6f; cc.true_stereo = 1;
  if (b200conv_chain_configure(h, &cc) != B200CONV_OK) { std::printf("chain: %s\n", b200conv_last_error(h)); return 2; }
  std::vector<float> outL(n), outR(n);
  for (size_t pos = 0; pos < n; pos += hostBlock)
  {
    // automation: dry/wet from 0.2 to 0.8 (equal-power gains, :1177-1182) and the low cut from 80 Hz to 600 Hz
    const float u = static_cast<float>(pos) / static_cast<float>(n - hostBlock);
    const float theta = (0.2f + 0.6f * u) * 1.57079632679f;
    b200conv_chain_config knob = cc;
    knob.drygain = std::cos(theta); knob.wetgain = std::sin(theta); knob.lowcut_hz = 80.0f + 520.0f * u;
    if (b200conv_chain_update(h, &knob) != B200CONV_OK) { std::printf("update: %s\n", b200conv_last_error(h)); return 2; }
    const float* dry[2] = { &L[pos], &R[pos] };
    float* out[2] = { &outL[pos], &outR[pos] };
    if (b200conv_chain_process(h, dry, &ysend[pos], &yrev[pos], out, hostBlock) != B200CONV_OK)
    {
      std::printf("process: %s\n", b200conv_last_error(h));
      return 2;
    }
  }

  // ---- the same thing with the shaped taps fetched back and the per-sample work on the host -----------------
  std::vector<std::vector<float>> shaped(4, std::vector<float>(taps));
  float* shp[4] = { shaped[0].data(), shaped[1].data(), shaped[2].data(), shaped[3].data() };
  size_t m = 0;
  if (b200conv_ir_shape(0, rawp, 4, taps, &sp, shp, &m) != B200CONV_OK) return 2;
  fftconvolver::TwoStageFFTConvolver conv[4];
  for (int c = 0; c < 4; ++c) conv[c].init(head, tail, shaped[c].data(), m);
  // cross-check of the wet path: device chain with neutral filters, no predelay, dry 0 / wet 1, against four drop-in
  // convolver objects whose outputs are mixed on the host exactly as src/PluginProcessor.cpp:1832-1856 does
  cc.lowcut_hz = 20.0f; cc.highcut_hz = 20000.0f; cc.predelay = 0; cc.drygain = 0.0f; cc.wetgain = 1.0f;
  b200conv_clear(h);
  b200conv_chain_configure(h, &cc);
  double maxerr = 0.0, peak = 0.0;
  std::vector<float> bLL(hostBlock), bRR(hostBlock), bLR(hostBlock), bRL(hostBlock), sL(hostBlock), sR(hostBlock), dL(hostBlock), dR(hostBlock);
  for (size_t pos = 0; pos < n; pos += hostBlock)
  {
    for (size_t i = 0; i < hostBlock; ++i) { sL[i] = L[pos + i] * ysend[pos + i]; sR[i] = R[pos + i] * ysend[pos + i]; }
    conv[0].process(sL.data(), bLL.data(), hostBlock);
    conv[1].process(sR.data(), bRR.data(), hostBlock);
    conv[2].process(sL.data(), bLR.data(), hostBlock);
    conv[3].process(sR.data(), bRL.data(), hostBlock);
    const float* dry[2] = { &L[pos], &R[pos] };
    float* out[2] = { dL.data(), dR.data() };
    b200conv_chain_process(h, dry, &ysend[pos], &yrev[pos], out, hostBlock);
    const float norm = 1.0f / (1.0f + cc.width);
    for (size_t i = 0; i < hostBlock; ++i)
    {
      const float lin = (bLL[i] + bRL[i]) * yrev[pos + i], rin = (bRR[i] + bLR[i]) * yrev[pos + i];
      const float mid = (lin + rin) * 0.5f, side = (lin - rin) * 0.5f;
      const float lo = (mid + side * cc.width) * norm, ro = (mid - side * cc.width) * norm;
      maxerr = std::max(maxerr, (double)std::fabs(lo - dL[i]));
      maxerr = std::max(maxerr, (double)std::fabs(ro - dR[i]));
      peak = std::max(peak, (double)std::fabs(lo));
    }
  }
  b200conv_destroy(h);
  std::printf("rendered %zu callbacks of %zu samples; device chain vs host-side mix: max err %.3g of peak %.3g (%.2e)\n",
              callbacks, hostBlock, maxerr, peak, maxerr / peak);
  return maxerr <= 1e-5 * peak ? 0 : 1;
}
