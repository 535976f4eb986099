// latency_dropin_test.cpp — the drop-in classes' setLatency: the output of a convolver with latency D equals the
// output of the same convolver at zero latency, delayed by D samples, for head-block calls and for ragged calls.
#include <cmath>
#include <cstdio>
#include <vector>

#include "FFTConvolver.h"
#include "TwoStageFFTConvolver.h"

static std::vector<float> signal(size_t n, unsigned seed) {
  std::vector<float> v(n);
  unsigned s = seed * 2654435761u + 1;
  for (size_t i = 0; i < n; ++i) {
    s = s * 1664525u + 1013904223u;
    v[i] = (float)((s >> 8) & 0xffff) / 32768.0f - 1.0f;
  }
  return v;
}

static std::vector<float> ir(size_t n, unsigned seed) {
  std::vector<float> v = signal(n, seed);
  for (size_t i = 0; i < n; ++i) v[i] *= std::exp(-4.0f * (float)i / (float)n);
  return v;
}

template <class Conv>
static std::vector<float> run(Conv& c, const std::vector<float>& x, const std::vector<size_t>& calls) {
  std::vector<float> y(x.size());
  size_t pos = 0;
  for (size_t m : calls) {
    c.process(x.data() + pos, y.data() + pos, m);
    pos += m;
  }
  return y;
}

// zero-latency output z, latency output y (delay D): y[:D] == 0 and y[D:] ~ z[:-D]
static bool shifted(const std::vector<float>& y, const std::vector<float>& z, size_t D, float tol, const char* what) {
  float peak = 0.0f, err = 0.0f;
  for (size_t i = 0; i < D; ++i)
    if (y[i] != 0.0f) { std::printf("%s: sample %zu before the latency is %g\n", what, i, y[i]); return false; }
  for (size_t i = D; i < y.size(); ++i) {
    peak = std::fmax(peak, std::fabs(z[i - D]));
    err = std::fmax(err, std::fabs(y[i] - z[i - D]));
  }
  if (err > tol * peak) { std::printf("%s: error %g of peak %g\n", what, err, peak); return false; }
  return true;
}

int main() {
  const size_t B = 64, n = 188 * B;
  const std::vector<float> x = signal(n, 3), h = ir(4000, 7);
  std::vector<size_t> even(n / B, B), ragged;
  const size_t pat[] = {B / 3, B - B / 3, 1, 2 * B + 5, B - 6, 700, B, 3};
  for (size_t tot = 0, i = 0; tot < n; ++i) {
    const size_t m = std::min(pat[i % 8], n - tot);
    ragged.push_back(m);
    tot += m;
  }
  bool ok = true;
  {
    fftconvolver::FFTConvolver z, f;
    z.init(B, h.data(), h.size());
    f.init(B, h.data(), h.size());
    ok = ok && !f.setLatency(B / 2) && f.getLatency() == 0;           // not a multiple of the block
    ok = ok && f.setLatency(2 * B) && f.getLatency() == 2 * B;
    const std::vector<float> yz = run(z, x, even), yf = run(f, x, even);
    ok = ok && shifted(yf, yz, 2 * B, 0.0f, "FFTConvolver");
    f.clear();
    ok = ok && f.getLatency() == 2 * B;
    fftconvolver::FFTConvolver z2;
    z2.init(B, h.data(), h.size());
    ok = ok && shifted(run(f, x, ragged), run(z2, x, even), 2 * B, 1e-6f, "FFTConvolver ragged");
    f.init(B, h.data(), h.size());
    ok = ok && f.getLatency() == 0;
  }
  {
    fftconvolver::TwoStageFFTConvolver z, f;
    z.init(B, 512, h.data(), h.size());
    f.init(B, 512, h.data(), h.size());
    ok = ok && f.setLatency(B) && f.getLatency() == B;
    ok = ok && shifted(run(f, x, ragged), run(z, x, even), B, 1e-6f, "TwoStageFFTConvolver");
    f.reset();
    ok = ok && f.getLatency() == 0;
  }
  std::printf(ok ? "ALL OK\n" : "FAILED\n");
  return ok ? 0 : 1;
}
