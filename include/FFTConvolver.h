// FFTConvolver.h — drop-in replacement for libs/FFTConvolver/FFTConvolver.h of tiagolr/reevr.
//
// Same namespace, class name and public surface as the reference
// (libs/FFTConvolver/FFTConvolver.h:62-80: init / process / clear / reset, `Sample` = float,
// Utilities.h:180); everything behind it runs on the GPU through the C ABI of b200conv.h.
// Header-only: put this directory on the include path instead of libs/FFTConvolver and link
// libb200conv.so (see INTEGRATION.md).  Written from scratch — no reference code.
//
// Behavioural contract kept from the reference:
//   * init() returns false only for blockSize == 0; an empty / all-below-1e-6 IR is a success and
//     process() then writes zeros (FFTConvolver.cpp:97-111,157-161);
//   * process() accepts any len, adds no latency, output complete on return, in/out must not alias;
//   * process()/clear()/reset() are void and never throw.  If the GPU call fails the output is
//     zero-filled, the error is kept (lastError()) and reported once on stderr — there is no CPU
//     fall-back path.
#ifndef B200CONV_FFTCONVOLVER_H
#define B200CONV_FFTCONVOLVER_H

#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "b200conv.h"

namespace fftconvolver
{

typedef float Sample;

namespace detail
{
inline int deviceFromEnv()
{
  const char* e = std::getenv("B200CONV_DEVICE");
  return e ? std::atoi(e) : 0;
}

// One C-ABI handle with a single channel; shared by both convolver classes.
class Handle
{
public:
  Handle() : _h(nullptr), _reported(false) {}
  ~Handle() { if (_h) b200conv_destroy(_h); }

  b200conv_t* get()
  {
    if (!_h)
    {
      b200conv_config cfg;
      std::memset(&cfg, 0, sizeof(cfg));
      cfg.n_channels = 1;
      cfg.device = deviceFromEnv();
      cfg.shard_count = 1;
      _h = b200conv_create(&cfg);
    }
    return _h;
  }

  // maps a C-ABI status to the reference's bool / void conventions
  bool ok(int status, const char* what)
  {
    if (status == B200CONV_OK)
      return true;
    _error = std::string(what) + ": " + (_h ? b200conv_last_error(_h) : "no handle");
    if (!_reported && status != B200CONV_EINVAL)
    {
      std::fprintf(stderr, "[b200conv] %s (status %d)\n", _error.c_str(), status);
      _reported = true;
    }
    return false;
  }

  const std::string& error() const { return _error; }

  // fixed-latency mode (b200conv_set_latency) of the handle; 0 without one
  bool setLatency(size_t samples) { return ok(b200conv_set_latency(get(), samples), "setLatency"); }
  size_t latency() const { return _h ? b200conv_latency(_h) : 0; }

private:
  b200conv_t* _h;
  std::string _error;
  bool _reported;
  Handle(const Handle&);
  Handle& operator=(const Handle&);
};
} // namespace detail


class FFTConvolver
{
public:
  FFTConvolver() {}
  virtual ~FFTConvolver() {}

  bool init(size_t blockSize, const Sample* ir, size_t irLen)
  {
    const float* irs[1] = { ir };
    const size_t lens[1] = { ir ? irLen : 0 };
    return _handle.ok(b200conv_init_uniform(_handle.get(), blockSize, irs, lens), "FFTConvolver::init");
  }

  void process(const Sample* input, Sample* output, size_t len)
  {
    if (len == 0)
      return;
    const float* in[1] = { input };
    float* out[1] = { output };
    if (!_handle.ok(b200conv_process(_handle.get(), in, out, len), "FFTConvolver::process"))
      std::memset(output, 0, len * sizeof(Sample));
  }

  void clear() { _handle.ok(b200conv_clear(_handle.get()), "FFTConvolver::clear"); }
  void reset() { _handle.ok(b200conv_reset(_handle.get()), "FFTConvolver::reset"); }

  // additions (not in the reference)
  const char* lastError() const { return _handle.error().c_str(); }
  // fixed-latency mode: process() returns its output `samples` later (0, or a multiple of the block size up to 16
  // blocks), so that the call never waits for the GPU while it keeps up; after init(), which returns to zero latency.
  // Clears the convolver.  Report getLatency() to the host (JUCE setLatencySamples).
  bool setLatency(size_t samples) { return _handle.setLatency(samples); }
  size_t getLatency() const { return _handle.latency(); }

private:
  detail::Handle _handle;
  FFTConvolver(const FFTConvolver&);
  FFTConvolver& operator=(const FFTConvolver&);
};

} // namespace fftconvolver

#endif
