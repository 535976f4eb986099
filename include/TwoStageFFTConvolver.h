// TwoStageFFTConvolver.h — drop-in replacement for libs/FFTConvolver/TwoStageFFTConvolver.h.
//
// Same namespace, class name, public surface (init / process / reset / clear,
// TwoStageFFTConvolver.h:65-83) and the same PROTECTED hooks the reference exposes for moving
// the tail into the background (startBackgroundProcessing / waitForBackgroundProcessing virtual,
// doBackgroundProcessing non-virtual, :94-106), so that REEV-R's `class Convolver : public
// fftconvolver::TwoStageFFTConvolver` (src/dsp/Convolver.h:28, Convolver.cpp:84-95) compiles and
// runs unchanged.  On the GPU the tail stage is just more kernels on the handle's stream — it is
// enqueued the moment a tail block completes and consumed (stream-ordered) one tail block
// later, so the hooks have nothing left to compute; they are still invoked at every tail-block
// boundary in the reference's order (wait, then start — TwoStageFFTConvolver.cpp:213-222) so a
// subclass's thread/event protocol (e.g. Convolver::isFinished()) keeps working.
#ifndef B200CONV_TWOSTAGEFFTCONVOLVER_H
#define B200CONV_TWOSTAGEFFTCONVOLVER_H

#include "FFTConvolver.h"

namespace fftconvolver
{

class TwoStageFFTConvolver
{
public:
  TwoStageFFTConvolver() : _tailBlockSize(0), _tailFill(0), _hasTail(false) {}
  virtual ~TwoStageFFTConvolver() {}

  bool init(size_t headBlockSize, size_t tailBlockSize, const Sample* ir, size_t irLen)
  {
    _tailBlockSize = 0;
    _tailFill = 0;
    _hasTail = false;
    const float* irs[1] = { ir };
    const size_t lens[1] = { ir ? irLen : 0 };
    b200conv_t* h = _handle.get();
    if (!_handle.ok(b200conv_init_twostage(h, headBlockSize, tailBlockSize, irs, lens), "TwoStageFFTConvolver::init"))
      return false;
    // a tail stage exists iff the (trimmed) IR is longer than two tail blocks (TwoStageFFTConvolver.cpp:131)
    if (b200conv_num_stages(h) == 2)
    {
      b200conv_stage_info info;
      if (b200conv_stage(h, 1, &info) == B200CONV_OK)
      {
        // hook cadence = the tail block size the caller asked for, rounded like the reference does
        // (TwoStageFFTConvolver.cpp:100-104,118); the engine may use smaller partitions internally
        size_t t = headBlockSize > tailBlockSize ? headBlockSize : tailBlockSize;
        size_t p = 1;
        while (p < t) p *= 2;
        _tailBlockSize = p > info.block ? p : info.block;
        _hasTail = true;
      }
    }
    return true;
  }

  void process(const Sample* input, Sample* output, size_t len)
  {
    if (len == 0)
      return;
    const float* in[1] = { input };
    float* out[1] = { output };
    if (!_handle.ok(b200conv_process(_handle.get(), in, out, len), "TwoStageFFTConvolver::process"))
      std::memset(output, 0, len * sizeof(Sample));
    if (_hasTail)
    {
      // one wait/start pair per completed tail block, as the reference issues them
      _tailFill += len;
      while (_tailFill >= _tailBlockSize)
      {
        _tailFill -= _tailBlockSize;
        waitForBackgroundProcessing();
        startBackgroundProcessing();
      }
    }
  }

  void reset()
  {
    _handle.ok(b200conv_reset(_handle.get()), "TwoStageFFTConvolver::reset");
    _tailBlockSize = 0;
    _tailFill = 0;
    _hasTail = false;
  }

  void clear()
  {
    _handle.ok(b200conv_clear(_handle.get()), "TwoStageFFTConvolver::clear");
    _tailFill = 0;
  }

  const char* lastError() const { return _handle.error().c_str(); }
  // fixed-latency mode (additions, not in the reference): see FFTConvolver::setLatency; a multiple of the head block
  bool setLatency(size_t samples) { return _handle.setLatency(samples); }
  size_t getLatency() const { return _handle.latency(); }

protected:
  virtual void startBackgroundProcessing() { doBackgroundProcessing(); }
  virtual void waitForBackgroundProcessing() {}
  void doBackgroundProcessing() {}   // tail work already queued on the GPU stream by process()

private:
  detail::Handle _handle;
  size_t _tailBlockSize;
  size_t _tailFill;
  bool _hasTail;
  TwoStageFFTConvolver(const TwoStageFFTConvolver&);
  TwoStageFFTConvolver& operator=(const TwoStageFFTConvolver&);
};

} // namespace fftconvolver

#endif
