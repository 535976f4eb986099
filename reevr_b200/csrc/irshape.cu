// irshape.cu — SURVEY 8f-3: REEV-R's IR recalculation (Impulse::recalcImpulse, src/dsp/Impulse.cpp:299-360) on the device.
//
// Impulse::applyDecay (src/dsp/Impulse.cpp:602-648): 4096-point STFT, hop 1024 (Impulse.h:21-22),
// analysis window of Impulse.cpp:65-69, per-bin decay that compounds once per block after the
// early-reflection blocks (:612, :626-633), inverse transform, overlap-add normalised by the summed
// window (:637-648).  On the device every STFT block is independent: the compounded decay of block b
// is lut[k]^(b - skip) in closed form, so all blocks are transformed, scaled and inverse-transformed
// in three batched launches and a fourth kernel gathers the (up to 4) overlapping blocks per sample.
// Reuses the Stockham passes / split functions of kernels.cuh (M = 2048 complex points per 4096 real).
//
// Around it, the rest of recalcImpulse in the reference's order (second half of this file): auto gain, reverse,
// resampling to the project rate and stretch (JUCE ResamplingAudioSource: closed-form linear interpolation, the second-
// order low pass as a chunked FP64 scan), trim, gain, the parametric EQ (SVF sections as chunked FP32 scans), the decay
// EQ with its table built from the bands on the host, clip and envelope.  Every kernel is a set of PC_HD phase
// functions, so the CPU emulation build (tests/emu) runs the same index arithmetic.
#if defined(PC_EMULATE)
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/b200conv.h"
#include "kernels.cuh"

namespace {

constexpr int kN = 4096;          // STFT size (Impulse.h:21)
constexpr int kM = kN / 2;        // complex points of the real transform
constexpr int kHop = kN / 4;      // Impulse.h:22

// analysis-windowed block straight from global memory: z[n] = (x[2n] w[2n], x[2n+1] w[2n+1])
struct StftIn {
  const float* src; const float* win; int nv;
  PC_HD int prep(int base) const { return base; }
  PC_HD float2 at(int tok, int off) const {
    const int i0 = 2 * (tok + off), i1 = i0 + 1;
    return make_float2(i0 < nv ? src[i0] * win[i0] : 0.0f, i1 < nv ? src[i1] * win[i1] : 0.0f);
  }
};
// last inverse pass: all 2M samples of the block, scaled, to a dense scratch row
struct StftOut {
  float* dst; float scale;
  PC_HD int prep(int base) const { return base; }
  PC_HD void put(int tok, int off, float2 v) const {
    const int n = tok + off;
    dst[2 * n] = v.x * scale;
    dst[2 * n + 1] = v.y * scale;
  }
};

// spectrum row of block b scaled by lut^m (m = b - skip > 0); entry 0 packs (DC, Nyquist): DC is left alone
// (the reference loop starts at k = 1, Impulse.cpp:627) and the Nyquist bin uses lut[M]
PC_HD void decay_scale(float2* row, const double* lut, int m, int k) {
  if (m <= 0) return;
  if (k == 0) { row[0].y *= (float)std::pow(lut[kM], (double)m); return; }
  const float g = (float)std::pow(lut[k], (double)m);
  row[k].x *= g;
  row[k].y *= g;
}

// out[i] = sum over the blocks covering i of scratch[b][i - b*hop], divided by the summed window (:637-648)
PC_HD float stft_gather(const float* scratch, const float* win, long long n, long long nblocks, long long i) {
  float acc = 0.0f, norm = 0.0f;
  const long long b_hi = i / kHop;
  for (long long b = b_hi; b >= 0 && b > b_hi - kN / kHop; --b) {
    if (b >= nblocks) continue;
    const long long off = i - b * kHop;
    if (off < kN) { acc += scratch[b * kN + off]; norm += win[off]; }
  }
  (void)n;
  return norm > 0.0f ? acc / norm : 0.0f;
}

#if !defined(PC_EMULATE)
__global__ void __launch_bounds__(512) k_stft_fwd(const float* x, long long n, const float* win, const float2* tw, float2* spec, long long nblocks) {
  extern __shared__ float2 sm[];
  const long long b = blockIdx.x;
  if (b >= nblocks) return;
  constexpr int NT = pc::fft_threads(kM);
  const int tx = threadIdx.x;
  float2* bufA = sm; float2* bufB = sm + kM;
  const long long start = b * kHop;
  const long long rem = n - start;
  const int nv = rem > kN ? kN : (int)rem;
  constexpr int R0 = pc::pass_radix(kM, 1);
  for (int i = tx; i < kM / R0; i += NT)
    pc::stockham_butterfly<false>(StftIn{x + start, win, nv}, pc::SmemOut{bufA}, tw + pc::tw_pass_offset(kM, 1), kM, 1, R0, i);
  __syncthreads();
  float2* res = pc::fft_mid_passes<false, kM, R0>(bufA, bufB, tw, tx, true);
  float2* row = spec + b * kM;
  for (int k = tx; k <= kM / 2; k += NT) pc::fwd_split(res, row, tw, kM, k);
}

__global__ void k_stft_decay(float2* spec, const double* lut, long long nblocks, int skip) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const long long b = blockIdx.y;
  if (k < kM && b < nblocks) decay_scale(spec + b * kM, lut, (int)(b - skip), k);
}

__global__ void __launch_bounds__(512) k_stft_inv(const float2* spec, const float2* zero_row, const float2* tw, float* scratch, long long nblocks) {
  extern __shared__ float2 sm[];
  const long long b = blockIdx.x;
  if (b >= nblocks) return;
  constexpr int NT = pc::fft_threads(kM);
  const int tx = threadIdx.x;
  float2* bufA = sm; float2* bufB = sm + kM;
  const float2* row = spec + b * kM;
  for (int k = tx; k <= kM / 2; k += NT) pc::inv_pre(row, zero_row, bufA, tw, kM, k, 1, 0);
  __syncthreads();
  float2* in = pc::fft_mid_passes<true, kM, 1>(bufA, bufB, tw, tx, true);
  // last pass (the one that reaches length M) writes all 2M samples of the block
  int p = 1;
  while (p * pc::pass_radix(kM, p) != kM) p *= pc::pass_radix(kM, p);
  const int R = pc::pass_radix(kM, p);
  for (int i = tx; i < kM / R; i += NT)
    pc::stockham_butterfly<true>(pc::SmemIn{in}, StftOut{scratch + b * kN, 1.0f / (float)kM}, tw + pc::tw_pass_offset(kM, p), kM, p, R, i);
}

__global__ void k_stft_gather(const float* scratch, const float* win, float* out, long long n, long long nblocks) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = stft_gather(scratch, win, n, nblocks, i);
}
#endif

// host reference of the per-block pipeline for the emulation build (same phase functions, loops for threads)
#if defined(PC_EMULATE)
void emu_stft(const float* x, long long n, const float* win, const float2* tw, const double* lut, int skip, float* out) {
  const long long nblocks = (n + kHop - 1) / kHop;
  std::vector<float2> spec((size_t)nblocks * kM), bufA(kM), bufB(kM), zero(kM, make_float2(0.f, 0.f));
  std::vector<float> scratch((size_t)nblocks * kN, 0.0f);
  for (long long b = 0; b < nblocks; ++b) {
    const long long start = b * kHop, rem = n - start;
    const int nv = rem > kN ? kN : (int)rem;
    const int R0 = pc::pass_radix(kM, 1);
    for (int i = 0; i < kM / R0; ++i)
      pc::stockham_butterfly<false>(StftIn{x + start, win, nv}, pc::SmemOut{bufA.data()}, tw + pc::tw_pass_offset(kM, 1), kM, 1, R0, i);
    float2* in = bufA.data(); float2* o = bufB.data();
    for (int p = R0; p < kM;) {
      const int R = pc::pass_radix(kM, p);
      for (int i = 0; i < kM / R; ++i) pc::stockham_butterfly<false>(pc::SmemIn{in}, pc::SmemOut{o}, tw + pc::tw_pass_offset(kM, p), kM, p, R, i);
      std::swap(in, o);
      p *= R;
    }
    float2* row = spec.data() + b * kM;
    for (int k = 0; k <= kM / 2; ++k) pc::fwd_split(in, row, tw, kM, k);
    for (int k = 0; k < kM; ++k) decay_scale(row, lut, (int)(b - skip), k);
    for (int k = 0; k <= kM / 2; ++k) pc::inv_pre(row, zero.data(), bufA.data(), tw, kM, k, 1, 0);
    in = bufA.data(); o = bufB.data();
    for (int p = 1; p < kM;) {
      const int R = pc::pass_radix(kM, p);
      const bool last = p * R == kM;
      for (int i = 0; i < kM / R; ++i) {
        if (!last) pc::stockham_butterfly<true>(pc::SmemIn{in}, pc::SmemOut{o}, tw + pc::tw_pass_offset(kM, p), kM, p, R, i);
        else pc::stockham_butterfly<true>(pc::SmemIn{in}, StftOut{scratch.data() + b * kN, 1.0f / (float)kM}, tw + pc::tw_pass_offset(kM, p), kM, p, R, i);
      }
      std::swap(in, o);
      p *= R;
    }
  }
  for (long long i = 0; i < n; ++i) out[i] = stft_gather(scratch.data(), win, n, nblocks, i);
}
#endif

}  // namespace

// window (Impulse.cpp:65-69) and twiddles on the host, in the layout of kernels.cuh
static void stft_tables(std::vector<float>& win, std::vector<float2>& tw) {
  win.resize(kN);
  const float step = 2.0f * 3.14159265358979323846f / (float)kN;
  for (int i = 0; i < kN / 2; ++i) win[i] = 0.42f - 0.50f * std::cos((float)i * step) + 0.08f * std::cos(2.0f * (float)i * step);
  for (int i = kN / 2; i < kN; ++i) win[i] = win[kN - 1 - i];
  tw.resize(pc::tw_table_len(kM));
  for (int k = 0; k <= kM / 2; ++k) {
    const double a = -2.0 * M_PI * (double)k / (2.0 * (double)kM);
    tw[k] = make_float2((float)std::cos(a), (float)std::sin(a));
  }
  for (int p = 1; p < kM;) {
    const int R = pc::pass_radix(kM, p);
    const int off = pc::tw_pass_offset(kM, p);
    for (int r = 1; r < R; ++r)
      for (int k = 0; k < p; ++k) {
        const double a = -2.0 * M_PI * (double)r * (double)k / ((double)p * (double)R);
        tw[off + (r - 1) * p + k] = make_float2((float)std::cos(a), (float)std::sin(a));
      }
    p *= R;
  }
}

// The decay-EQ STFT on DEVICE-resident taps, in place, C channels of n taps at dx + c * stride: one set of tables and
// scratch buffers for all channels, everything on stream st (no host synchronisation inside).
struct DecayScratch {
  float* dwin = nullptr; float* dscratch = nullptr; float* dtmp = nullptr;
  float2* dtw = nullptr; float2* dspec = nullptr; float2* dzero = nullptr; double* dlut = nullptr;
  void release() {
    cudaFree(dwin); cudaFree(dscratch); cudaFree(dtmp); cudaFree(dtw); cudaFree(dspec); cudaFree(dzero); cudaFree(dlut);
    *this = DecayScratch();
  }
};

static bool decay_eq_device(float* dx, size_t stride, int C, size_t n, const double* lut, double srate, cudaStream_t st,
                            DecayScratch& sc, std::vector<float>& win, std::vector<float2>& tw) {
  if (n == 0) return true;
  stft_tables(win, tw);
  const int skip = (int)std::ceil(100.0 * srate / (1000.0 * (double)kN));       // EARLY_REFLECTIONS_MS = 100, :612
  const long long nblocks = ((long long)n + kHop - 1) / kHop;
#if defined(PC_EMULATE)
  (void)st; (void)sc;
  std::vector<float> out(n);
  for (int c = 0; c < C; ++c) {
    emu_stft(dx + (size_t)c * stride, (long long)n, win.data(), tw.data(), lut, skip, out.data());
    std::memcpy(dx + (size_t)c * stride, out.data(), n * sizeof(float));
  }
  return true;
#else
  const size_t smem = 2 * kM * sizeof(float2);
  if (!sc.dtmp) {        // scratch and tables once per shaping job, shared by all channels (same n)
    bool ok = cudaMalloc(&sc.dtmp, n * sizeof(float)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dwin, kN * sizeof(float)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dtw, tw.size() * sizeof(float2)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dlut, (kM + 1) * sizeof(double)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dspec, (size_t)nblocks * kM * sizeof(float2)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dzero, kM * sizeof(float2)) == cudaSuccess;
    ok = ok && cudaMalloc(&sc.dscratch, (size_t)nblocks * kN * sizeof(float)) == cudaSuccess;
    if (!ok) return false;
    cudaFuncSetAttribute(k_stft_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(k_stft_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaMemcpyAsync(sc.dwin, win.data(), kN * sizeof(float), cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(sc.dtw, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(sc.dlut, lut, (kM + 1) * sizeof(double), cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(sc.dzero, 0, kM * sizeof(float2), st);
  }
  const int NT = pc::fft_threads(kM);
  for (int c = 0; c < C; ++c) {
    float* x = dx + (size_t)c * stride;
    k_stft_fwd<<<(unsigned)nblocks, NT, smem, st>>>(x, (long long)n, sc.dwin, sc.dtw, sc.dspec, nblocks);
    k_stft_decay<<<dim3((kM + 255) / 256, (unsigned)nblocks), 256, 0, st>>>(sc.dspec, sc.dlut, nblocks, skip);
    k_stft_inv<<<(unsigned)nblocks, NT, smem, st>>>(sc.dspec, sc.dzero, sc.dtw, sc.dscratch, nblocks);
    k_stft_gather<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(sc.dscratch, sc.dwin, sc.dtmp, (long long)n, nblocks);
    cudaMemcpyAsync(x, sc.dtmp, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
  }
  return cudaGetLastError() == cudaSuccess;
#endif
}

extern "C" int b200conv_ir_decay_eq(int device, float* ir, size_t n, const double* lut, double srate) {
  if (!ir || !lut) return B200CONV_EINVAL;
  if (n == 0) return B200CONV_OK;
  std::vector<float> win; std::vector<float2> tw;
#if defined(PC_EMULATE)
  (void)device;
  DecayScratch sc;
  decay_eq_device(ir, n, 1, n, lut, srate, nullptr, sc, win, tw);
  return B200CONV_OK;
#else
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return B200CONV_ECUDA; }
  float* dx = nullptr;
  cudaStream_t st = nullptr;
  DecayScratch sc;
  bool ok = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaMalloc(&dx, n * sizeof(float)) == cudaSuccess;
  if (ok) {
    cudaMemcpyAsync(dx, ir, n * sizeof(float), cudaMemcpyHostToDevice, st);
    ok = decay_eq_device(dx, n, 1, n, lut, srate, st, sc, win, tw);
    cudaMemcpyAsync(ir, dx, n * sizeof(float), cudaMemcpyDeviceToHost, st);
    ok = ok && cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess;
  }
  sc.release();
  cudaFree(dx);
  if (st) cudaStreamDestroy(st);
  if (!ok) { cudaGetLastError(); return B200CONV_ECUDA; }
  return B200CONV_OK;
#endif
}

// ---------------------------------------------------------------------------------------------------------
// Impulse::recalcImpulse (src/dsp/Impulse.cpp:299-360) on the device, in the reference's order:
// auto gain (:313-324, calculateAutoGain :691-709) -> reverse (:326-334) -> resampling to the project rate (:362-389) ->
// stretch (:391-434) -> trim (:436-470) -> gain (:472-486) -> parametric EQ (:503-537) -> decay EQ (:539-648) ->
// clip (:488-501) -> attack / decay envelope (:651-680).
// Without resampling and stretch, auto gain, reverse, trim and gain are one fused gather (k_ir_pick); with either, the
// gather splits around them so that (v * autogain) is rounded before the resampler, as in the reference.
// ---------------------------------------------------------------------------------------------------------
namespace {
// dst[i] = (raw[src index of i] * autogain) * gain, src index = trim start + i, mirrored when reversed
PC_HD float ir_pick(const float* raw, long long n_raw, long long start, int reverse, float ag, float g, long long i) {
  const long long j = start + i;
  const float v = raw[reverse ? n_raw - 1 - j : j];
  return (v * ag) * g;
}
PC_HD float ir_clip_env(float v, int clip, long long i, long long n, long long attack_n, long long decay_n) {
  if (clip) v = v < -1.0f ? -1.0f : (v > 1.0f ? 1.0f : v);
  if (i < attack_n) v *= (float)i / (float)attack_n;
  if (i >= n - decay_n) {
    const float t = (float)(i - (n - decay_n)) / (float)decay_n;
    v *= 1.0f - (float)std::pow((double)t, 0.5);
  }
  return v;
}

// ---- JUCE ResamplingAudioSource (juce_ResamplingAudioSource.cpp:92-275) ----
// createLowPass (:210-243), normalised by c4 = 1: y = c0 x + c1 x1 + c2 x2 - c4 y1 - c5 y2, in double (applyFilter :251-275)
struct RsLowPass { double c0, c1, c2, c4, c5; };

// the low pass over one stream x (zero beyond nx) as a linear recursion in the two past outputs s = (y1, y2); the past
// inputs are read from x.  Writes scale * (float)y.
struct RsFilterRec {
  using T = double;
  const float* x; long long x_stride, nx;
  float* y; long long y_stride;
  float scale;
  RsLowPass f;
  PC_HD double in(int ch, long long i) const { return i >= 0 && i < nx ? (double)x[ch * x_stride + i] : 0.0; }
  PC_HD double step(int ch, long long i, double* s) const {
    double out = f.c0 * in(ch, i) + f.c1 * in(ch, i - 1) + f.c2 * in(ch, i - 2) - f.c4 * s[0] - f.c5 * s[1];
    if (!(out < -1.0e-8 || out > 1.0e-8)) out = 0.0;          // JUCE_INTEL flush (:263-266)
    s[1] = s[0];
    s[0] = out;
    return out;
  }
  PC_HD void free_step(double* s) const {
    const double out = -f.c4 * s[0] - f.c5 * s[1];
    s[1] = s[0];
    s[0] = out;
  }
  PC_HD void put(int ch, long long i, double v) const { y[ch * y_stride + i] = (float)v * scale; }
};

// output m of the linear interpolator (:155-177) at the input position m * ratio in closed form.  JUCE accumulates the
// position serially (subSampleOffset); the two can only disagree where it crosses an integer, where the interpolant is
// continuous, so the outputs still agree.
PC_HD float rs_interp(const float* x, long long nx, double ratio, long long m) {
  const double pos = (double)m * ratio;
  const long long i = (long long)pos;
  const float alpha = (float)(pos - (double)i);
  const float a = i < nx ? x[i] : 0.0f, b = i + 1 < nx ? x[i + 1] : 0.0f;
  return a + alpha * (b - a);
}

// ---- SVF sections of the parametric EQ (src/dsp/SVF.cpp:113-137, processBlock :139-209, processBlock6dB :211-245) ----
// applyParamEQ passes each filter its own freq / q / gain, so the interpolation steps are zero: constant coefficients
struct SvfCoeffs {
  int mode;                          // SVF::Mode after Impulse.cpp's mapping (Off and unknown -> PK)
  float g, r2, a1, a2, a3, cl, cb, ch;
};
constexpr int kSvfHP6 = 7, kSvfLP6 = 8;
// F = float: the reference's arithmetic.  F = double: the same equations from the same float coefficients (A^L)
template <class F>
PC_HD F svf_step(const SvfCoeffs& f, F* s, F x) {
  if (f.mode == kSvfHP6 || f.mode == kSvfLP6) {
    const F delta = (F)f.g * (x - s[0]);
    s[0] += delta;
    return f.mode == kSvfLP6 ? s[0] : x - s[0];
  }
  const F v3 = x - s[1];
  const F v1 = (F)f.a1 * s[0] + (F)f.a2 * v3;
  const F v2 = s[1] + (F)f.a2 * s[0] + (F)f.a3 * v3;
  s[0] = (F)2 * v1 - s[0];
  s[1] = (F)2 * v2 - s[1];
  return (F)f.cl * v2 + (F)f.cb * v1 + (F)f.ch * (x - (F)f.r2 * v1 - v2);
}
// one section in place over C channels (channel stride `stride`), state s = (s1, s2) from zero (SVF::clear(0), :247-251)
struct SvfRec {
  using T = float;
  float* x; long long stride;
  SvfCoeffs f;
  PC_HD float step(int ch, long long i, float* s) const { return svf_step<float>(f, s, x[ch * stride + i]); }
  PC_HD void free_step(double* s) const { (void)svf_step<double>(f, s, 0.0); }
  PC_HD void put(int ch, long long i, float v) const { x[ch * stride + i] = v; }
};

// ---- chunked form of a 2-state linear recursion, the scheme of k_chain_send (kernels_chain.cuh:14-33) ----
// kScanThreads chunks of L = ceil(n / kScanThreads) samples per channel: pass 1 runs every chunk from a zero state,
// A^L comes from the zero-input response to the unit states, one thread scans S_{t+1} = A^L S_t + Z_t from S_0 = 0
// (every channel starts from a zero state), pass 2 re-runs every chunk from its true state and writes.
// Precision: the chunks run in the recursion's own type (float for the SVF, in the reference's order; double for the
// resampler); A^L (the zero-input response of the same step equations) and the scan always run in double, and the
// states handed to pass 2 are rounded to the chunk type.  A low band at 96 / 192 kHz puts the poles within ~1e-4 of
// the unit circle, where an error in S_t persists for tens of chunks: with A^L and the scan in float the SVF chunked
// form was up to 5e-5 of peak from a float64 serial filter, 20-30x the serial float filter's own error; with them in
// double it was 3e-7 for a 20 Hz, Q 8, +24 dB low shelf at 96 kHz (serial float: 1.6e-6) and never more than 1.7x
// the serial float filter's error (tests/test_scan_precision.py).  The resampler's flush of |y| <= 1e-8 to zero is
// the one non-linear step; it is applied inside the chunks (both passes), so the chunked form can differ from the
// serial one there by less than 1e-8 per sample, fed into a stable filter.
constexpr int kScanThreads = 1024;

PC_HD void scan_bounds(int t, long long L, long long n, long long& i0, long long& i1) {
  i0 = (long long)t * L < n ? (long long)t * L : n;
  i1 = i0 + L < n ? i0 + L : n;
}
template <class R>
PC_HD void scan_chunk(const R& rec, int ch, long long i0, long long i1, typename R::T* s, bool write) {
  for (long long i = i0; i < i1; ++i) {
    const typename R::T y = rec.step(ch, i, s);
    if (write) rec.put(ch, i, y);
  }
}
template <class R>
PC_HD void scan_power_column(const R& rec, long long L, int j, double* col) {
  col[0] = j == 0 ? 1 : 0;
  col[1] = j == 1 ? 1 : 0;
  for (long long i = 0; i < L; ++i) rec.free_step(col);
}
// Z[t]: zero-state end point of chunk t on entry, the initial state of chunk t (rounded to T) on exit;
// AL[q][j] = (A^L)_qj; the scan runs in double
template <class T>
PC_HD void scan_states(T (*Z)[2], const double (*AL)[2], int nt, long long L, long long n) {
  double s0 = 0, s1 = 0;
  for (int c = 0; c < nt; ++c) {
    const double n0 = (double)Z[c][0] + AL[0][0] * s0 + AL[0][1] * s1;
    const double n1 = (double)Z[c][1] + AL[1][0] * s0 + AL[1][1] * s1;
    Z[c][0] = (T)s0;
    Z[c][1] = (T)s1;
    if ((long long)c * L + L <= n) { s0 = n0; s1 = n1; }      // a ragged / empty last chunk does not advance by A^L
  }
}

#if !defined(PC_EMULATE)
// grid = C channels, block = kScanThreads
template <class R>
__global__ void __launch_bounds__(kScanThreads) k_scan2(R rec, long long n) {
  using T = typename R::T;
  __shared__ double AL[2][2];
  __shared__ T Z[kScanThreads][2];
  const int ch = blockIdx.x, t = threadIdx.x;
  const long long L = (n + kScanThreads - 1) / kScanThreads;
  long long i0, i1;
  scan_bounds(t, L, n, i0, i1);
  T s[2] = {0, 0};
  scan_chunk(rec, ch, i0, i1, s, false);
  Z[t][0] = s[0];
  Z[t][1] = s[1];
  if (t < 2) {
    double col[2];
    scan_power_column(rec, L, t, col);
    AL[0][t] = col[0];
    AL[1][t] = col[1];
  }
  __syncthreads();
  if (t == 0) scan_states<T>(Z, AL, kScanThreads, L, n);
  __syncthreads();
  s[0] = Z[t][0];
  s[1] = Z[t][1];
  scan_chunk(rec, ch, i0, i1, s, true);
}

__global__ void k_rs_interp(const float* x, long long x_stride, long long nx, float* y, long long y_stride, long long M,
                            double ratio, float scale) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int ch = blockIdx.y;
  if (m < M) y[ch * y_stride + m] = rs_interp(x + ch * x_stride, nx, ratio, m) * scale;
}

__global__ void k_ir_energy(const float* l, const float* r, long long n, double* out) {
  __shared__ double red[256];
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double a = (double)l[i], b = (double)r[i];
    acc += a * a + b * b;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) { if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s]; __syncthreads(); }
  if (threadIdx.x == 0) atomicAdd(out, red[0]);
}
__global__ void k_ir_pick(float* dst, const float* raw, long long n_raw, long long start, long long n, int reverse, float ag, float g) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = ir_pick(raw, n_raw, start, reverse, ag, g, i);
}
__global__ void k_ir_clip_env(float* x, long long n, int clip, long long attack_n, long long decay_n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = ir_clip_env(x[i], clip, i, n, attack_n, decay_n);
}
// 1 + index of the last tap with |h| >= 1e-6 (the trim rule of FFTConvolver.cpp:103-106), 0 if none
__global__ void k_ir_last_significant(const float* x, long long n, unsigned long long* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(fabsf(x[i]) < 0.000001f)) atomicMax(out, (unsigned long long)(i + 1));
}
#else
// CPU emulation (tests/emu): same chunks, same two passes, threads as loops
template <class R>
void emu_scan2(const R& rec, int C, long long n) {
  using T = typename R::T;
  const long long L = (n + kScanThreads - 1) / kScanThreads;
  std::vector<T> zbuf(2 * kScanThreads);
  T (*Z)[2] = reinterpret_cast<T (*)[2]>(zbuf.data());
  double AL[2][2];
  for (int ch = 0; ch < C; ++ch) {
    long long i0, i1;
    for (int t = 0; t < kScanThreads; ++t) {
      scan_bounds(t, L, n, i0, i1);
      T s[2] = {0, 0};
      scan_chunk(rec, ch, i0, i1, s, false);
      Z[t][0] = s[0];
      Z[t][1] = s[1];
    }
    for (int j = 0; j < 2; ++j) {
      double col[2];
      scan_power_column(rec, L, j, col);
      AL[0][j] = col[0];
      AL[1][j] = col[1];
    }
    scan_states<T>(Z, AL, kScanThreads, L, n);
    for (int t = 0; t < kScanThreads; ++t) {
      scan_bounds(t, L, n, i0, i1);
      T s[2] = {Z[t][0], Z[t][1]};
      scan_chunk(rec, ch, i0, i1, s, true);
    }
  }
}
#endif

// launches (device) or loops (emulation) over the same phase functions
template <class R>
void launch_scan(const R& rec, int C, long long n, cudaStream_t st) {
  if (n <= 0) return;
#if defined(PC_EMULATE)
  (void)st;
  emu_scan2(rec, C, n);
#else
  k_scan2<R><<<C, kScanThreads, 0, st>>>(rec, n);
#endif
}
void launch_interp(const float* x, long long x_stride, long long nx, float* y, long long y_stride, int C, long long M, double ratio,
                   float scale, cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)st;
  for (int ch = 0; ch < C; ++ch)
    for (long long m = 0; m < M; ++m) y[ch * y_stride + m] = rs_interp(x + ch * x_stride, nx, ratio, m) * scale;
#else
  k_rs_interp<<<dim3((unsigned)((M + 255) / 256), (unsigned)C), 256, 0, st>>>(x, x_stride, nx, y, y_stride, M, ratio, scale);
#endif
}
void launch_pick(float* dst, const float* raw, long long n_raw, long long start, long long n, int reverse, float ag, float g,
                 cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)st;
  for (long long i = 0; i < n; ++i) dst[i] = ir_pick(raw, n_raw, start, reverse, ag, g, i);
#else
  k_ir_pick<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dst, raw, n_raw, start, n, reverse, ag, g);
#endif
}
// clip + envelope in place, then dlast = 1 + index of the last tap with |h| >= 1e-6
void launch_clip_env_last(float* x, long long n, int clip, long long attack_n, long long decay_n, unsigned long long* dlast,
                          cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)st;
  for (long long i = 0; i < n; ++i) {
    x[i] = ir_clip_env(x[i], clip, i, n, attack_n, decay_n);
    if (!(std::fabs(x[i]) < 0.000001f)) *dlast = (unsigned long long)(i + 1);
  }
#else
  const unsigned gb = (unsigned)((n + 255) / 256);
  k_ir_clip_env<<<gb, 256, 0, st>>>(x, n, clip, attack_n, decay_n);
  k_ir_last_significant<<<gb, 256, 0, st>>>(x, n, dlast);
#endif
}
}  // namespace

// ---- host side: coefficients, lengths and the plan of one recalculation ----
static const float kPiF = 3.14159265358979323846f;          // MathConstants<float>::pi

static RsLowPass rs_lowpass(double ratio) {                  // createLowPass + setFilterCoefficients (:210-243)
  const double prop = ratio > 1.0 ? 0.5 / ratio : 0.5 * ratio;
  const double n = 1.0 / std::tan(M_PI * std::max(0.001, prop));
  const double n2 = n * n;
  const double c1 = 1.0 / (1.0 + M_SQRT2 * n + n2);
  return RsLowPass{c1, c1 * 2.0f, c1, c1 * 2.0 * (1.0 - n2), c1 * (1.0 - M_SQRT2 * n + n2)};
}

// taps of the low-passed input stream that the interpolator reads when down-sampling to M outputs
static long long rs_stream_len(long long M, double ratio) { return (long long)((double)(M - 1) * ratio) + 2; }

// one ResamplingAudioSource pass over C channels (channel stride cap): src (ns taps) -> dst (M taps), `ratio` input samples
// per output sample, times `scale`; tmp is scratch of the same layout
static void rs_stage(const float* src, long long ns, float* dst, float* tmp, long long cap, int C, double ratio, long long M,
                     float scale, cudaStream_t st) {
  const RsLowPass f = rs_lowpass(ratio);
  if (ratio > 1.0001) {                // down-sampling: the filter runs on the zero-padded input first (:135-141)
    const long long ls = rs_stream_len(M, ratio);
    launch_scan(RsFilterRec{src, cap, ns, tmp, cap, 1.0f, f}, C, ls, st);
    launch_interp(tmp, cap, ls, dst, cap, C, M, ratio, scale, st);
  } else if (ratio < 0.9999) {         // up-sampling: on the interpolated output (:179-184)
    launch_interp(src, cap, ns, tmp, cap, C, M, ratio, 1.0f, st);
    launch_scan(RsFilterRec{tmp, cap, M, dst, cap, scale, f}, C, M, st);
  } else {                             // no filter in between
    launch_interp(src, cap, ns, dst, cap, C, M, ratio, scale, st);
  }
}

// SVF::lp / bp / hp / ls / hs / pk / bs / hp6 / lp6 (src/dsp/SVF.cpp:4-111) chosen as Impulse.cpp:511-519 does
static SvfCoeffs svf_coeffs(const b200conv_eq_band& b, float srate) {
  SvfCoeffs f{};
  auto setup = [&](float freq, float q, float resfactor) {
    f.g = std::tan(kPiF * std::fmin(freq / srate, 0.49f));
    f.r2 = (1.0f / q) * resfactor;
    f.a1 = 1.0f / (1.0f + f.g * (f.g + f.r2));
    f.a2 = f.g * f.a1;
    f.a3 = f.g * f.a2;
  };
  f.mode = b.mode;
  switch (b.mode) {
    case 0: setup(b.freq, b.q, 1.f); f.cl = 1.f; f.cb = 0.f; f.ch = 0.f; break;                           // LP
    case 1: setup(b.freq, b.q, 1.f); f.cl = 0.f; f.cb = 1.f / b.q; f.ch = 0.f; break;                     // BP
    case 2: setup(b.freq, b.q, 1.f); f.cl = 0.f; f.cb = 0.f; f.ch = 1.f; break;                           // HP
    case 3: setup(b.freq * std::pow(b.gain, -0.25f), b.q, 1.f);                                           // LS
            f.cl = b.gain; f.cb = f.r2 * std::sqrt(b.gain); f.ch = 1.f; break;
    case 4: setup(b.freq * std::pow(b.gain, 0.25f), b.q, 1.f);                                            // HS
            f.cl = 1.f; f.cb = f.r2 * std::sqrt(b.gain); f.ch = b.gain; break;
    case 6: setup(b.freq, b.q, 1.f); f.cl = 1.f; f.cb = 0.f; f.ch = 1.f; break;                           // BS
    case kSvfHP6:
    case kSvfLP6: f.g = std::tan(kPiF * std::fmin(b.freq / srate, 0.49f)); f.g = f.g / (1.0f + f.g); break;
    default:                                                                                              // PK, Off
      f.mode = 5;
      setup(b.freq, b.q, b.gain < 1.f ? 7.5f : 1.f);
      f.cl = 1.f; f.cb = f.r2 * b.gain; f.ch = 1.f;
  }
  return f;
}

static float svf_magnitude(const SvfCoeffs& f, float srate, float freq) {      // SVF::getMagnitude (:253-284)
  freq = std::min(freq, 0.49f * srate);
  if (f.mode == kSvfHP6 || f.mode == kSvfLP6) {
    const float omega = 2.0f * kPiF * freq / srate;
    const float a = f.g, b = 1.0f - a, c = std::cos(omega);
    float denom = 1.0f + b * b - 2.0f * b * c;
    denom = std::max(denom, 1e-12f);
    const float num = f.mode == kSvfLP6 ? a * a : 2.0f - 2.0f * c;
    return std::sqrt(num / denom);
  }
  const float g_eval = std::tan(kPiF * std::fmin(freq / srate, 0.49f));
  const float g_norm = g_eval / f.g;
  const std::complex<float> denom(g_norm * g_norm - 1.0f, g_norm * f.r2);
  const std::complex<float> num = -f.cl * std::complex<float>(1.0f, 0.0f) + f.cb * std::complex<float>(0.0f, g_norm) +
                                  f.ch * std::complex<float>(g_norm * g_norm, 0.0f);
  return std::abs(num / denom);
}

// the 2049-entry decay table of Impulse::applyDecayEQ (Impulse.cpp:562-591) from the bands
static void decay_lut_from_bands(const b200conv_eq_band* bands, int nb, double srate, float decay_rate, double* lut) {
  std::vector<SvfCoeffs> eq;
  for (int i = 0; i < nb; ++i) eq.push_back(svf_coeffs(bands[i], (float)srate));
  const int size = kM + 1;
  const float max_gain = 24.f;                                 // EQ_MAX_GAIN (src/Globals.h:36)
  const double decay_per_s = 1.0 - (double)0.9f, grow_per_s = 1.0 + (double)2.f;   // EQ_MAX_DECAY_RATE_NEG / _POS
  const double ln_decay = std::log(std::pow(decay_per_s, ((double)kN / srate) * (double)decay_rate));
  const double ln_grow = std::log(std::pow(grow_per_s, ((double)kN / srate) * (double)decay_rate));
  for (int i = 0; i < size; ++i) {
    float freq = (float)i / (float)(size - 1) * (float)srate * 0.5f;
    freq = std::clamp(freq, 20.f, 20000.f);
    float mag = 1.f;
    for (const SvfCoeffs& f : eq) mag *= svf_magnitude(f, (float)srate, freq);
    const float db = 20.0f * std::log10(mag);
    float norm = std::clamp((max_gain - db) / (2.f * max_gain), 0.f, 1.f);
    norm = (norm * 2.f - 1.f) * -1.f;
    double d = 1.0;
    if (norm > 0.f) d = std::exp(norm * ln_grow);
    else if (norm < 0.f) d = std::exp(-norm * ln_decay);
    lut[i] = d;
  }
}

// internal (tests): the decay table the library builds from the bands
extern "C" void pc_ir_decay_lut(const b200conv_eq_band* bands, int nb, double srate, float decay_rate, double* lut) {
  decay_lut_from_bands(bands, nb, srate, decay_rate, lut);
}

struct RecalcPlan {
  int autogain = 0, reverse = 0;
  size_t n = 0, n1 = 0, n2 = 0;        // taps of the raw IR, after resampling, after stretch
  double rs_ratio = 0.0;               // resampling: input samples per output sample (0: off)
  double st_ratio = 0.0;               // stretch (0: off)
  size_t start = 0, m = 0;             // trim of the n2 taps
  float gain = 1.0f;
  std::vector<SvfCoeffs> param_eq;
  const double* lut = nullptr;         // decay table (nullptr: no decay EQ)
  std::vector<double> lut_store;
  double srate = 0.0;
  int clip = 0;
  float attack = 0.0f, decay = 0.0f;
};

static void plan_trim(RecalcPlan& P, float trim_left, float trim_right) {     // applyTrim (:436-452)
  const size_t n = P.n2;
  const size_t start = (size_t)(trim_left * (float)n);
  const size_t end = n - (size_t)(trim_right * (float)n);
  P.start = 0;
  P.m = 0;
  if (n == 0 || start >= end || start >= n || end > n) return;
  P.start = start;
  P.m = end - start;
}

static bool bands_ok(int nb, const b200conv_eq_band* b) {
  if (nb < 0 || nb > 8 || (nb > 0 && !b)) return false;
  for (int i = 0; i < nb; ++i)
    if (b[i].mode < 0 || b[i].mode > 9) return false;
  return true;
}

static int recalc_plan(size_t n, const b200conv_ir_recalc_params* p, RecalcPlan& P) {
  if (!p || !(p->srate > 0.0) || !(p->ir_srate > 0.0)) return B200CONV_EINVAL;
  if (!bands_ok(p->n_param_eq, p->param_eq) || !bands_ok(p->n_decay_eq, p->decay_eq)) return B200CONV_EINVAL;
  P.autogain = p->autogain;
  P.reverse = p->reverse;
  P.n = P.n1 = P.n2 = n;
  if (n > 0 && std::fabs(p->ir_srate - p->srate) >= 1e-6) {   // resampleIRToProjectRate (:364-373)
    P.rs_ratio = p->ir_srate / p->srate;
    P.n1 = (size_t)std::ceil((double)n / P.rs_ratio);
  }
  P.n2 = P.n1;
  if (p->stretch != 0.f && P.n1 > 0) {                          // applyStretch (:393-409)
    const double ss = std::pow(2.0, (double)p->stretch) * p->srate;
    if (!(std::fabs(ss - p->srate) < 1e-6 || ss < 1.0 || p->srate < 1.0)) {
      P.st_ratio = p->srate / ss;
      P.n2 = (size_t)std::ceil((double)P.n1 * ss / p->srate);
    }
  }
  plan_trim(P, p->trim_left, p->trim_right);
  P.gain = p->gain;
  for (int i = 0; i < p->n_param_eq; ++i) P.param_eq.push_back(svf_coeffs(p->param_eq[i], (float)p->srate));
  if (p->n_decay_eq > 0) {
    P.lut_store.resize(kM + 1);
    decay_lut_from_bands(p->decay_eq, p->n_decay_eq, p->srate, p->decay_rate, P.lut_store.data());
    P.lut = P.lut_store.data();
  }
  P.srate = p->srate;
  P.clip = p->clip;
  P.attack = p->attack;
  P.decay = p->decay;
  return B200CONV_OK;
}

// shapes C raw channels (host) into C device buffers dev_out[c] = dev_out[0] + c * (*out_len) (one cudaMalloc here,
// *out_len taps each, the caller frees with pc_ir_shape_free)
// and reports the post-trim lengths trimmed[c] that FFTConvolver::init would use.  One upload; scratch once for all channels.
static int ir_pipeline(int device, const float* const* raw, int C, const RecalcPlan& P, float** dev_out, size_t* out_len,
                       size_t* trimmed) {
  for (int c = 0; c < C; ++c) dev_out[c] = nullptr;
  const size_t n = P.n, m = P.m;
  *out_len = m;
  if (m == 0) { for (int c = 0; c < C; ++c) if (trimmed) trimmed[c] = 0; return B200CONV_OK; }
  const long long attack_n = (long long)(int)(P.attack * (float)(int)m), decay_n = (long long)(int)(P.decay * (float)(int)m);
  const bool moved = P.rs_ratio != 0.0 || P.st_ratio != 0.0;
  const size_t cap = std::max(n, std::max(P.n1, P.n2)) + 4;      // channel stride of the resampling buffers
#if defined(PC_EMULATE)
  (void)device;
#else
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return B200CONV_ECUDA; }
#endif
  cudaStream_t st = nullptr;
  float* draw = nullptr; float* work = nullptr; double* denergy = nullptr; unsigned long long* dlast = nullptr;
  DecayScratch sc;
  std::vector<float> win; std::vector<float2> tw;
  bool ok = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaMalloc(&draw, (size_t)C * n * sizeof(float)) == cudaSuccess;
  if (moved) ok = ok && cudaMalloc(&work, 3 * (size_t)C * cap * sizeof(float)) == cudaSuccess;
  ok = ok && cudaMalloc(&denergy, sizeof(double)) == cudaSuccess;
  ok = ok && cudaMalloc(&dlast, C * sizeof(unsigned long long)) == cudaSuccess;
  float* dout = nullptr;
  ok = ok && cudaMalloc(&dout, (size_t)C * m * sizeof(float)) == cudaSuccess;
  if (ok) for (int c = 0; c < C; ++c) dev_out[c] = dout + (size_t)c * m;
  float ag = 1.0f;
  if (ok) {
    for (int c = 0; c < C; ++c) cudaMemcpyAsync(draw + (size_t)c * n, raw[c], n * sizeof(float), cudaMemcpyHostToDevice, st);   // the ONE upload
    if (P.autogain) {
      double energy = 0.0;
#if defined(PC_EMULATE)
      for (size_t i = 0; i < n; ++i) { const double a = draw[i], b = draw[n + i]; energy += a * a + b * b; }
#else
      cudaMemsetAsync(denergy, 0, sizeof(double), st);
      k_ir_energy<<<296, 256, 0, st>>>(draw, draw + n, (long long)n, denergy);
      cudaMemcpyAsync(&energy, denergy, sizeof(double), cudaMemcpyDeviceToHost, st);
      ok = cudaStreamSynchronize(st) == cudaSuccess;
#endif
      if (ok && energy > 0.0) ag = (float)std::min(1.0 / std::sqrt(energy), 1.0);
    }
  }
  if (ok) {
    if (!moved) {
      for (int c = 0; c < C; ++c)
        launch_pick(dev_out[c], draw + (size_t)c * n, (long long)n, (long long)P.start, (long long)m, P.reverse, ag, P.gain, st);
    } else {
      float* buf[3] = {work, work + (size_t)C * cap, work + 2 * (size_t)C * cap};
      int cur = 0, nxt = 1;
      const int tmp = 2;
      for (int c = 0; c < C; ++c)                 // auto gain + reverse, rounded before the resampler
        launch_pick(buf[cur] + (size_t)c * cap, draw + (size_t)c * n, (long long)n, 0, (long long)n, P.reverse, ag, 1.0f, st);
      long long len = (long long)n;
      if (P.rs_ratio != 0.0) {                    // the output is scaled by (float)ratio (:385-388)
        rs_stage(buf[cur], len, buf[nxt], buf[tmp], (long long)cap, C, P.rs_ratio, (long long)P.n1, (float)P.rs_ratio, st);
        std::swap(cur, nxt);
        len = (long long)P.n1;
      }
      if (P.st_ratio != 0.0) {
        rs_stage(buf[cur], len, buf[nxt], buf[tmp], (long long)cap, C, P.st_ratio, (long long)P.n2, 1.0f, st);
        std::swap(cur, nxt);
        len = (long long)P.n2;
      }
      for (int c = 0; c < C; ++c)                 // trim + gain
        launch_pick(dev_out[c], buf[cur] + (size_t)c * cap, len, (long long)P.start, (long long)m, 0, 1.0f, P.gain, st);
    }
    if (!P.param_eq.empty()) {                    // band after band over the whole buffer, as applyParamEQ
      SvfRec rec{dout, (long long)m, {}};
      for (const SvfCoeffs& f : P.param_eq) {
        rec.f = f;
        launch_scan(rec, C, (long long)m, st);
      }
    }
    if (P.lut)
      for (int c = 0; c < C && ok; ++c)
        ok = decay_eq_device(dev_out[c], m, 1, m, P.lut, P.srate, st, sc, win, tw);   // one scratch set for all channels
    cudaMemsetAsync(dlast, 0, C * sizeof(unsigned long long), st);
    for (int c = 0; c < C; ++c) launch_clip_env_last(dev_out[c], (long long)m, P.clip, attack_n, decay_n, dlast + c, st);
    unsigned long long last[8] = {};
    cudaMemcpyAsync(last, dlast, C * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
    ok = ok && cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess;
    if (trimmed) for (int c = 0; c < C; ++c) trimmed[c] = (size_t)last[c];
  }
  sc.release();
  cudaFree(draw); cudaFree(work); cudaFree(denergy); cudaFree(dlast);
  if (st) cudaStreamDestroy(st);
  if (!ok) {
    cudaFree(dout);
    for (int c = 0; c < C; ++c) dev_out[c] = nullptr;
    cudaGetLastError();
    return B200CONV_ECUDA;
  }
  return B200CONV_OK;
}

// internal (not part of the C ABI): the b200conv_ir_shape subset — no resampling, stretch or parametric EQ, a given table
extern "C" int pc_ir_shape_to_device(int device, const float* const* raw, int C, size_t n, const b200conv_ir_shape_params* sp,
                                     float** dev_out, size_t* out_len, size_t* trimmed) {
  if (!raw || !sp || !dev_out || !out_len || C < 2 || C > 8) return B200CONV_EINVAL;
  RecalcPlan P;
  P.autogain = sp->autogain;
  P.reverse = sp->reverse;
  P.n = P.n1 = P.n2 = n;
  plan_trim(P, sp->trim_left, sp->trim_right);
  P.gain = sp->gain;
  P.lut = sp->decay_lut;
  P.srate = sp->srate;
  P.clip = sp->clip;
  P.attack = sp->attack;
  P.decay = sp->decay;
  return ir_pipeline(device, raw, C, P, dev_out, out_len, trimmed);
}

// internal: the whole recalculation into device buffers (b200conv_init_*_recalc)
extern "C" int pc_ir_recalc_to_device(int device, const float* const* raw, int C, size_t n, const b200conv_ir_recalc_params* p,
                                      float** dev_out, size_t* out_len, size_t* trimmed) {
  if (!raw || !p || !dev_out || !out_len || C < 2 || C > 8) return B200CONV_EINVAL;
  for (int c = 0; c < C && n > 0; ++c) if (!raw[c]) return B200CONV_EINVAL;
  RecalcPlan P;
  if (int rc = recalc_plan(n, p, P)) return rc;
  return ir_pipeline(device, raw, C, P, dev_out, out_len, trimmed);
}

extern "C" void pc_ir_shape_free(float** dev_out, int C) {
  cudaFree(dev_out[0]);                    // one allocation for all channels (ir_pipeline)
  for (int c = 0; c < C; ++c) dev_out[c] = nullptr;
}

// the shaped taps back on the host (m per channel), then the device buffers freed
static int download_and_free(float** dev, int C, size_t m, float* const* out) {
  bool ok = true;
  for (int c = 0; c < C && m > 0; ++c) {
#if defined(PC_EMULATE)
    std::memcpy(out[c], dev[c], m * sizeof(float));
#else
    ok = ok && cudaMemcpy(out[c], dev[c], m * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
#endif
  }
  pc_ir_shape_free(dev, C);
  return ok ? B200CONV_OK : B200CONV_ECUDA;
}

// stand-alone: the shaped taps back on the host (tests, waveform display)
extern "C" int b200conv_ir_shape(int device, const float* const* raw, int n_channels, size_t n, const b200conv_ir_shape_params* sp,
                                 float* const* out, size_t* out_len) {
  if (!out || !out_len) return B200CONV_EINVAL;
  float* dev[8] = {};
  size_t m = 0;
  const int rc = pc_ir_shape_to_device(device, raw, n_channels, n, sp, dev, &m, nullptr);
  if (rc != B200CONV_OK) return rc;
  *out_len = m;
  return download_and_free(dev, n_channels, m, out);
}

extern "C" size_t b200conv_ir_recalc_len(size_t n, const b200conv_ir_recalc_params* p) {
  RecalcPlan P;
  return recalc_plan(n, p, P) == B200CONV_OK ? P.m : 0;
}

extern "C" int b200conv_ir_recalc(int device, const float* const* raw, int n_channels, size_t n, const b200conv_ir_recalc_params* p,
                                  float* const* out, size_t out_cap, size_t* out_len) {
  if (!out || !out_len || !p || n_channels < 2 || n_channels > 8) return B200CONV_EINVAL;
  const size_t need = b200conv_ir_recalc_len(n, p);
  if (need > out_cap) return B200CONV_EINVAL;
  for (int c = 0; c < n_channels && need > 0; ++c) if (!out[c]) return B200CONV_EINVAL;
  float* dev[8] = {};
  size_t m = 0;
  const int rc = pc_ir_recalc_to_device(device, raw, n_channels, n, p, dev, &m, nullptr);
  if (rc != B200CONV_OK) return rc;
  *out_len = m;
  return download_and_free(dev, n_channels, m, out);
}
