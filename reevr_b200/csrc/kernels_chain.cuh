// kernels_chain.cuh — SURVEY 8f-4 and the remainder of 8f-1: the per-sample work REEV-R does on the host around the
// convolver, moved to the device so that the device boundary sits at the plugin's dry input / final output:
//
//   k_chain_send   send = dry * ysend ; low cut / high cut state-variable filters ; predelay ring
//                  (src/PluginProcessor.cpp:1639-1653 + src/dsp/Filter.cpp:23-68 ; :1766-1790)
//   k_chain_wet    wet L = LL (+ RL), R = RR (+ LR) ; * yrev ; mid/side width ; out = drygain * dry + wetgain * wet
//                  (src/PluginProcessor.cpp:1832-1876)
//   k_chain_wet_xfade  the same during an IR hot swap: outgoing and incoming convolvers crossfaded per sample before
//                  the mixdown (src/PluginProcessor.cpp:1799-1838)
// The IR hot swap's warm-up (src/PluginProcessor.cpp:1694-1756) runs k_chain_send in replay mode (replay_w > 0): the
// input is gathered from the predelay ring, which holds the filtered, undelayed send, with the reference's warmer index
// map; the filters start from a zero state; nothing is written to the ring.
//
// The filters are recursive (two TPT state-variable sections per 24 dB filter), i.e. sequential in time — on a GPU the
// block of n samples is cut into T chunks, one per thread:
//   pass 1  every thread runs the whole cascade (low cut, high cut: up to 8 state variables) over its chunk from a ZERO
//           state and keeps the final state — the zero-state response end point Z_t
//   powers  the cascade is linear and time-invariant: state' = A state + b x.  Column j of A^L (L = chunk length) is the
//           state after L steps with zero input from the unit state e_j — 8 threads run that once per launch
//   scan    S_{t+1} = A^L S_t + Z_t  gives every chunk's true initial state (one thread, T small steps of an 8x8
//           matrix-vector product); S_0 is the state carried over from the previous call
// Each filter keeps the reference's five state variables (src/dsp/Filter.h:52-55, 79): ic1..ic4 of the 12 / 24 dB
// sections and the separate 6 dB `state`, so that a slope switch by b200conv_chain_update resumes whatever each
// variable last held.  The cascade works on four slots per filter: ic1..ic4 at 12 / 24 dB; `state`, ic2, ic3, ic4 at
// 6 dB (the 6 dB filter touches slot 0 only).  The variable slot 0 does not hold (`state` at 12 / 24 dB, ic1 at 6 dB)
// waits in a fifth, stash slot; a launch whose slope crossed 6 dB <-> 12 / 24 dB exchanges slot 0 and the stash before
// the scan (swap_lc / swap_hc).  Slots the current slopes do not use, and those of a filter that is off, are identity
// rows of A^L, which the scan carries over unchanged.
//   pass 2  every thread re-runs its chunk from its true initial state and writes the filtered samples
// The arithmetic inside a chunk is the reference's (same order, float32).  A^L (the zero-input response of the same
// equations from the same float coefficients) and the scan run in double; the initial states handed to pass 2 are
// rounded to float.  A 20 Hz cut at 96 / 192 kHz has poles within ~1e-4 of the unit circle, so an error in S_t
// persists for tens of chunks: with A^L and the scan in float the chunked form was up to 1.2e-4 of peak from a float64
// serial filter, several times the serial float filter's own error; in double it is never more than 1.7x that error
// (tests/test_scan_precision.py).  The predelay ring is written after the filters and read `predelay` samples back, in
// the same launch.
#pragma once

#include "kernels.cuh"

namespace pc {

constexpr int kChainStates = 8;      // scan slots: low cut 4 + high cut 4
constexpr int kChainStateStride = 10; // per channel in memory: the 8 scan slots, then the low-cut and high-cut stash

// coefficients of one reference Filter (src/dsp/Filter.h:53-70), computed on the host as Filter::init does
struct ChainFilter {
  int on, slope, mode;               // slope 0/1/2 = 6/12/24 dB ; mode 0 = LP, 2 = HP
  float g, k, k2, a1, a2, a3, a12, a22, a32;
};

struct ChainSendParams {
  const float* dry; long long dry_stride;       // 2 channels
  const float* ysend;                           // send envelope, n samples (nullptr: 1)
  float* conv_in; long long conv_stride;        // output: the convolver's input, 2 channels
  float* filt; long long filt_stride;           // scratch: filtered samples of this call, 2 channels
  float* state;                                 // [2][kChainStateStride] filter state carried between calls
  int swap_lc, swap_hc;                         // exchange slot 0 and the stash of the low / high cut first
  // predelay ring (power of two), indexed by absolute sample position: ring_pos = position of the call's first sample;
  // delay reads below delay_floor (the last growth of the delay line) return zero
  float* ring; long long ring_stride; long long ring_mask; long long ring_pos;
  long long delay_floor;
  int predelay;
  long long n;
  ChainFilter lc, hc;
  long long replay_w, replay_off;               // warm-up replay: warmer length W (0: normal send), first replay index
};

// one sample through one Filter: Filter::eval (src/dsp/Filter.cpp:23-68); s = its 4 slots (ic1..ic4, 6 dB: state in s[0]).
// F = float: the reference's arithmetic.  F = double: the same equations from the same float coefficients (A^L)
template <class F>
PC_HD F chain_filter_eval(const ChainFilter& f, F* s, F sample) {
  if (f.slope == 0) {
    const F delta = (F)f.g * (sample - s[0]);
    s[0] += delta;
    return f.mode == 0 ? s[0] : sample - s[0];
  }
  F v3 = sample - s[1];
  F v1 = (F)f.a1 * s[0] + (F)f.a2 * v3;
  F v2 = s[1] + (F)f.a2 * s[0] + (F)f.a3 * v3;
  s[0] = (F)2 * v1 - s[0];
  s[1] = (F)2 * v2 - s[1];
  F out = f.mode == 0 ? v2 : (f.mode == 1 ? v1 : sample - (F)f.k * v1 - v2);
  if (f.slope == 1) return out;
  v3 = out - s[3];
  v1 = (F)f.a12 * s[2] + (F)f.a22 * v3;
  v2 = s[3] + (F)f.a22 * s[2] + (F)f.a32 * v3;
  s[2] = (F)2 * v1 - s[2];
  s[3] = (F)2 * v2 - s[3];
  return f.mode == 0 ? v2 : (f.mode == 1 ? v1 : out - (F)f.k2 * v1 - v2);
}

// the cascade of the send path for one sample (s: 8 state variables)
template <class F>
PC_HD F chain_cascade(const ChainSendParams& P, F* s, F x) {
  if (P.lc.on) x = chain_filter_eval<F>(P.lc, s, x);
  if (P.hc.on) x = chain_filter_eval<F>(P.hc, s + 4, x);
  return x;
}

PC_HD float chain_send_in(const ChainSendParams& P, int ch, long long i) {
  if (P.replay_w) {
    // replay index j reads warmer[(warmwritepos + 1 + j) % W] (:1698-1731): the samples W-1 .. 1 calls back, then the
    // oldest one (W back); ring_pos is the next write slot, so age a lives at ring_pos - a
    const long long j = P.replay_off + i;
    const long long age = j < P.replay_w - 1 ? P.replay_w - 1 - j : P.replay_w;
    return P.ring[(long long)ch * P.ring_stride + ((P.ring_pos - age) & P.ring_mask)];
  }
  const float v = P.dry[(long long)ch * P.dry_stride + i];
  return P.ysend ? v * P.ysend[i] : v;
}

// chunk [i0, i1) of channel ch from state s (updated); out != nullptr: write the filtered samples
PC_HD void chain_run_chunk(const ChainSendParams& P, int ch, long long i0, long long i1, float* s, float* out) {
  for (long long i = i0; i < i1; ++i) {
    const float y = chain_cascade<float>(P, s, chain_send_in(P, ch, i));
    if (out) out[i] = y;
  }
}

// a slope switch across 6 dB <-> 12 / 24 dB: slot 0 of the filter and its stash trade places (S: the scan's initial state)
PC_HD void chain_state_unstash(const ChainSendParams& P, int ch, float* S) {
  float* st = P.state + (long long)ch * kChainStateStride + kChainStates;
  if (P.swap_lc) { const float v = S[0]; S[0] = st[0]; st[0] = v; }
  if (P.swap_hc) { const float v = S[4]; S[4] = st[1]; st[1] = v; }
}

// zero-input response in double: column j of A^L
PC_HD void chain_power_column(const ChainSendParams& P, long long L, int j, double* col) {
  for (int q = 0; q < kChainStates; ++q) col[q] = (q == j) ? 1.0 : 0.0;
  for (long long i = 0; i < L; ++i) (void)chain_cascade<double>(P, col, 0.0);
}

// the scan's initial state: the state carried over from the previous call, slot 0 and the stash exchanged if needed
PC_HD void chain_scan_start(const ChainSendParams& P, int ch, double* S) {
  float s[kChainStates];
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) s[q] = P.state[ch * kChainStateStride + q];
  chain_state_unstash(P, ch, s);
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) S[q] = s[q];
}

// one scan step over chunk c: S <- A^L S + Z[c] in double (unless the chunk is ragged or empty), Z[c] <- the chunk's
// initial state rounded to float.  A^L is read through a volatile pointer: otherwise the compiler hoists its 64 loads
// out of the scan loop into registers it does not have and spills them (an 808-byte stack frame)
PC_HD void chain_scan_step(const volatile double (*AL)[kChainStates], float* Zc, double* S, bool full) {
  double nx[kChainStates];
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) {
    double a = Zc[q];
#pragma unroll
    for (int r = 0; r < kChainStates; ++r) a = fma(AL[q][r], S[r], a);
    nx[q] = a;
  }
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) { Zc[q] = (float)S[q]; if (full) S[q] = nx[q]; }
}

// predelay: conv_in[i] = ring[(pos + i - predelay) & mask] after ring[(pos + i) & mask] = filtered[i]; positions
// below the delay floor were cleared by a growth of the delay line (src/PluginProcessor.cpp:1184-1188) and read zero,
// while the ring keeps them for the warm-up replay of an IR hot swap
PC_HD void chain_ring_write(const ChainSendParams& P, int ch, long long i) {
  P.ring[(long long)ch * P.ring_stride + ((P.ring_pos + i) & P.ring_mask)] = P.filt[(long long)ch * P.filt_stride + i];
}
PC_HD void chain_ring_read(const ChainSendParams& P, int ch, long long i) {
  const long long p = P.ring_pos + i - P.predelay;
  P.conv_in[(long long)ch * P.conv_stride + i] =
      p < P.delay_floor ? 0.0f : P.ring[(long long)ch * P.ring_stride + (p & P.ring_mask)];
}

struct ChainWetParams {
  const float* dry; long long dry_stride;       // 2 channels
  const float* conv; long long conv_stride;     // per-convolver outputs: LL, RR[, LR, RL]
  const float* yrev;                            // reverb envelope (nullptr: 1)
  float* out; long long out_stride;             // 2 channels
  long long n;
  int quad_ts;                                  // add RL / LR (quad IR and true stereo enabled)
  float width, drygain, wetgain;
  // k_chain_wet_xfade: conv = outgoing convolvers, conv_in = incoming LL, RR (stride conv_stride); xfade0 = the
  // reference's `xfade` counter at sample 0 of this launch, xfadelen its start value
  const float* conv_in;
  long long xfade0, xfadelen;
  // fixed-latency steps: completion word in pinned host memory (nullptr: none), raised to done_val by the last CTA to
  // finish (ticket: a device word that is 0 between launches) after every CTA's output stores
  unsigned int* done_flag; unsigned int done_val;
  unsigned int* ticket;
};

// * yrev ; mid/side width ; dry / wet mix of one sample of the summed wet signal (src/PluginProcessor.cpp:1840-1876)
PC_HD void chain_wet_mix(const ChainWetParams& P, long long i, float wl, float wr) {
  const float e = P.yrev ? P.yrev[i] : 1.0f;
  const float lin = wl * e, rin = wr * e;
  const float mid = (lin + rin) * 0.5f, side = (lin - rin) * 0.5f;
  const float norm = 1.0f / (1.0f + P.width);
  const float lout = (mid + side * P.width) * norm;
  const float rout = (mid - side * P.width) * norm;
  P.out[i] = P.dry[i] * P.drygain + lout * P.wetgain;
  P.out[P.out_stride + i] = P.dry[P.dry_stride + i] * P.drygain + rout * P.wetgain;
}

PC_HD void chain_wet_sample(const ChainWetParams& P, long long i) {     // src/PluginProcessor.cpp:1832-1838
  float wl = P.conv[i], wr = P.conv[P.conv_stride + i];
  if (P.quad_ts) { wl += P.conv[3 * P.conv_stride + i]; wr += P.conv[2 * P.conv_stride + i]; }
  chain_wet_mix(P, i, wl, wr);
}

// src/PluginProcessor.cpp:1808-1838: the alpha expression of :1809 and the summation order of the wet buffer
// (0 + incoming, + outgoing LL / RR, + outgoing RL / LR); quad_ts = 0 in the call that completes the swap
PC_HD void chain_wet_xfade_sample(const ChainWetParams& P, long long i) {
  float alpha = 1.f - (float)(P.xfade0 - i) / (float)P.xfadelen;
  alpha = alpha < 0.f ? 0.f : (alpha > 1.f ? 1.f : alpha);
  const float beta = 1.f - alpha;
  float wl = 0.f + P.conv_in[i] * alpha, wr = 0.f + P.conv_in[P.conv_stride + i] * alpha;
  wl += P.conv[i] * beta;
  wr += P.conv[P.conv_stride + i] * beta;
  if (P.quad_ts) { wl += P.conv[3 * P.conv_stride + i] * beta; wr += P.conv[2 * P.conv_stride + i] * beta; }
  chain_wet_mix(P, i, wl, wr);
}

#if defined(__CUDACC__)
// grid (2 channels), block T threads (T = 64 for real-time calls, 1024 for batches); static smem
static __global__ void __launch_bounds__(1024) k_chain_send(ChainSendParams P) {
  __shared__ double AL[kChainStates][kChainStates];    // A^L, column j in AL[.][j]
  __shared__ float Z[1024][kChainStates];              // pass 1: zero-state end points ; after the scan: initial states
  const int ch = blockIdx.x, t = threadIdx.x, T = blockDim.x;
  const long long L = (P.n + T - 1) / T;
  const long long i0 = (long long)t * L < P.n ? (long long)t * L : P.n;
  const long long i1 = i0 + L < P.n ? i0 + L : P.n;
  const bool filtered = P.lc.on || P.hc.on;
  float* filt = P.filt + (long long)ch * P.filt_stride;
  if (filtered) {
    float s[kChainStates];
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) s[q] = 0.0f;
    chain_run_chunk(P, ch, i0, i1, s, nullptr);
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) Z[t][q] = s[q];
    if (t < kChainStates) {
      double col[kChainStates];
      chain_power_column(P, L, t, col);
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) AL[q][t] = col[q];
    }
    __syncthreads();
    if (t == 0) {       // S_{t+1} = A^L S_t + Z_t ; Z[t] becomes the initial state of chunk t
      double S[kChainStates];
      chain_scan_start(P, ch, S);
      for (int c = 0; c < T; ++c)                      // a ragged / empty last chunk does not advance by A^L
        chain_scan_step(AL, Z[c], S, (long long)c * L + L <= P.n);
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) s[q] = Z[t][q];
    chain_run_chunk(P, ch, i0, i1, s, filt);
    // the state after the LAST sample of the call belongs to the thread whose chunk ends at n
    if (i1 == P.n && i0 < P.n) {
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
    }
  } else {
    for (long long i = i0; i < i1; ++i) filt[i] = chain_send_in(P, ch, i);
  }
  if (P.replay_w) return;
  __syncthreads();
  for (long long i = t; i < P.n; i += T) chain_ring_write(P, ch, i);
  __syncthreads();
  for (long long i = t; i < P.n; i += T) chain_ring_read(P, ch, i);
}

// the pattern of k_rt_block's done_flag across the CTAs of a grid: every thread's stores are released system-wide, the
// CTA meets, and the CTA that draws the last ticket raises the word
static __device__ __forceinline__ void chain_wet_done(const ChainWetParams& P) {
  if (!P.done_flag) return;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(P.ticket, 1u) == gridDim.x - 1) {
    atomicExch(P.ticket, 0u);
    __threadfence_system();
    *reinterpret_cast<volatile unsigned int*>(P.done_flag) = P.done_val;
    __threadfence_system();
  }
}

static __global__ void k_chain_wet(ChainWetParams P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n) chain_wet_sample(P, i);
  chain_wet_done(P);
}

static __global__ void k_chain_wet_xfade(ChainWetParams P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n) chain_wet_xfade_sample(P, i);
  chain_wet_done(P);
}
#else
// CPU emulation (tests/emu): same chunking, same two passes
inline void emu_chain_send(const ChainSendParams& P, int T) {
  for (int ch = 0; ch < 2; ++ch) {
    const long long L = (P.n + T - 1) / T;
    float* filt = P.filt + (long long)ch * P.filt_stride;
    if (P.lc.on || P.hc.on) {
      float (*Z)[kChainStates] = new float[T][kChainStates];
      double AL[kChainStates][kChainStates];
      for (int t = 0; t < T; ++t) {
        const long long i0 = (long long)t * L < P.n ? (long long)t * L : P.n;
        const long long i1 = i0 + L < P.n ? i0 + L : P.n;
        float s[kChainStates] = {0, 0, 0, 0, 0, 0, 0, 0};
        chain_run_chunk(P, ch, i0, i1, s, nullptr);
        for (int q = 0; q < kChainStates; ++q) Z[t][q] = s[q];
      }
      for (int j = 0; j < kChainStates; ++j) {
        double col[kChainStates];
        chain_power_column(P, L, j, col);
        for (int q = 0; q < kChainStates; ++q) AL[q][j] = col[q];
      }
      double S[kChainStates];
      chain_scan_start(P, ch, S);
      for (int c = 0; c < T; ++c) chain_scan_step(AL, Z[c], S, (long long)c * L + L <= P.n);
      for (int t = 0; t < T; ++t) {
        const long long i0 = (long long)t * L < P.n ? (long long)t * L : P.n;
        const long long i1 = i0 + L < P.n ? i0 + L : P.n;
        float s[kChainStates];
        for (int q = 0; q < kChainStates; ++q) s[q] = Z[t][q];
        chain_run_chunk(P, ch, i0, i1, s, filt);
        if (i1 == P.n && i0 < P.n)
          for (int q = 0; q < kChainStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
      }
      delete[] Z;
    } else {
      for (long long i = 0; i < P.n; ++i) filt[i] = chain_send_in(P, ch, i);
    }
    if (P.replay_w) continue;
    for (long long i = 0; i < P.n; ++i) chain_ring_write(P, ch, i);
    for (long long i = 0; i < P.n; ++i) chain_ring_read(P, ch, i);
  }
}
inline void emu_chain_wet(const ChainWetParams& P) {
  for (long long i = 0; i < P.n; ++i) chain_wet_sample(P, i);
  if (P.done_flag) *P.done_flag = P.done_val;
}
inline void emu_chain_wet_xfade(const ChainWetParams& P) {
  for (long long i = 0; i < P.n; ++i) chain_wet_xfade_sample(P, i);
  if (P.done_flag) *P.done_flag = P.done_val;
}
#endif

}  // namespace pc
