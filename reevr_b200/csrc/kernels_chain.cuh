// kernels_chain.cuh — SURVEY 8f-4 and the remainder of 8f-1: the per-sample work REEV-R does on the host around the
// convolver, moved to the device so that the device boundary sits at the plugin's dry input / final output:
//
//   k_chain_send   send = dry * ysend ; low cut / high cut state-variable filters ; predelay ring
//                  (src/PluginProcessor.cpp:1639-1653 + src/dsp/Filter.cpp:23-68 ; :1766-1790)
//   k_chain_wet    wet L = LL (+ RL), R = RR (+ LR) ; * yrev ; mid/side width ; out = drygain * dry + wetgain * wet
//                  (src/PluginProcessor.cpp:1832-1876)
//   k_chain_wet_xfade  the same during an IR hot swap: outgoing and incoming convolvers crossfaded per sample before
//                  the mixdown (src/PluginProcessor.cpp:1799-1838)
//   k_chain_send_group / k_chain_wet_group  the same for the chain calls of a group of handles
//                  (b200conv_chain_group_process): one launch of each for up to kChainGroupMax members
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

// The chain calls of up to kChainGroupMax handles in one send and one wet launch (b200conv_chain_group_process),
// passed by value like RtGroupParams (kernels_rt.cuh).  In a zero-latency group call the members' wet parameters carry
// no completion word of their own: the wet launch raises the group's.  In a fixed-latency group call each member's
// carries its ring word and ticket, and the launch has no group word.
constexpr int kChainGroupMax = 32;
struct ChainSendGroupParams {
  int n;
  ChainSendParams p[kChainGroupMax];
};
struct ChainWetGroupParams {
  int n;
  unsigned int* done_flag; unsigned int done_val;     // pinned word (nullptr: none), raised after every CTA's stores
  unsigned int* ticket;                               // device word, 0 between launches
  ChainWetParams p[kChainGroupMax];
};
static_assert(sizeof(ChainSendGroupParams) <= 32764, "k_chain_send_group's parameter table exceeds the kernel-parameter limit");
static_assert(sizeof(ChainWetGroupParams) <= 32764, "k_chain_wet_group's parameter table exceeds the kernel-parameter limit");

// ---- the whole-GPU send form of long device-pointer pieces (b200conv_chain_process_device) -------------------------
// The math of k_chain_send, spread over as many CTAs as the piece needs, both channels in one grid: chunks of a fixed
// kWideLc samples, one per thread, kWideT chunks per CTA.  Four launches:
//   powers  k_chain_wide_powers: A from one zero-input step (chain_power_column), squared in double to
//           P_j = A^(kWideLc * 2^j), j < kWidePowers (once per call: the filters do not change within a call)
//   pass 1  k_chain_wide_pass1: every chunk from a zero state gives its end state Z_c (FP32, as chain_run_chunk runs
//           it); the CTA folds its Z_c in double into its aggregate sum_c M^(last - c) Z_c (M = P_0 = A^Lc) by a tree
//   carry   k_chain_wide_carry: one CTA per channel scans the aggregates, G_{b+1} = M^kWideT G_b + agg_b from
//           G_0 = chain_scan_start (the stash exchange and the carried state as in k_chain_send), Hillis-Steele in
//           tiles of kWideCarryT with P_{log2 kWideT + j} as the multipliers
//   pass 2  k_chain_wide_pass2: the CTA scans its Z_c again, seeded with G_b, for every chunk's true initial state
//           (rounded to float), re-runs the chunks and writes the ring and the predelayed convolver input
// Only the last chunk of a piece can be ragged; nothing downstream of it is read, so no chunk advances by less than M.
// The send is staged through shared memory (row per chunk, padded against bank conflicts), so every global access is
// coalesced.  Pass 2 needs no grid barrier for the predelay: conv_in[i] for i >= predelay is the pass-2 value of sample
// i - predelay, written by whichever thread owns that sample; conv_in[i] for i < predelay reads a ring slot of an
// earlier piece, at a distance of at most predelay + n - 1 < ring size (chain_ring_len: >= D + Lmax + 1, predelay <=
// D, n <= Lmax) from every slot this piece writes.  Deterministic: fixed chunking, fixed reduction and scan order.
constexpr int kWideLc = 64;                // samples per chunk
constexpr int kWideT = 128;                // chunks (threads) per CTA
constexpr int kWideSpan = kWideLc * kWideT;
constexpr int kWideLogT = 7;
constexpr int kWideCarryT = 512;           // threads of the carry scan: a tile carries 511 aggregates
constexpr int kWideLogCarry = 9;
constexpr int kWideLogLc = 6;
constexpr int kWidePowers = kWideLogT + kWideLogCarry;

// scratch of the whole-GPU form, sized for Lmax (b200conv_chain_configure)
struct ChainWideScratch {
  double* pw;                              // [kWidePowers][8][8] P_j
  double* agg;                             // [2][nb_cap][8] CTA aggregates
  double* carry;                           // [2][nb_cap][8] G_b: the state entering CTA b
  float* z;                                // [2][nb_cap * kWideT][8] zero-state end points
  long long nb_cap;
};

inline long long chain_wide_ctas(long long n) { return (n + kWideSpan - 1) / kWideSpan; }

// entry (q, r) of M * M
PC_HD double chain_square_entry(const double (*M)[kChainStates], int q, int r) {
  double a = 0.0;
#pragma unroll
  for (int k = 0; k < kChainStates; ++k) a = fma(M[q][k], M[k][r], a);
  return a;
}

// acc += M x.  M is not read through a volatile pointer (unlike chain_scan_step's A^L): every scan step uses another
// power, so there is nothing to hoist, and volatile loads would serialise the 64 shared-memory reads of each step
PC_HD void chain_affine_acc(const double (*M)[kChainStates], const double* x, double* acc) {
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) {
    double a = acc[q];
#pragma unroll
    for (int r = 0; r < kChainStates; ++r) a = fma(M[q][r], x[r], a);
    acc[q] = a;
  }
}

// one combine step over a [kChainStates][N] array of double states: nx = V[t] + M V[t - d]  (t >= d), or
// V[t] + M V[t + d] read as "left then right" when `tree` (pass 1: V[t] <- M V[t] + V[t + d])
PC_HD void chain_combine(const double (*M)[kChainStates], const double* V, int N, int t, int d, bool tree,
                         double* nx) {
  double x[kChainStates];
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) {
    nx[q] = tree ? V[q * N + t + d] : V[q * N + t];
    x[q] = tree ? V[q * N + t] : V[q * N + t - d];
  }
  chain_affine_acc(M, x, nx);
}

// the send sample i of channel ch (no replay: the whole-GPU form is never a warm-up)
PC_HD float chain_wide_send(const ChainSendParams& P, int ch, long long i) {
  const float v = P.dry[(long long)ch * P.dry_stride + i];
  return P.ysend ? v * P.ysend[i] : v;
}

// pass 2's output of sample i (y): ring slot, predelayed convolver input, and the undelayed send while a swap fades
PC_HD void chain_wide_store(const ChainSendParams& P, int ch, long long i, float y) {
  P.ring[(long long)ch * P.ring_stride + ((P.ring_pos + i) & P.ring_mask)] = y;
  if (i + P.predelay < P.n) P.conv_in[(long long)ch * P.conv_stride + i + P.predelay] = y;
  if (i < P.predelay) {
    const long long p = P.ring_pos + i - P.predelay;
    P.conv_in[(long long)ch * P.conv_stride + i] =
        p < P.delay_floor ? 0.0f : P.ring[(long long)ch * P.ring_stride + (p & P.ring_mask)];
  }
  if (P.filt) P.filt[(long long)ch * P.filt_stride + i] = y;
}

// ---- parameter events inside one device call (b200conv_chain_process_device_events) --------------------------------
// The call carries a table of segments, one row per stretch of samples with one parameter set; a piece of the call
// overlaps a contiguous run of rows.  A piece inside one row runs the kernels above with that row's parameters.  A long
// piece that spans several rows runs the segmented whole-GPU form, in five launches:
//   maps   k_chain_seg_maps: per CTA, either (uniform CTA: one row, no slope exchange at its first sample) the powers
//          P_j = A^(kWideLc * 2^j) of that row's A, squared exactly as k_chain_wide_powers squares them, and
//          M_b = P_kWideLogT; or (mixed CTA) every chunk's transfer matrix T_c from kSegStates zero-input runs in double
//          over its samples, switching coefficients and exchanging slot 0 and the stash where a row starts, and
//          M_b = T_last ... T_0 composed in order
//   pass 1 k_chain_seg_pass1: every chunk from a zero state (FP32, switching as above) gives Z_c; a uniform CTA folds
//          them by k_chain_wide_pass1's tree with its P_j, a mixed one by S <- T_c S + Z_c in double, in order
//   carry  k_chain_seg_carry: G_{b+1} = M_b G_b + agg_b in double from the carried state, CTA after CTA
//   pass 2 k_chain_seg_pass2: a uniform CTA seeds and scans as k_chain_wide_pass2 does; a mixed one runs
//          S <- T_c S + Z_c from G_b; both re-run the chunks from the rounded seeds and write the ring
//   read   k_chain_seg_read: the predelayed convolver input, each sample at its row's predelay and delay floor
// The state is kSegStates wide: the 8 scan slots and the two stash slots, which only slope exchanges move (a
// permutation, exact in double), so the stash a row leaves is the FP32 value the serial filter would leave.  The
// double scan has the precision argument of the event-free form: every T_c and M_b is the exact-coefficient transfer
// of its samples, rounded once per entry, and each chunk's seed is rounded to float once; nothing accumulates across
// rows beyond the scan's own rounding.  The ring is read only after pass 2 has written the whole piece, in its own
// launch: with a predelay that changes inside the piece, the sample a convolver input needs may belong to another CTA.
// The slots it reads lie at most predelay + n - 1 < ring size behind every slot the piece writes, as in the event-free
// form.
constexpr int kSegStates = kChainStates + 2;

struct ChainSeg {                  // one row: parameters from sample `start` of the call on
  long long start;
  long long delay_floor;           // absolute ring position below which the delay reads zero
  ChainFilter lc, hc;
  int swap_lc, swap_hc;            // the slope crossed 6 dB <-> 12 / 24 dB at `start`: slot 0 and the stash trade places
  int predelay;
  int quad_ts;
  float width, drygain, wetgain;
};

struct ChainSegs {                 // the rows one piece overlaps
  const ChainSeg* seg;             // the row in force at the piece's first sample
  int nseg;
  long long off;                   // the piece's first sample in the call
};

// scratch of the segmented form, sized for Lmax (grown by the first events call that needs it, before its first launch)
struct ChainSegScratch {
  double* pw;                      // [nb_cap][kWideLogT][8][8] P_j of uniform CTAs
  double* mb;                      // [nb_cap][kSegStates][kSegStates] M_b
  double* tc;                      // [nb_cap * kWideT][kSegStates][kSegStates] T_c of mixed CTAs
  double* agg;                     // [2][nb_cap][kSegStates]
  double* carry;                   // [2][nb_cap][kSegStates] G_b
  float* z;                        // [2][nb_cap * kWideT][kSegStates] zero-state end points
  long long nb_cap;
};

// samples of the chunk starting at sample i0 of an n-sample piece (0 .. kWideLc)
PC_HD int chain_seg_len(long long n, long long i0) {
  return i0 >= n ? 0 : (n - i0 < kWideLc ? (int)(n - i0) : kWideLc);
}

// the row in force at sample i of the piece
PC_HD int chain_seg_at(const ChainSegs& S, long long i) {
  const long long a = S.off + i;
  int lo = 0, hi = S.nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (S.seg[mid].start <= a) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// the CTA [base, end) lies inside one row and starts with no slope exchange: that row, else -1
PC_HD int chain_seg_uniform(const ChainSegs& S, long long base, long long end) {
  const int k = chain_seg_at(S, base);
  if (k + 1 < S.nseg && S.seg[k + 1].start < S.off + end) return -1;
  if (S.seg[k].start == S.off + base && (S.seg[k].swap_lc || S.seg[k].swap_hc)) return -1;
  return k;
}

// chain_cascade with a row's filters (the same arithmetic)
template <class F>
PC_HD F chain_seg_cascade(const ChainSeg& g, F* s, F x) {
  if (g.lc.on) x = chain_filter_eval<F>(g.lc, s, x);
  if (g.hc.on) x = chain_filter_eval<F>(g.hc, s + 4, x);
  return x;
}

// m samples from sample i0 of the piece on the kSegStates-wide state s; x: input (nullptr: zeros), y: output or nullptr
// (may be x).  Where a row starts, its slope exchange happens before its first sample.
template <class F>
PC_HD void chain_seg_run(const ChainSegs& S, long long i0, int m, F* s, const float* x, float* y) {
  int k = chain_seg_at(S, i0);
  for (int j = 0; j < m; ++j) {
    const long long a = S.off + i0 + j;
    if (k + 1 < S.nseg && S.seg[k + 1].start <= a) ++k;
    const ChainSeg& g = S.seg[k];
    if (g.start == a) {
      if (g.swap_lc) { const F v = s[0]; s[0] = s[kChainStates]; s[kChainStates] = v; }
      if (g.swap_hc) { const F v = s[4]; s[4] = s[kChainStates + 1]; s[kChainStates + 1] = v; }
    }
    const F v = chain_seg_cascade<F>(g, s, x ? (F)x[j] : (F)0);
    if (y) y[j] = (float)v;
  }
}

// column j of chunk c's transfer matrix T_c (a zero-input run from the unit state e_j)
PC_HD void chain_seg_column(const ChainSegs& S, long long i0, int m, int j, double* col) {
  for (int q = 0; q < kSegStates; ++q) col[q] = (q == j) ? 1.0 : 0.0;
  chain_seg_run<double>(S, i0, m, col, nullptr, nullptr);
}

// the convolver input of sample i: the ring at the row's predelay, zero below the row's delay floor
PC_HD void chain_seg_ring_read(const ChainSendParams& P, const ChainSeg& g, int ch, long long i) {
  const long long p = P.ring_pos + i - g.predelay;
  P.conv_in[(long long)ch * P.conv_stride + i] =
      p < g.delay_floor ? 0.0f : P.ring[(long long)ch * P.ring_stride + (p & P.ring_mask)];
}

// chain_wet_mix with a row's width and gains
PC_HD void chain_wet_seg_sample(const ChainWetParams& P, const ChainSeg& g, long long i) {
  float wl = P.conv[i], wr = P.conv[P.conv_stride + i];
  if (g.quad_ts) { wl += P.conv[3 * P.conv_stride + i]; wr += P.conv[2 * P.conv_stride + i]; }
  const float e = P.yrev ? P.yrev[i] : 1.0f;
  const float lin = wl * e, rin = wr * e;
  const float mid = (lin + rin) * 0.5f, side = (lin - rin) * 0.5f;
  const float norm = 1.0f / (1.0f + g.width);
  const float lout = (mid + side * g.width) * norm;
  const float rout = (mid - side * g.width) * norm;
  P.out[i] = P.dry[i] * g.drygain + lout * g.wetgain;
  P.out[P.out_stride + i] = P.dry[P.dry_stride + i] * g.drygain + rout * g.wetgain;
}

#if defined(__CUDACC__)
// grid (2 channels), block T threads (T = 64 for real-time calls, 1024 for batches); static smem
static __global__ void __launch_bounds__(1024) k_chain_send(ChainSendParams P) {
  const int ch = blockIdx.x;
#include "kernels_chain_send.inc"
}

// The send of up to kChainGroupMax handles' chain calls of one length (b200conv_chain_group_process): grid (2, n),
// block chain_send_threads(n samples); CTA (ch, i) runs channel ch of G.p[i] exactly as k_chain_send would.
static __global__ void __launch_bounds__(1024) k_chain_send_group(const __grid_constant__ ChainSendGroupParams G) {
  const ChainSendParams& P = G.p[blockIdx.y];
  const int ch = blockIdx.x;
#include "kernels_chain_send.inc"
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

// The wet mix of up to kChainGroupMax handles' chain calls (b200conv_chain_group_process): grid (blocks of 256
// samples, n), row i of the grid mixes G.p[i] as k_chain_wet would.  The CTA that draws the last ticket of the whole
// grid raises the group's one completion word.  Without one (G.done_flag nullptr), each row whose G.p[i].done_flag is
// set raises that word once all gridDim.x CTAs of the row have stored (fixed-latency group steps: every member's ring
// word carries its own sequence value); every CTA of the row counts, also those past a shorter row's n.
static __global__ void __launch_bounds__(256) k_chain_wet_group(const __grid_constant__ ChainWetGroupParams G) {
  const ChainWetParams& P = G.p[blockIdx.y];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n) chain_wet_sample(P, i);
  if (!G.done_flag) {
    chain_wet_done(P);
    return;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(G.ticket, 1u) == gridDim.x * gridDim.y - 1) {
    atomicExch(G.ticket, 0u);
    __threadfence_system();
    *reinterpret_cast<volatile unsigned int*>(G.done_flag) = G.done_val;
    __threadfence_system();
  }
}

// whole-GPU send form (see above).  One CTA of 64 threads: A, then kWideLogLc + kWidePowers - 1 squarings
static __global__ void __launch_bounds__(64) k_chain_wide_powers(ChainSendParams P, double* pw) {
  __shared__ double M[kChainStates][kChainStates];
  const int t = threadIdx.x, q = t / kChainStates, r = t % kChainStates;
  if (t < kChainStates) {
    double col[kChainStates];
    chain_power_column(P, 1, t, col);
#pragma unroll
    for (int k = 0; k < kChainStates; ++k) M[k][t] = col[k];
  }
  __syncthreads();
  for (int s = 1; s < kWideLogLc + kWidePowers; ++s) {      // M = A^(2^s)
    const double a = chain_square_entry(M, q, r);
    __syncthreads();
    M[q][r] = a;
    if (s >= kWideLogLc) pw[(s - kWideLogLc) * kChainStates * kChainStates + t] = a;
    __syncthreads();
  }
}

// the CTA's kWideSpan send samples of channel ch into shared memory, one padded row per chunk (coalesced loads)
static __device__ __forceinline__ void chain_wide_stage(const ChainSendParams& P, int ch, long long base,
                                                        float (*buf)[kWideLc + 1]) {
  for (int j = threadIdx.x; j < kWideSpan; j += kWideT) {
    const long long i = base + j;
    buf[j / kWideLc][j % kWideLc] = i < P.n ? chain_wide_send(P, ch, i) : 0.0f;
  }
}

// inclusive Hillis-Steele scan of V[kChainStates][N] with multipliers Mj[j] = M^(2^j): V[t] <- sum_k M^(t-k) V[k]
template <int N>
static __device__ __forceinline__ void chain_wide_scan(const double (*Mj)[kChainStates][kChainStates], double* V) {
  const int t = threadIdx.x;
#pragma unroll 1
  for (int j = 0, d = 1; d < N; ++j, d *= 2) {
    double nx[kChainStates];
    if (t >= d) chain_combine(Mj[j], V, N, t, d, false, nx);
    __syncthreads();
    if (t >= d) {
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) V[q * N + t] = nx[q];
    }
    __syncthreads();
  }
}

// samples of chunk t (0 .. kWideLc) of the CTA starting at base
static __device__ __forceinline__ int chain_wide_len(long long n, long long i0) {
  return i0 >= n ? 0 : (n - i0 < kWideLc ? (int)(n - i0) : kWideLc);
}

// pass 1: zero-state end points Z_c and the CTA aggregate.  grid (CTAs, 2 channels)
static __global__ void __launch_bounds__(kWideT) k_chain_wide_pass1(ChainSendParams P, ChainWideScratch W) {
  __shared__ float buf[kWideT][kWideLc + 1];
  __shared__ double V[kChainStates * kWideT];
  __shared__ double PW[kWideLogT][kChainStates][kChainStates];
  const int ch = blockIdx.y, b = blockIdx.x, t = threadIdx.x;
  const long long base = (long long)b * kWideSpan;
  chain_wide_stage(P, ch, base, buf);
  for (int j = t; j < kWideLogT * kChainStates * kChainStates; j += kWideT) (&PW[0][0][0])[j] = W.pw[j];
  __syncthreads();
  float s[kChainStates];
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) s[q] = 0.0f;
  const int m = chain_wide_len(P.n, base + (long long)t * kWideLc);
  for (int k = 0; k < m; ++k) (void)chain_cascade<float>(P, s, buf[t][k]);
  float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kChainStates;
#pragma unroll
  for (int q = 0; q < kChainStates; ++q) { z[q] = s[q]; V[q * kWideT + t] = s[q]; }
  __syncthreads();
  // tree: the segment at t (length d) absorbs the one at t + d: V[t] <- M^d V[t] + V[t + d]
#pragma unroll 1
  for (int j = 0, d = 1; d < kWideT; ++j, d *= 2) {
    double nx[kChainStates];
    const bool act = (t & (2 * d - 1)) == 0;
    if (act) chain_combine(PW[j], V, kWideT, t, d, true, nx);
    __syncthreads();
    if (act) {
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = nx[q];
    }
    __syncthreads();
  }
  if (t < kChainStates) W.agg[((long long)ch * W.nb_cap + b) * kChainStates + t] = V[t * kWideT];
}

// carry: G_0 = the scan's initial state, G_{b+1} = M^kWideT G_b + agg_b.  grid (2 channels)
static __global__ void __launch_bounds__(kWideCarryT) k_chain_wide_carry(ChainSendParams P, ChainWideScratch W, long long nb) {
  __shared__ double V[kChainStates * kWideCarryT];
  __shared__ double Q[kWideLogCarry][kChainStates][kChainStates];
  const int ch = blockIdx.x, t = threadIdx.x;
  for (int j = t; j < kWideLogCarry * kChainStates * kChainStates; j += kWideCarryT)
    (&Q[0][0][0])[j] = W.pw[kWideLogT * kChainStates * kChainStates + j];
  __shared__ double c[kChainStates];      // G at the start of the tile (in shared memory: no registers across tiles)
  if (t == 0) chain_scan_start(P, ch, c);
  const double* agg = W.agg + (long long)ch * W.nb_cap * kChainStates;
  double* G = W.carry + (long long)ch * W.nb_cap * kChainStates;
  // tile: slot 0 holds G_g0, slot k > 0 agg_{g0 + k - 1}; after the scan slot k holds G_{g0 + k}
#pragma unroll 1
  for (long long g0 = 0; g0 < nb; g0 += kWideCarryT - 1) {
    __syncthreads();
    const long long a = g0 + t - 1;
#pragma unroll
    for (int q = 0; q < kChainStates; ++q)
      V[q * kWideCarryT + t] = t == 0 ? c[q] : (a < nb - 1 ? agg[a * kChainStates + q] : 0.0);
    __syncthreads();
    chain_wide_scan<kWideCarryT>(Q, V);
    if (g0 + t < nb) {
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) G[(g0 + t) * kChainStates + q] = V[q * kWideCarryT + t];
    }
    if (t < kChainStates) c[t] = V[t * kWideCarryT + kWideCarryT - 1];
  }
}

// pass 2: true initial states, the filtered chunks, ring + predelayed convolver input (+ the undelayed send while a
// swap fades).  grid (CTAs, 2 channels)
static __global__ void __launch_bounds__(kWideT) k_chain_wide_pass2(ChainSendParams P, ChainWideScratch W) {
  __shared__ float buf[kWideT][kWideLc + 1];
  __shared__ double V[kChainStates * kWideT];
  __shared__ double PW[kWideLogT][kChainStates][kChainStates];
  const int ch = blockIdx.y, b = blockIdx.x, t = threadIdx.x;
  const long long base = (long long)b * kWideSpan;
  chain_wide_stage(P, ch, base, buf);
  if (P.lc.on || P.hc.on) {
    for (int j = t; j < kWideLogT * kChainStates * kChainStates; j += kWideT) (&PW[0][0][0])[j] = W.pw[j];
    const float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kChainStates;
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = z[q];
    __syncthreads();
    double G[kChainStates] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (t == 0) {                       // seed: V[0] = M G_b + Z_0, so that V[t] becomes the state after chunk t
      const double* g = W.carry + ((long long)ch * W.nb_cap + b) * kChainStates;
      double acc[kChainStates];
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) { G[q] = g[q]; acc[q] = V[q * kWideT]; }
      chain_affine_acc(PW[0], G, acc);
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) V[q * kWideT] = acc[q];
    }
    __syncthreads();
    chain_wide_scan<kWideT>(PW, V);
    float s[kChainStates];
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) s[q] = (float)(t == 0 ? G[q] : V[q * kWideT + t - 1]);
    const long long i0 = base + (long long)t * kWideLc;
    const int m = chain_wide_len(P.n, i0);
    for (int k = 0; k < m; ++k) buf[t][k] = chain_cascade<float>(P, s, buf[t][k]);
    if (m > 0 && i0 + m == P.n) {       // the state after the piece's last sample
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
    }
  }
  __syncthreads();
  for (int j = t; j < kWideSpan; j += kWideT) {
    const long long i = base + j;
    if (i < P.n) chain_wide_store(P, ch, i, buf[j / kWideLc][j % kWideLc]);
  }
}

// segmented whole-GPU send form (see above).  S <- T_c S + V[., c] for the CTA's chunks in order, thread q < kSegStates
// one row; `seeds`: V[q][c] becomes S[q] entering chunk c.  Sv: S in shared memory
static __device__ __forceinline__ void chain_seg_serial(const double* tc, double* V, double* Sv, bool seeds) {
  const int q = threadIdx.x;
#pragma unroll 1
  for (int c = 0; c < kWideT; ++c) {
    double a = 0.0;
    if (q < kSegStates) {
      a = V[q * kWideT + c];
      if (seeds) V[q * kWideT + c] = Sv[q];
      const double* row = tc + ((long long)c * kSegStates + q) * kSegStates;
#pragma unroll
      for (int r = 0; r < kSegStates; ++r) a = fma(row[r], Sv[r], a);
    }
    __syncthreads();
    if (q < kSegStates) Sv[q] = a;
    __syncthreads();
  }
}

// maps: per CTA the powers of its row (uniform) or its chunks' T_c and their product (mixed).  grid (CTAs)
static __global__ void __launch_bounds__(kWideT) k_chain_seg_maps(ChainSegs S, long long n, ChainSegScratch W) {
  __shared__ double M[kSegStates][kSegStates];
  const int b = blockIdx.x, t = threadIdx.x;
  const long long base = (long long)b * kWideSpan, end = base + kWideSpan < n ? base + kWideSpan : n;
  const int k = chain_seg_uniform(S, base, end);
  double* mb = W.mb + (long long)b * kSegStates * kSegStates;
  if (k >= 0) {                         // k_chain_wide_powers' squarings, P_0 .. P_kWideLogT
    const int q = t / kChainStates, r = t % kChainStates;
    if (t < kChainStates) {
      double col[kChainStates];
      for (int p = 0; p < kChainStates; ++p) col[p] = (p == t) ? 1.0 : 0.0;
      (void)chain_seg_cascade<double>(S.seg[k], col, 0.0);
#pragma unroll
      for (int p = 0; p < kChainStates; ++p) M[p][t] = col[p];
    }
    __syncthreads();
    double* pw = W.pw + (long long)b * kWideLogT * kChainStates * kChainStates;
    for (int s = 1; s <= kWideLogLc + kWideLogT; ++s) {
      double a = 0.0;
      if (t < kChainStates * kChainStates) {
#pragma unroll
        for (int p = 0; p < kChainStates; ++p) a = fma(M[q][p], M[p][r], a);
      }
      __syncthreads();
      if (t < kChainStates * kChainStates) {
        M[q][r] = a;
        if (s >= kWideLogLc && s < kWideLogLc + kWideLogT) pw[(s - kWideLogLc) * kChainStates * kChainStates + t] = a;
      }
      __syncthreads();
    }
    for (int j = t; j < kSegStates * kSegStates; j += kWideT) {
      const int p = j / kSegStates, c = j % kSegStates;
      mb[j] = (p < kChainStates && c < kChainStates) ? M[p][c] : (p == c ? 1.0 : 0.0);
    }
    return;
  }
  const long long i0 = base + (long long)t * kWideLc;
  const int m = chain_seg_len(n, i0);
  double* tc = W.tc + ((long long)b * kWideT + t) * kSegStates * kSegStates;
#pragma unroll 1
  for (int j = 0; j < kSegStates; ++j) {
    double col[kSegStates];
    chain_seg_column(S, i0, m, j, col);
#pragma unroll
    for (int p = 0; p < kSegStates; ++p) tc[p * kSegStates + j] = col[p];
  }
  __syncthreads();
  const double* T = W.tc + (long long)b * kWideT * kSegStates * kSegStates;
  const int q = t / kSegStates, r = t % kSegStates;
  const bool act = t < kSegStates * kSegStates;
  if (act) M[q][r] = T[t];
  __syncthreads();
#pragma unroll 1
  for (int c = 1; c < kWideT; ++c) {    // M <- T_c M
    double a = 0.0;
    if (act) {
      const double* Tc = T + (long long)c * kSegStates * kSegStates + q * kSegStates;
#pragma unroll
      for (int p = 0; p < kSegStates; ++p) a = fma(Tc[p], M[p][r], a);
    }
    __syncthreads();
    if (act) M[q][r] = a;
    __syncthreads();
  }
  if (act) mb[t] = M[q][r];
}

// pass 1: zero-state end points and the CTA aggregate.  grid (CTAs, 2 channels)
static __global__ void __launch_bounds__(kWideT) k_chain_seg_pass1(ChainSendParams P, ChainSegs S, ChainSegScratch W) {
  __shared__ float buf[kWideT][kWideLc + 1];
  __shared__ double V[kSegStates * kWideT];
  __shared__ double PW[kWideLogT][kChainStates][kChainStates];
  __shared__ double Sv[kSegStates];
  const int ch = blockIdx.y, b = blockIdx.x, t = threadIdx.x;
  const long long base = (long long)b * kWideSpan, end = base + kWideSpan < P.n ? base + kWideSpan : P.n;
  const int k = chain_seg_uniform(S, base, end);
  chain_wide_stage(P, ch, base, buf);
  if (k >= 0)
    for (int j = t; j < kWideLogT * kChainStates * kChainStates; j += kWideT)
      (&PW[0][0][0])[j] = W.pw[(long long)b * kWideLogT * kChainStates * kChainStates + j];
  if (t < kSegStates) Sv[t] = 0.0;
  __syncthreads();
  float s[kSegStates];
#pragma unroll
  for (int q = 0; q < kSegStates; ++q) s[q] = 0.0f;
  const long long i0 = base + (long long)t * kWideLc;
  chain_seg_run<float>(S, i0, chain_seg_len(P.n, i0), s, buf[t], nullptr);
  float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kSegStates;
#pragma unroll
  for (int q = 0; q < kSegStates; ++q) { z[q] = s[q]; V[q * kWideT + t] = s[q]; }
  __syncthreads();
  double* agg = W.agg + ((long long)ch * W.nb_cap + b) * kSegStates;
  if (k >= 0) {                         // k_chain_wide_pass1's tree
#pragma unroll 1
    for (int j = 0, d = 1; d < kWideT; ++j, d *= 2) {
      double nx[kChainStates];
      const bool act = (t & (2 * d - 1)) == 0;
      if (act) chain_combine(PW[j], V, kWideT, t, d, true, nx);
      __syncthreads();
      if (act) {
#pragma unroll
        for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = nx[q];
      }
      __syncthreads();
    }
    if (t < kSegStates) agg[t] = t < kChainStates ? V[t * kWideT] : 0.0;
  } else {
    chain_seg_serial(W.tc + (long long)b * kWideT * kSegStates * kSegStates, V, Sv, false);
    if (t < kSegStates) agg[t] = Sv[t];
  }
}

// carry: G_0 = the carried state (scan slots and stash), G_{b+1} = M_b G_b + agg_b.  grid (2 channels), 32 threads
static __global__ void __launch_bounds__(32) k_chain_seg_carry(ChainSendParams P, ChainSegScratch W, long long nb) {
  __shared__ double G[kSegStates];
  const int ch = blockIdx.x, q = threadIdx.x;
  if (q < kSegStates) G[q] = P.state[ch * kChainStateStride + q];
  __syncwarp();
  double* out = W.carry + (long long)ch * W.nb_cap * kSegStates;
  const double* agg = W.agg + (long long)ch * W.nb_cap * kSegStates;
#pragma unroll 1
  for (long long b = 0; b < nb; ++b) {
    double a = 0.0;
    if (q < kSegStates) {
      out[b * kSegStates + q] = G[q];
      a = agg[b * kSegStates + q];
      const double* row = W.mb + (b * kSegStates + q) * kSegStates;
#pragma unroll
      for (int r = 0; r < kSegStates; ++r) a = fma(row[r], G[r], a);
    }
    __syncwarp();
    if (q < kSegStates) G[q] = a;
    __syncwarp();
  }
}

// pass 2: every chunk's true initial state, the filtered chunks, the ring.  grid (CTAs, 2 channels)
static __global__ void __launch_bounds__(kWideT) k_chain_seg_pass2(ChainSendParams P, ChainSegs S, ChainSegScratch W) {
  __shared__ float buf[kWideT][kWideLc + 1];
  __shared__ double V[kSegStates * kWideT];
  __shared__ double PW[kWideLogT][kChainStates][kChainStates];
  __shared__ double Sv[kSegStates];
  const int ch = blockIdx.y, b = blockIdx.x, t = threadIdx.x;
  const long long base = (long long)b * kWideSpan, end = base + kWideSpan < P.n ? base + kWideSpan : P.n;
  const int k = chain_seg_uniform(S, base, end);
  chain_wide_stage(P, ch, base, buf);
  const double* g = W.carry + ((long long)ch * W.nb_cap + b) * kSegStates;
  const float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kSegStates;
#pragma unroll
  for (int q = 0; q < kSegStates; ++q) V[q * kWideT + t] = z[q];
  if (t < kSegStates) Sv[t] = g[t];
  float s[kSegStates];
  if (k >= 0) {                         // k_chain_wide_pass2's seed and scan
    for (int j = t; j < kWideLogT * kChainStates * kChainStates; j += kWideT)
      (&PW[0][0][0])[j] = W.pw[(long long)b * kWideLogT * kChainStates * kChainStates + j];
    __syncthreads();
    double G[kChainStates] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (t == 0) {
      double acc[kChainStates];
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) { G[q] = Sv[q]; acc[q] = V[q * kWideT]; }
      chain_affine_acc(PW[0], G, acc);
#pragma unroll
      for (int q = 0; q < kChainStates; ++q) V[q * kWideT] = acc[q];
    }
    __syncthreads();
    chain_wide_scan<kWideT>(PW, V);
#pragma unroll
    for (int q = 0; q < kChainStates; ++q) s[q] = (float)(t == 0 ? G[q] : V[q * kWideT + t - 1]);
    s[kChainStates] = (float)Sv[kChainStates];
    s[kChainStates + 1] = (float)Sv[kChainStates + 1];
  } else {
    __syncthreads();
    chain_seg_serial(W.tc + (long long)b * kWideT * kSegStates * kSegStates, V, Sv, true);
#pragma unroll
    for (int q = 0; q < kSegStates; ++q) s[q] = (float)V[q * kWideT + t];
  }
  const long long i0 = base + (long long)t * kWideLc;
  const int m = chain_seg_len(P.n, i0);
  chain_seg_run<float>(S, i0, m, s, buf[t], buf[t]);
  if (m > 0 && i0 + m == P.n) {         // the state after the piece's last sample, stash included
#pragma unroll
    for (int q = 0; q < kSegStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
  }
  __syncthreads();
  for (int j = t; j < kWideSpan; j += kWideT) {
    const long long i = base + j;
    if (i < P.n) {
      const float y = buf[j / kWideLc][j % kWideLc];
      P.ring[(long long)ch * P.ring_stride + ((P.ring_pos + i) & P.ring_mask)] = y;
      if (P.filt) P.filt[(long long)ch * P.filt_stride + i] = y;
    }
  }
}

// read: the predelayed convolver input per sample.  grid (blocks of 256 samples, 2 channels); the block finds its first
// row once, each thread walks from there
static __global__ void __launch_bounds__(256) k_chain_seg_read(ChainSendParams P, ChainSegs S) {
  __shared__ int k0;
  const long long base = (long long)blockIdx.x * blockDim.x, i = base + threadIdx.x;
  if (threadIdx.x == 0) k0 = chain_seg_at(S, base);
  __syncthreads();
  if (i >= P.n) return;
  int k = k0;
  while (k + 1 < S.nseg && S.seg[k + 1].start <= S.off + i) ++k;
  chain_seg_ring_read(P, S.seg[k], blockIdx.y, i);
}

// k_chain_wet with the row of each sample.  grid (blocks of 256 samples)
static __global__ void __launch_bounds__(256) k_chain_wet_seg(ChainWetParams P, ChainSegs S) {
  __shared__ int k0;
  const long long base = (long long)blockIdx.x * blockDim.x, i = base + threadIdx.x;
  if (threadIdx.x == 0) k0 = chain_seg_at(S, base);
  __syncthreads();
  if (i >= P.n) return;
  int k = k0;
  while (k + 1 < S.nseg && S.seg[k + 1].start <= S.off + i) ++k;
  chain_wet_seg_sample(P, S.seg[k], i);
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
// the whole-GPU send form: the same chunking, reduction tree and scan order, one CTA / thread after another
inline void emu_chain_wide_scan(const double (*Mj)[kChainStates][kChainStates], double* V, int N) {
  double* nx = new double[(size_t)N * kChainStates];
  for (int j = 0, d = 1; d < N; ++j, d *= 2) {
    for (int t = d; t < N; ++t) chain_combine(Mj[j], V, N, t, d, false, nx + (size_t)t * kChainStates);
    for (int t = d; t < N; ++t)
      for (int q = 0; q < kChainStates; ++q) V[q * N + t] = nx[(size_t)t * kChainStates + q];
  }
  delete[] nx;
}
inline void emu_chain_wide(const ChainSendParams& P, const ChainWideScratch& W, bool powers) {
  const bool filtered = P.lc.on || P.hc.on;
  const long long nb = chain_wide_ctas(P.n);
  constexpr int S2 = kChainStates * kChainStates;
  if (filtered && powers) {
    double M[kChainStates][kChainStates], nx[kChainStates][kChainStates];
    for (int j = 0; j < kChainStates; ++j) {
      double col[kChainStates];
      chain_power_column(P, 1, j, col);
      for (int k = 0; k < kChainStates; ++k) M[k][j] = col[k];
    }
    for (int s = 1; s < kWideLogLc + kWidePowers; ++s) {
      for (int q = 0; q < kChainStates; ++q)
        for (int r = 0; r < kChainStates; ++r) nx[q][r] = chain_square_entry(M, q, r);
      for (int q = 0; q < kChainStates; ++q)
        for (int r = 0; r < kChainStates; ++r) {
          M[q][r] = nx[q][r];
          if (s >= kWideLogLc) W.pw[(s - kWideLogLc) * S2 + q * kChainStates + r] = nx[q][r];
        }
    }
  }
  const double (*PW)[kChainStates][kChainStates] = reinterpret_cast<const double (*)[kChainStates][kChainStates]>(W.pw);
  float (*buf)[kWideLc + 1] = new float[kWideT][kWideLc + 1];
  double* V = new double[(size_t)kChainStates * kWideCarryT];
  auto stage = [&](int ch, long long base) {
    for (int j = 0; j < kWideSpan; ++j) {
      const long long i = base + j;
      buf[j / kWideLc][j % kWideLc] = i < P.n ? chain_wide_send(P, ch, i) : 0.0f;
    }
  };
  auto len = [&](long long i0) { return i0 >= P.n ? 0 : (P.n - i0 < kWideLc ? (int)(P.n - i0) : kWideLc); };
  if (filtered) {
    for (int ch = 0; ch < 2; ++ch)                 // pass 1
      for (long long b = 0; b < nb; ++b) {
        const long long base = b * kWideSpan;
        stage(ch, base);
        for (int t = 0; t < kWideT; ++t) {
          float s[kChainStates] = {0, 0, 0, 0, 0, 0, 0, 0};
          const int m = len(base + (long long)t * kWideLc);
          for (int k = 0; k < m; ++k) (void)chain_cascade<float>(P, s, buf[t][k]);
          float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kChainStates;
          for (int q = 0; q < kChainStates; ++q) { z[q] = s[q]; V[q * kWideT + t] = s[q]; }
        }
        for (int j = 0, d = 1; d < kWideT; ++j, d *= 2)
          for (int t = 0; t < kWideT; t += 2 * d) {
            double nx[kChainStates];
            chain_combine(PW[j], V, kWideT, t, d, true, nx);
            for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = nx[q];
          }
        for (int q = 0; q < kChainStates; ++q) W.agg[((long long)ch * W.nb_cap + b) * kChainStates + q] = V[q * kWideT];
      }
    for (int ch = 0; ch < 2; ++ch) {               // carry
      double c[kChainStates];
      chain_scan_start(P, ch, c);
      const double* agg = W.agg + (long long)ch * W.nb_cap * kChainStates;
      double* G = W.carry + (long long)ch * W.nb_cap * kChainStates;
      for (long long g0 = 0; g0 < nb; g0 += kWideCarryT - 1) {
        for (int t = 0; t < kWideCarryT; ++t) {
          const long long a = g0 + t - 1;
          for (int q = 0; q < kChainStates; ++q)
            V[q * kWideCarryT + t] = t == 0 ? c[q] : (a < nb - 1 ? agg[a * kChainStates + q] : 0.0);
        }
        emu_chain_wide_scan(PW + kWideLogT, V, kWideCarryT);
        for (int t = 0; t < kWideCarryT && g0 + t < nb; ++t)
          for (int q = 0; q < kChainStates; ++q) G[(g0 + t) * kChainStates + q] = V[q * kWideCarryT + t];
        for (int q = 0; q < kChainStates; ++q) c[q] = V[q * kWideCarryT + kWideCarryT - 1];
      }
    }
  }
  for (int ch = 0; ch < 2; ++ch)                   // pass 2
    for (long long b = 0; b < nb; ++b) {
      const long long base = b * kWideSpan;
      stage(ch, base);
      if (filtered) {
        for (int t = 0; t < kWideT; ++t) {
          const float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kChainStates;
          for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = z[q];
        }
        double G[kChainStates], acc[kChainStates];
        for (int q = 0; q < kChainStates; ++q) {
          G[q] = W.carry[((long long)ch * W.nb_cap + b) * kChainStates + q];
          acc[q] = V[q * kWideT];
        }
        chain_affine_acc(PW[0], G, acc);
        for (int q = 0; q < kChainStates; ++q) V[q * kWideT] = acc[q];
        emu_chain_wide_scan(PW, V, kWideT);
        for (int t = 0; t < kWideT; ++t) {
          float s[kChainStates];
          for (int q = 0; q < kChainStates; ++q) s[q] = (float)(t == 0 ? G[q] : V[q * kWideT + t - 1]);
          const long long i0 = base + (long long)t * kWideLc;
          const int m = len(i0);
          for (int k = 0; k < m; ++k) buf[t][k] = chain_cascade<float>(P, s, buf[t][k]);
          if (m > 0 && i0 + m == P.n)
            for (int q = 0; q < kChainStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
        }
      }
      for (int j = 0; j < kWideSpan; ++j) {
        const long long i = base + j;
        if (i < P.n) chain_wide_store(P, ch, i, buf[j / kWideLc][j % kWideLc]);
      }
    }
  delete[] buf;
  delete[] V;
}
// the segmented form: the same maps, chunking, folds and scan order, one CTA / thread after another
inline void emu_chain_seg_serial(const double* tc, double* V, double* Sv, bool seeds) {
  for (int c = 0; c < kWideT; ++c) {
    double a[kSegStates];
    for (int q = 0; q < kSegStates; ++q) {
      a[q] = V[q * kWideT + c];
      if (seeds) V[q * kWideT + c] = Sv[q];
      const double* row = tc + ((long long)c * kSegStates + q) * kSegStates;
      for (int r = 0; r < kSegStates; ++r) a[q] = fma(row[r], Sv[r], a[q]);
    }
    for (int q = 0; q < kSegStates; ++q) Sv[q] = a[q];
  }
}
inline void emu_chain_seg(const ChainSendParams& P, const ChainSegs& S, const ChainSegScratch& W) {
  constexpr int S2 = kChainStates * kChainStates, T2 = kSegStates * kSegStates;
  const long long nb = chain_wide_ctas(P.n);
  auto cta_end = [&](long long base) { return base + kWideSpan < P.n ? base + kWideSpan : P.n; };
  for (long long b = 0; b < nb; ++b) {             // maps
    const long long base = b * kWideSpan;
    const int k = chain_seg_uniform(S, base, cta_end(base));
    double* mb = W.mb + b * T2;
    if (k >= 0) {
      double M[kChainStates][kChainStates], nx[kChainStates][kChainStates];
      for (int j = 0; j < kChainStates; ++j) {
        double col[kChainStates];
        for (int p = 0; p < kChainStates; ++p) col[p] = (p == j) ? 1.0 : 0.0;
        (void)chain_seg_cascade<double>(S.seg[k], col, 0.0);
        for (int p = 0; p < kChainStates; ++p) M[p][j] = col[p];
      }
      for (int s = 1; s <= kWideLogLc + kWideLogT; ++s) {
        for (int q = 0; q < kChainStates; ++q)
          for (int r = 0; r < kChainStates; ++r) nx[q][r] = chain_square_entry(M, q, r);
        for (int q = 0; q < kChainStates; ++q)
          for (int r = 0; r < kChainStates; ++r) {
            M[q][r] = nx[q][r];
            if (s >= kWideLogLc && s < kWideLogLc + kWideLogT) W.pw[(b * kWideLogT + s - kWideLogLc) * S2 + q * kChainStates + r] = nx[q][r];
          }
      }
      for (int p = 0; p < kSegStates; ++p)
        for (int c = 0; c < kSegStates; ++c)
          mb[p * kSegStates + c] = (p < kChainStates && c < kChainStates) ? M[p][c] : (p == c ? 1.0 : 0.0);
      continue;
    }
    const double* T = W.tc + b * kWideT * T2;
    for (int t = 0; t < kWideT; ++t) {
      const long long i0 = base + (long long)t * kWideLc;
      double* tc = W.tc + (b * kWideT + t) * T2;
      for (int j = 0; j < kSegStates; ++j) {
        double col[kSegStates];
        chain_seg_column(S, i0, chain_seg_len(P.n, i0), j, col);
        for (int p = 0; p < kSegStates; ++p) tc[p * kSegStates + j] = col[p];
      }
    }
    double M[kSegStates][kSegStates], nx[kSegStates][kSegStates];
    for (int j = 0; j < T2; ++j) M[j / kSegStates][j % kSegStates] = T[j];
    for (int c = 1; c < kWideT; ++c) {
      for (int q = 0; q < kSegStates; ++q)
        for (int r = 0; r < kSegStates; ++r) {
          double a = 0.0;
          for (int p = 0; p < kSegStates; ++p) a = fma(T[c * T2 + q * kSegStates + p], M[p][r], a);
          nx[q][r] = a;
        }
      std::memcpy(M, nx, sizeof(M));
    }
    for (int j = 0; j < T2; ++j) mb[j] = M[j / kSegStates][j % kSegStates];
  }
  float (*buf)[kWideLc + 1] = new float[kWideT][kWideLc + 1];
  double* V = new double[(size_t)kSegStates * kWideT];
  const double (*PWall)[kChainStates][kChainStates] = reinterpret_cast<const double (*)[kChainStates][kChainStates]>(W.pw);
  auto stage = [&](int ch, long long base) {
    for (int j = 0; j < kWideSpan; ++j) {
      const long long i = base + j;
      buf[j / kWideLc][j % kWideLc] = i < P.n ? chain_wide_send(P, ch, i) : 0.0f;
    }
  };
  for (int ch = 0; ch < 2; ++ch)                   // pass 1
    for (long long b = 0; b < nb; ++b) {
      const long long base = b * kWideSpan;
      const int k = chain_seg_uniform(S, base, cta_end(base));
      stage(ch, base);
      for (int t = 0; t < kWideT; ++t) {
        float s[kSegStates] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        const long long i0 = base + (long long)t * kWideLc;
        chain_seg_run<float>(S, i0, chain_seg_len(P.n, i0), s, buf[t], nullptr);
        float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kSegStates;
        for (int q = 0; q < kSegStates; ++q) { z[q] = s[q]; V[q * kWideT + t] = s[q]; }
      }
      double* agg = W.agg + ((long long)ch * W.nb_cap + b) * kSegStates;
      if (k >= 0) {
        const double (*PW)[kChainStates][kChainStates] = PWall + b * kWideLogT;
        for (int j = 0, d = 1; d < kWideT; ++j, d *= 2)
          for (int t = 0; t < kWideT; t += 2 * d) {
            double nx[kChainStates];
            chain_combine(PW[j], V, kWideT, t, d, true, nx);
            for (int q = 0; q < kChainStates; ++q) V[q * kWideT + t] = nx[q];
          }
        for (int q = 0; q < kSegStates; ++q) agg[q] = q < kChainStates ? V[q * kWideT] : 0.0;
      } else {
        double Sv[kSegStates] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        emu_chain_seg_serial(W.tc + b * kWideT * T2, V, Sv, false);
        for (int q = 0; q < kSegStates; ++q) agg[q] = Sv[q];
      }
    }
  for (int ch = 0; ch < 2; ++ch) {                 // carry
    double G[kSegStates];
    for (int q = 0; q < kSegStates; ++q) G[q] = P.state[ch * kChainStateStride + q];
    double* out = W.carry + (long long)ch * W.nb_cap * kSegStates;
    const double* agg = W.agg + (long long)ch * W.nb_cap * kSegStates;
    for (long long b = 0; b < nb; ++b) {
      double a[kSegStates];
      for (int q = 0; q < kSegStates; ++q) {
        out[b * kSegStates + q] = G[q];
        a[q] = agg[b * kSegStates + q];
        for (int r = 0; r < kSegStates; ++r) a[q] = fma(W.mb[(b * kSegStates + q) * kSegStates + r], G[r], a[q]);
      }
      for (int q = 0; q < kSegStates; ++q) G[q] = a[q];
    }
  }
  for (int ch = 0; ch < 2; ++ch)                   // pass 2
    for (long long b = 0; b < nb; ++b) {
      const long long base = b * kWideSpan;
      const int k = chain_seg_uniform(S, base, cta_end(base));
      stage(ch, base);
      const double* g = W.carry + ((long long)ch * W.nb_cap + b) * kSegStates;
      for (int t = 0; t < kWideT; ++t) {
        const float* z = W.z + (((long long)ch * W.nb_cap + b) * kWideT + t) * kSegStates;
        for (int q = 0; q < kSegStates; ++q) V[q * kWideT + t] = z[q];
      }
      double G[kChainStates];
      if (k >= 0) {
        const double (*PW)[kChainStates][kChainStates] = PWall + b * kWideLogT;
        double acc[kChainStates];
        for (int q = 0; q < kChainStates; ++q) { G[q] = g[q]; acc[q] = V[q * kWideT]; }
        chain_affine_acc(PW[0], G, acc);
        for (int q = 0; q < kChainStates; ++q) V[q * kWideT] = acc[q];
        emu_chain_wide_scan(PW, V, kWideT);
      } else {
        double Sv[kSegStates];
        for (int q = 0; q < kSegStates; ++q) Sv[q] = g[q];
        emu_chain_seg_serial(W.tc + b * kWideT * T2, V, Sv, true);
      }
      for (int t = 0; t < kWideT; ++t) {
        float s[kSegStates];
        if (k >= 0) {
          for (int q = 0; q < kChainStates; ++q) s[q] = (float)(t == 0 ? G[q] : V[q * kWideT + t - 1]);
          s[kChainStates] = (float)g[kChainStates];
          s[kChainStates + 1] = (float)g[kChainStates + 1];
        } else {
          for (int q = 0; q < kSegStates; ++q) s[q] = (float)V[q * kWideT + t];
        }
        const long long i0 = base + (long long)t * kWideLc;
        const int m = chain_seg_len(P.n, i0);
        chain_seg_run<float>(S, i0, m, s, buf[t], buf[t]);
        if (m > 0 && i0 + m == P.n)
          for (int q = 0; q < kSegStates; ++q) P.state[ch * kChainStateStride + q] = s[q];
      }
      for (int j = 0; j < kWideSpan; ++j) {
        const long long i = base + j;
        if (i < P.n) {
          const float y = buf[j / kWideLc][j % kWideLc];
          P.ring[(long long)ch * P.ring_stride + ((P.ring_pos + i) & P.ring_mask)] = y;
          if (P.filt) P.filt[(long long)ch * P.filt_stride + i] = y;
        }
      }
    }
  delete[] buf;
  delete[] V;
}
inline void emu_chain_seg_read(const ChainSendParams& P, const ChainSegs& S) {
  for (int ch = 0; ch < 2; ++ch)
    for (long long i = 0; i < P.n; ++i) chain_seg_ring_read(P, S.seg[chain_seg_at(S, i)], ch, i);
}
inline void emu_chain_wet_seg(const ChainWetParams& P, const ChainSegs& S) {
  for (long long i = 0; i < P.n; ++i) chain_wet_seg_sample(P, S.seg[chain_seg_at(S, i)], i);
}
inline void emu_chain_wet(const ChainWetParams& P) {
  for (long long i = 0; i < P.n; ++i) chain_wet_sample(P, i);
  if (P.done_flag) *P.done_flag = P.done_val;
}
inline void emu_chain_wet_xfade(const ChainWetParams& P) {
  for (long long i = 0; i < P.n; ++i) chain_wet_xfade_sample(P, i);
  if (P.done_flag) *P.done_flag = P.done_val;
}
inline void emu_chain_send_group(const ChainSendGroupParams& G, int T) {
  for (int i = 0; i < G.n; ++i) emu_chain_send(G.p[i], T);
}
inline void emu_chain_wet_group(const ChainWetGroupParams& G) {
  for (int i = 0; i < G.n; ++i) {
    for (long long j = 0; j < G.p[i].n; ++j) chain_wet_sample(G.p[i], j);
    if (!G.done_flag && G.p[i].done_flag) *G.p[i].done_flag = G.p[i].done_val;
  }
  if (G.done_flag) *G.done_flag = G.done_val;
}
#endif

}  // namespace pc
