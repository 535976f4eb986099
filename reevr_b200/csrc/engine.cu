// engine.cu — host side of the H100 partitioned-convolution engine + the C ABI (include/b200conv.h).
//
// One handle = C mono convolvers sharing a stage schedule.  Stage s = uniform partitioned
// convolver with block B_s over the IR taps [off_s, off_{s+1}) whose contribution is delayed by
// q_s = off_s / B_s blocks (the scheme TwoStageFFTConvolver.cpp:120-138,166-222 uses for its
// tails, generalised): stage 0 is the zero-latency head (handles partially filled blocks like
// FFTConvolver.cpp:164-193), stages >= 1 work on completed blocks only and deposit their
// output into a look-ahead ring the head's inverse-FFT epilogue adds on top.
//
// Device state per stage (all float32 / float2, resident for the handle's lifetime):
//   H   [C][Prows][B]   IR partition spectra (this shard's partition range), zero padded
//   X   [C][R][B]       input-spectrum timeline = the frequency-domain delay line, linear:
//                       row `head` is the open block; partition p of output block t reads row
//                       head + t - p.  Compacted (history moved to the front) when full.
//   Y[2] [1+T][C][B]    spectra of the current launch group (double-buffered by group so that reduce +
//                       inverse FFT of group i overlap the sweep of group i+1); row 0 = last completed
//                       block of the previous group (the overlap state, FFTConvolver.cpp:204 kept in
//                       the frequency domain)
//   inbuf [C][B + Lmax] time-domain input of the open block + this call's samples
//   fut [C][ring]       (stages >= 1) look-ahead output ring, indexed by absolute position
// Streams: s_main (forward FFT + sweep), s_post (exchange/reduce + inverse FFT + mixdown), s_in / s_out
// (PCIe copies of the pipelined host path).  Multi-GPU: partition-range shards with either a reduce hook
// (NCCL) or the fused slot exchange over peer memory (run_group_p2p).
#if defined(PC_EMULATE)
#include "cuda_emu.h"      // tests/emu: host stand-in for the CUDA runtime (test infrastructure)
#else
#include <cuda_runtime.h>
#endif

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200conv.h"
#include "kernels.cuh"
#include "kernels_stream.cuh"
#include "kernels_fft512.cuh"
#include "kernels_rt.cuh"
#include "kernels_chain.cuh"
#include "kernels_tc.cuh"
#include "kernels_lfft.cuh"
#include "kernels_fourstep.cuh"

namespace {

constexpr int kDPre = 8;          // max prefetch distance of the CMAC kernels (rows readable past the end)
constexpr int kPadP = 96;         // H / history rows are padded to a multiple of this = lcm of every sweep tile height TT in use (8, 12, 16, 24, 32)
constexpr int kMaxTT = 32;        // slack rows after the newest X row
constexpr int kDefaultBatch = 4224;   // 132 SMs * 32
constexpr int kMaxBlockLog2 = 13;     // B <= 8192 (two M-point ping-pong buffers = 128 KB smem)

inline size_t next_pow2(size_t v) { size_t p = 1; while (p < v) p *= 2; return p; }
inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// grow-only device scratch of the long sweep forms (reserve)
template <class T>
struct Scratch {
  T* p = nullptr;
  size_t bytes = 0;
  void release() { cudaFree(p); *this = Scratch(); }
};

// An operand a long sweep form builds once from one stage's partition spectra H and keeps until the IR changes
template <class T>
struct IrCache {
  Scratch<T> buf;
  const void* H = nullptr;           // the H (with its partition rows, block size and channels) it was built from
  int P = 0, B = 0, C = 0;
  bool holds(const pc::CmacParams& cp, int c) const { return H == cp.H && P == cp.Ppad && B == cp.B && C == c; }
  void built_from(const pc::CmacParams& cp, int c) { H = cp.H; P = cp.Ppad; B = cp.B; C = c; }
  void release() { buf.release(); H = nullptr; }
};

struct Stage {
  int B = 0;
  size_t tap_off = 0;      // first IR tap of this stage
  size_t tap_end = 0;      // one past the last tap (over all channels)
  int q = 0;               // output delay in blocks (tap_off / B)
  int P_full = 0;          // partitions of the stage (max over channels)
  int p_begin = 0, p_end = 0;   // this shard's partition range
  int P = 0;               // p_end - p_begin
  int Prows = 0;           // allocated H rows
  int hist = 0;            // X rows kept before the open block
  int Tcap = 0;            // max blocks per launch group
  int R = 0;               // X rows allocated
  long long head = 0;      // X row of the open block
  long long blocks_done = 0;   // completed blocks since init/clear
  int fill = 0;            // samples of the open block already buffered
  float2* H = nullptr;
  float2* X = nullptr;
  float2* Y[2] = {nullptr, nullptr};   // double buffer: the sweep of group i+1 may overlap reduce+IFFT of group i
  // B = 512 groups on the tensor-core sweep: its bin-major complex result, read by the inverse FFT (paired with Y[b])
  Scratch<float2> tcY[2];
  int ybuf = 0;
  cudaEvent_t ev_sweep[2] = {nullptr, nullptr};   // Y[b] rows written by the sweep
  cudaEvent_t ev_post[2] = {nullptr, nullptr};    // Y[b] no longer needed by reduce / inverse FFT
  float2* tw = nullptr;
  float2* tab512 = nullptr;   // B == 512: tables of the register-resident FFT kernels
  float* inbuf = nullptr;           // open block of this stage (+ the current call's samples on the batch path)
  float* inbuf_alt = nullptr;       // stages >= 1: second buffer — a tail block enqueued on s_tail keeps reading the
                                    // one it completed while the following calls already fill the other
  size_t in_stride = 0;
  // tail blocks enqueued on the low-priority stream by the real-time path (stages >= 1)
  cudaEvent_t ev_job[2] = {nullptr, nullptr};
  long long job_out_start[2] = {0, 0};   // absolute sample position where the job's output is first needed
  bool job_waited[2] = {true, true};
  unsigned long long njobs = 0;
  float* fut = nullptr;
  size_t ring = 0;
};

struct EventPair { cudaEvent_t a, b; int kind; };

// Fixed-latency mode (b200conv_set_latency): pinned rings of `nslots` head blocks the steps read their input from and
// write their output into, zero-copy.  Block k lives in slot k % nslots of both rings.  Each step raises the ring's
// sequence word to its own value in stream order; the host compares wrap-safely, (int)(word - want) >= 0.
struct LatRing {
  int rows_in = 0, rows_out = 0;
  size_t B = 0, nslots = 0, len = 0;      // len = nslots * B samples per row
  size_t piece = 0;                       // samples per channel one pass of a call takes in (a multiple of B)
  float* in = nullptr; float* in_dev = nullptr;     // [rows_in][len], pinned, + its device address
  float* out = nullptr; float* out_dev = nullptr;   // [rows_out][len]
  unsigned int* word = nullptr; unsigned int* word_dev = nullptr;   // pinned sequence word
  unsigned int* ticket = nullptr;         // device word: last-CTA ticket of the chain's wet kernel
  unsigned int seq = 0;                   // last sequence value issued
  std::vector<unsigned int> slot_seq;     // value of the step that last wrote each output slot
  long long pos = 0;                      // input samples taken in since set_latency / clear
  cudaStream_t last_st = nullptr;         // stream of the last step (every earlier step is ordered before it)
};

// What the rows of a chain call carry from one to the next, and the chain from one call to the next
struct ChainCarry {
  bool six[2] = {false, false};    // slot 0 of the low / high cut's state holds the 6 dB `state` (else ic1)
  long long delay_len = 0;         // the reference's delay-line length D (src/PluginProcessor.cpp:640, 1184-1188)
  long long delay_floor = 0;       // absolute position of the last growth of D: older samples read zero as delay
};

// The send / wet chain around a handle's convolvers (b200conv_chain_*, kernels_chain.cuh): one object, so that the
// end of an IR hot swap (chain_move) hands all of it to the incoming handle
struct Chain {
  bool on = false;
  b200conv_chain_config cfg{};
  pc::ChainFilter lc{}, hc{};
  float* io = nullptr;             // [dry L, dry R, ysend, yrev, out L, out R][Lmax] staging
  float* conv_in = nullptr;        // [2][Lmax] convolver input (after filters + predelay)
  float* filt = nullptr;           // [3][Lmax]: filtered send of the call ; row 2 stays zero (LR / RL input of a
                                   // quad handle being crossfaded in)
  float* state = nullptr;          // [4][kChainStateStride] filter states: rows 0-1 the send, rows 2-3 the warm-up replay of a swap
  void* wide = nullptr;            // scratch of the whole-GPU send form (pc::ChainWideScratch), sized for Lmax
  float* hpin = nullptr;           // pinned [dry L, dry R, ysend, yrev, out L, out R][hpin_cap]: zero-copy I/O of real-time chain calls
  float* hpin_dev = nullptr;
  float* ring = nullptr;           // [2][ring] predelay ring; also the warmer of an IR hot swap (>= W samples of history)
  size_t ring_size = 0;
  long long ring_pos = 0;          // absolute position of the next sample written (ring index: & (ring_size - 1))
  ChainCarry carry;
  LatRing* lat = nullptr;          // fixed latency (b200conv_chain_process): dry L, dry R, ysend, yrev in; L, R out
  // parameter events inside device calls (b200conv_chain_process_device_events), allocated by the first call that needs
  // them and grown before a call's first launch: the segmented send form's scratch (pc::ChainSegScratch, sized for
  // Lmax), the call's segment table on the device and its pinned staging, and the event that ends the table's copy
  void* seg = nullptr;
  pc::ChainSeg* segtab = nullptr;
  pc::ChainSeg* segpin = nullptr;
  size_t segcap = 0;
  cudaEvent_t segev = nullptr;
  bool segev_live = false;
};

}  // namespace

struct b200conv {
  b200conv_config cfg{};
  int C = 1;
  std::string err;
  bool sticky_cuda_error = false;
  std::vector<Stage> stages;
  std::vector<size_t> ir_len;     // post-trim
  size_t Lmax = 0;                // max samples per launch group
  long long abs_pos = 0;          // absolute stream position (samples since init/clear)
  cudaStream_t s_main = nullptr, s_post = nullptr, s_in = nullptr, s_out = nullptr;
  cudaStream_t s_tail = nullptr;     // lowest priority: tail-stage blocks of the real-time path (run_tail_block)
  cudaStream_t s_launch = nullptr;   // stream the kernel launchers use: s_main, or s_tail while a tail block is enqueued
  cudaEvent_t ev_rt = nullptr;       // real-time kernel of the current call done (s_main)
  float* hpin_in_dev = nullptr;      // device-side addresses of the pinned staging buffers (zero-copy I/O)
  float* hpin_out_dev = nullptr;
  unsigned long long* stream_ticket = nullptr;   // ticket counters of the dynamic streaming sweep (device, 256 words)
  unsigned long long stream_ticket_base = 0;
  unsigned int stream_launches = 0;             // alternates the walk direction of the streaming sweep
  bool opt_stream_alt = std::getenv("B200CONV_NO_STREAM_ALT") == nullptr;
  unsigned int* hflag = nullptr;     // pinned completion word of the real-time kernel (+ its device-side address)
  unsigned int* hflag_dev = nullptr;
  unsigned int flag_epoch = 0;
  cudaEvent_t ev_h2d[2]{}, ev_comp[2]{}, ev_d2h[2]{}, ev_din[2]{};
  cudaEvent_t ev_join = nullptr;
  float* din[2] = {nullptr, nullptr};
  float* dout[2] = {nullptr, nullptr};
  float* hpin_in = nullptr;       // pinned host staging of the latency path: all channels of a call in ONE copy
  float* hpin_out = nullptr;
  size_t hpin_cap = 0;            // samples per channel the staging holds
  unsigned long long launches = 0;
  // timing
  bool timing = false;
  std::vector<EventPair> ev_pool;
  size_t ev_used = 0;
  float t_cmac = 0, t_fft = 0, t_ifft = 0;
  int n_cmac = 0;
  // sharding
  b200conv_reduce_fn reduce = nullptr;
  void* reduce_user = nullptr;
  int n_sm = 132;
  // I/O routing + mixdown (b200conv_set_routing)
  bool route_on = false;
  int n_in = 0, n_out = 0;
  int in_map[8] = {};
  float mix[64] = {};
  float* dch[1] = {nullptr};                // per-convolver outputs [C][Lmax] before the mixdown
  // time-slice sharding: Y row 0 (the overlap state, spectrum of the last completed block) does not belong to
  // the block in front of the open one any more (the timeline was advanced by forward FFTs only)
  bool yprev_stale = false;
  // send / wet chain around the convolver (b200conv_chain_*, kernels_chain.cuh)
  Chain chain;
  bool route_in_only = false;        // chain calls: convolver c reads chain input c & 1, outputs stay per convolver
  // IR hot swap inside the chain (b200conv_chain_swap): swap_peer links the two handles of a pending swap
  b200conv* swap_peer = nullptr;
  int swap_state = 0;                // 0 none, 1 armed, 2 fading, 3 this handle gave its chain away
  bool swap_live = false;            // the live side of the pending swap (holds the fade state below)
  size_t swap_block = 0;             // host block of the warm-up replay
  long long swap_xfade = 0, swap_xfadelen = 0;   // the reference's xfade / xfadelen counters
  // b200conv_init_*_shaped: the taps handed to init are DEVICE buffers (shaped there) with known post-trim lengths
  bool ir_on_device = false;
  const size_t* ir_trimmed = nullptr;
  // tuning / A-B switches (b200conv_set_option; defaults from the environment)
  bool opt_rt = std::getenv("B200CONV_NO_RT") == nullptr;
  bool opt_fft512 = std::getenv("B200CONV_NO_FFT512") == nullptr;
  bool opt_slice_tail = true;        // sliced calls: also transform the last P blocks of the call (full-state contract)
  // tensor-core sweep (kernels_tc.cuh): Toeplitz tile images of one stage's H, per-bin time lines, the bin-major
  // complex result of the groups that merge it into Y rows
  bool opt_tc = std::getenv("B200CONV_NO_TC") == nullptr;
  IrCache<void> tc_A;                // FP16 images, then the per-line scale exponents (kernels_tc.cuh a_image_bytes_gauss)
  Scratch<float> tc_Xt;
  Scratch<float2> tc_Yt;
  int* tc_err = nullptr;             // mapped pinned word: a barrier wait of k_tc_sweep gave up
  int* tc_err_dev = nullptr;
  // line-FFT sweep (kernels_lfft.cuh): kN-point spectra of every line of one stage's H
  IrCache<float2> lf_S;
  // four-step sweep (kernels_fourstep.cuh): the IR spectrum, the column spectra of a group, and the taps / the history
  // in front of a group
  IrCache<float2> fs_S;
  Scratch<float2> fs_X;
  Scratch<float> fs_hist;
  unsigned fs_rows_ctas[2] = {0, 0};  // resident CTAs of k_fs_rows<false> / <true> on the device (persistent grid)
  // the scratch of a long form (40, 41 or 42) did not fit once: automatic selection stays on the FFMA sweep
  bool tc_alloc_failed = false;
  int last_variant = 0;              // sweep form the last launch_cmac resolved to (b200conv_last_sweep_variant)
  // slot exchange (fused multi-GPU path), stage 0 of a single-stage handle
  bool p2p_on = false;
  int p2p_mode = 0;
  int xSR = 0;                       // rows per slot (slice rows + halo + spare)
  size_t xslot = 0;                  // float2 per slot
  float2* Yx[2] = {nullptr, nullptr};       // [G slots][xSR][C][B]
  float2* Hh = nullptr;                     // [3][G][C][B] halo of the next group's first slice (owner 0)
  float* xout[2] = {nullptr, nullptr};      // [C][Lmax] output exchange (used on shard 0)
  unsigned int* xflags = nullptr;           // 8 barrier words + 1 error word
  int hidx = 0;                             // halo buffer in use (mod 3)
  unsigned int bar_epoch = 0;
  float2* peerYx[8][2] = {};
  float2* peerHh0 = nullptr;
  float* peer_xout0[2] = {nullptr, nullptr};
  unsigned int* peer_flags[8] = {};
  bool bcast_in = false;                    // shard 0 uploads the input and stores it into the peers' staging (NVLink)
  float* peer_din[8][2] = {};               // every shard's din[0..1] (mapped on shard 0 when the broadcast is enabled)
  std::vector<unsigned char> din_records;   // the peers' exported din records, opened lazily
  unsigned int in_epoch = 0;                // epoch of the "input landed" barrier (flag words 16..23)
  unsigned long long xgrp = 0;              // slot-exchange groups issued so far
  cudaEvent_t ev_b1[2] = {nullptr, nullptr};   // first barrier of group (xgrp & 1) passed: peers finished reading din
  std::vector<void*> ipc_opened;
  b200conv_barrier_fn host_barrier = nullptr;
  void* host_barrier_user = nullptr;
  // tail-stage sharding (option "shard_head" = 0): rank 0 holds the head stage whole, only the stages >= 1 are
  // partition-range sharded; their partial spectra reach rank 0 through the reduce hook or the tail slot exchange
  bool opt_shard_head = true;
  bool p2p_tail = false;                    // tail slot exchange attached
  float2* Tx[4] = {};                       // stage s >= 1: [2 parities][G slots][2 rows][C][B] (used on rank 0)
  float2* peerTx0[4] = {};                  // rank 0's Tx (mapped)
  unsigned int* ttick = nullptr;            // tickets + tile counter of the exchange sweep (tail_tick_words)
  unsigned long long tx_blocks[4] = {};     // tail blocks exchanged per stage since the attach (flag epochs)
  bool rt_tail_joined = false;              // the last real-time call waited for a tail block (and its barrier)
  // fixed-latency mode (b200conv_set_latency): D samples, a multiple of the head block; 0 = zero latency
  size_t lat_D = 0;
  LatRing* lat = nullptr;                   // b200conv_process: C rows each way (routing uses n_in / n_out of them)
  unsigned long long lat_waits = 0;         // waits for a step that had not completed (since set_latency)
  // groups (b200conv_group_process): s_main may hold work the host has not seen complete (every entry point sets it in
  // set_device, a real-time call that saw its completion word clears it); a group's event this handle's next own call
  // orders s_main and s_post behind (nullptr: none)
  bool main_unsynced = false;
  cudaEvent_t grp_ev = nullptr;
  // a device-buffer group call leaves no event behind: grp_ev is recorded on grp_st (the group's stream) by this
  // handle's next own call, in set_device (nullptr: nothing to record)
  cudaStream_t grp_st = nullptr;
};

namespace {

// Only errors that poison the CUDA context (or mean there is no usable device) make the handle fail for
// good; everything else — out of memory while loading a long IR, CUDA IPC not permitted in this container,
// an invalid argument — is cleared from the runtime, reported through the status code and leaves the
// handle usable (the caller can fall back to the reduce hook, load a shorter IR, ...).
bool cuda_error_is_sticky(cudaError_t e) {
#if defined(PC_EMULATE)
  (void)e;
  return false;
#else
  switch (e) {
    case cudaErrorIllegalAddress: case cudaErrorLaunchFailure: case cudaErrorLaunchTimeout:
    case cudaErrorIllegalInstruction: case cudaErrorMisalignedAddress: case cudaErrorInvalidAddressSpace:
    case cudaErrorInvalidPc: case cudaErrorHardwareStackError: case cudaErrorAssert:
    case cudaErrorECCUncorrectable: case cudaErrorNoDevice: case cudaErrorInsufficientDriver:
    case cudaErrorDevicesUnavailable: case cudaErrorCudartUnloading: case cudaErrorUnknown:
      return true;
    default:
      return false;
  }
#endif
}

int cuda_fail(b200conv* h, cudaError_t e, const char* what) {
  h->err = std::string(what) + ": " + cudaGetErrorString(e);
  cudaGetLastError();                                   // clear the runtime's (non-sticky) last error
  if (cuda_error_is_sticky(e)) h->sticky_cuda_error = true;
  return e == cudaErrorMemoryAllocation ? B200CONV_ENOMEM : B200CONV_ECUDA;
}

#define CU_CHECK(h, expr)                                                                  \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) return cuda_fail((h), e__, #expr);                             \
  } while (0)

int fail(b200conv* h, int code, const std::string& msg) { h->err = msg; return code; }

void free_stage(Stage& s) {
  cudaFree(s.H); cudaFree(s.X); cudaFree(s.Y[0]); cudaFree(s.Y[1]); s.tcY[0].release(); s.tcY[1].release(); cudaFree(s.tw); cudaFree(s.tab512); cudaFree(s.inbuf); cudaFree(s.inbuf_alt); cudaFree(s.fut);
  for (int i = 0; i < 2; ++i) {
    if (s.ev_job[i]) cudaEventDestroy(s.ev_job[i]);
    if (s.ev_sweep[i]) cudaEventDestroy(s.ev_sweep[i]);
    if (s.ev_post[i]) cudaEventDestroy(s.ev_post[i]);
  }
  s = Stage();
}

void p2p_release(b200conv* h) {
#if !defined(PC_EMULATE)
  for (void* p : h->ipc_opened) cudaIpcCloseMemHandle(p);
#endif
  h->ipc_opened.clear();
  cudaFree(h->Yx[0]); cudaFree(h->Yx[1]); cudaFree(h->Hh); cudaFree(h->xout[0]); cudaFree(h->xout[1]); cudaFree(h->xflags);
  h->Yx[0] = h->Yx[1] = nullptr; h->Hh = nullptr; h->xout[0] = h->xout[1] = nullptr; h->xflags = nullptr;
  h->p2p_on = false; h->hidx = 0; h->bar_epoch = 0; h->in_epoch = 0; h->xgrp = 0; h->bcast_in = false;
  for (int s = 0; s < 4; ++s) { cudaFree(h->Tx[s]); h->Tx[s] = h->peerTx0[s] = nullptr; h->tx_blocks[s] = 0; }
  cudaFree(h->ttick); h->ttick = nullptr;
  h->p2p_tail = false;
  for (int i = 0; i < 2; ++i) { if (h->ev_b1[i]) cudaEventDestroy(h->ev_b1[i]); h->ev_b1[i] = nullptr; }
}

void lat_free(LatRing*& r) {
  if (!r) return;
  if (r->in) cudaFreeHost(r->in);
  if (r->out) cudaFreeHost(r->out);
  if (r->word) cudaFreeHost(r->word);
  cudaFree(r->ticket);
  delete r;
  r = nullptr;
}

// a fresh stream: the next D output samples are zeros; every slot counts as consumed
void lat_restart(LatRing* r) {
  if (!r) return;
  r->pos = 0;
  r->slot_seq.assign(r->nslots, r->seq);
}

// Rings for latency D and head block B: D / B blocks in flight behind the input, one pass of a call (`piece` samples),
// the open block and one spare.  A slot is then rewritten only after the host has consumed its block, so the reuse
// check never waits while the device keeps up.
int lat_alloc(b200conv* h, LatRing** out, int rows_in, int rows_out, size_t D, size_t B, size_t piece) {
  LatRing* r = new (std::nothrow) LatRing();
  if (!r) return fail(h, B200CONV_ENOMEM, "out of host memory");
  *out = r;
  r->rows_in = rows_in; r->rows_out = rows_out; r->B = B; r->piece = piece;
  r->nslots = D / B + piece / B + 2;
  r->len = r->nslots * B;
  CU_CHECK(h, cudaMallocHost((void**)&r->in, (size_t)rows_in * r->len * sizeof(float)));
  CU_CHECK(h, cudaMallocHost((void**)&r->out, (size_t)rows_out * r->len * sizeof(float)));
  CU_CHECK(h, cudaMallocHost((void**)&r->word, 64));
  CU_CHECK(h, cudaMalloc(&r->ticket, sizeof(unsigned int)));
  CU_CHECK(h, cudaMemsetAsync(r->ticket, 0, sizeof(unsigned int), h->s_main));
  *r->word = 0;
#if defined(PC_EMULATE)
  r->in_dev = r->in; r->out_dev = r->out; r->word_dev = r->word;
#else
  if (cudaHostGetDevicePointer((void**)&r->in_dev, r->in, 0) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&r->out_dev, r->out, 0) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&r->word_dev, r->word, 0) != cudaSuccess) {
    cudaGetLastError();
    return fail(h, B200CONV_ECUDA, "fixed-latency mode needs mapped pinned memory");
  }
#endif
  lat_restart(r);
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return 0;
}

// frees everything the chain holds and leaves it unconfigured
void chain_free(Chain& c) {
  lat_free(c.lat);
  cudaFree(c.io); cudaFree(c.conv_in); cudaFree(c.filt); cudaFree(c.state); cudaFree(c.ring); cudaFree(c.wide);
  cudaFree(c.seg); cudaFree(c.segtab);
  if (c.segpin) cudaFreeHost(c.segpin);
  if (c.segev) cudaEventDestroy(c.segev);
  if (c.hpin) cudaFreeHost(c.hpin);
  c = Chain();
}

void free_all(b200conv* h) {
  lat_free(h->lat);
  chain_free(h->chain);
  h->lat_D = 0;
  p2p_release(h);
  for (auto& s : h->stages) free_stage(s);
  h->stages.clear();
  for (int i = 0; i < 2; ++i) {
    cudaFree(h->din[i]); cudaFree(h->dout[i]);
    h->din[i] = h->dout[i] = nullptr;
  }
  cudaFree(h->dch[0]); h->dch[0] = nullptr;
  h->tc_A.release(); h->tc_Xt.release(); h->tc_Yt.release(); h->lf_S.release();
  h->fs_S.release(); h->fs_X.release(); h->fs_hist.release();
  if (h->tc_err) cudaFreeHost(h->tc_err);
  h->tc_err = h->tc_err_dev = nullptr; h->tc_alloc_failed = false;
  h->route_in_only = false;
  if (h->swap_state == 3) h->swap_state = 0;
  if (h->hpin_in) cudaFreeHost(h->hpin_in);
  if (h->hpin_out) cudaFreeHost(h->hpin_out);
  if (h->hflag) cudaFreeHost(h->hflag);
  h->hflag = h->hflag_dev = nullptr;
  h->hpin_in = h->hpin_out = nullptr; h->hpin_cap = 0;
  h->hpin_in_dev = h->hpin_out_dev = nullptr;
  h->ir_len.assign(h->C, 0);
  h->abs_pos = 0;
  h->Lmax = 0;
}

// ---- timing helpers ------------------------------------------------------------------------
enum { kKindFft = 0, kKindCmac = 1, kKindIfft = 2 };

int timing_begin(b200conv* h, int kind, cudaStream_t st = nullptr) {
  if (!st) st = h->s_launch;
  if (!h->timing) return -1;
  if (h->ev_used == h->ev_pool.size()) {
    EventPair p;
    if (cudaEventCreate(&p.a) != cudaSuccess || cudaEventCreate(&p.b) != cudaSuccess) return -1;
    h->ev_pool.push_back(p);
  }
  int id = (int)h->ev_used++;
  h->ev_pool[id].kind = kind;
  cudaEventRecord(h->ev_pool[id].a, st);
  return id;
}
void timing_end(b200conv* h, int id, cudaStream_t st = nullptr) {
  if (id >= 0) cudaEventRecord(h->ev_pool[id].b, st ? st : h->s_launch);
}
void timing_collect(b200conv* h) {
  h->t_cmac = h->t_fft = h->t_ifft = 0;
  h->n_cmac = 0;
  for (size_t i = 0; i < h->ev_used; ++i) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, h->ev_pool[i].a, h->ev_pool[i].b) != cudaSuccess) continue;
    if (h->ev_pool[i].kind == kKindCmac) { h->t_cmac += ms; h->n_cmac++; }
    else if (h->ev_pool[i].kind == kKindFft) h->t_fft += ms;
    else h->t_ifft += ms;
  }
}

// ---- kernel launchers ----------------------------------------------------------------------
// block (NT, ty): NT threads per transform, ty transforms per CTA; see k_fwd_fft
struct FftGeom { dim3 grid, block; size_t smem; bool tws; };

FftGeom fft_geometry(int M, int nblocks, int C) {
  FftGeom g;
  const int nt = pc::fft_threads(M);
  int ty = 1;
  if (pc::fft_warp_mode(M)) {            // one warp per transform
    ty = std::max(1, std::min(8, 4096 / std::max(M, 1)));
    ty = std::min(ty, std::max(1, nblocks));
    g.tws = (long long)nblocks * C >= 64;    // real-time calls: a few transforms, table read through L1 instead
  } else {
    g.tws = (M <= 4096);
  }
  g.block = dim3(nt, ty, 1);
  g.grid = dim3((nblocks + ty - 1) / ty, C, 1);
  const size_t tl = g.tws ? (((size_t)pc::tw_table_len(M) + 15) & ~(size_t)15) : 0;
  g.smem = (tl + (size_t)ty * 2 * std::max(M, 16)) * sizeof(float2);
  return g;
}

#if !defined(PC_EMULATE)
template <int L>
void launch_fwd_l(const pc::FwdParams& P, const FftGeom& g, cudaStream_t st) {
  if (g.tws) pc::k_fwd_fft<(1 << L), true><<<g.grid, g.block, g.smem, st>>>(P);
  else pc::k_fwd_fft<(1 << L), false><<<g.grid, g.block, g.smem, st>>>(P);
}
template <int L>
void launch_inv_l(const pc::InvParams& P, const FftGeom& g, cudaStream_t st) {
  if (P.n_partials > 1) {
    if (g.tws) pc::k_inv_fft_ola<(1 << L), true, true><<<g.grid, g.block, g.smem, st>>>(P);
    else pc::k_inv_fft_ola<(1 << L), false, true><<<g.grid, g.block, g.smem, st>>>(P);
  } else {
    if (g.tws) pc::k_inv_fft_ola<(1 << L), true, false><<<g.grid, g.block, g.smem, st>>>(P);
    else pc::k_inv_fft_ola<(1 << L), false, false><<<g.grid, g.block, g.smem, st>>>(P);
  }
}
// loads the FFT kernels of block size 2^L a tail block of the slot exchange launches (lazy module loading)
template <int L>
cudaError_t fft_preload() {
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, pc::k_fwd_fft<(1 << L), true>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, pc::k_fwd_fft<(1 << L), false>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, pc::k_inv_fft_ola<(1 << L), true, true>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, pc::k_inv_fft_ola<(1 << L), false, true>);
  return e;
}
template <int L>
bool fft_set_smem_attr() {
  const int kSmem = 200 * 1024;   // B = 4096: 48 KB table + 64 KB ping-pong buffers; B = 8192: 128 KB buffers
  bool ok = cudaFuncSetAttribute(pc::k_fwd_fft<(1 << L), true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_fwd_fft<(1 << L), false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_inv_fft_ola<(1 << L), true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_inv_fft_ola<(1 << L), false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_inv_fft_ola<(1 << L), true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_inv_fft_ola<(1 << L), false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) == cudaSuccess;
  return ok;
}
bool stream_set_smem_attr() {
  bool ok = true;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * pc::kStreamStageBytes + 64) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * pc::kStreamStageBytes + 64) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * pc::kStreamStageBytes + 128) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * pc::kStreamStageBytes + 256) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<6, pc::StreamXchParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * pc::kStreamStageBytes + 128) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma<12, pc::StreamXchParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * pc::kStreamStageBytes + 256) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma_dyn<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * pc::kStreamStageBytes + 256) == cudaSuccess;
  ok = ok && cudaFuncSetAttribute(pc::k_cmac_stream_tma_dyn<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * pc::kStreamStageBytes + 512) == cudaSuccess;
  return ok;
}
#define PC_FOR_EACH_LOG2(X) X(0) X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13)
#endif

// register-resident kernels for B = 512 (kernels_fft512.cuh): batches only — a real-time call of a few transforms
// would pay the per-CTA table staging for nothing
constexpr int kF512MinTransforms = 32;
constexpr size_t kF512Smem = (size_t)(pc::kF512_TabLen + 8 * pc::kF512_Xch) * sizeof(float2);
// k_fwd_fft512_lines: + the [re / im][512][16] time-line tile (2 CTAs per SM)
constexpr size_t kF512LinesSmem = kF512Smem + (size_t)2 * pc::kF512_M * pc::kF512_LineR * sizeof(float);

bool use_fft512(const b200conv* h, int M, int nblocks, int C, const float2* tab) {
  return h->opt_fft512 && M == pc::kF512_M && tab != nullptr && (long long)nblocks * C >= kF512MinTransforms;
}

int launch_fwd(b200conv* h, const pc::FwdParams& P, int C) {
  if (use_fft512(h, P.M, P.nblocks, C, P.tab512)) {
    int id = timing_begin(h, kKindFft);
#if defined(PC_EMULATE)
    if (P.lines) return fail(h, B200CONV_EINVAL, "time-line output is not part of the CPU emulation");
    pc::emu_fwd_fft512(P.nblocks, C, P, P.tab512);
#else
    if (P.lines) {
      const long long R = pc::kF512_LineR;
      const int tiles = (int)((P.line_tau0 + P.nblocks - 1) / R - P.line_tau0 / R + 1);
      const int gx = std::max(1, std::min(tiles, (2 * h->n_sm + C - 1) / C));
      pc::k_fwd_fft512_lines<<<dim3(gx, C, 1), dim3(32, 8, 1), kF512LinesSmem, h->s_launch>>>(P, P.tab512);
    } else {
      const int gx = std::max(1, std::min((P.nblocks + 7) / 8, (4 * h->n_sm + C - 1) / C));
      pc::k_fwd_fft512<<<dim3(gx, C, 1), dim3(32, 8, 1), kF512Smem, h->s_launch>>>(P, P.tab512);
    }
#endif
    timing_end(h, id);
    h->launches++;
    CU_CHECK(h, cudaGetLastError());
    return 0;
  }
  const FftGeom g = fft_geometry(P.M, P.nblocks, C);
  int id = timing_begin(h, kKindFft);
#if defined(PC_EMULATE)
  pc::emu_fwd_fft({(int)g.grid.x, (int)g.grid.y, 1}, {(int)g.block.x, (int)g.block.y, 1}, P);
#else
  switch (pc::ilog2(P.M)) {
#define PC_CASE(L) case L: launch_fwd_l<L>(P, g, h->s_launch); break;
    PC_FOR_EACH_LOG2(PC_CASE)
#undef PC_CASE
    default: return fail(h, B200CONV_EINVAL, "unsupported transform size");
  }
#endif
  timing_end(h, id);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

int launch_inv(b200conv* h, const pc::InvParams& P, int C, cudaStream_t st) {
  if (P.n_partials <= 1 && use_fft512(h, P.M, P.nblocks, C, P.tab512)) {
    // whole blocks inside the destination, nothing added on top, linear and 8-byte aligned: float2 stores
    const bool fast = P.n_add == 0 && P.mask == -1 && P.lo <= P.index0 && P.hi >= P.index0 + (long long)P.nblocks * P.M &&
                      (P.index0 & 1) == 0 && (P.dst_cstride & 1) == 0 && (reinterpret_cast<size_t>(P.dst) & 7) == 0;
    int id = timing_begin(h, kKindIfft, st);
#if defined(PC_EMULATE)
    if (P.yc) return fail(h, B200CONV_EINVAL, "bin-major input is not part of the CPU emulation");
    pc::emu_inv_fft512(P.nblocks, C, P, P.tab512, fast);
#else
    const int gx = std::max(1, std::min((P.nblocks + 7) / 8, (3 * h->n_sm + C - 1) / C));
    const dim3 grid(gx, C, 1), block(32, 8, 1);
    if (P.yc) {
      if (fast) pc::k_inv_fft512<true, true><<<grid, block, kF512Smem, st>>>(P, P.tab512);
      else pc::k_inv_fft512<false, true><<<grid, block, kF512Smem, st>>>(P, P.tab512);
    } else {
      if (fast) pc::k_inv_fft512<true, false><<<grid, block, kF512Smem, st>>>(P, P.tab512);
      else pc::k_inv_fft512<false, false><<<grid, block, kF512Smem, st>>>(P, P.tab512);
    }
#endif
    timing_end(h, id, st);
    h->launches++;
    CU_CHECK(h, cudaGetLastError());
    return 0;
  }
  if (P.yc) return fail(h, B200CONV_EINVAL, "bin-major input needs the B = 512 inverse FFT");
  const FftGeom g = fft_geometry(P.M, P.nblocks, C);
  int id = timing_begin(h, kKindIfft, st);
#if defined(PC_EMULATE)
  pc::emu_inv_fft_ola({(int)g.grid.x, (int)g.grid.y, 1}, {(int)g.block.x, (int)g.block.y, 1}, P);
#else
  switch (pc::ilog2(P.M)) {
#define PC_CASE(L) case L: launch_inv_l<L>(P, g, st); break;
    PC_FOR_EACH_LOG2(PC_CASE)
#undef PC_CASE
    default: return fail(h, B200CONV_EINVAL, "unsupported transform size");
  }
#endif
  timing_end(h, id, st);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

template <int TT, int D, int TW, int BS = 0>
void launch_cmac_t(b200conv* h, pc::CmacParams P, int C) {
  P.Ppad = round_up(P.Ppad, TT);
  dim3 block(32, TW, 1);
  dim3 grid((P.B + 31) / 32, (P.nblocks + TT * TW - 1) / (TT * TW), C);
#if defined(PC_EMULATE)
  (void)block;
  pc::emu_cmac_batch<TT, D, TW>({(int)grid.x, (int)grid.y, (int)grid.z}, P);
#else
  pc::k_cmac_batch<TT, D, TW, BS><<<grid, block, 0, h->s_launch>>>(P);
#endif
}

template <int TT, int D, int TW, int BS, int MINB>
void launch_cmac2_t(b200conv* h, pc::CmacParams P, int C) {
  P.Ppad = round_up(P.Ppad, TT);
  dim3 block(32, TW, 1);
  dim3 grid((P.B + 31) / 32, (P.nblocks + TT * TW - 1) / (TT * TW), C);
#if defined(PC_EMULATE)
  (void)block;
  pc::emu_cmac_batch2<TT, D, TW>({(int)grid.x, (int)grid.y, (int)grid.z}, P);
#else
  pc::k_cmac_batch2<TT, D, TW, BS, MINB><<<grid, block, 0, h->s_launch>>>(P);
#endif
}

template <int TT, int D, int TW, int MINB>
void launch_cmac2_bs(b200conv* h, const pc::CmacParams& P, int C) {
  switch (P.B) {
    case 128: launch_cmac2_t<TT, D, TW, 128, MINB>(h, P, C); break;
    case 512: launch_cmac2_t<TT, D, TW, 512, MINB>(h, P, C); break;
    case 8192: launch_cmac2_t<TT, D, TW, 8192, MINB>(h, P, C); break;
    default: launch_cmac2_t<TT, D, TW, 0, MINB>(h, P, C); break;
  }
}

// compile-time row pitch for the common block sizes (immediate load offsets), runtime pitch otherwise
template <int TT, int D, int TW>
void launch_cmac_bs(b200conv* h, const pc::CmacParams& P, int C) {
  switch (P.B) {
    case 128: launch_cmac_t<TT, D, TW, 128>(h, P, C); break;
    case 512: launch_cmac_t<TT, D, TW, 512>(h, P, C); break;
    case 8192: launch_cmac_t<TT, D, TW, 8192>(h, P, C); break;
    default: launch_cmac_t<TT, D, TW, 0>(h, P, C); break;
  }
}

constexpr int kStreamNBS = 4;      // blocks per launch the streaming sweep handles
constexpr int kStreamPW = 8;       // warps per CTA, each striding over the CTA's partition slice

pc::StreamParams stream_params(const pc::CmacParams& P) {
  pc::StreamParams S{};
  S.H = P.H; S.h_cstride = P.h_cstride;
  S.X = P.X; S.x_cstride = P.x_cstride; S.xrow0 = P.xrow0;
  S.Y = P.Y; S.y_cstride = P.y_cstride; S.y_rstride = P.y_rstride; S.yrow0 = P.yrow0;
  S.B = P.B; S.P = P.Ppad; S.nblocks = P.nblocks;
  return S;
}

int launch_cmac_stream(b200conv* h, const pc::CmacParams& P, int C) {
  pc::StreamParams S = stream_params(P);
  const int ktiles = (P.B / 2 + 31) / 32;
  // enough CTAs for ~2 per SM, but at least kStreamPW*4 partitions per CTA
  int nsplit = std::max(1, (2 * h->n_sm) / std::max(1, ktiles * C));
  nsplit = std::max(1, std::min(nsplit, P.Ppad / (kStreamPW * 4)));
  S.nsplit = nsplit;
  if (nsplit > 1) {
    // rows [yrow0, yrow0+nb) of every channel are contiguous (row pitch C*B)
    CU_CHECK(h, cudaMemsetAsync(S.Y + S.yrow0 * S.y_rstride, 0, (size_t)P.nblocks * S.y_rstride * sizeof(float2), h->s_launch));
  }
  dim3 grid(ktiles, nsplit, C), block(32, kStreamPW, 1);
  int id = timing_begin(h, kKindCmac);
#if defined(PC_EMULATE)
  (void)block;
  pc::emu_cmac_stream<kStreamNBS, kStreamPW>({(int)grid.x, (int)grid.y, (int)grid.z}, S);
#else
  pc::k_cmac_stream<kStreamNBS, kStreamPW><<<grid, block, 0, h->s_launch>>>(S);
#endif
  timing_end(h, id);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

template <int NB, int U>
void launch_stream_rows_t(b200conv* h, const pc::StreamParams& S, dim3 grid, int threads) {
#if defined(PC_EMULATE)
  pc::emu_cmac_stream_rows<NB, U>({(int)grid.x, (int)grid.y, (int)grid.z}, threads, S);
#else
  pc::k_cmac_stream_rows<NB, U><<<grid, dim3(threads, 1, 1), 0, h->s_launch>>>(S);
#endif
}

// row-walking streaming sweep (B >= 64): see k_cmac_stream_rows
int launch_cmac_stream_rows(b200conv* h, const pc::CmacParams& P, int C) {
  pc::StreamParams S = stream_params(P);
  const int threads = std::min(256, P.B / 2);
  const int xt = (P.B / 2 + threads - 1) / threads;
  // ~3 CTAs per SM, but no CTA with fewer than 8 partitions (one unrolled load batch)
  int nsplit = std::max(1, (3 * h->n_sm) / std::max(1, xt * C));
  nsplit = std::max(1, std::min(nsplit, std::max(1, P.Ppad / 8)));
  S.nsplit = nsplit;
  if (nsplit > 1)
    CU_CHECK(h, cudaMemsetAsync(S.Y + S.yrow0 * S.y_rstride, 0, (size_t)P.nblocks * S.y_rstride * sizeof(float2), h->s_launch));
  dim3 grid(xt, nsplit, C);
  int id = timing_begin(h, kKindCmac);
  if (P.nblocks <= 1) launch_stream_rows_t<1, 8>(h, S, grid, threads);
  else if (P.nblocks == 2) launch_stream_rows_t<2, 4>(h, S, grid, threads);
  else launch_stream_rows_t<4, 2>(h, S, grid, threads);
  timing_end(h, id);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

// TMA-fed streaming sweep (one block per launch, B >= 64): see kernels_stream.cuh.  S ring stages of 16 KB per
// CTA, `per_sm` CTAs per SM (S * per_sm * 16 KB <= 192 KB of shared memory per SM in flight).
template <int S>
int launch_stream_tma_dyn_s(b200conv* h, const pc::StreamParams& S_, dim3 grid) {
#if defined(PC_EMULATE)
  pc::emu_cmac_stream_tma_dyn({(int)grid.x, (int)grid.y, (int)grid.z}, S_);
#else
  const size_t smem = (size_t)S * pc::kStreamStageBytes + 16 * S + 8 * S;
  pc::k_cmac_stream_tma_dyn<S><<<grid, dim3(288, 1, 1), smem, h->s_launch>>>(S_);
#endif
  return 0;
}

template <int S>
int launch_stream_tma_s(b200conv* h, const pc::StreamParams& S_, dim3 grid) {
#if defined(PC_EMULATE)
  pc::emu_cmac_stream_tma({(int)grid.x, (int)grid.y, (int)grid.z}, S_);
#else
  const size_t smem = (size_t)S * pc::kStreamStageBytes + 16 * S;
  pc::k_cmac_stream_tma<S><<<grid, dim3(288, 1, 1), smem, h->s_launch>>>(S_);
#endif
  return 0;
}

// the same sweep with the tail slot exchange epilogue
template <int S>
int launch_stream_tma_xch_s(b200conv* h, const pc::StreamParams& S_, const pc::StreamXchParams& X, dim3 grid) {
#if defined(PC_EMULATE)
  pc::emu_cmac_stream_tma({(int)grid.x, (int)grid.y, (int)grid.z}, S_, &X);
#else
  const size_t smem = (size_t)S * pc::kStreamStageBytes + 16 * S;
  pc::k_cmac_stream_tma<S, pc::StreamXchParams><<<grid, dim3(288, 1, 1), smem, h->s_launch>>>(S_, X);
#endif
  return 0;
}

// destination of the tail slot exchange epilogue (launch_cmac_stream_tma with xch != nullptr)
struct TailXch { float2* dst; unsigned int* flag; unsigned int epoch; };

int launch_cmac_stream_tma(b200conv* h, const pc::CmacParams& P, int C, int stages, int per_sm, bool dynamic = false, float skew = -1.0f,
                           const TailXch* xch = nullptr) {
  pc::StreamParams S = stream_params(P);
  S.nblocks = 1;
  const int W = pc::stream_tma_w(P.B), PP = pc::stream_tma_pp(P.B), RG = pc::stream_tma_rg(P.B);
  const int xt = P.B / W;
  // per_sm CTAs per SM, but no CTA with fewer than two ring stages of partitions
  int nsplit = std::max(1, (per_sm * h->n_sm) / std::max(1, xt * C));
  nsplit = std::max(1, std::min(nsplit, std::max(1, P.Ppad / (2 * PP))));
  S.nsplit = nsplit;
  if (!dynamic && (nsplit > 1 || RG > 1))
    CU_CHECK(h, cudaMemsetAsync(S.Y + S.yrow0 * S.y_rstride, 0, (size_t)S.y_rstride * sizeof(float2), h->s_launch));
  dim3 grid(xt, nsplit, C);
  if (!dynamic && h->opt_stream_alt) S.descending = (int)(h->stream_launches++ & 1u);
  if (skew >= 0.0f && !dynamic) {        // skewed static slices, channels interleaved in launch order
    S.interleave = 1; S.skew = skew;
    grid = dim3(xt, nsplit * C, 1);
  }
  if (dynamic) {
    if (xt * C > 256) return fail(h, B200CONV_EINVAL, "too many ticket counters");
    if (!h->stream_ticket) {
      CU_CHECK(h, cudaMalloc(&h->stream_ticket, 256 * sizeof(unsigned long long)));
      CU_CHECK(h, cudaMemsetAsync(h->stream_ticket, 0, 256 * sizeof(unsigned long long), h->s_launch));
      h->stream_ticket_base = 0;
    }
    nsplit = std::max(1, std::min((per_sm * h->n_sm) / std::max(1, xt * C), std::max(1, P.Ppad / (2 * PP))));
    S.nsplit = nsplit;
    grid = dim3(xt, nsplit, C);
    S.ticket = h->stream_ticket; S.ticket_base = h->stream_ticket_base; S.chunk_stages = 2;
    h->stream_ticket_base += (unsigned long long)pc::stream_dyn_chunks(S.P, PP, S.chunk_stages) + (unsigned long long)nsplit;
    CU_CHECK(h, cudaMemsetAsync(S.Y + S.yrow0 * S.y_rstride, 0, (size_t)S.y_rstride * sizeof(float2), h->s_launch));   // always RED.ADD
    int idd = timing_begin(h, kKindCmac);
    if (stages == 12) launch_stream_tma_dyn_s<12>(h, S, grid); else launch_stream_tma_dyn_s<6>(h, S, grid);
    timing_end(h, idd);
    h->launches++;
    CU_CHECK(h, cudaGetLastError());
    return 0;
  }
  int id = timing_begin(h, kKindCmac);
  if (xch) {
    const pc::StreamXchParams X{xch->dst, h->ttick, xch->flag, xch->epoch};
    if (stages == 12) launch_stream_tma_xch_s<12>(h, S, X, grid);
    else launch_stream_tma_xch_s<6>(h, S, X, grid);
  } else {
    switch (stages) {
      case 2: launch_stream_tma_s<2>(h, S, grid); break;
      case 6: launch_stream_tma_s<6>(h, S, grid); break;
      case 12: launch_stream_tma_s<12>(h, S, grid); break;
      default: launch_stream_tma_s<4>(h, S, grid); break;
    }
  }
  timing_end(h, id);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

// streaming sweep of one block: 12 stages x 1 CTA/SM for rows below 512 bins and single-tile shapes of at most 32 MB,
// which stay resident in the 50 MB L2 (fewer CTAs to ramp up); 6 stages x 2 CTAs/SM beyond
int stream_variant(const pc::CmacParams& P, int C) {
  const size_t bytes = (size_t)P.Ppad * P.B * 16 * (size_t)C;
  return (P.B < 512 || (P.B == 512 && bytes <= (size_t)32 << 20)) ? 104 : 103;
}

// the TMA streaming sweep of one block as form 102 - 105; xch: with the tail slot exchange epilogue (103 / 104)
int launch_stream_ring(b200conv* h, const pc::CmacParams& P, int C, int variant, const TailXch* xch = nullptr) {
  // 102: 4 stages x 3 CTAs/SM   103: 6 x 2   104: 12 x 1   105: 2 x 6    (all 192 KB in flight per SM)
  static const int cfg[4][2] = {{4, 3}, {6, 2}, {12, 1}, {2, 6}};
  return launch_cmac_stream_tma(h, P, C, cfg[variant - 102][0], cfg[variant - 102][1], false, -1.0f, xch);
}

// ---- the sweep form of a launch; long launch groups: tensor-core (40), line-FFT (41) and four-step (42) sweeps -------
constexpr int kTcMinBlocks = 4096;      // below that a 128-segment tile is mostly padding: the FFMA sweep is faster
// from here on the line-FFT sweep (kernels_lfft.cuh) replaces the tensor-core one; between the two thresholds the
// Toeplitz form stays (its crossover with the line FFTs is not settled below this length)
constexpr int kLfftMinBlocks = 16384;
// from here on the four-step sweep (kernels_fourstep.cuh) replaces the line FFTs for the groups it takes
constexpr int kFourStepMinBlocks = 32768;

// The sweep form select_cmac chose.  In the B = 512 direct form of a tensor-core or line-FFT launch group (run_group)
// the sweep's bin-major complex result stays in yc for the inverse FFT, lines yc_stride apart; output 0 of the sweep
// is block -extra of the group (extra = 1: the sweep computes the overlap state)
struct Sweep {
  int variant = 0;
  float2* yc = nullptr;              // nullptr: the result lines are merged into Y rows
  long long yc_stride = 0;
  int extra = 0;
};

// How the n samples of a launch group enter a stage's open block: `complete` blocks to transform from `src`, `partial`
// samples left over as the next open block.
struct Intake { int complete, partial; bool direct; const float* src; size_t src_stride; size_t total; };
// the launch-group helpers run_group_fourstep shares with run_group (defined with them below)
pc::CmacParams sweep_params(const Stage& s, int C, float2* Y, int nblocks, int extra = 0);
pc::FwdParams fwd_params(const b200conv* h, const Stage& s, const float* src, size_t src_stride, long long nvalid,
                         int nblocks, bool direct);
int launch_mix(b200conv* h, const float* in, size_t in_stride, float* out, size_t out_stride, size_t n, cudaStream_t st);

#if !defined(PC_EMULATE)
// can this sweep run on the tensor cores or the line FFTs?  (geometry only; the scratch is reserve_form's)
bool tc_eligible(const pc::CmacParams& P, int C) {
  if (P.xg > 0 || P.Ppad < 1 || P.nblocks < 1) return false;
  const pc::tc::Geom g = pc::tc::make_geom(P.Ppad, P.nblocks);
  if (!pc::tc::geom_ok(g, P.B)) return false;
  return (unsigned long long)C * P.B * 4ull * (unsigned long long)g.rows < (1ull << 31);
}

// Can this launch group of stage s run as four-step FFT convolutions of its samples (variant 42)?  extra: the sweep
// would start early (a time-slice rank's overlap state)
bool fourstep_ok(const b200conv* h, const Stage& s, const Intake& it, int extra, int C) {
  return h->cfg.shard_count == 1 && h->stages.size() == 1 && extra == 0 && s.fill == 0 && it.partial == 0 &&
         it.complete > 0 && pc::fs::plan_ok(s.P) && use_fft512(h, s.B, it.complete, C, s.tab512);
}

// Grows s to `need` bytes.  A failed allocation is not an error of the call: the CUDA error is cleared and the caller
// falls back to another form.  It also sets tc_alloc_failed, so a failure of any long form's scratch, the four-step
// form's included, keeps 40, 41 and 42 out of automatic selection for the life of the handle.
template <class T>
bool reserve(b200conv* h, Scratch<T>& s, size_t need) {
  if (s.bytes >= need) return true;
  s.release();
  if (cudaMalloc((void**)&s.p, need) != cudaSuccess) { cudaGetLastError(); s.p = nullptr; h->tc_alloc_failed = true; return false; }
  s.bytes = need;
  return true;
}

// room for an operand of `need` bytes built from this IR; a cache that holds another one or is too small is marked empty
template <class T>
bool reserve(b200conv* h, IrCache<T>& c, const pc::CmacParams& P, int C, size_t need) {
  if (c.holds(P, C) && c.buf.bytes >= need) return true;
  c.H = nullptr;
  return reserve(h, c.buf, need);
}

// The scratch of sweep form `variant`: for 40 / 41 the time lines, the result lines (yc) and the Toeplitz images (40)
// or the line spectra (41); for 42 the column spectra, the history and the IR spectrum.  false: not enough memory
bool reserve_form(b200conv* h, const pc::CmacParams& P, int C, int variant, Scratch<float2>& yc) {
  if (variant == 42) {
    namespace fs = pc::fs;
    const fs::Plan plan = fs::make_plan(P.Ppad, (long long)P.nblocks * P.B);
    return reserve(h, h->fs_X, fs::work_bytes(plan, C)) && reserve(h, h->fs_hist, fs::hist_bytes(P.Ppad, C)) &&
           reserve(h, h->fs_S, P, C, fs::spectrum_bytes(C));
  }
  namespace tc = pc::tc;
  const tc::Geom g = tc::make_geom(P.Ppad, P.nblocks);
  const size_t lines = (size_t)C * P.B;
  if (!reserve(h, h->tc_Xt, lines * 2 * (size_t)g.Lt * sizeof(float)) ||
      !reserve(h, yc, lines * (size_t)tc::yc_stride(g) * sizeof(float2))) return false;
  if (variant == 41) return reserve(h, h->lf_S, P, C, pc::lfft::spectra_bytes(lines, C));
  return reserve(h, h->tc_A, P, C, tc::a_image_bytes_gauss(lines, tc::nchunk_f16(g.Q)) + lines * 2 * sizeof(int));
}

// the time lines of a tensor-core or line-FFT sweep.  The direct form's forward FFT wrote the group's own blocks
// (tau = Q + extra ... Q + nblocks - 1) into them: the split only fills the history in front of them and zeroes the
// tail behind them
void launch_split_x(b200conv* h, const pc::CmacParams& P, int C, const pc::tc::Geom& g, const Sweep& sw) {
  namespace tc = pc::tc;
  tc::SplitXParams sp{P.X, P.x_cstride, P.xrow0 - g.Q, std::max<long long>(0, P.xrow0 - (P.Ppad - 1)), P.xrow0 + P.nblocks, P.B, g.rows, h->tc_Xt.p,
                      sw.yc ? g.Q + sw.extra : g.Lt, sw.yc ? g.Q + P.nblocks : g.Lt, 0, 0};
  tc::split_x_chunks(g.rows, sp.skip_lo, sp.skip_hi, &sp.nchunk_lo, &sp.chunk_hi);
  const int split_chunks = sp.nchunk_lo + g.rows * 2 - sp.chunk_hi;
  tc::k_tc_split_x<<<dim3((unsigned)split_chunks, P.B / 32, C), dim3(32, 8), 0, h->s_launch>>>(sp);
}

// the tensor-core sweep (kernels_tc.cuh); the scratch is in place (reserve_form)
int launch_cmac_tc(b200conv* h, const pc::CmacParams& P, int C, const Sweep& sw) {
  namespace tc = pc::tc;
  const tc::Geom g = tc::make_geom(P.Ppad, P.nblocks);
  const size_t lines = (size_t)C * P.B;
  if (!h->tc_err) {
    CU_CHECK(h, cudaHostAlloc((void**)&h->tc_err, sizeof(int), cudaHostAllocMapped));
    *h->tc_err = 0;
    CU_CHECK(h, cudaHostGetDevicePointer((void**)&h->tc_err_dev, h->tc_err, 0));
  }
  if (*reinterpret_cast<volatile int*>(h->tc_err) != 0)
    return fail(h, B200CONV_ECUDA, "tensor-core sweep: a pipeline barrier timed out (code " + std::to_string(*h->tc_err) + ")");
  const int nchunk = tc::nchunk_f16(g.Q);
  const size_t img_bytes = tc::a_image_bytes_gauss(lines, nchunk);
  __half* A = static_cast<__half*>(h->tc_A.buf.p);
  int* eh = reinterpret_cast<int*>(static_cast<unsigned char*>(h->tc_A.buf.p) + img_bytes);
  cudaStream_t st = h->s_launch;
  int id = timing_begin(h, kKindCmac);
  if (!h->tc_A.holds(P, C)) {     // once per IR (and stage): H -> scaled FP16 hi / lo Toeplitz tile images and their exponents
    tc::BuildAParams bp{P.H, P.h_cstride, P.B, P.Ppad, g.Q, nchunk, A, eh};
    tc::k_tc_build_a<<<dim3(nchunk, P.B, C), 256, 0, st>>>(bp);
    h->tc_A.built_from(P, C);
    h->launches++;
  }
  launch_split_x(h, P, C, g, sw);
  float2* Yc = sw.yc ? sw.yc : h->tc_Yt.p;
  tc::SweepParams wp{A, eh, h->tc_Xt.p, Yc, tc::yc_stride(g), (int)lines, g.ntile, tc::npair(g), nchunk, g.rows, P.B, h->tc_err_dev};
  const int total = (int)lines * tc::npair(g);
  tc::k_tc_sweep<<<std::min(total, h->n_sm), tc::kThreads, tc::kSmemBytesGauss, st>>>(wp);
  if (!sw.yc) {
    tc::MergeYParams mp{Yc, tc::yc_stride(g), P.B, P.nblocks, P.Y, P.y_cstride, P.y_rstride, P.yrow0};
    tc::k_tc_merge_y<<<dim3((P.nblocks + 31) / 32, P.B / 32, C), dim3(32, 8), 0, st>>>(mp);
  }
  timing_end(h, id);
  h->launches += sw.yc ? 2 : 3;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

// the line-FFT sweep (kernels_lfft.cuh); the scratch is in place (reserve_form)
int launch_cmac_lfft(b200conv* h, const pc::CmacParams& P, int C, const Sweep& sw) {
  namespace tc = pc::tc;
  namespace lf = pc::lfft;
  const tc::Geom g = tc::make_geom(P.Ppad, P.nblocks);
  const lf::Plan plan = lf::make_plan(P.Ppad, P.nblocks);
  const int lines = C * P.B;
  cudaStream_t st = h->s_launch;
  int id = timing_begin(h, kKindCmac);
  if (!h->lf_S.holds(P, C)) {   // once per IR (and stage)
    lf::k_lfft_build_h<<<dim3(P.B, C), lf::kThreads, 0, st>>>(lf::BuildHParams{P.H, P.h_cstride, P.B, P.Ppad, C, h->lf_S.buf.p});
    h->lf_S.built_from(P, C);
    h->launches++;
  }
  launch_split_x(h, P, C, g, sw);
  float2* Yc = sw.yc ? sw.yc : h->tc_Yt.p;
  const lf::SweepParams wp{h->tc_Xt.p, h->lf_S.buf.p, Yc, tc::yc_stride(g), g.rows, P.B, C, plan};
  lf::k_lfft_sweep<<<(unsigned)lines * (unsigned)plan.nseg, lf::kThreads, 0, st>>>(wp);
  if (!sw.yc) {
    tc::MergeYParams mp{Yc, tc::yc_stride(g), P.B, P.nblocks, P.Y, P.y_cstride, P.y_rstride, P.yrow0};
    tc::k_tc_merge_y<<<dim3((P.nblocks + 31) / 32, P.B / 32, C), dim3(32, 8), 0, st>>>(mp);
  }
  timing_end(h, id);
  h->launches += sw.yc ? 2 : 3;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

// A four-step group (kernels_fourstep.cuh) in place of forward FFT, sweep and inverse FFT: history from the X rows in
// front of the group, passes 1 and 2 on s_main, pass 3 into the output on ps.  Then the handle is left as a
// line-FFT group leaves it: the X rows of the last s.hist blocks, and row 0 of the next Y buffer = sum_p H[p] X[last - p]
// (a one-block streaming sweep), so that any form can follow.  The scratch is in place (reserve_form).
int run_group_fourstep(b200conv* h, Stage& s, const Intake& it, float* out_dev, size_t out_stride, size_t n, bool overlap) {
  namespace fs = pc::fs;
  const int C = h->C, B = s.B, P = s.P, complete = it.complete;
  const fs::Plan plan = fs::make_plan(P, (long long)n);
  const long long hl = (long long)P * B;
  const int yb = s.ybuf, nxt = overlap ? (yb ^ 1) : yb;
  cudaStream_t st = h->s_launch, ps = overlap ? h->s_post : st;
  // the one-block sweep of the overlap state at the end; its H and geometry are also the IR spectrum's
  pc::CmacParams op = sweep_params(s, C, s.Y[nxt], 1);
  // the previous groups' post work may still read the column spectra (a four-step pass 3) and Y[nxt] row 0
  if (overlap) {
    CU_CHECK(h, cudaStreamWaitEvent(st, s.ev_post[0], 0));
    CU_CHECK(h, cudaStreamWaitEvent(st, s.ev_post[1], 0));
  }
  const dim3 taps_block(32, 8), cols_grid(fs::kN2 / fs::kCols, plan.nseg, C);
  if (!h->fs_S.holds(op, C)) {   // once per IR: taps -> spectrum
    int id = timing_begin(h, kKindCmac);
    fs::k_fs_taps<<<dim3((P + 7) / 8, C), taps_block, kF512Smem, st>>>(
        fs::TapsParams{s.H, (long long)s.Prows * B, P, h->fs_hist.p, hl}, s.tab512);
    fs::ColsParams tp{};
    tp.src = h->fs_hist.p; tp.src_cstride = hl; tp.nsrc = hl; tp.nseg = 1; tp.dst = h->fs_S.buf.p;
    fs::k_fs_cols<<<dim3(fs::kN2 / fs::kCols, 1, C), fs::kColThreads, fs::kColSmem, st>>>(tp, s.tab512);
    const unsigned items = (unsigned)(C * fs::kRows);
    fs::k_fs_rows<false><<<std::min(items, h->fs_rows_ctas[0]), pc::lfft::kThreads, fs::rows_smem<false>(), st>>>(
        fs::RowsParams{h->fs_S.buf.p, nullptr, 1, items});
    timing_end(h, id);
    h->fs_S.built_from(op, C);
    h->launches += 3;
  }
  // pass 1, its negative positions from the X rows [head - P, head)
  int id = timing_begin(h, kKindFft);
  fs::k_fs_taps<<<dim3((P + 7) / 8, C), taps_block, kF512Smem, st>>>(
      fs::TapsParams{s.X + (s.head - P) * B, (long long)s.R * B, P, h->fs_hist.p, hl}, s.tab512);
  fs::ColsParams cp{};
  cp.src = it.src; cp.src_cstride = (long long)it.src_stride;
  cp.use_cmap = (h->route_on || h->route_in_only) ? 1 : 0;
  for (int c = 0; c < 8; ++c) cp.cmap[c] = h->in_map[c];
  cp.nsrc = (long long)n; cp.hist = h->fs_hist.p; cp.hist_len = hl;
  cp.w0 = fs::window_start(plan, 0); cp.L = plan.L; cp.nseg = plan.nseg; cp.dst = h->fs_X.p;
  fs::k_fs_cols<<<cols_grid, fs::kColThreads, fs::kColSmem, st>>>(cp, s.tab512);
  timing_end(h, id);
  id = timing_begin(h, kKindCmac);
  const unsigned items = (unsigned)(C * fs::kRows * plan.nseg);
  fs::k_fs_rows<true><<<std::min(items, h->fs_rows_ctas[1]), pc::lfft::kThreads, fs::rows_smem<true>(), st>>>(
      fs::RowsParams{h->fs_X.p, h->fs_S.buf.p, plan.nseg, items});
  timing_end(h, id);
  h->launches += 3;
  CU_CHECK(h, cudaGetLastError());
  CU_CHECK(h, cudaEventRecord(s.ev_sweep[yb], st));
  if (overlap) CU_CHECK(h, cudaStreamWaitEvent(ps, s.ev_sweep[yb], 0));

  // pass 3 into the output (through the mixdown with routing on)
  id = timing_begin(h, kKindIfft, ps);
  const fs::ColsInvParams ip{h->fs_X.p, plan.nseg, plan, h->route_on ? h->dch[0] : out_dev,
                             h->route_on ? (long long)h->Lmax : (long long)out_stride};
  fs::k_fs_cols_inv<<<cols_grid, fs::kColThreads, fs::kColSmem, ps>>>(ip, s.tab512);
  timing_end(h, id, ps);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  if (h->route_on) { if (int rc = launch_mix(h, h->dch[0], h->Lmax, out_dev, out_stride, n, ps)) return rc; }
  if (overlap) CU_CHECK(h, cudaEventRecord(s.ev_post[yb], ps));

  // the state every other form reads: the X rows of the last s.hist blocks ...
  const int from = std::max(0, complete - s.hist);
  pc::FwdParams fp = fwd_params(h, s, it.src + (size_t)from * B, it.src_stride, (long long)(complete - from) * B,
                                complete - from, it.direct);
  fp.dst_row0 = s.head + from;
  if (int rc = launch_fwd(h, fp, C)) return rc;
  // ... and the overlap state of the next group, the spectrum of the last block
  op.xrow0 = s.head + complete - 1;
  op.yrow0 = 0;
  if (int rc = launch_stream_ring(h, op, C, stream_variant(op, C))) return rc;
  s.ybuf = nxt;
  s.head += complete;
  s.blocks_done += complete;
  return 0;
}
#else   // the CPU emulation has none of these forms: no shape qualifies, so select_cmac refuses a forced 40 / 41 / 42
bool tc_eligible(const pc::CmacParams&, int) { return false; }
bool fourstep_ok(const b200conv*, const Stage&, const Intake&, int, int) { return false; }
bool reserve_form(b200conv*, const pc::CmacParams&, int, int, Scratch<float2>&) { return false; }
int launch_cmac_tc(b200conv* h, const pc::CmacParams&, int, const Sweep&) {
  return fail(h, B200CONV_EINVAL, "the tensor-core sweep is not part of the CPU emulation");
}
int launch_cmac_lfft(b200conv* h, const pc::CmacParams&, int, const Sweep&) {
  return fail(h, B200CONV_EINVAL, "the line-FFT sweep is not part of the CPU emulation");
}
int run_group_fourstep(b200conv* h, Stage&, const Intake&, float*, size_t, size_t, bool) {
  return fail(h, B200CONV_EINVAL, "the four-step sweep is not part of the CPU emulation");
}
#endif

// The sweep form of a launch (*sw).  A launch group decides it before its forward FFT: the long forms reserve their
// scratch here, so that when the memory is not there the fallback still finds the X rows it reads.  yc: where the
// result lines of a tensor-core or line-FFT sweep go in the B = 512 direct form, whose sweep starts `extra` blocks
// early; nullptr: the handle's lines, merged into Y rows.  fs_ok: the launch group may run as a four-step group
// (fourstep_ok).  P.Ppad enters as the number of real (unpadded) partition rows of this shard
int select_cmac(b200conv* h, const pc::CmacParams& P, int C, Sweep* sw, Scratch<float2>* yc = nullptr, int extra = 0,
                bool fs_ok = false) {
  const int forced = h->cfg.cmac_variant, ffma = (P.nblocks >= 64) ? 22 : 26;
  int variant = P.xg > 0 ? ffma : forced;     // slot exchange: only the packed-FMA sweeps carry the exchange epilogue
  if (variant == 0) {
    // streaming sweep for real-time calls; packed-FMA batched sweep otherwise (TT = 16 when the
    // launch group is long enough to fill 16-block tiles, TT = 8 below that)
    if (P.nblocks == 1 && P.B >= 64 && P.Ppad >= 1) variant = stream_variant(P, C);   // TMA ring
    else if (P.nblocks <= kStreamNBS && P.B >= 64 && P.Ppad >= 1) variant = 101;
    else if (P.nblocks <= kStreamNBS && P.B >= 2 && P.Ppad >= 1) variant = 100;
    else if (h->opt_tc && !h->tc_alloc_failed && P.nblocks >= kTcMinBlocks && tc_eligible(P, C))
      variant = fs_ok && P.nblocks >= kFourStepMinBlocks ? 42 : P.nblocks >= kLfftMinBlocks ? 41 : 40;
    else variant = ffma;
  }
  // 42: four-step FFTs of the samples; 40 / 41: wgmma 3xFP16 block-Toeplitz sweep / FP32 line FFTs
  if (variant == 42 && !fs_ok) return fail(h, B200CONV_EINVAL, "four-step sweep: unsupported launch group (needs whole blocks from a block boundary, B = 512, at most 961 partitions, an unsharded single-stage handle)");
  if ((variant == 40 || variant == 41) && !tc_eligible(P, C)) return fail(h, B200CONV_EINVAL, "tensor-core / line-FFT sweep: unsupported shape (needs B % 32 == 0, at most 961 partitions, no slot exchange)");
  // when the scratch does not fit: 42 -> 41 -> FFMA sweep, 40 -> FFMA, 41 -> FFMA; a forced form fails
  Scratch<float2>& lines = yc ? *yc : h->tc_Yt;
  if (variant == 42 && !reserve_form(h, P, C, 42, lines)) {
    if (forced == 42) return fail(h, B200CONV_ENOMEM, "four-step sweep: scratch allocation failed");
    variant = 41;
  }
  if ((variant == 40 || variant == 41) && !reserve_form(h, P, C, variant, lines)) {
    if (forced == variant) return fail(h, B200CONV_ENOMEM, "tensor-core / line-FFT sweep: scratch allocation failed");
    variant = ffma;
  }
  *sw = Sweep{variant};
  if (yc && (variant == 40 || variant == 41)) {
    sw->yc = yc->p;
    sw->yc_stride = pc::tc::yc_stride(pc::tc::make_geom(P.Ppad, P.nblocks));
    sw->extra = extra;
  }
  h->last_variant = variant;
  return 0;
}

// runs the sweep form select_cmac chose
int launch_cmac_as(b200conv* h, const pc::CmacParams& P, int C, const Sweep& sw) {
  const int variant = sw.variant;
  if (variant == 40) return launch_cmac_tc(h, P, C, sw);
  if (variant == 41) return launch_cmac_lfft(h, P, C, sw);
  if (variant == 108) {                        // 6 stages x 2 CTAs/SM, skewed static slices (B200CONV_STREAM_SKEW percent, default 8)
    if (P.nblocks != 1 || P.B < 64) return fail(h, B200CONV_EINVAL, "TMA streaming sweep needs nblocks == 1 and B >= 64");
    static const float skew = [] { const char* e = std::getenv("B200CONV_STREAM_SKEW"); return e ? (float)std::atof(e) / 100.0f : 0.08f; }();
    return launch_cmac_stream_tma(h, P, C, 6, 2, false, skew);
  }
  if (variant == 106 || variant == 107) {      // dynamic chunk tickets: 106 = 6 stages x 2 CTAs/SM, 107 = 12 x 1
    if (P.nblocks != 1 || P.B < 64) return fail(h, B200CONV_EINVAL, "TMA streaming sweep needs nblocks == 1 and B >= 64");
    return launch_cmac_stream_tma(h, P, C, variant == 106 ? 6 : 12, variant == 106 ? 2 : 1, true);
  }
  if (variant >= 102 && variant <= 105) {
    if (P.nblocks != 1 || P.B < 64) return fail(h, B200CONV_EINVAL, "TMA streaming sweep needs nblocks == 1 and B >= 64");
    return launch_stream_ring(h, P, C, variant);
  }
  if (variant == 101) {
    if (P.nblocks > kStreamNBS || P.B < 4) return fail(h, B200CONV_EINVAL, "streaming sweep needs nblocks <= 4 and B >= 4");
    return launch_cmac_stream_rows(h, P, C);
  }
  if (variant == 100) {
    if (P.nblocks > kStreamNBS || P.B < 2) return fail(h, B200CONV_EINVAL, "streaming sweep needs nblocks <= 4 and B >= 2");
    return launch_cmac_stream(h, P, C);
  }
  int id = timing_begin(h, kKindCmac);
  switch (variant) {
    case 1: launch_cmac_t<16, 4, 8>(h, P, C); break;
    case 2: launch_cmac_t<16, 4, 4>(h, P, C); break;
    case 3: launch_cmac_t<8, 4, 4>(h, P, C); break;
    case 4: launch_cmac_t<8, 4, 8>(h, P, C); break;
    case 5: launch_cmac_t<16, 2, 8>(h, P, C); break;
    case 6: launch_cmac_t<32, 4, 4>(h, P, C); break;
    case 7: launch_cmac_t<4, 4, 8>(h, P, C); break;
    case 11: launch_cmac_bs<16, 4, 8>(h, P, C); break;
    case 12: launch_cmac_bs<16, 4, 4>(h, P, C); break;
    case 16: launch_cmac_bs<32, 4, 4>(h, P, C); break;
    case 21: launch_cmac2_bs<16, 4, 4, 4>(h, P, C); break;    // packed-pair FMA, 128 thr/CTA, <=128 regs
    case 22: launch_cmac2_bs<16, 4, 4, 3>(h, P, C); break;    // packed-pair FMA, 128 thr/CTA, <=168 regs
    case 23: launch_cmac2_bs<16, 4, 8, 2>(h, P, C); break;    // packed-pair FMA, 256 thr/CTA, <=128 regs
    case 24: launch_cmac2_bs<16, 2, 4, 4>(h, P, C); break;
    case 25: launch_cmac2_bs<12, 4, 4, 4>(h, P, C); break;
    case 26: launch_cmac2_bs<8, 4, 4, 4>(h, P, C); break;
    case 27: launch_cmac2_bs<16, 4, 2, 8>(h, P, C); break;    // 64 thr/CTA
    case 28: launch_cmac2_bs<24, 4, 4, 2>(h, P, C); break;
    // banked for the next tuning round (functionally verified, not yet timed):
    case 33: launch_cmac2_bs<16, 8, 4, 3>(h, P, C); break;    // deeper software prefetch
    case 34: launch_cmac2_bs<16, 4, 2, 6>(h, P, C); break;    // 64-thread CTAs, 6 per SM: finer load balance
    default: return fail(h, B200CONV_EINVAL, "unknown cmac_variant");
  }
  timing_end(h, id);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
}

int launch_cmac(b200conv* h, const pc::CmacParams& P, int C) {
  Sweep sw;
  if (int rc = select_cmac(h, P, C, &sw)) return rc;
  return launch_cmac_as(h, P, C, sw);
}

// the single-block sweep of a tail block whose partial spectrum goes to rank 0 through the slot exchange: the TMA
// streaming form launch_cmac selects for nblocks == 1 (also for an empty partition range: the zero slot is published too)
int launch_cmac_exchange(b200conv* h, const pc::CmacParams& P, int C, const TailXch& x) {
  h->last_variant = stream_variant(P, C);
  return launch_stream_ring(h, P, C, h->last_variant, &x);
}

// First thing of every entry point that enqueues device work.  After a group call that recorded its event this
// handle's streams are ordered behind the group's shared launch and the tail-output waits it queued (the lazy wait of
// b200conv_group_process).
int set_device(b200conv* h) {
  CU_CHECK(h, cudaSetDevice(h->cfg.device));
  h->main_unsynced = true;
  if (h->grp_st) {
    CU_CHECK(h, cudaEventRecord(h->grp_ev, h->grp_st));
    h->grp_st = nullptr;
  }
  if (h->grp_ev) {
    CU_CHECK(h, cudaStreamWaitEvent(h->s_main, h->grp_ev, 0));
    CU_CHECK(h, cudaStreamWaitEvent(h->s_post, h->grp_ev, 0));
    h->grp_ev = nullptr;
  }
  return 0;
}

// shard_head = 0 on a sharded handle: the head stage stays whole on rank 0, the stages >= 1 are sharded
bool tail_layout(const b200conv* h) { return !h->opt_shard_head && h->cfg.shard_count > 1; }

// ---- IR load -------------------------------------------------------------------------------
size_t trimmed_len(const float* ir, size_t n) {
  // FFTConvolver.cpp:103-106 / TwoStageFFTConvolver.cpp:107-110: absolute 1e-6 threshold
  while (n > 0 && std::fabs(ir[n - 1]) < 0.000001f) --n;
  return n;
}

int build_stage(b200conv* h, Stage& s, const float* const* ir, const std::vector<size_t>& L) {
  const int C = h->C;
  const int B = s.B;
  // partitions of this stage (max over channels)
  size_t maxlen = 0;
  std::vector<int> len_c(C, 0);
  for (int c = 0; c < C; ++c) {
    size_t e = std::min(L[c], s.tap_end);
    size_t n = e > s.tap_off ? e - s.tap_off : 0;
    len_c[c] = (int)n;
    maxlen = std::max(maxlen, n);
  }
  s.P_full = (int)((maxlen + B - 1) / B);
  s.q = (int)(s.tap_off / B);
  // shard range
  const int G = std::max(1, h->cfg.shard_count), g = h->cfg.shard_rank;
  const int per = (s.P_full + G - 1) / G;
  s.p_begin = std::min(s.P_full, g * per);
  s.p_end = std::min(s.P_full, (g + 1) * per);
  if (tail_layout(h) && &s == &h->stages.front()) {     // the head: whole on rank 0, nothing on the other ranks
    s.p_begin = 0;
    s.p_end = g == 0 ? s.P_full : 0;
  }
  s.P = s.p_end - s.p_begin;
  s.Prows = round_up(std::max(s.P, 1), kPadP) + kDPre;
  s.hist = s.p_begin + round_up(std::max(s.P, 1), kPadP) + kDPre;

  // twiddle table (layout: kernels.cuh tw_pass_offset), computed in double
  const int N = pc::tw_table_len(B);
  std::vector<float2> tw(N);
  for (int k = 0; k <= B / 2; ++k) {                       // split twiddles exp(-2*pi*i*k/(2B))
    const double a = -2.0 * M_PI * (double)k / (2.0 * (double)B);
    tw[k] = make_float2((float)std::cos(a), (float)std::sin(a));
  }
  for (int p = 1; p < B;) {                                // pass twiddles exp(-2*pi*i*r*k/(p*R))
    const int R = pc::pass_radix(B, p);
    const int off = pc::tw_pass_offset(B, p);
    for (int r = 1; r < R; ++r)
      for (int k = 0; k < p; ++k) {
        const double a = -2.0 * M_PI * (double)r * (double)k / ((double)p * (double)R);
        tw[off + (r - 1) * p + k] = make_float2((float)std::cos(a), (float)std::sin(a));
      }
    p *= R;
  }
  CU_CHECK(h, cudaMalloc(&s.tw, N * sizeof(float2)));
  CU_CHECK(h, cudaMemcpyAsync(s.tw, tw.data(), N * sizeof(float2), cudaMemcpyHostToDevice, h->s_main));
  std::vector<float2> t512;
  if (B == pc::kF512_M) {       // tables of kernels_fft512.cuh, in double
    t512.resize(pc::kF512_TabLen);
    auto w = [](double num, double den) {
      const double a = -2.0 * M_PI * num / den;
      return make_float2((float)std::cos(a), (float)std::sin(a));
    };
    for (int k2 = 0; k2 < 8; ++k2)
      for (int m = 0; m < 64; ++m) t512[pc::kF512_T1 + k2 * 64 + m] = w((double)m * k2, 512.0);
    for (int a = 0; a < 8; ++a)
      for (int b = 0; b < 8; ++b) t512[pc::kF512_T2 + a * 8 + b] = w((double)a * b, 64.0);
    for (int k = 0; k < 512; ++k) t512[pc::kF512_TS + k] = w((double)k, 1024.0);
    CU_CHECK(h, cudaMalloc(&s.tab512, t512.size() * sizeof(float2)));
    CU_CHECK(h, cudaMemcpyAsync(s.tab512, t512.data(), t512.size() * sizeof(float2), cudaMemcpyHostToDevice, h->s_main));
  }
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));

  // H: upload this shard's taps, transform
  const size_t hrow = (size_t)B;
  CU_CHECK(h, cudaMalloc(&s.H, (size_t)C * s.Prows * hrow * sizeof(float2)));
  CU_CHECK(h, cudaMemsetAsync(s.H, 0, (size_t)C * s.Prows * hrow * sizeof(float2), h->s_main));
  if (s.P > 0) {
    const size_t taps_per_c = (size_t)s.P * B;
    std::vector<float> host((size_t)C * taps_per_c, 0.0f);
    std::vector<int> nvalid(C, 0);
    for (int c = 0; c < C; ++c) {
      const long long first = (long long)s.p_begin * B;            // within the stage
      long long n = (long long)len_c[c] - first;
      n = std::max(0LL, std::min(n, (long long)taps_per_c));
      nvalid[c] = (int)n;
      if (n > 0 && !h->ir_on_device) std::memcpy(&host[(size_t)c * taps_per_c], ir[c] + s.tap_off + first, (size_t)n * sizeof(float));
    }
    float* dtaps = nullptr; int* dnv = nullptr;
    CU_CHECK(h, cudaMalloc(&dtaps, host.size() * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&dnv, C * sizeof(int)));
    if (h->ir_on_device) {        // taps shaped on the device: no host round trip
      CU_CHECK(h, cudaMemsetAsync(dtaps, 0, host.size() * sizeof(float), h->s_main));
      for (int c = 0; c < C; ++c)
        if (nvalid[c] > 0)
          CU_CHECK(h, cudaMemcpyAsync(dtaps + (size_t)c * taps_per_c, ir[c] + s.tap_off + (size_t)s.p_begin * B,
                                      (size_t)nvalid[c] * sizeof(float), cudaMemcpyDeviceToDevice, h->s_main));
    } else
    CU_CHECK(h, cudaMemcpyAsync(dtaps, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice, h->s_main));
    CU_CHECK(h, cudaMemcpyAsync(dnv, nvalid.data(), C * sizeof(int), cudaMemcpyHostToDevice, h->s_main));
    pc::FwdParams fp{};
    fp.src = dtaps; fp.src_cstride = (long long)taps_per_c;
    fp.nvalid_c = dnv; fp.nvalid = 0;
    fp.dst = s.H; fp.dst_cstride = (long long)s.Prows * B; fp.dst_row0 = 0;
    fp.tw = s.tw; fp.tab512 = s.tab512; fp.M = B; fp.nblocks = s.P;
    int rc = launch_fwd(h, fp, C);
    if (rc) { cudaFree(dtaps); cudaFree(dnv); return rc; }
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    cudaFree(dtaps); cudaFree(dnv);
  }
  return 0;
}

int alloc_stage_state(b200conv* h, Stage& s) {
  const int C = h->C, B = s.B;
  s.Tcap = (int)(h->Lmax / B) + 2;
  s.R = 2 * s.hist + s.Tcap + kMaxTT;
  CU_CHECK(h, cudaMalloc(&s.X, (size_t)C * s.R * B * sizeof(float2)));
  for (int i = 0; i < 2; ++i) {
    CU_CHECK(h, cudaMalloc(&s.Y[i], (size_t)(1 + s.Tcap) * C * B * sizeof(float2)));
    CU_CHECK(h, cudaEventCreateWithFlags(&s.ev_sweep[i], cudaEventDisableTiming));
    CU_CHECK(h, cudaEventCreateWithFlags(&s.ev_post[i], cudaEventDisableTiming));
  }
  s.in_stride = (size_t)B + h->Lmax;
  CU_CHECK(h, cudaMalloc(&s.inbuf, (size_t)C * s.in_stride * sizeof(float)));
  if (s.q > 0) {
    s.ring = next_pow2((size_t)(s.q + 2) * B + h->Lmax + B);
    CU_CHECK(h, cudaMalloc(&s.fut, (size_t)C * s.ring * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&s.inbuf_alt, (size_t)C * s.in_stride * sizeof(float)));
    for (int i = 0; i < 2; ++i) CU_CHECK(h, cudaEventCreateWithFlags(&s.ev_job[i], cudaEventDisableTiming));
  }
  return 0;
}

int clear_state(b200conv* h) {
  if (h->s_tail) CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
  CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  for (auto& s : h->stages) {
    const int C = h->C, B = s.B;
    CU_CHECK(h, cudaMemsetAsync(s.X, 0, (size_t)C * s.R * B * sizeof(float2), h->s_main));
    for (int i = 0; i < 2; ++i)
      CU_CHECK(h, cudaMemsetAsync(s.Y[i], 0, (size_t)(1 + s.Tcap) * C * B * sizeof(float2), h->s_main));
    s.ybuf = 0;
    CU_CHECK(h, cudaMemsetAsync(s.inbuf, 0, (size_t)C * s.in_stride * sizeof(float), h->s_main));
    if (s.inbuf_alt) CU_CHECK(h, cudaMemsetAsync(s.inbuf_alt, 0, (size_t)C * s.in_stride * sizeof(float), h->s_main));
    if (s.fut) CU_CHECK(h, cudaMemsetAsync(s.fut, 0, (size_t)C * s.ring * sizeof(float), h->s_main));
    s.job_waited[0] = s.job_waited[1] = true;
    s.njobs = 0;
    s.head = s.hist;
    s.blocks_done = 0;
    s.fill = 0;
  }
  h->abs_pos = 0;
  h->yprev_stale = false;
  if (h->Yx[0]) {
    const Stage& s0 = h->stages[0];
    const size_t row = (size_t)h->C * s0.B;
    for (int i = 0; i < 2; ++i) CU_CHECK(h, cudaMemsetAsync(h->Yx[i], 0, (size_t)h->cfg.shard_count * h->xslot * sizeof(float2), h->s_main));
    CU_CHECK(h, cudaMemsetAsync(h->Hh, 0, (size_t)3 * h->cfg.shard_count * row * sizeof(float2), h->s_main));
    h->hidx = 0;
  }
  // tail slot exchange: the summed overlap rows (slot 0, row 0, both parities) on rank 0.  The peers' rows 1 are
  // overwritten by every block, their rows 0 stay zero; the flag epochs keep counting on every rank alike.
  for (size_t si = 1; si < h->stages.size() && h->cfg.shard_rank == 0; ++si)
    if (h->Tx[si]) {
      const size_t row = (size_t)h->C * h->stages[si].B;
      for (int par = 0; par < 2; ++par)
        CU_CHECK(h, cudaMemsetAsync(h->Tx[si] + (size_t)par * h->cfg.shard_count * 2 * row, 0, row * sizeof(float2), h->s_main));
    }
  return 0;
}

int init_impl(b200conv* h, int n_stages, const size_t* blocks, const size_t* offsets,
              const float* const* ir, const size_t* ir_len) {
  if (int rc = set_device(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  if (h->s_tail) CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
  free_all(h);
  const int C = h->C;
  for (int s = 0; s < n_stages; ++s)
    if (blocks[s] == 0) return fail(h, B200CONV_EINVAL, "block size 0");
  std::vector<size_t> L(C);
  size_t Lir = 0;
  for (int c = 0; c < C; ++c) {
    if (h->ir_on_device) L[c] = (ir && ir[c] && h->ir_trimmed) ? std::min(h->ir_trimmed[c], ir_len[c]) : 0;
    else L[c] = (ir && ir[c] && ir_len) ? trimmed_len(ir[c], ir_len[c]) : 0;
    Lir = std::max(Lir, L[c]);
  }
  h->ir_len = L;
  if (Lir == 0) return B200CONV_OK;      // empty IR: legal, process() writes zeros (FFTConvolver.cpp:108-111)

  std::vector<Stage> st;
  for (int s = 0; s < n_stages; ++s) {
    Stage x;
    // FFTConvolver.cpp:113 rounds up to a power of two.  Partition sizes above 8192 are clamped to 8192: the
    // output of a partitioned convolver is the same linear convolution whatever the partition size, and
    // every offset that is a multiple of a larger power of two is a multiple of 8192 too (REEV-R asks for
    // tail = max(8192, 2*head), StereoConvolver.cpp:15, i.e. 16384 for host blocks above 4096 samples).
    const size_t b = std::min(next_pow2(blocks[s]), size_t(1) << kMaxBlockLog2);
    x.B = (int)b;
    x.tap_off = offsets ? offsets[s] : 0;
    x.tap_end = (s + 1 < n_stages) ? offsets[s + 1] : Lir;
    if (x.tap_off >= Lir) break;                              // IR shorter than this stage's offset
    x.tap_end = std::min(x.tap_end, Lir);
    if (s > 0 && (x.tap_off % b != 0 || x.tap_off < b))
      return fail(h, B200CONV_EINVAL, "stage offset must be a multiple of (and >=) its block size");
    st.push_back(x);
  }
  const int B0 = st[0].B;
  // default launch-group size: kDefaultBatch head blocks, but no more than ~4 M samples of staging per channel
  int batch = h->cfg.max_batch_blocks > 0 ? h->cfg.max_batch_blocks
                                          : std::max(64, std::min(kDefaultBatch, (int)((size_t)4194304 / (size_t)B0)));
  h->Lmax = (size_t)batch * B0;
  for (auto& x : st) h->Lmax = std::max(h->Lmax, (size_t)2 * x.B);
  h->stages = st;
  for (auto& s : h->stages) {
    if (int rc = build_stage(h, s, ir, L)) return rc;
    if (int rc = alloc_stage_state(h, s)) return rc;
  }
  for (int i = 0; i < 2; ++i) {
    CU_CHECK(h, cudaMalloc(&h->din[i], (size_t)C * h->Lmax * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&h->dout[i], (size_t)C * h->Lmax * sizeof(float)));
  }
  CU_CHECK(h, cudaMalloc(&h->dch[0], (size_t)C * h->Lmax * sizeof(float)));
  // latency path staging (calls of up to max(64 head blocks, 16384) samples)
  h->hpin_cap = std::min(h->Lmax, std::max((size_t)64 * B0, (size_t)16384));
  CU_CHECK(h, cudaMallocHost((void**)&h->hpin_in, (size_t)C * h->hpin_cap * sizeof(float)));
  CU_CHECK(h, cudaMallocHost((void**)&h->hpin_out, (size_t)C * h->hpin_cap * sizeof(float)));
  CU_CHECK(h, cudaMallocHost((void**)&h->hflag, 64));
  *h->hflag = 0; h->flag_epoch = 0;
#if defined(PC_EMULATE)
  h->hpin_in_dev = h->hpin_in; h->hpin_out_dev = h->hpin_out; h->hflag_dev = h->hflag;
#else
  if (cudaHostGetDevicePointer((void**)&h->hflag_dev, h->hflag, 0) != cudaSuccess) { cudaGetLastError(); h->hflag_dev = nullptr; }
  if (cudaHostGetDevicePointer((void**)&h->hpin_in_dev, h->hpin_in, 0) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&h->hpin_out_dev, h->hpin_out, 0) != cudaSuccess) {
    cudaGetLastError();
    h->hpin_in_dev = h->hpin_out_dev = nullptr;       // no zero-copy I/O: the real-time path stays on the copy path
  }
#endif
  if (int rc = clear_state(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return B200CONV_OK;
}

// A failed load (e.g. B200CONV_ENOMEM for an IR that does not fit) leaves the handle in the "no IR" state:
// nothing half-allocated, later init / process calls work.
int init_common(b200conv* h, int n_stages, const size_t* blocks, const size_t* offsets,
                const float* const* ir, const size_t* ir_len) {
  if (h->swap_peer) return fail(h, B200CONV_ESTATE, "an IR hot swap is pending on this handle");
  const int rc = init_impl(h, n_stages, blocks, offsets, ir, ir_len);
  if (rc != B200CONV_OK && !h->sticky_cuda_error) {
    const std::string keep = h->err;
    free_all(h);
    h->err = keep;
  }
  return rc;
}

// copies `count` samples of every convolver channel from the caller's device buffer (n_in routed inputs or
// C plain channels) into a C-channel staging buffer
int copy_in(b200conv* h, float* dst, size_t dstride, const float* src, size_t sstride, size_t count) {
  if (count == 0) return 0;
  if (!h->route_on && !h->route_in_only) {
    CU_CHECK(h, cudaMemcpy2DAsync(dst, dstride * sizeof(float), src, sstride * sizeof(float), count * sizeof(float), h->C,
                                  cudaMemcpyDeviceToDevice, h->s_main));
  } else {
    for (int c = 0; c < h->C; ++c)
      CU_CHECK(h, cudaMemcpyAsync(dst + (size_t)c * dstride, src + (size_t)h->in_map[c] * sstride, count * sizeof(float),
                                  cudaMemcpyDeviceToDevice, h->s_main));
  }
  return 0;
}

#if !defined(PC_EMULATE)
#define PC_LAUNCH_MIX(mp, grid, st) pc::k_mix<<<grid, 256, 0, st>>>(mp)
#endif

// per-convolver outputs (C channels in `in`) -> n_out mixed outputs
int launch_mix(b200conv* h, const float* in, size_t in_stride, float* out, size_t out_stride, size_t n, cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)st;
  for (int o = 0; o < h->n_out; ++o)
    for (size_t i = 0; i < n; ++i) {
      float acc = 0.0f;
      for (int c = 0; c < h->C; ++c) {
        const float m = h->mix[o * h->C + c];
        if (m != 0.0f) acc = std::fmaf(m, in[(size_t)c * in_stride + i], acc);
      }
      out[(size_t)o * out_stride + i] = acc;
    }
#else
  pc::MixParams mp{};
  mp.in = in; mp.in_stride = (long long)in_stride; mp.out = out; mp.out_stride = (long long)out_stride;
  mp.n = (long long)n; mp.C = h->C; mp.n_out = h->n_out;
  std::memcpy(mp.mix, h->mix, sizeof(mp.mix));
  dim3 grid((unsigned)((n + 255) / 256), h->n_out, 1);
  PC_LAUNCH_MIX(mp, grid, st);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
#endif
  return 0;
}

// ---- one launch group: n <= Lmax samples, device-resident ------------------------------------
int compact_timeline(b200conv* h, Stage& s, cudaStream_t st) {
  const int C = h->C, B = s.B;
  const size_t bytes = (size_t)s.hist * B * sizeof(float2);
  for (int c = 0; c < C; ++c) {
    float2* base = s.X + (size_t)c * s.R * B;
    CU_CHECK(h, cudaMemcpyAsync(base, base + (size_t)(s.head - s.hist) * B, bytes, cudaMemcpyDeviceToDevice, st));
  }
  s.head = s.hist;
  return 0;
}

// room for nb more X rows from the open block on (plus the sweeps' slack rows); a compaction is queued on st
int ensure_rows(b200conv* h, Stage& s, int nb, cudaStream_t st) {
  return s.head + nb + kMaxTT > s.R ? compact_timeline(h, s, st) : 0;
}

// How a Stage maps onto the kernels' parameter blocks.  The sweep of `nblocks` blocks from the open one on writes Y
// rows 1..; with `extra` it starts that many blocks early (row 0, see run_group).
pc::CmacParams sweep_params(const Stage& s, int C, float2* Y, int nblocks, int extra) {
  pc::CmacParams cp{};
  cp.H = s.H; cp.h_cstride = (long long)s.Prows * s.B;
  cp.X = s.X; cp.x_cstride = (long long)s.R * s.B; cp.xrow0 = s.head - s.p_begin - extra;
  cp.Y = Y; cp.y_cstride = s.B; cp.y_rstride = (long long)C * s.B; cp.yrow0 = 1 - extra;
  cp.B = s.B; cp.Ppad = s.P; cp.nblocks = nblocks + extra;
  return cp;
}

// forward FFT of `nblocks` blocks (`nvalid` samples, zero-padded) into the X rows from the open block on; `direct`: src
// is the caller's buffer, whose channels go through the input routing
pc::FwdParams fwd_params(const b200conv* h, const Stage& s, const float* src, size_t src_stride, long long nvalid,
                         int nblocks, bool direct) {
  pc::FwdParams fp{};
  fp.src = src; fp.src_cstride = (long long)src_stride;
  fp.nvalid_c = nullptr; fp.nvalid = nvalid;
  fp.use_cmap = (direct && (h->route_on || h->route_in_only)) ? 1 : 0;
  for (int c = 0; c < 8; ++c) fp.cmap[c] = h->in_map[c];
  fp.dst = s.X; fp.dst_cstride = (long long)s.R * s.B; fp.dst_row0 = s.head;
  fp.tw = s.tw; fp.tab512 = s.tab512; fp.M = s.B; fp.nblocks = nblocks;
  return fp;
}

// inverse FFT of Y rows 1..nblocks (row 0 is the overlap state); the caller adds the destination
pc::InvParams inv_params(const Stage& s, int C, float2* Y, int nblocks) {
  pc::InvParams ip{};
  ip.Y = Y; ip.y_cstride = s.B; ip.y_rstride = (long long)C * s.B; ip.yrow0 = 1;
  ip.tw = s.tw; ip.tab512 = s.tab512; ip.M = s.B; ip.nblocks = nblocks; ip.scale = 1.0f / (float)s.B;
  return ip;
}

// ... into the look-ahead ring of a stage >= 1, q blocks ahead of the stage's input
void inv_into_ring(pc::InvParams& ip, const Stage& s) {
  ip.dst = s.fut; ip.dst_cstride = (long long)s.ring;
  ip.index0 = (s.blocks_done + s.q) * (long long)s.B;
  ip.lo = 0; ip.hi = (long long)1 << 62; ip.mask = (long long)s.ring - 1;
}

// With an empty open block the forward FFT reads the caller's buffer directly; only a trailing partial block is
// buffered.  Otherwise the new samples are appended behind the open block's.
int intake_begin(b200conv* h, Stage& s, const float* in_dev, size_t in_stride, size_t n, Intake* it) {
  it->total = (size_t)s.fill + n;
  it->complete = (int)(it->total / s.B);
  it->partial = (int)(it->total % s.B);
  it->direct = s.fill == 0;
  it->src = it->direct ? in_dev : s.inbuf;
  it->src_stride = it->direct ? in_stride : s.in_stride;
  return it->direct ? 0 : copy_in(h, s.inbuf + s.fill, s.in_stride, in_dev, in_stride, n);
}

// the trailing partial block goes to the front of inbuf (with nothing completed and samples appended it is there already)
int intake_end(b200conv* h, Stage& s, const Intake& it) {
  const size_t off = (size_t)it.complete * s.B;
  if (it.partial > 0 && it.direct) {
    if (int rc = copy_in(h, s.inbuf, s.in_stride, it.src + off, it.src_stride, it.partial)) return rc;
  } else if (it.partial > 0 && it.complete > 0) {
    CU_CHECK(h, cudaMemcpy2DAsync(s.inbuf, s.in_stride * sizeof(float), s.inbuf + off, s.in_stride * sizeof(float),
                                  it.partial * sizeof(float), h->C, cudaMemcpyDeviceToDevice, h->s_main));
  }
  s.fill = it.partial;
  return 0;
}


// ---- slot exchange (fused multi-GPU path) ------------------------------------------------------
struct P2PRecord { unsigned long long kind; unsigned long long ptr; unsigned char ipc[64]; };
constexpr int kP2PBuffers = 8;    // Yx[0], Yx[1], Hh, xout[0], xout[1], flags, din[0], din[1]

int p2p_alloc(b200conv* h) {
  if (h->Yx[0]) return 0;
  const Stage& s = h->stages[0];
  const int G = h->cfg.shard_count, C = h->C, B = s.B;
  const size_t row = (size_t)C * B;
  h->xSR = (s.Tcap + G - 1) / G + 2;
  h->xslot = (size_t)h->xSR * row;
  for (int i = 0; i < 2; ++i) {
    CU_CHECK(h, cudaMalloc(&h->Yx[i], (size_t)G * h->xslot * sizeof(float2)));
    CU_CHECK(h, cudaMemsetAsync(h->Yx[i], 0, (size_t)G * h->xslot * sizeof(float2), h->s_main));
    CU_CHECK(h, cudaMalloc(&h->xout[i], (size_t)C * h->Lmax * sizeof(float)));
  }
  CU_CHECK(h, cudaMalloc(&h->Hh, (size_t)3 * G * row * sizeof(float2)));
  CU_CHECK(h, cudaMemsetAsync(h->Hh, 0, (size_t)3 * G * row * sizeof(float2), h->s_main));
  CU_CHECK(h, cudaMalloc(&h->xflags, 32 * sizeof(unsigned int)));
  CU_CHECK(h, cudaMemsetAsync(h->xflags, 0, 32 * sizeof(unsigned int), h->s_main));
  for (int i = 0; i < 2; ++i)
    if (!h->ev_b1[i]) CU_CHECK(h, cudaEventCreateWithFlags(&h->ev_b1[i], cudaEventDisableTiming));
#if !defined(PC_EMULATE)
  // Load every kernel / driver copy routine the exchange flow launches NOW: a lazy module load
  // synchronises the context and must not happen while a peer's flag barrier is spinning on this device.
  {
    cudaFuncAttributes fa;
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_p2p_barrier));
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_copy_rows));
#define PC_PRELOAD(BS) \
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_cmac_batch2<16, 4, 4, BS, 3>)); \
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_cmac_batch2<8, 4, 4, BS, 4>));
    PC_PRELOAD(0) PC_PRELOAD(128) PC_PRELOAD(512) PC_PRELOAD(8192)
#undef PC_PRELOAD
    // strided device-to-device copies and memsets as used by run_group_p2p / compact_timeline
    CU_CHECK(h, cudaMemcpy2DAsync(h->Yx[1], h->xslot * sizeof(float2), h->Hh, row * sizeof(float2), row * sizeof(float2), G,
                                  cudaMemcpyDeviceToDevice, h->s_main));
    CU_CHECK(h, cudaMemcpy2DAsync(h->xout[1], h->Lmax * sizeof(float), h->xout[0], h->Lmax * sizeof(float), sizeof(float), C,
                                  cudaMemcpyDeviceToDevice, h->s_post));
    CU_CHECK(h, cudaMemcpyAsync(h->Yx[1], h->Yx[0], row * sizeof(float2), cudaMemcpyDeviceToDevice, h->s_main));
    CU_CHECK(h, cudaMemsetAsync(h->Yx[1], 0, (size_t)G * h->xslot * sizeof(float2), h->s_main));
    CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  }
#endif
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return 0;
}

// after a host synchronisation: did a flag barrier give up waiting for a peer?
int p2p_check(b200conv* h) {
#if !defined(PC_EMULATE)
  if (h->xflags && (h->bar_epoch + h->in_epoch > 0 || h->p2p_tail)) {
    unsigned int err = 0;
    CU_CHECK(h, cudaMemcpy(&err, h->xflags + 8, sizeof(err), cudaMemcpyDeviceToHost));
    if (err != 0) {
      // report once, then re-arm: one slow peer must not fail every later call
      CU_CHECK(h, cudaMemset(h->xflags + 8, 0, sizeof(unsigned int)));
      return fail(h, B200CONV_ECUDA, "slot-exchange barrier timed out waiting for a peer GPU (audio of this call is incomplete)");
    }
  }
#else
  (void)h;
#endif
  return 0;
}

#if !defined(PC_EMULATE)
unsigned long long p2p_timeout_ns() {
  static const unsigned long long timeout_ms = [] {
    const char* e = std::getenv("B200CONV_P2P_TIMEOUT_MS");
    const long long v = e ? std::atoll(e) : 0;
    return (unsigned long long)(v > 0 ? v : 4000);       // default 4 s (every kernel of the exchange is pre-loaded at attach)
  }();
  return timeout_ms * 1000000ull;
}
#endif

// bank 0: exchange barriers (flag words 0..7, issued on s_post); bank 1: "input landed" barriers (words 16..23)
int p2p_barrier(b200conv* h, cudaStream_t st, int bank = 0) {
  unsigned int& epoch = bank == 0 ? h->bar_epoch : h->in_epoch;
  epoch++;
#if defined(PC_EMULATE)
  (void)st;
  if (!h->host_barrier) return fail(h, B200CONV_ESTATE, "emulated slot exchange needs a host barrier");
  if (h->host_barrier(h->host_barrier_user) != 0) return fail(h, B200CONV_ECUDA, "host barrier failed");
#else
  if (h->host_barrier) {
    // all shards in ONE process on one device (tests): spinning flag kernels of several handles share the
    // device's hardware queues / copy engines and can block each other, so synchronise through the host
    CU_CHECK(h, cudaStreamSynchronize(st));
    if (h->host_barrier(h->host_barrier_user) != 0) return fail(h, B200CONV_ECUDA, "host barrier failed");
    return 0;
  }
  pc::BarrierParams bp{};
  for (int g = 0; g < h->cfg.shard_count; ++g) bp.peer_flags[g] = h->peer_flags[g] + 16 * bank;
  bp.my_flags = h->xflags + 16 * bank;
  bp.error_word = h->xflags + 8;
  bp.rank = h->cfg.shard_rank; bp.G = h->cfg.shard_count; bp.epoch = epoch;
  bp.timeout_ns = p2p_timeout_ns();
  pc::k_p2p_barrier<<<1, 32, 0, st>>>(bp);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
#endif
  return 0;
}

// device-to-device row copy as a kernel (never a copy-engine copy: see k_copy_rows)
int copy_rows_kernel(b200conv* h, float* dst, size_t dpitch, const float* src, size_t spitch, size_t width, int rows, cudaStream_t st) {
  if (width == 0 || rows == 0) return 0;
#if defined(PC_EMULATE)
  (void)st;
  for (int r = 0; r < rows; ++r) std::memmove(dst + (size_t)r * dpitch, src + (size_t)r * spitch, width * sizeof(float));
#else
  dim3 grid((unsigned)((width + 255) / 256), rows, 1);
  pc::k_copy_rows<<<grid, 256, 0, st>>>(dst, (long long)dpitch, src, (long long)spitch, (long long)width, rows);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
#endif
  return 0;
}

// ---- tail slot exchange (stages >= 1 of a tail-sharded handle) ------------------------------------------------------
// Rank 0 owns, per tail stage, Tx = [2 parities][G slots][2 rows][C][B]: rank g stores the partial spectrum of a
// block into row 1 of slot g of the block's parity (sweep epilogue, peer store) and raises its flag in the stage's
// bank.  Row 0 of slot 0 is the summed spectrum of the previous block (the overlap state), rows 0 of the other slots
// stay zero, so that the inverse FFT summing the G slots (n_partials = G) sees the full sums of both rows.  A slot is
// written again two blocks later: rank g first waits until rank 0 has reached the barrier of the block in between,
// which it issues after the inverse FFT that read the slot.
constexpr int kFlagWords = 96;           // bank 0 words 0..7 + error word 8, bank 1 words 16..23, tail banks below
int tail_bank(int si) { return 32 + 16 * (si - 1); }

// ticket words of the exchange sweep: one per (channel, bin tile) of the widest tail stage (its grid is
// B / stream_tma_w(B) x nsplit x C) + the tile counter
size_t tail_tick_words(const b200conv* h) {
  int tiles = 1;
  for (size_t si = 1; si < h->stages.size(); ++si) tiles = std::max(tiles, h->stages[si].B / pc::stream_tma_w(h->stages[si].B));
  return (size_t)h->C * tiles + 1;
}

int p2p_alloc_tail(b200conv* h) {
  if (h->ttick) return 0;
  const int G = h->cfg.shard_count, C = h->C;
  CU_CHECK(h, cudaMalloc(&h->xflags, kFlagWords * sizeof(unsigned int)));
  CU_CHECK(h, cudaMemsetAsync(h->xflags, 0, kFlagWords * sizeof(unsigned int), h->s_main));
  const size_t ticks = tail_tick_words(h);
  CU_CHECK(h, cudaMalloc(&h->ttick, ticks * sizeof(unsigned int)));
  CU_CHECK(h, cudaMemsetAsync(h->ttick, 0, ticks * sizeof(unsigned int), h->s_main));
  for (size_t si = 1; si < h->stages.size() && h->cfg.shard_rank == 0; ++si) {
    const size_t bytes = (size_t)2 * G * 2 * C * h->stages[si].B * sizeof(float2);
    CU_CHECK(h, cudaMalloc(&h->Tx[si], bytes));
    CU_CHECK(h, cudaMemsetAsync(h->Tx[si], 0, bytes, h->s_main));
  }
#if !defined(PC_EMULATE)
  // every kernel a tail block launches, loaded now (see p2p_alloc)
  {
    cudaFuncAttributes fa;
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_p2p_barrier));
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_sum_slots));
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_cmac_stream_tma<6, pc::StreamXchParams>));
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_cmac_stream_tma<12, pc::StreamXchParams>));
    CU_CHECK(h, cudaFuncGetAttributes(&fa, pc::k_fwd_fft512));
    for (size_t si = 1; si < h->stages.size(); ++si) {
      cudaError_t e = cudaErrorInvalidValue;
      switch (pc::ilog2(h->stages[si].B)) {
#define PC_CASE(L) case L: e = fft_preload<L>(); break;
        PC_FOR_EACH_LOG2(PC_CASE)
#undef PC_CASE
        default: break;
      }
      CU_CHECK(h, e);
    }
  }
#endif
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return 0;
}

// host-side rendezvous of all shards (emulation build, shards sharing one device in one process)
int host_rendezvous(b200conv* h, cudaStream_t st) {
  CU_CHECK(h, cudaStreamSynchronize(st));
  if (h->host_barrier(h->host_barrier_user) != 0) return fail(h, B200CONV_ECUDA, "host barrier failed");
  return 0;
}

// rank 0: every rank's flag of block e is up (it publishes e in the peers' banks first); rank g >= 1: rank 0 has
// published e (this waits only: the scratch word 8 of the bank takes the publish)
int tail_flag_wait(b200conv* h, cudaStream_t st, int si, unsigned int e) {
#if defined(PC_EMULATE)
  (void)st; (void)si; (void)e;
  return fail(h, B200CONV_ESTATE, "emulated slot exchange needs a host barrier");
#else
  const int off = tail_bank(si);
  pc::BarrierParams bp{};
  bp.my_flags = h->xflags + off;
  bp.error_word = h->xflags + 8;
  bp.rank = 0; bp.epoch = e;
  bp.timeout_ns = p2p_timeout_ns();
  if (h->cfg.shard_rank == 0) {
    bp.G = h->cfg.shard_count;
    for (int g = 0; g < bp.G; ++g) bp.peer_flags[g] = h->peer_flags[g] + off;
  } else {
    bp.G = 1;
    bp.peer_flags[0] = h->xflags + off + 8;
  }
  pc::k_p2p_barrier<<<1, 32, 0, st>>>(bp);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
  return 0;
#endif
}

int launch_sum_slots(b200conv* h, float2* dst, const float2* src, size_t n, int np, size_t ps, cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)h; (void)st;
  for (size_t i = 0; i < n; ++i) dst[i] = pc::sum_partials(src + i, 0, np, (long long)ps);
#else
  pc::k_sum_slots<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dst, src, (long long)n, np, (long long)ps);
  h->launches++;
  CU_CHECK(h, cudaGetLastError());
#endif
  return 0;
}

// One completed block of a stage >= 1, spectrum in X row s.head (output block s.blocks_done), everything on
// h->s_launch: the sweep over this rank's partitions, on a tail-sharded handle the partial spectra of all ranks summed
// on rank 0 (slot exchange, else the reduce hook), and on rank 0 (the only rank of an unsharded handle) the inverse
// FFT into the stage's look-ahead ring.
int tail_block(b200conv* h, Stage& s, int si) {
  const int C = h->C, B = s.B, G = h->cfg.shard_count, g = h->cfg.shard_rank;
  const size_t row = (size_t)C * B;
  cudaStream_t st = h->s_launch;
  float2* Yb = s.Y[s.ybuf];
  const pc::CmacParams cp = sweep_params(s, C, Yb, 1);
  pc::InvParams ip = inv_params(s, C, Yb, 1);
  inv_into_ring(ip, s);
  if (!h->p2p_tail) {
    if (s.P > 0) { if (int rc = launch_cmac(h, cp, C)) return rc; }
    else CU_CHECK(h, cudaMemsetAsync(Yb + row, 0, row * sizeof(float2), st));
    if (tail_layout(h)) {                   // reduce hook: once per tail block, never for the head
      if (!h->reduce) return fail(h, B200CONV_ESTATE, "sharded handle without a reduce hook");
      if (h->reduce(h->reduce_user, reinterpret_cast<float*>(Yb + row), row * 2, st) != 0)
        return fail(h, B200CONV_ECUDA, "reduce hook failed");
    }
    if (g == 0) {
      if (int rc = launch_inv(h, ip, C, st)) return rc;
      CU_CHECK(h, cudaMemcpyAsync(Yb, Yb + row, row * sizeof(float2), cudaMemcpyDeviceToDevice, st));   // overlap state
    }
    return 0;
  }
  const unsigned long long e = ++h->tx_blocks[si];
  const size_t par = (size_t)G * 2 * row;                      // float2 per parity
  if (g > 0 && !h->host_barrier && e > 1) { if (int rc = tail_flag_wait(h, st, si, (unsigned int)(e - 1))) return rc; }
  const TailXch x{h->peerTx0[si] + (size_t)(e & 1) * par + (size_t)g * 2 * row + row,
                  h->peer_flags[0] + tail_bank(si) + g, (unsigned int)e};
  if (int rc = launch_cmac_exchange(h, cp, C, x)) return rc;
  if (h->host_barrier) { if (int rc = host_rendezvous(h, st)) return rc; }
  else if (g == 0) { if (int rc = tail_flag_wait(h, st, si, (unsigned int)e)) return rc; }
  if (g == 0) {
    float2* mine = h->Tx[si] + (size_t)(e & 1) * par;
    ip.Y = mine; ip.n_partials = G; ip.partial_stride = (long long)(2 * row);
    if (int rc = launch_inv(h, ip, C, st)) return rc;
    // the summed spectrum -> overlap row of the next block (the other parity)
    if (int rc = launch_sum_slots(h, h->Tx[si] + (size_t)((e + 1) & 1) * par, mine + row, row, G, 2 * row, st)) return rc;
  }
  return 0;
}

// Stages >= 1 of a tail-sharded handle for one launch group of n samples: forward FFT of the completed blocks, then
// tail_block for each, stage by stage in ascending order (the same sequence of exchanges / hook calls on every rank
// and on every path, the real-time one included).
int run_tail_stages(b200conv* h, const float* in_dev, size_t in_stride, size_t n) {
  const int C = h->C;
  for (size_t si = 1; si < h->stages.size(); ++si) {
    Stage& s = h->stages[si];
    Intake it;
    if (int rc = intake_begin(h, s, in_dev, in_stride, n, &it)) return rc;
    if (it.complete > 0) {
      if (int rc = ensure_rows(h, s, it.complete, h->s_launch)) return rc;
      const pc::FwdParams fp = fwd_params(h, s, it.src, it.src_stride, (long long)it.total, it.complete, it.direct);
      if (int rc = launch_fwd(h, fp, C)) return rc;
      for (int j = 0; j < it.complete; ++j) {
        if (int rc = tail_block(h, s, (int)si)) return rc;
        s.head += 1;
        s.blocks_done += 1;
      }
    }
    if (int rc = intake_end(h, s, it)) return rc;
  }
  return 0;
}

// one launch group of a single-stage sharded handle through the slot exchange
int run_group_p2p(b200conv* h, const float* in_dev, size_t in_stride, float* out_dev, size_t out_stride, size_t n) {
  const int C = h->C, G = h->cfg.shard_count, g = h->cfg.shard_rank;
  Stage& s = h->stages[0];
  const int B = s.B;
  const size_t row = (size_t)C * B;
  cudaStream_t ps = h->s_post;
  if (n == 0) return 0;
  if (n + B > h->Lmax) return fail(h, B200CONV_ESTATE, "launch group larger than the staging buffers");
  Intake it;
  if (int rc = intake_begin(h, s, in_dev, in_stride, n, &it)) return rc;
  const int complete = it.complete;
  const int nb = complete + (it.partial > 0 ? 1 : 0);
  const int yb = s.ybuf;
  const int per = (nb + G - 1) / G;
  if (int rc = ensure_rows(h, s, nb, h->s_launch)) return rc;
  // (routing is refused on this path: the input map stays unused)
  const pc::FwdParams fp = fwd_params(h, s, it.src, it.src_stride, (long long)it.total, nb, it.direct);
  if (int rc = launch_fwd(h, fp, C)) return rc;

  // the exchange buffers of parity yb are free once every GPU finished the inverse FFT of two groups ago
  CU_CHECK(h, cudaStreamWaitEvent(h->s_main, s.ev_post[yb], 0));
  pc::CmacParams cp = sweep_params(s, C, nullptr, nb);    // the rows go to the ranks' exchange slots
  cp.yrow0 = 0;
  cp.xg = G; cp.xrank = g; cp.xper = per; cp.xslot = (long long)h->xslot;
  cp.xhalo_block = complete > 0 ? complete - 1 : -1;
  for (int r = 0; r < G; ++r) cp.xbase[r] = h->peerYx[r][yb];
  cp.xhalo = h->peerHh0 + (size_t)((h->hidx + 1) % 3) * G * row;
  if (int rc = launch_cmac(h, cp, C)) return rc;
  CU_CHECK(h, cudaEventRecord(s.ev_sweep[yb], h->s_main));
  CU_CHECK(h, cudaStreamWaitEvent(ps, s.ev_sweep[yb], 0));

  if (int rc = p2p_barrier(h, ps)) return rc;          // every GPU's partial rows have landed
  CU_CHECK(h, cudaEventRecord(h->ev_b1[h->xgrp & 1], ps));   // ... hence every GPU is done reading this group's input
  h->xgrp++;

  const int j0 = std::min(nb, g * per), j1 = std::min(nb, (g + 1) * per);
  if (j1 > j0) {
    if (g == 0) { // halo of the first slice = last completed row of the previous group (all G partials)
      if (int rc = copy_rows_kernel(h, reinterpret_cast<float*>(h->Yx[yb]), h->xslot * 2,
                                    reinterpret_cast<const float*>(h->Hh + (size_t)h->hidx * G * row), row * 2, row * 2, G, ps)) return rc;
    }
    pc::InvParams ip = inv_params(s, C, h->Yx[yb], j1 - j0);
    ip.n_partials = G; ip.partial_stride = (long long)h->xslot;
    ip.dst = h->peer_xout0[yb]; ip.dst_cstride = (long long)h->Lmax;
    ip.index0 = -(long long)s.fill + (long long)j0 * B; ip.lo = 0; ip.hi = (long long)n; ip.mask = -1;
    if (int rc = launch_inv(h, ip, C, ps)) return rc;
  }
  if (int rc = p2p_barrier(h, ps)) return rc;          // every slice of the audio is in shard 0's exchange buffer
  if (g == 0 && out_dev) {
    if (int rc = copy_rows_kernel(h, out_dev, out_stride, h->xout[yb], h->Lmax, n, C, ps)) return rc;
  }
  CU_CHECK(h, cudaEventRecord(s.ev_post[yb], ps));

  if (complete > 0) {
    s.ybuf = yb ^ 1;
    h->hidx = (h->hidx + 1) % 3;
    s.head += complete;
    s.blocks_done += complete;
  }
  if (int rc = intake_end(h, s, it)) return rc;
  h->abs_pos += (long long)n;
  return 0;
}

int drain_tail(b200conv* h);
int join_post(b200conv* h);

// `overlap`: reduce + inverse FFT go to s_post so that they overlap the next group's forward
// FFT + sweep on s_main (double-buffered Y); otherwise everything is issued on s_main.
int run_group(b200conv* h, const float* in_dev, size_t in_stride, float* out_dev, size_t out_stride, size_t n,
              bool overlap) {
  const int C = h->C;
  const bool root = h->cfg.shard_rank == 0;
  if (h->p2p_on) {
    if (h->route_on) return fail(h, B200CONV_ESTATE, "I/O routing is not available on the slot-exchange path");
    return run_group_p2p(h, in_dev, in_stride, out_dev, out_stride, n);
  }
  cudaStream_t ps = overlap ? h->s_post : h->s_main;
  if (n == 0) return 0;
  if (n + h->stages[0].B > h->Lmax) return fail(h, B200CONV_ESTATE, "launch group larger than the staging buffers");
  if (int rc = drain_tail(h)) return rc;
  const bool tails = tail_layout(h);
  if (tails) {
    // stages >= 1 block by block on s_main, behind the previous group's head output (which reads their rings)
    if (overlap) { if (int rc = join_post(h)) return rc; }
    if (int rc = run_tail_stages(h, in_dev, in_stride, n)) return rc;
    if (!root) { h->abs_pos += (long long)n; return 0; }     // no head partitions on this rank
  }
  // stages >= 1 first (their look-ahead output may be consumed by the head within this group)
  for (int si = tails ? 0 : (int)h->stages.size() - 1; si >= 0; --si) {
    Stage& s = h->stages[si];
    const int B = s.B;
    const size_t row = (size_t)C * B;           // float2 per Y row (all channels)
    Intake it;
    if (int rc = intake_begin(h, s, in_dev, in_stride, n, &it)) return rc;
    const int complete = it.complete;
    const int nb = (si == 0) ? complete + (it.partial > 0 ? 1 : 0) : complete;
    const int yb = s.ybuf;
    float2* Yb = s.Y[yb];
    // B = 512 groups on the tensor-core sweep (unsharded): the inverse FFT reads the sweep's bin-major result
    // (tcY[yb], sw.yc); the transpose into Y rows is left out
    Sweep sw;
    if (nb > 0) {
      if (int rc = ensure_rows(h, s, nb, h->s_launch)) return rc;
      // overlap state after a forward-FFT-only advance (time-slice sharding): Y row 0 must become
      // sum_p H[p] X[head-1-p], the spectrum of the block in front of this group — its input spectra are in the
      // timeline, so the sweep simply starts one block early and writes that block as row 0
      const int extra = (si == 0 && h->yprev_stale) ? 1 : 0;
      const pc::CmacParams cp = sweep_params(s, C, Yb, nb, extra);
      const bool direct_ok = h->cfg.shard_count == 1 && use_fft512(h, B, nb, C, s.tab512);
      if (int rc = select_cmac(h, cp, C, &sw, direct_ok ? &s.tcY[yb] : nullptr, extra,
                               si == 0 && fourstep_ok(h, s, it, extra, C))) return rc;
      if (sw.variant == 42) {
        if (int rc = run_group_fourstep(h, s, it, out_dev, out_stride, n, overlap)) return rc;
        if (int rc = intake_end(h, s, it)) return rc;
        continue;
      }

      pc::FwdParams fp = fwd_params(h, s, it.src, it.src_stride, (long long)it.total, nb, it.direct);
      if (sw.yc) {
        const pc::tc::Geom tg = pc::tc::make_geom(cp.Ppad, cp.nblocks);
        // the spectra go straight into the sweep's time lines (block b at tau = Q + extra + b).  X rows are still what
        // everything after this group reads the history from: the next group's split, real-time calls and the
        // streaming sweeps, FFMA groups, a time-slice rank's early block (its sweep starts one row back) and
        // compact_timeline.  None of them reads further back than s.hist rows behind the head (compact_timeline
        // keeps exactly those), so only the blocks from complete - s.hist on write their rows
        fp.lines = h->tc_Xt.p; fp.line_tau0 = tg.Q + extra; fp.line_rows = tg.rows;
        fp.xrow_from = std::max(0, complete - s.hist);
      }
      if (int rc = launch_fwd(h, fp, C)) return rc;

      // Y[yb] rows >= 1 (and tcY[yb]) may still be read by the post work of two groups ago
      if (overlap) CU_CHECK(h, cudaStreamWaitEvent(h->s_main, s.ev_post[yb], 0));
      if (extra) {
        if (overlap) CU_CHECK(h, cudaStreamWaitEvent(h->s_main, s.ev_post[yb ^ 1], 0));   // row 0 was written on s_post
        h->yprev_stale = false;
      }
      if (int rc = launch_cmac_as(h, cp, C, sw)) return rc;
      if (overlap) {
        CU_CHECK(h, cudaEventRecord(s.ev_sweep[yb], h->s_main));
        CU_CHECK(h, cudaStreamWaitEvent(ps, s.ev_sweep[yb], 0));
      }

      if (h->cfg.shard_count > 1 && !tails) {
        if (!h->reduce) return fail(h, B200CONV_ESTATE, "sharded handle without a reduce hook");
        if (h->reduce(h->reduce_user, reinterpret_cast<float*>(Yb + row), (size_t)nb * row * 2, ps) != 0)
          return fail(h, B200CONV_ECUDA, "reduce hook failed");
      }
      if (root) {
        pc::InvParams ip = inv_params(s, C, Yb, nb);
        if (sw.yc) {   // block t at slot kYLead + extra + t; block -1 is the overlap state (Y row 0) unless swept
          ip.yc = sw.yc; ip.yc_stride = sw.yc_stride; ip.yc_slot0 = pc::tc::kYLead + sw.extra;
          ip.yc_prev_row = sw.extra == 0;
        }
        if (si == 0) {
          ip.dst = h->route_on ? h->dch[0] : out_dev;
          ip.dst_cstride = h->route_on ? (long long)h->Lmax : (long long)out_stride;
          ip.index0 = -(long long)s.fill; ip.lo = 0; ip.hi = (long long)n; ip.mask = -1;
          ip.abs0 = h->abs_pos - s.fill;
          int na = 0;
          for (size_t sj = 1; sj < h->stages.size() && na < 3; ++sj) {
            ip.add[na] = h->stages[sj].fut; ip.add_cstride[na] = (long long)h->stages[sj].ring;
            ip.add_mask[na] = (long long)h->stages[sj].ring - 1;
            ++na;
          }
          ip.n_add = na;
        } else {
          inv_into_ring(ip, s);
        }
        if (int rc = launch_inv(h, ip, C, ps)) return rc;
        if (si == 0 && h->route_on) { if (int rc = launch_mix(h, h->dch[0], h->Lmax, out_dev, out_stride, n, ps)) return rc; }
      }
    }
    // state update
    if (complete > 0) {
      // overlap state for the next group: last completed row -> row 0 of the buffer it will use
      const int nxt = overlap ? (yb ^ 1) : yb;
      if (sw.yc)     // block complete - 1 of every line
        CU_CHECK(h, cudaMemcpy2DAsync(s.Y[nxt], sizeof(float2), sw.yc + pc::tc::kYLead + sw.extra + (complete - 1),
                                      (size_t)sw.yc_stride * sizeof(float2), sizeof(float2), row, cudaMemcpyDeviceToDevice, ps));
      else
        CU_CHECK(h, cudaMemcpyAsync(s.Y[nxt], Yb + (size_t)complete * row, row * sizeof(float2),
                                    cudaMemcpyDeviceToDevice, ps));
      if (overlap) CU_CHECK(h, cudaEventRecord(s.ev_post[yb], ps));
      s.ybuf = nxt;
      s.head += complete;
      s.blocks_done += complete;
    }
    if (int rc = intake_end(h, s, it)) return rc;
    // a group that completed no block releases Y[yb] here (one that did, above)
    if (complete == 0 && overlap && nb > 0) CU_CHECK(h, cudaEventRecord(s.ev_post[yb], ps));
  }
  h->abs_pos += (long long)n;
  return 0;
}

// Forward FFTs only (uniform handle, no open block): the spectra of `nblocks` input blocks go into the timeline,
// no sweep, no output.  Used by the time-slice sharding for the history in front of a slice and for the tail of
// the call every GPU keeps.
int advance_fft_only(b200conv* h, const float* in_dev, size_t in_stride, long long nblocks) {
  Stage& s = h->stages[0];
  const int C = h->C, B = s.B;
  for (long long done = 0; done < nblocks;) {
    const int nb = (int)std::min<long long>(nblocks - done, s.Tcap);
    if (int rc = ensure_rows(h, s, nb, h->s_launch)) return rc;
    const pc::FwdParams fp = fwd_params(h, s, in_dev + (size_t)done * B, in_stride, (long long)nb * B, nb, false);
    if (int rc = launch_fwd(h, fp, C)) return rc;
    s.head += nb;
    s.blocks_done += nb;
    done += nb;
  }
  if (nblocks > 0) h->yprev_stale = true;
  h->abs_pos += nblocks * B;
  return 0;
}

// Time-slice sharding of one block-aligned call of T blocks (see b200conv_process_sliced): which blocks this
// GPU transforms only ([lo, a) in front of its slice, [tail_lo, T) behind it) and which it convolves ([a, b)).
struct SlicePlan { long long T, a, b, lo, tail_lo; };

int plan_slice(b200conv* h, size_t len, int rank, int count, SlicePlan* sp) {
  if (count < 1 || rank < 0 || rank >= count) return fail(h, B200CONV_EINVAL, "slice_rank / slice_count out of range");
  if (h->stages.size() != 1) return fail(h, B200CONV_ESTATE, "time-slice sharding needs a uniform (single-stage) handle");
  if (h->cfg.shard_count != 1) return fail(h, B200CONV_ESTATE, "time-slice sharding needs an unsharded handle (the full IR on every GPU)");
  if (h->route_on) return fail(h, B200CONV_ESTATE, "time-slice sharding is not available with I/O routing");
  const Stage& s = h->stages[0];
  if (s.fill != 0 || len % (size_t)s.B != 0)
    return fail(h, B200CONV_ESTATE, "time-slice sharding needs block-aligned calls (len a multiple of the block size, no open block)");
  const long long T = (long long)(len / (size_t)s.B), P = s.P_full;
  const long long per = (T + count - 1) / count;
  sp->T = T;
  sp->a = std::min(T, rank * per);
  sp->b = std::min(T, (rank + 1) * per);
  // block t needs X[t-p], p < P, and the overlap-add needs the spectrum of block t-1 as well: P blocks of history
  sp->lo = sp->b > sp->a ? std::max(0LL, sp->a - P) : sp->a;
  sp->tail_lo = std::max(sp->b, T - P);
  // Without the tail the handle's history ends with its own slice: enough for a following sliced call whose slice
  // starts at least P blocks into the call (it uploads its own history then) — what every rank but 0 of a steady
  // batch job needs; saves P blocks of H2D + forward FFT per call.
  if (!h->opt_slice_tail && sp->b > sp->a) sp->tail_lo = T;
  if (sp->b <= sp->a) { sp->a = sp->b = sp->lo = std::max(0LL, T - P); sp->tail_lo = sp->a; }   // empty slice: only keep the tail
  return 0;
}

// ---- real-time path: one cluster kernel per call (kernels_rt.cuh) + tail blocks on the low-priority stream -----
// every batch-path entry point first orders s_main (and s_post) behind all tail blocks still in flight on s_tail
int drain_tail(b200conv* h) {
  for (auto& s : h->stages)
    for (int j = 0; j < 2; ++j)
      if (!s.job_waited[j]) {
        CU_CHECK(h, cudaStreamWaitEvent(h->s_main, s.ev_job[j], 0));
        CU_CHECK(h, cudaStreamWaitEvent(h->s_post, s.ev_job[j], 0));
        s.job_waited[j] = true;
      }
  return 0;
}

// ONE completed block of a stage >= 1 (its samples are in s.inbuf), everything on h->s_launch: forward FFT into the
// timeline, streaming sweep, inverse FFT into the stage's look-ahead ring (TwoStageFFTConvolver.cpp:201-222)
int run_tail_block(b200conv* h, Stage& s) {
  if (int rc = ensure_rows(h, s, 1, h->s_launch)) return rc;
  const pc::FwdParams fp = fwd_params(h, s, s.inbuf, s.in_stride, s.B, 1, false);
  if (int rc = launch_fwd(h, fp, h->C)) return rc;
  // on rank 0 of a tail-sharded handle the other ranks' partial spectra join here
  if (int rc = tail_block(h, s, (int)(&s - h->stages.data()))) return rc;
  s.head += 1;
  s.blocks_done += 1;
  s.fill = 0;
  return 0;
}

constexpr size_t kRtMaxBytesPerCta = 384 * 1024;      // H + FDL bytes one CTA of the cluster may have to stream

// CTAs per convolver for the cluster kernel; -1 = split mode (head stage too large for one cluster); 0 = the call does not qualify
int rt_cluster_ctas(const b200conv* h, size_t len) {
  if (!h->opt_rt || h->stages.empty() || h->stages.size() > 4) return 0;
  // rank 0 of a tail-sharded handle holds the head whole: its tail blocks are exchanged by run_tail_block
  const bool whole_head = h->cfg.shard_count == 1 || (tail_layout(h) && h->cfg.shard_rank == 0);
  if (!whole_head || h->p2p_on || h->timing || h->yprev_stale) return 0;
  const Stage& s0 = h->stages[0];
  const int M = s0.B, C = h->C;
  if (M < 16 || M > 1024 || C > 8 || len == 0 || len > (size_t)M) return 0;
  if (h->route_on && (h->n_out * (int)len > 8 * 1024)) return 0;
  // A call that completes the open block and starts the next one runs as two segments.  Every later stage's block must
  // then end on head-block boundaries only, and a stage whose block completes at this boundary must not be needed
  // before the call ends: its block is enqueued after the launch, and with q = 1 its output starts at the boundary.
  const bool cross = (size_t)s0.fill + len > (size_t)M;
  if (cross)
    for (size_t si = 1; si < h->stages.size(); ++si) {
      const Stage& s = h->stages[si];
      if (s.B % M != 0 || (s.q < 2 && s.fill + (M - s0.fill) == s.B)) return 0;
    }
  int max_nc = 1;
  while (max_nc * 2 * C <= 16 && max_nc * 2 <= M / 32) max_nc *= 2;     // cluster <= 16 CTAs, tile >= 16 bin pairs
  int nc = 1;
  while (M / nc / 2 > 256) nc *= 2;                                      // at most 256 bin pairs per CTA
  const size_t bytes = (size_t)s0.P * M * 16;                            // H + FDL rows of one convolver
  // one SM pulls ~20-50 GB/s out of L2 with this access pattern: spread a convolver over as many CTAs as the
  // cluster allows until a CTA streams <= 64 KB; beyond kRtMaxBytesPerCta the all-SM streaming sweep wins
  while (nc < max_nc && bytes / nc > 64 * 1024) nc *= 2;
  if (nc > max_nc || bytes / nc > kRtMaxBytesPerCta)      // -1: split mode (front kernel, all-SM TMA sweep, back
    return (!cross && C <= 8 && M >= 64) ? -1 : 0;        // kernel) for calls inside the open block
  return nc;
}

#if !defined(PC_EMULATE)
// grid of `nctas` CTAs in clusters of `cluster`
template <class Arg>
cudaError_t rt_launch_kernel(void (*k)(Arg), const Arg& a, int nctas, int cluster, size_t smem, cudaStream_t st) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(nctas, 1, 1);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k, a);
}
template <int M>
cudaError_t rt_launch_m(const pc::RtParams& P, int cluster, size_t smem, cudaStream_t st) {
  return rt_launch_kernel(pc::k_rt_block<M>, P, cluster, cluster, smem, st);
}
template <int M>
cudaError_t rt_launch_m(const pc::RtGroupParams& G, int cluster, size_t smem, cudaStream_t st) {
  return rt_launch_kernel(pc::k_rt_group<M>, G, G.n * cluster, cluster, smem, st);
}
template <int M>
cudaError_t rt_launch_m(const pc::RtStepGroupParams& G, int cluster, size_t smem, cudaStream_t st) {
  return rt_launch_kernel(pc::k_rt_group_steps<M>, G, G.n * cluster, cluster, smem, st);
}
// k_rt_block<M> (one call), k_rt_group<M> or k_rt_group_steps<M> (a group's shape class) with clusters of C * NC CTAs
template <class Arg>
cudaError_t rt_launch(const Arg& a, int M, int C, int NC, cudaStream_t st) {
  const size_t smem = (size_t)pc::rt_smem_layout(M, C).bytes;
  switch (M) {
    case 16: return rt_launch_m<16>(a, C * NC, smem, st);
    case 32: return rt_launch_m<32>(a, C * NC, smem, st);
    case 64: return rt_launch_m<64>(a, C * NC, smem, st);
    case 128: return rt_launch_m<128>(a, C * NC, smem, st);
    case 256: return rt_launch_m<256>(a, C * NC, smem, st);
    case 512: return rt_launch_m<512>(a, C * NC, smem, st);
    case 1024: return rt_launch_m<1024>(a, C * NC, smem, st);
    default: return cudaErrorInvalidValue;
  }
}
template <int M>
bool rt_set_attr() {
  const int smem = pc::rt_smem_layout(M, 16).bytes;
  return cudaFuncSetAttribute(pc::k_rt_block<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
         cudaFuncSetAttribute(pc::k_rt_block<M>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess &&
         cudaFuncSetAttribute(pc::k_rt_group<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
         cudaFuncSetAttribute(pc::k_rt_group<M>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess &&
         cudaFuncSetAttribute(pc::k_rt_group_steps<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
         cudaFuncSetAttribute(pc::k_rt_group_steps<M>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess;
}
#endif

// A real-time call (rt_cluster_ctas() > 0) runs as prepare, launch, commit; b200conv_group_process prepares several
// handles, launches them together and commits them.  `in` / `out` are device-accessible (pinned host or device memory).
// Prepare: the waits for tail outputs the call needs and room in the timeline, both queued on `st`, the stream the launch
// goes to (*waited is set if there was a wait), and the call's parameters.  Split mode (nc < 0) is set up by rt_call.
// With T (the step form of the device-buffer group calls, group_step_ctas() > 0), P is T->p and the call of up to
// kRtMaxSteps head blocks becomes one step record: the kernel derives its segments from the call's start.
int rt_prepare(b200conv* h, int nc, const float* in, size_t in_stride, float* out, size_t out_stride, size_t len,
               cudaStream_t st, pc::RtParams& P, bool* waited, pc::RtStepParams* T = nullptr) {
  const int C = h->C;
  Stage& s0 = h->stages[0];
  const int M = s0.B;
  // tail blocks whose output this call needs must have landed in their look-ahead rings
  for (size_t si = 1; si < h->stages.size(); ++si) {
    Stage& s = h->stages[si];
    for (int j = 0; j < 2; ++j)
      if (!s.job_waited[j] && h->abs_pos + (long long)len > s.job_out_start[j]) {
        CU_CHECK(h, cudaStreamWaitEvent(st, s.ev_job[j], 0));
        s.job_waited[j] = true;
        h->rt_tail_joined = true;
        *waited = true;
      }
  }
  // a call that crosses the block boundary: len1 samples complete the open block, the other r start the next one
  const int len1 = std::min((int)len, M - s0.fill), r = (int)len - len1;
  const int nrows = T ? 1 + (r + M - 1) / M : (r ? 2 : 1);
  if (int rc = ensure_rows(h, s0, nrows, st)) return rc;
  if (T) *T = pc::RtStepParams{};
  P = pc::RtParams{};
  P.M = M; P.C = C; P.NC = nc; P.P = s0.P;
  P.len = (int)len; P.nseg = T ? 0 : (r ? 2 : 1);
  pc::RtSeg& S1 = P.seg[0];
  pc::RtSeg& S2 = P.seg[1];
  S1.fill = s0.fill; S1.len = len1; S1.complete = (s0.fill + len1 == M) ? 1 : 0; S1.off = 0;
  S1.head = s0.head; S1.abs0 = h->abs_pos - s0.fill;
  S2.fill = 0; S2.len = r; S2.complete = 0; S2.off = len1;
  S2.head = s0.head + 1; S2.abs0 = h->abs_pos + len1;
  P.in = in; P.in_stride = (long long)in_stride;
  for (int c = 0; c < 8; ++c) P.in_map[c] = (h->route_on || h->route_in_only) ? h->in_map[c] : c;
  P.inbuf0 = s0.inbuf; P.inbuf0_stride = (long long)s0.in_stride;
  P.H = s0.H; P.h_cstride = (long long)s0.Prows * M;
  P.X = s0.X; P.x_cstride = (long long)s0.R * M;
  // the step form stores only the last completed block's spectrum, where the one-launch calls would have left it
  const int ncomplete = (s0.fill + (int)len) / M;
  P.Yprev = s0.Y[s0.ybuf]; P.Ynext = s0.Y[T ? s0.ybuf ^ (ncomplete & 1) : s0.ybuf ^ 1]; P.y_cstride = M;
  P.tw = s0.tw;
  int na = 0;
  for (size_t si = 1; si < h->stages.size(); ++si) {
    Stage& s = h->stages[si];
    P.later_stride[na] = (long long)s.in_stride;
    S1.later_inbuf[na] = s.inbuf; S1.later_fill[na] = s.fill;
    // a stage whose block completes at the boundary takes the samples after it at the front of its other buffer (the
    // step form: at the one boundary group_step_ctas allows inside the call)
    const bool at_boundary = T ? s.fill + (int)len > s.B : (r && s.fill + len1 == s.B);
    S2.later_inbuf[na] = at_boundary ? s.inbuf_alt : s.inbuf; S2.later_fill[na] = at_boundary ? 0 : s.fill + len1;
    if (T) {
      T->later_inbuf[na] = s.inbuf; T->later_alt[na] = s.inbuf_alt;
      T->later_fill[na] = s.fill; T->later_B[na] = s.B;
    }
    // That buffer was read by the stage's previous tail block on s_tail, so s_main must be ordered behind it.  With
    // q <= 2 (every two-stage handle) the loop above has already waited for it, as it does for the first call after the
    // buffer swap below: that block's output starts at (blocks_done - 1 + q) * B, at or before the boundary, and this
    // call ends after the boundary.  Deeper stages of b200conv_init_stages wait here.
    const int jp = (int)((s.njobs + 1) & 1);
    if (at_boundary && s.njobs && !s.job_waited[jp]) {
      CU_CHECK(h, cudaStreamWaitEvent(st, s.ev_job[jp], 0));
      s.job_waited[jp] = true;
      h->rt_tail_joined = true;
      *waited = true;
    }
    P.add[na] = s.fut; P.add_cstride[na] = (long long)s.ring; P.add_mask[na] = (long long)s.ring - 1;
    ++na;
  }
  P.n_later = na; P.n_add = na;
  P.out = out; P.out_stride = (long long)out_stride;
  P.mix_on = h->route_on ? 1 : 0; P.n_out = h->route_on ? h->n_out : C;
  std::memcpy(P.mix, h->mix, sizeof(P.mix));
  if (T) {
    P.seg[0] = P.seg[1] = pc::RtSeg{};
    T->fill = s0.fill; T->head = s0.head; T->abs_pos = h->abs_pos;
  }
  return 0;
}

// Commit: the bookkeeping of a launched call of len samples, as the one-launch calls of its head-block pieces would
// leave it, and the tail blocks it completes (at most one per stage).  They go to the low-priority stream behind event
// `ev`, which is recorded on `st` (behind the call's launch) by the first of them unless *recorded.
int rt_commit(b200conv* h, int len, cudaEvent_t ev, cudaStream_t st, bool* recorded) {
  Stage& s0 = h->stages[0];
  // bookkeeping of the head stage: every completed block advances the timeline and flips the overlap buffer
  const int ncomplete = (s0.fill + len) / s0.B;
  s0.head += ncomplete; s0.blocks_done += ncomplete; s0.ybuf ^= ncomplete & 1;
  s0.fill = (s0.fill + len) % s0.B;
  h->abs_pos += (long long)len;
  // later stages: the kernel appended the samples; a completed block goes to the low-priority stream
  for (size_t si = 1; si < h->stages.size(); ++si) {
    Stage& s = h->stages[si];
    s.fill += len;
    if (s.fill < s.B) continue;
    const int rest = s.fill - s.B;
    if (!*recorded) { CU_CHECK(h, cudaEventRecord(ev, st)); *recorded = true; }
    CU_CHECK(h, cudaStreamWaitEvent(h->s_tail, ev, 0));
    const int j = (int)(s.njobs & 1);
    s.job_out_start[j] = (s.blocks_done + s.q) * (long long)s.B;
    h->s_launch = h->s_tail;
    const int rc = run_tail_block(h, s);
    h->s_launch = h->s_main;
    if (rc) return rc;
    CU_CHECK(h, cudaEventRecord(s.ev_job[j], h->s_tail));
    s.job_waited[j] = false;
    s.njobs++;
    std::swap(s.inbuf, s.inbuf_alt);              // the following calls fill the other buffer
    s.fill = rest;                                // ... which holds the samples after the boundary
  }
  return 0;
}

// one launch of the cluster kernel on s_main
int rt_launch_one(b200conv* h, const pc::RtParams& P) {
#if defined(PC_EMULATE)
  pc::emu_rt_block(P);
#else
  CU_CHECK(h, rt_launch(P, P.M, P.C, P.NC, h->s_main));
#endif
  h->launches++;
  return 0;
}

// One real-time call of one handle on its s_main.  done_flag (device address of a pinned word, or nullptr): raised to
// done_val once every output sample is written.
int rt_call(b200conv* h, int nc, const float* in, size_t in_stride, float* out, size_t out_stride, size_t len,
            unsigned int* done_flag, unsigned int done_val) {
  const bool split = nc < 0;
  pc::RtParams P;
  bool waited = false;
  if (int rc = rt_prepare(h, split ? 1 : nc, in, in_stride, out, out_stride, len, h->s_main, P, &waited)) return rc;
  if (!split) {
    P.done_flag = done_flag; P.done_val = done_val;
    if (int rc = rt_launch_one(h, P)) return rc;
  } else {
    // head stage too large for one cluster: FRONT (assemble + forward FFT + timeline row), the TMA streaming sweep
    // over all SMs into Y row 1, BACK (overlap-add + inverse FFT + output) — still zero-copy I/O and no D2H/H2D
    Stage& s0 = h->stages[0];
    float2* Yb = s0.Y[s0.ybuf];
    const size_t row = (size_t)h->C * s0.B;
    P.mode = 1;
    if (int rc = rt_launch_one(h, P)) return rc;
    if (int rc = launch_cmac(h, sweep_params(s0, h->C, Yb, 1), h->C)) return rc;
    P.mode = 2; P.Yt = Yb + row;
    P.done_flag = done_flag; P.done_val = done_val;
    if (int rc = rt_launch_one(h, P)) return rc;
  }
  bool recorded = false;
  return rt_commit(h, P.len, h->ev_rt, h->s_main, &recorded);
}

// Waits until the pinned completion word *f reached `want`: spins, and after 20 ms synchronises st, the stream that
// holds the work raising it, so that a device error is reported from there.  False if the word is still not raised
// then, with *e the synchronise's error (cudaSuccess: st completed without raising it).
bool wait_word(const volatile unsigned int* f, unsigned int want, cudaStream_t st, cudaError_t* e) {
  const auto t0 = std::chrono::steady_clock::now();
  for (unsigned spins = 1; (int)(*f - want) < 0; ++spins)
    if ((spins & 0x3ff) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(20)) {
      *e = cudaStreamSynchronize(st);
      return !*e && (int)(*f - want) >= 0;
    }
  return true;
}

// b200conv_reset / b200conv_destroy of either handle of a pending IR hot swap: the live handle continues alone
void swap_cancel(b200conv* h) {
  if (!h->swap_peer) return;
  b200conv* p = h->swap_peer;
  p->swap_peer = nullptr; p->swap_state = 0; p->swap_live = false;
  h->swap_peer = nullptr; h->swap_state = 0; h->swap_live = false;
}

// make s_main wait for everything queued on s_post (end of an overlapped call)
int join_post(b200conv* h) {
  CU_CHECK(h, cudaEventRecord(h->ev_join, h->s_post));
  CU_CHECK(h, cudaStreamWaitEvent(h->s_main, h->ev_join, 0));
  return 0;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

const char* b200conv_version(void) {
#if defined(PC_EMULATE)
  return "b200conv 0.1 EMULATED-ON-CPU (tests only)";
#else
  return "b200conv 0.1 (sm_90a, hand-written Stockham FFT + register-tiled FDL sweep)";
#endif
}

b200conv_t* b200conv_create(const b200conv_config* cfg) {
  if (!cfg || cfg->n_channels < 1) return nullptr;
  b200conv* h = new (std::nothrow) b200conv();
  if (!h) return nullptr;
  h->cfg = *cfg;
  if (h->cfg.shard_count < 1) h->cfg.shard_count = 1;
  if (h->cfg.shard_rank < 0 || h->cfg.shard_rank >= h->cfg.shard_count) h->cfg.shard_rank = 0;
  h->C = cfg->n_channels;
  h->ir_len.assign(h->C, 0);
  // CUDA resources; failures are recorded and reported by the first real call
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) {
    h->err = "cudaSetDevice failed: no usable CUDA device";
    h->sticky_cuda_error = true;
    cudaGetLastError();
    return h;
  }
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
#if !defined(PC_EMULATE)
  {
    int sm = 0;
    if (cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, h->cfg.device) == cudaSuccess && sm > 0) h->n_sm = sm;
  }
#endif
  bool ok = cudaStreamCreateWithPriority(&h->s_main, cudaStreamNonBlocking, hi) == cudaSuccess;
  ok = ok && cudaStreamCreateWithPriority(&h->s_post, cudaStreamNonBlocking, hi) == cudaSuccess;
  // tail blocks have a whole tail period (8192 samples = 171 ms at 48 kHz) to finish: lowest priority, so that they
  // never delay the head-stage kernels of this or any other handle (TwoStageFFTConvolver.cpp:213-222, Convolver.cpp:84-95)
  ok = ok && cudaStreamCreateWithPriority(&h->s_tail, cudaStreamNonBlocking, lo) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&h->ev_rt, cudaEventDisableTiming) == cudaSuccess;
  h->s_launch = h->s_main;
  ok = ok && cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; i < 2 && ok; ++i) {
    ok = ok && cudaEventCreateWithFlags(&h->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&h->ev_comp[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&h->ev_d2h[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&h->ev_din[i], cudaEventDisableTiming) == cudaSuccess;
  }
#if !defined(PC_EMULATE)
  if (ok) {
    // function attributes are per device: set them once per device ordinal
    static std::once_flag once[64];
    static bool attr_ok = true;
    std::call_once(once[h->cfg.device & 63], [] {
#define PC_CASE(L) attr_ok = attr_ok && fft_set_smem_attr<L>();
      PC_FOR_EACH_LOG2(PC_CASE)
#undef PC_CASE
      attr_ok = attr_ok && stream_set_smem_attr();
      attr_ok = attr_ok && rt_set_attr<16>() && rt_set_attr<32>() && rt_set_attr<64>() && rt_set_attr<128>() &&
                rt_set_attr<256>() && rt_set_attr<512>() && rt_set_attr<1024>();
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_fwd_fft512, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512Smem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_inv_fft512<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512Smem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_inv_fft512<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512Smem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_fwd_fft512_lines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512LinesSmem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_inv_fft512<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512Smem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::k_inv_fft512<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF512Smem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::tc::k_tc_sweep, cudaFuncAttributeMaxDynamicSharedMemorySize, pc::tc::kSmemBytesGauss) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::fs::k_fs_cols, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pc::fs::kColSmem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::fs::k_fs_cols_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pc::fs::kColSmem) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::fs::k_fs_rows<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pc::fs::rows_smem<false>()) == cudaSuccess;
      attr_ok = attr_ok && cudaFuncSetAttribute(pc::fs::k_fs_rows<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pc::fs::rows_smem<true>()) == cudaSuccess;
    });
    ok = attr_ok;
    // the four-step row pass is persistent: its grid is the CTAs that fit on the device at once
    int per_sm[2] = {0, 0};
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[0], pc::fs::k_fs_rows<false>, pc::lfft::kThreads, pc::fs::rows_smem<false>()) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[1], pc::fs::k_fs_rows<true>, pc::lfft::kThreads, pc::fs::rows_smem<true>()) == cudaSuccess;
    h->fs_rows_ctas[0] = (unsigned)(per_sm[0] * h->n_sm);
    h->fs_rows_ctas[1] = (unsigned)(per_sm[1] * h->n_sm);
  }
#endif
  if (!ok) {
    h->err = std::string("CUDA resource creation failed: ") + cudaGetErrorString(cudaGetLastError());
    h->sticky_cuda_error = true;
  }
  return h;
}

void b200conv_destroy(b200conv_t* h) {
  if (!h) return;
  swap_cancel(h);
  if (!h->sticky_cuda_error || h->s_main) {
    cudaSetDevice(h->cfg.device);
    if (h->s_main) cudaStreamSynchronize(h->s_main);
    if (h->s_post) cudaStreamSynchronize(h->s_post);
    if (h->s_tail) cudaStreamSynchronize(h->s_tail);
    free_all(h);
    if (h->ev_rt) cudaEventDestroy(h->ev_rt);
    cudaFree(h->stream_ticket); h->stream_ticket = nullptr;
    if (h->s_tail) cudaStreamDestroy(h->s_tail);
    for (auto& p : h->ev_pool) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
    for (int i = 0; i < 2; ++i) {
      if (h->ev_h2d[i]) cudaEventDestroy(h->ev_h2d[i]);
      if (h->ev_comp[i]) cudaEventDestroy(h->ev_comp[i]);
      if (h->ev_d2h[i]) cudaEventDestroy(h->ev_d2h[i]);
      if (h->ev_din[i]) cudaEventDestroy(h->ev_din[i]);
    }
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->s_post) cudaStreamDestroy(h->s_post);
    if (h->s_main) cudaStreamDestroy(h->s_main);
    if (h->s_in) cudaStreamDestroy(h->s_in);
    if (h->s_out) cudaStreamDestroy(h->s_out);
  }
  delete h;
}

const char* b200conv_last_error(const b200conv_t* h) { return h ? h->err.c_str() : "null handle"; }

#define REQUIRE_CUDA(h)                                                   \
  do {                                                                    \
    if (!(h)) return B200CONV_EINVAL;                                     \
    if ((h)->sticky_cuda_error) return B200CONV_ECUDA;                    \
  } while (0)

int b200conv_init_uniform(b200conv_t* h, size_t block, const float* const* ir, const size_t* ir_len) {
  REQUIRE_CUDA(h);
  const size_t off = 0;
  return init_common(h, 1, &block, &off, ir, ir_len);
}

int b200conv_init_twostage(b200conv_t* h, size_t head_block, size_t tail_block,
                           const float* const* ir, const size_t* ir_len) {
  REQUIRE_CUDA(h);
  if (head_block == 0 || tail_block == 0) {                       // TwoStageFFTConvolver.cpp:94-97
    if (h->swap_peer) return fail(h, B200CONV_ESTATE, "an IR hot swap is pending on this handle");
    if (int rc = set_device(h)) return rc;
    cudaStreamSynchronize(h->s_main);
    free_all(h);
    return fail(h, B200CONV_EINVAL, "block size 0");
  }
  if (head_block > tail_block) std::swap(head_block, tail_block);  // :100-104
  const size_t hb = next_pow2(head_block), tb = next_pow2(tail_block);   // :117-118
  // head covers taps [0, T), tail0 (same block size as the head, :123-129) taps [T, 2T): the two
  // are one uniform stage of block hb over [0, 2T); the tail runs block T over [2T, L) (:131-138).
  const size_t blocks[2] = {hb, tb};
  const size_t offsets[2] = {0, 2 * tb};
  return init_common(h, 2, blocks, offsets, ir, ir_len);
}

int b200conv_init_stages(b200conv_t* h, int n_stages, const size_t* blocks, const size_t* offsets,
                         const float* const* ir, const size_t* ir_len) {
  REQUIRE_CUDA(h);
  if (n_stages < 1 || n_stages > 4 || !blocks || !offsets || offsets[0] != 0)
    return fail(h, B200CONV_EINVAL, "need 1..4 stages with offsets[0] == 0");
  return init_common(h, n_stages, blocks, offsets, ir, ir_len);
}

// irshape.cu (internal): shape / recalculate raw host taps into device buffers
int pc_ir_shape_to_device(int device, const float* const* raw, int C, size_t n, const b200conv_ir_shape_params* sp,
                          float** dev_out, size_t* out_len, size_t* trimmed);
int pc_ir_recalc_to_device(int device, const float* const* raw, int C, size_t n, const b200conv_ir_recalc_params* p,
                           float** dev_out, size_t* out_len, size_t* trimmed);
void pc_ir_shape_free(float** dev_out, int C);

// exactly one of sp (b200conv_init_*_shaped) and rp (b200conv_init_*_recalc) is set
static int init_shaped(b200conv_t* h, int n_stages, const size_t* blocks, const size_t* offsets,
                       const float* const* raw, size_t n, const b200conv_ir_shape_params* sp,
                       const b200conv_ir_recalc_params* rp = nullptr) {
  if (!raw || (!sp && !rp)) return fail(h, B200CONV_EINVAL, "null argument");
  if (h->swap_peer) return fail(h, B200CONV_ESTATE, "an IR hot swap is pending on this handle");
  if (h->C < 2 || h->C > 8) return fail(h, B200CONV_ESTATE, "IR shaping works on 2..8 channel handles (LL, RR[, LR, RL])");
  float* dev[8] = {};
  size_t m = 0, trimmed[8] = {}, lens[8] = {};
  if (int rc = sp ? pc_ir_shape_to_device(h->cfg.device, raw, h->C, n, sp, dev, &m, trimmed)
                  : pc_ir_recalc_to_device(h->cfg.device, raw, h->C, n, rp, dev, &m, trimmed))
    return fail(h, rc, "IR shaping on the device failed");
  for (int c = 0; c < h->C; ++c) lens[c] = m;
  h->ir_on_device = true; h->ir_trimmed = trimmed;
  const int rc = init_common(h, n_stages, blocks, offsets, dev, lens);
  h->ir_on_device = false; h->ir_trimmed = nullptr;
  pc_ir_shape_free(dev, h->C);
  return rc;
}

int b200conv_init_uniform_shaped(b200conv_t* h, size_t block, const float* const* raw, size_t n, const b200conv_ir_shape_params* sp) {
  REQUIRE_CUDA(h);
  const size_t off = 0;
  return init_shaped(h, 1, &block, &off, raw, n, sp);
}

int b200conv_init_twostage_shaped(b200conv_t* h, size_t head_block, size_t tail_block, const float* const* raw, size_t n,
                                  const b200conv_ir_shape_params* sp) {
  REQUIRE_CUDA(h);
  if (head_block == 0 || tail_block == 0) return fail(h, B200CONV_EINVAL, "block size 0");
  if (head_block > tail_block) std::swap(head_block, tail_block);
  const size_t hb = next_pow2(head_block), tb = next_pow2(tail_block);
  const size_t blocks[2] = {hb, tb};
  const size_t offsets[2] = {0, 2 * tb};
  return init_shaped(h, 2, blocks, offsets, raw, n, sp);
}

int b200conv_init_uniform_recalc(b200conv_t* h, size_t block, const float* const* raw, size_t n, const b200conv_ir_recalc_params* p) {
  REQUIRE_CUDA(h);
  const size_t off = 0;
  return init_shaped(h, 1, &block, &off, raw, n, nullptr, p);
}

int b200conv_init_twostage_recalc(b200conv_t* h, size_t head_block, size_t tail_block, const float* const* raw, size_t n,
                                  const b200conv_ir_recalc_params* p) {
  REQUIRE_CUDA(h);
  if (head_block == 0 || tail_block == 0) return fail(h, B200CONV_EINVAL, "block size 0");
  if (head_block > tail_block) std::swap(head_block, tail_block);
  const size_t hb = next_pow2(head_block), tb = next_pow2(tail_block);
  const size_t blocks[2] = {hb, tb};
  const size_t offsets[2] = {0, 2 * tb};
  return init_shaped(h, 2, blocks, offsets, raw, n, nullptr, p);
}

int b200conv_process_device(b200conv_t* h, const float* in_dev, size_t in_stride,
                            float* out_dev, size_t out_stride, size_t len, int sync) {
  REQUIRE_CUDA(h);
  if (h->lat_D) return fail(h, B200CONV_ESTATE, "device-pointer calls are not available in fixed-latency mode");
  if (int rc = set_device(h)) return rc;
  if (h->timing) h->ev_used = 0;
  if (h->stages.empty()) {      // no IR: zeros (FFTConvolver.cpp:157-161)
    if (len) CU_CHECK(h, cudaMemset2DAsync(out_dev, out_stride * sizeof(float), 0, len * sizeof(float),
                                           h->route_on ? h->n_out : h->C, h->s_main));
  } else {
    const size_t B0 = h->stages[0].B;
    const size_t chunk = h->Lmax - B0;     // keeps fill + n <= Lmax for every stage (inbuf holds B + Lmax samples)
    const bool overlap = len > chunk || h->cfg.shard_count > 1;    // (slot-exchange groups always use s_post)
    size_t done = 0;
    if (const int nc = rt_cluster_ctas(h, len)) {       // a call of at most one head block: one cluster kernel
      if (int rc = rt_call(h, nc, in_dev, in_stride, out_dev, out_stride, len, nullptr, 0)) return rc;
      done = len;
    }
    while (done < len) {
      size_t n = std::min(len - done, chunk);
      if (int rc = run_group(h, in_dev + done, in_stride, out_dev + done, out_stride, n, overlap)) return rc;
      done += n;
    }
    if (overlap) { if (int rc = join_post(h)) return rc; }
  }
  if (sync || h->timing) {
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    if (h->timing) timing_collect(h);
    if (int rc = p2p_check(h)) return rc;
  }
  return B200CONV_OK;
}

// Host -> device staging of one launch group (n samples per channel from in[c] + off into din[b], channel pitch
// `pitch`) on stream st.  With the slot exchange's input broadcast only shard 0 touches PCIe: it uploads the
// group, stores it into every peer's din[b] over NVLink and an "input landed" flag barrier releases the peers.
// Launch-group sizes of a pipelined host-pointer call: the H2D copy of the FIRST group and the D2H copy of the LAST one
// cannot overlap with compute, so the sequence ramps up from one sweep wave (w, 2w, 4w, ...), runs steady groups of
// `grp` samples and ramps down again; every group but the last is a whole number of waves / 64-block tiles, the last
// one carries whatever is left (incl. a ragged tail).
// Long calls are split into groups so that the PCIe copies overlap with compute: only the first group's H2D
// and the last group's D2H are exposed, so aim for ~`parts` groups — but keep every group a whole number of
// sweep WAVES (n_sm x 3 CTAs x 64 blocks per CTA over ceil(B/32) x C tile columns), otherwise a
// partially filled last wave costs more than the overlap gains.  `cap` is the staging capacity; the steady group
// size goes to *grp_out.
static std::vector<size_t> ramped_groups(const b200conv_t* h, size_t B, size_t len, size_t parts, size_t cap,
                                         size_t* grp_out = nullptr) {
  const size_t tile = B * 64;
  const size_t cols = (size_t)((B + 31) / 32) * (size_t)h->C;
  size_t wave = ((size_t)h->n_sm * 3 * 64 + cols - 1) / cols * B;       // samples per full wave
  wave = std::max(tile, wave / tile * tile);
  size_t grp = std::max(wave, (len / parts) / wave * wave);
  grp = std::min(grp, cap >= tile ? cap / tile * tile : cap);
  if (grp_out) *grp_out = grp;
  std::vector<size_t> g, up;
  size_t tot = 0;
  for (size_t r = wave; r * 2 <= grp && 2 * (tot + r) + 2 * grp <= len; r *= 2) { up.push_back(r); tot += r; }
  size_t remaining = len;
  for (size_t r : up) { g.push_back(r); remaining -= r; }
  while (remaining > tot + grp) { g.push_back(grp); remaining -= grp; }
  if (!up.empty()) {
    const size_t mid = (remaining - tot) / tile * tile;
    if (mid) { g.push_back(mid); remaining -= mid; }
    for (size_t i = up.size(); i-- > 1;) { g.push_back(up[i]); remaining -= up[i]; }
  }
  if (remaining) g.push_back(remaining);
  std::vector<size_t> out;                      // no group above the staging capacity
  for (size_t v : g) { while (v > cap) { out.push_back(cap); v -= cap; } if (v) out.push_back(v); }
  return out;
}

static int stage_input(b200conv_t* h, int b, const float* const* in, size_t off, size_t n, size_t pitch, int Cin,
                       const float* packed_src, cudaStream_t st) {
  const bool bc = h->p2p_on && h->bcast_in;
  if (!bc || h->cfg.shard_rank == 0) {
    if (packed_src) {
      CU_CHECK(h, cudaMemcpyAsync(h->din[b], packed_src, (size_t)Cin * n * sizeof(float), cudaMemcpyHostToDevice, st));
    } else {
      for (int c = 0; c < Cin; ++c)
        CU_CHECK(h, cudaMemcpyAsync(h->din[b] + (size_t)c * pitch, in[c] + off, n * sizeof(float), cudaMemcpyHostToDevice, st));
    }
  }
  if (bc) {
    if (h->cfg.shard_rank == 0) {
      // the peers read din[b] in the forward FFT of the group two exchange groups ago: its first barrier has passed
      CU_CHECK(h, cudaStreamWaitEvent(st, h->ev_b1[h->xgrp & 1], 0));
      for (int r = 1; r < h->cfg.shard_count; ++r)
        if (int rc = copy_rows_kernel(h, h->peer_din[r][b], pitch, h->din[b], pitch, n, Cin, st)) return rc;
    }
    if (int rc = p2p_barrier(h, st, 1)) return rc;
  }
  return 0;
}

static int process_impl(b200conv_t* h, const float* const* in, float* const* out_user, size_t len) {
  REQUIRE_CUDA(h);
  if (len == 0) return B200CONV_OK;
  if (!in) return fail(h, B200CONV_EINVAL, "null buffer");
  // only shard 0 of a sharded handle produces audio; the other shards leave `out` untouched (no D2H, and
  // no host memset either: that would cost more than the whole step on the throughput path)
  float* const* out = (out_user && h->cfg.shard_rank != 0) ? nullptr : out_user;
  if (int rc = set_device(h)) return rc;
  if (h->timing) h->ev_used = 0;
  const int C = h->C;
  const int Cin = h->route_on ? h->n_in : C, Cout = h->route_on ? h->n_out : C;
  if (h->stages.empty()) {
    if (out) for (int c = 0; c < Cout; ++c) std::memset(out[c], 0, len * sizeof(float));
    return B200CONV_OK;
  }
  const size_t B0 = h->stages[0].B;
  const size_t chunk = h->Lmax - B0;
  if (len <= chunk && len <= std::max((size_t)64 * B0, (size_t)16384)) {
    if (const int nc = (len <= h->hpin_cap && h->hpin_in_dev && h->hpin_out_dev) ? rt_cluster_ctas(h, len) : 0) {
      // real-time path: the cluster kernel reads the samples straight from the pinned staging buffer and writes the
      // result into it (zero-copy over PCIe): one launch + one synchronise per call
      for (int c = 0; c < Cin; ++c) std::memcpy(h->hpin_in + (size_t)c * len, in[c], len * sizeof(float));
      if (int rc = rt_call(h, nc, h->hpin_in_dev, len, h->hpin_out_dev, len, len, h->hflag_dev,
                           h->hflag_dev ? ++h->flag_epoch : 0)) return rc;
      // wait for the kernel's completion word (set after all output stores) instead of the driver's stream
      // synchronise; wait_word falls back to the synchronise (and its error report)
      cudaError_t e = cudaSuccess;
      if (!h->hflag_dev) e = cudaStreamSynchronize(h->s_main);
      else wait_word(h->hflag, h->flag_epoch, h->s_main, &e);
      if (e) return cuda_fail(h, e, "cudaStreamSynchronize(h->s_main)");
      h->main_unsynced = false;           // the kernel was the last work on s_main
      if (out)
        for (int c = 0; c < Cout; ++c) std::memcpy(out[c], h->hpin_out + (size_t)c * len, len * sizeof(float));
      if (h->p2p_tail && h->rt_tail_joined) {     // a tail block's barrier has run: did it give up on a peer?
        h->rt_tail_joined = false;
        return p2p_check(h);
      }
      return B200CONV_OK;
    }
    // latency path: one stream, one group; all channels travel in ONE pinned H2D and ONE D2H copy
    // (channel pitch = len), which matters for the 2-4 channel handles of a StereoConvolver
    const bool packed = len <= h->hpin_cap;
    const size_t pitch = packed ? len : h->Lmax;
    const bool uploads = !(h->p2p_on && h->bcast_in) || h->cfg.shard_rank == 0;
    if (packed && uploads)
      for (int c = 0; c < Cin; ++c) std::memcpy(h->hpin_in + (size_t)c * len, in[c], len * sizeof(float));
    if (int rc = stage_input(h, 0, in, 0, len, pitch, Cin, packed ? h->hpin_in : nullptr, h->s_main)) return rc;
    const bool ov = h->cfg.shard_count > 1;
    if (int rc = run_group(h, h->din[0], pitch, h->dout[0], pitch, len, ov)) return rc;
    if (ov) { if (int rc = join_post(h)) return rc; }
    if (out) {
      if (packed) {
        CU_CHECK(h, cudaMemcpyAsync(h->hpin_out, h->dout[0], (size_t)Cout * len * sizeof(float), cudaMemcpyDeviceToHost, h->s_main));
      } else {
        for (int c = 0; c < Cout; ++c)
          CU_CHECK(h, cudaMemcpyAsync(out[c], h->dout[0] + (size_t)c * h->Lmax, len * sizeof(float), cudaMemcpyDeviceToHost, h->s_main));
      }
    }
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    if (out && packed)
      for (int c = 0; c < Cout; ++c) std::memcpy(out[c], h->hpin_out + (size_t)c * len, len * sizeof(float));
    return p2p_check(h);
  }
  // throughput path: H2D / compute / D2H of successive groups overlap on three streams
  size_t done = 0;
  int i = 0;
  const std::vector<size_t> groups = ramped_groups(h, B0, len, 8, chunk);
  for (size_t gi = 0; gi < groups.size() && done < len; ++gi, ++i) {
    const int b = i & 1;
    const size_t n = std::min(len - done, groups[gi]);
    if (i >= 2) CU_CHECK(h, cudaStreamWaitEvent(h->s_in, h->ev_din[b], 0));     // din[b] free again
    if (int rc = stage_input(h, b, in, done, n, h->Lmax, Cin, nullptr, h->s_in)) return rc;
    CU_CHECK(h, cudaEventRecord(h->ev_h2d[b], h->s_in));
    CU_CHECK(h, cudaStreamWaitEvent(h->s_main, h->ev_h2d[b], 0));
    if (i >= 2) CU_CHECK(h, cudaStreamWaitEvent(h->s_post, h->ev_d2h[b], 0));    // dout[b] drained
    if (int rc = run_group(h, h->din[b], h->Lmax, h->dout[b], h->Lmax, n, true)) return rc;
    CU_CHECK(h, cudaEventRecord(h->ev_din[b], h->s_main));    // every read of din[b] is queued on s_main
    CU_CHECK(h, cudaEventRecord(h->ev_comp[b], h->s_post));    // dout[b] complete
    CU_CHECK(h, cudaStreamWaitEvent(h->s_out, h->ev_comp[b], 0));
    if (out)
      for (int c = 0; c < Cout; ++c)
        CU_CHECK(h, cudaMemcpyAsync(out[c] + done, h->dout[b] + (size_t)c * h->Lmax, n * sizeof(float), cudaMemcpyDeviceToHost, h->s_out));
    CU_CHECK(h, cudaEventRecord(h->ev_d2h[b], h->s_out));
    done += n;
  }
  CU_CHECK(h, cudaStreamSynchronize(h->s_out));
  if (int rc = join_post(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return p2p_check(h);
}

// ---- fixed-latency mode (b200conv_set_latency) ---------------------------------------------------------------------
// the completion word of a step that ran as several launches and copies, queued behind them on st
static int launch_seq_flag(b200conv_t* h, unsigned int* flag, unsigned int v, cudaStream_t st) {
#if defined(PC_EMULATE)
  (void)st;
  pc::emu_seq_flag(flag, v);
#else
  pc::k_seq_flag<<<1, 1, 0, st>>>(flag, v);
  CU_CHECK(h, cudaGetLastError());
#endif
  h->launches++;
  return 0;
}

// Waits until ring r's sequence word reached `want`, with the stream of the ring's last step behind wait_word's
// fallback (every earlier step is ordered before it).  *waited: a wait was needed.
static int lat_wait(b200conv_t* h, LatRing* r, unsigned int want, bool* waited) {
  const volatile unsigned int* f = r->word;
  if ((int)(*f - want) >= 0) return 0;
  *waited = true;
  cudaError_t e = cudaSuccess;
  if (wait_word(f, want, r->last_st, &e)) return 0;
  if (e) return cuda_fail(h, e, "cudaStreamSynchronize(r->last_st)");
  return fail(h, B200CONV_ECUDA, "a fixed-latency step did not raise its completion word");
}

// A call in fixed-latency mode runs in passes of at most r->piece samples.  Input half of a pass of n samples, samples
// [done, done + n) of the call: waits until the ring slots the pass writes are free, copies the samples into the input
// ring (in[i] == nullptr: row i reads 1) and moves r->pos past them.
static int lat_in(b200conv_t* h, LatRing* r, const float* const* in, int n_in, size_t done, long long n, bool* waited) {
  const long long B = (long long)r->B, L = (long long)r->len, NS = (long long)r->nslots;
  const long long p0 = r->pos;
  // the slots this pass writes are free once the steps that last read them completed
  for (long long k = p0 / B; k <= (p0 + n - 1) / B; ++k)
    if (int rc = lat_wait(h, r, r->slot_seq[k % NS], waited)) return rc;
  for (long long p = p0; p < p0 + n;) {
    const long long i = p % L, seg = std::min(p0 + n - p, L - i);
    for (int c = 0; c < n_in; ++c) {
      float* dst = r->in + (size_t)c * L + i;
      if (in[c]) std::memcpy(dst, in[c] + done + (p - p0), (size_t)seg * sizeof(float));
      else std::fill(dst, dst + seg, 1.0f);
    }
    p += seg;
  }
  r->pos = p0 + n;
  return 0;
}

// Output half of the pass whose input began at ring position p0: the output ring read D samples behind the input, into
// samples [done, done + n) of the call; output before sample 0 is zero.  Every block it reads has been enqueued by
// the pass's steps, since D >= B; it waits only for one that has not completed.
static int lat_out(b200conv_t* h, LatRing* r, float* const* out, int n_out, size_t done, long long p0, long long n,
                   bool* waited) {
  const long long B = (long long)r->B, D = (long long)h->lat_D, L = (long long)r->len, NS = (long long)r->nslots;
  const long long q0 = p0 - D, q1 = p0 + n - D;
  for (long long q = q0; q < q1;) {
    const size_t o = done + (size_t)(q - q0);
    if (q < 0) {
      const long long z = std::min(q1, 0LL) - q;
      for (int c = 0; c < n_out; ++c) std::memset(out[c] + o, 0, (size_t)z * sizeof(float));
      q += z;
      continue;
    }
    const long long k = q / B, slot = k % NS, seg = std::min(q1, (k + 1) * B) - q;
    if (int rc = lat_wait(h, r, r->slot_seq[slot], waited)) return rc;
    for (int c = 0; c < n_out; ++c)
      std::memcpy(out[c] + o, r->out + (size_t)c * L + (size_t)(slot * B + (q - k * B)), (size_t)seg * sizeof(float));
    q += seg;
  }
  return 0;
}

// One call in fixed-latency mode: per pass the input half, one step(k, v) with sequence value v per head block k the
// pass completes (a group call runs these steps in shared launches instead), and the output half.
extern "C++" {
template <class Step>
static int lat_run(b200conv_t* h, LatRing* r, const float* const* in, int n_in, float* const* out, int n_out, size_t len,
                   Step step) {
  const long long B = (long long)r->B, NS = (long long)r->nslots;
  bool waited = false;                                     // a call that waited counts once in latency_waits
  struct Count { b200conv_t* h; const bool& w; ~Count() { if (w) h->lat_waits++; } } count{h, waited};
  for (size_t done = 0; done < len;) {
    const long long n = (long long)std::min(len - done, r->piece);
    const long long p0 = r->pos;
    if (int rc = lat_in(h, r, in, n_in, done, n, &waited)) return rc;
    for (long long k = p0 / B; k < (p0 + n) / B; ++k) {      // one step per completed head block
      const unsigned int v = ++r->seq;
      if (int rc = step(k, v)) return rc;
      r->slot_seq[k % NS] = v;
    }
    if (int rc = lat_out(h, r, out, n_out, done, p0, n, &waited)) return rc;
    done += (size_t)n;
  }
  return 0;
}
}  // extern "C++"

// Head block k of a b200conv_process call in fixed-latency mode: exactly the zero-latency step of a call of B0 samples.
// One k_rt_block launch reading the input slot and writing the output slot zero-copy when the shape allows it (its
// completion word carries v), otherwise the launch-group path through the staging buffers, then the flag kernel.
static int lat_step(b200conv_t* h, long long k, unsigned int v) {
  LatRing* r = h->lat;
  const size_t B = r->B, L = r->len, off = (size_t)(k % (long long)r->nslots) * B;
  const int Cin = h->route_on ? h->n_in : h->C, Cout = h->route_on ? h->n_out : h->C;
  r->last_st = h->s_main;
  if (const int nc = (h->hpin_in_dev && h->hpin_out_dev) ? rt_cluster_ctas(h, B) : 0)
    return rt_call(h, nc, r->in_dev + off, L, r->out_dev + off, L, B, r->word_dev, v);
  CU_CHECK(h, cudaMemcpy2DAsync(h->din[0], B * sizeof(float), r->in + off, L * sizeof(float), B * sizeof(float), Cin,
                                cudaMemcpyHostToDevice, h->s_main));
  if (int rc = run_group(h, h->din[0], B, h->dout[0], B, B, false)) return rc;
  CU_CHECK(h, cudaMemcpy2DAsync(r->out + off, L * sizeof(float), h->dout[0], B * sizeof(float), B * sizeof(float), Cout,
                                cudaMemcpyDeviceToHost, h->s_main));
  return launch_seq_flag(h, r->word_dev, v, h->s_main);
}

static int process_latency(b200conv_t* h, const float* const* in, float* const* out, size_t len) {
  REQUIRE_CUDA(h);
  if (len == 0) return B200CONV_OK;
  const int Cin = h->route_on ? h->n_in : h->C, Cout = h->route_on ? h->n_out : h->C;
  if (!in) return fail(h, B200CONV_EINVAL, "null buffer");
  for (int c = 0; c < Cin; ++c)
    if (!in[c]) return fail(h, B200CONV_EINVAL, "null buffer");
  if (int rc = set_device(h)) return rc;
  if (h->timing) h->ev_used = 0;
  return lat_run(h, h->lat, in, Cin, out, Cout, len, [h](long long k, unsigned int v) { return lat_step(h, k, v); });
}

int b200conv_process(b200conv_t* h, const float* const* in, float* const* out, size_t len) {
  if (h && len && !out) return fail(h, B200CONV_EINVAL, "null buffer");
  if (h && h->lat_D) return process_latency(h, in, out, len);
  return process_impl(h, in, out, len);
}

int b200conv_prime(b200conv_t* h, const float* const* in, size_t len) {
  if (h && h->lat_D) return fail(h, B200CONV_ESTATE, "b200conv_prime is not available in fixed-latency mode");
  return process_impl(h, in, nullptr, len);
}

int b200conv_process_device_sliced(b200conv_t* h, const float* in_dev, size_t in_stride, float* out_dev, size_t out_stride,
                                   size_t len, int slice_rank, int slice_count, int sync) {
  REQUIRE_CUDA(h);
  if (h->lat_D) return fail(h, B200CONV_ESTATE, "time-slice calls are not available in fixed-latency mode");
  if (int rc = set_device(h)) return rc;
  if (h->timing) h->ev_used = 0;
  if (h->stages.empty()) {
    if (len) CU_CHECK(h, cudaMemset2DAsync(out_dev, out_stride * sizeof(float), 0, len * sizeof(float), h->C, h->s_main));
  } else {
    SlicePlan sp;
    if (int rc = plan_slice(h, len, slice_rank, slice_count, &sp)) return rc;
    Stage& s = h->stages[0];
    const size_t B = (size_t)s.B;
    const long long done0 = s.blocks_done, pos0 = h->abs_pos;
    if (int rc = advance_fft_only(h, in_dev + (size_t)sp.lo * B, in_stride, sp.a - sp.lo)) return rc;
    const size_t chunk = (h->Lmax - B) / B * B;
    const size_t n_slice = (size_t)(sp.b - sp.a) * B;
    const bool overlap = n_slice > chunk;
    for (size_t done = 0; done < n_slice;) {
      const size_t n = std::min(n_slice - done, chunk);
      const size_t off = (size_t)sp.a * B + done;
      if (int rc = run_group(h, in_dev + off, in_stride, out_dev + off, out_stride, n, overlap)) return rc;
      done += n;
    }
    if (overlap) { if (int rc = join_post(h)) return rc; }
    if (int rc = advance_fft_only(h, in_dev + (size_t)sp.tail_lo * B, in_stride, sp.T - sp.tail_lo)) return rc;
    s.blocks_done = done0 + sp.T;               // the state is that of the whole call
    h->abs_pos = pos0 + (long long)len;
  }
  if (sync || h->timing) {
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    if (h->timing) timing_collect(h);
  }
  return B200CONV_OK;
}

int b200conv_process_sliced(b200conv_t* h, const float* const* in, float* const* out, size_t len, int slice_rank, int slice_count) {
  REQUIRE_CUDA(h);
  if (h->lat_D) return fail(h, B200CONV_ESTATE, "time-slice calls are not available in fixed-latency mode");
  if (len == 0) return B200CONV_OK;
  if (!in || !out) return fail(h, B200CONV_EINVAL, "null buffer");
  if (int rc = set_device(h)) return rc;
  if (h->timing) h->ev_used = 0;
  const int C = h->C;
  if (h->stages.empty()) {                      // no IR: zeros (FFTConvolver.cpp:157-161); every GPU writes the same value
    for (int c = 0; c < C; ++c) std::memset(out[c], 0, len * sizeof(float));
    return B200CONV_OK;
  }
  SlicePlan sp;
  if (int rc = plan_slice(h, len, slice_rank, slice_count, &sp)) return rc;
  Stage& s = h->stages[0];
  const size_t B = (size_t)s.B;
  const long long done0 = s.blocks_done, pos0 = h->abs_pos;
  // pieces of at most `grp` samples, each one H2D -> (forward FFTs | full group) -> D2H, pipelined over the three
  // streams like b200conv_process: [lo, a) and [tail_lo, T) are transformed only, [a, b) is convolved
  const size_t chunk = (h->Lmax - B) / B * B;
  const size_t n_slice = (size_t)(sp.b - sp.a) * B;
  size_t grp = 0;
  const std::vector<size_t> slice_groups = ramped_groups(h, B, n_slice, 4, chunk, &grp);
  struct Piece { size_t off, n; bool conv; };
  std::vector<Piece> pieces;
  auto add = [&](long long b0, long long b1, bool conv) {
    for (size_t o = (size_t)b0 * B, e = (size_t)b1 * B; o < e; o += grp) pieces.push_back({o, std::min(grp, e - o), conv});
  };
  add(sp.lo, sp.a, false);
  {   // the slice itself: ramped groups (short first H2D, short last D2H)
    size_t o = (size_t)sp.a * B;
    for (size_t gsz : slice_groups) { pieces.push_back({o, gsz, true}); o += gsz; }
  }
  add(sp.tail_lo, sp.T, false);
  int i = 0;
  bool used_out[2] = {false, false};
  for (const Piece& pc_ : pieces) {
    const int b = i & 1;
    if (i >= 2) CU_CHECK(h, cudaStreamWaitEvent(h->s_in, h->ev_din[b], 0));
    for (int c = 0; c < C; ++c)
      CU_CHECK(h, cudaMemcpyAsync(h->din[b] + (size_t)c * h->Lmax, in[c] + pc_.off, pc_.n * sizeof(float), cudaMemcpyHostToDevice, h->s_in));
    CU_CHECK(h, cudaEventRecord(h->ev_h2d[b], h->s_in));
    CU_CHECK(h, cudaStreamWaitEvent(h->s_main, h->ev_h2d[b], 0));
    if (!pc_.conv) {
      if (int rc = advance_fft_only(h, h->din[b], h->Lmax, (long long)(pc_.n / B))) return rc;
      CU_CHECK(h, cudaEventRecord(h->ev_din[b], h->s_main));
    } else {
      if (used_out[b]) CU_CHECK(h, cudaStreamWaitEvent(h->s_post, h->ev_d2h[b], 0));
      if (int rc = run_group(h, h->din[b], h->Lmax, h->dout[b], h->Lmax, pc_.n, true)) return rc;
      CU_CHECK(h, cudaEventRecord(h->ev_din[b], h->s_main));
      CU_CHECK(h, cudaEventRecord(h->ev_comp[b], h->s_post));
      CU_CHECK(h, cudaStreamWaitEvent(h->s_out, h->ev_comp[b], 0));
      for (int c = 0; c < C; ++c)
        CU_CHECK(h, cudaMemcpyAsync(out[c] + pc_.off, h->dout[b] + (size_t)c * h->Lmax, pc_.n * sizeof(float), cudaMemcpyDeviceToHost, h->s_out));
      CU_CHECK(h, cudaEventRecord(h->ev_d2h[b], h->s_out));
      used_out[b] = true;
    }
    ++i;
  }
  CU_CHECK(h, cudaStreamSynchronize(h->s_out));
  if (int rc = join_post(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  s.blocks_done = done0 + sp.T;
  h->abs_pos = pos0 + (long long)len;
  return B200CONV_OK;
}

int b200conv_register_host(void* p, size_t bytes) {
#if defined(PC_EMULATE)
  (void)p; (void)bytes;
  return B200CONV_OK;
#else
  if (cudaHostRegister(p, bytes, cudaHostRegisterPortable) != cudaSuccess) { cudaGetLastError(); return B200CONV_ECUDA; }
  return B200CONV_OK;
#endif
}

int b200conv_unregister_host(void* p) {
#if defined(PC_EMULATE)
  (void)p;
  return B200CONV_OK;
#else
  if (cudaHostUnregister(p) != cudaSuccess) { cudaGetLastError(); return B200CONV_ECUDA; }
  return B200CONV_OK;
#endif
}

int b200conv_process_xfade(b200conv_t* ho, b200conv_t* hn, const float* const* in, float* const* out,
                           size_t len, float alpha0, float alpha_step) {
  REQUIRE_CUDA(ho);
  REQUIRE_CUDA(hn);
  if (ho->lat_D || hn->lat_D) return fail(hn, B200CONV_ESTATE, "b200conv_process_xfade is not available in fixed-latency mode");
  if (len == 0) return B200CONV_OK;
  if (!in || !out) return fail(hn, B200CONV_EINVAL, "null buffer");
  if (ho == hn || ho->cfg.device != hn->cfg.device || ho->C != hn->C || ho->route_on != hn->route_on ||
      (ho->route_on && (ho->n_in != hn->n_in || ho->n_out != hn->n_out)) ||
      ho->cfg.shard_count > 1 || hn->cfg.shard_count > 1)
    return fail(hn, B200CONV_EINVAL, "crossfade needs two different unsharded handles with the same device, channels and routing");
  if (int rc = set_device(hn)) return rc;
  const int C = hn->C;
  const int Cin = hn->route_on ? hn->n_in : C, Cout = hn->route_on ? hn->n_out : C;
  if (ho->stages.empty() || hn->stages.empty()) {   // one side has no IR: its output is silence
    b200conv_t* live = ho->stages.empty() ? hn : ho;
    if (int rc = process_impl(live, in, out, len)) return rc;
    for (int c = 0; c < Cout; ++c)
      for (size_t i = 0; i < len; ++i) {
        const float al = std::fmin(1.0f, std::fmax(0.0f, alpha0 + alpha_step * (float)i));
        out[c][i] *= (live == hn) ? al : (1.0f - al);
      }
    return B200CONV_OK;
  }
#if !defined(PC_EMULATE)
  if (ho->Lmax != hn->Lmax) return fail(hn, B200CONV_EINVAL, "crossfade needs equal staging sizes (same head block and batch size)");
#endif
  if (ho->timing) ho->ev_used = 0;
  if (hn->timing) hn->ev_used = 0;
  const size_t chunk = std::min(ho->Lmax - ho->stages[0].B, hn->Lmax - hn->stages[0].B);
  for (size_t done = 0; done < len;) {
    const size_t n = std::min(len - done, chunk);
    // input once (old handle's staging), both convolvers read it
    for (int c = 0; c < Cin; ++c)
      CU_CHECK(ho, cudaMemcpyAsync(ho->din[0] + (size_t)c * ho->Lmax, in[c] + done, n * sizeof(float), cudaMemcpyHostToDevice, ho->s_main));
    CU_CHECK(ho, cudaEventRecord(ho->ev_h2d[0], ho->s_main));
    if (int rc = run_group(ho, ho->din[0], ho->Lmax, ho->dout[0], ho->Lmax, n, false)) return rc;
    CU_CHECK(ho, cudaEventRecord(ho->ev_comp[0], ho->s_main));
    CU_CHECK(hn, cudaStreamWaitEvent(hn->s_main, ho->ev_h2d[0], 0));
    if (int rc = run_group(hn, ho->din[0], ho->Lmax, hn->dout[0], hn->Lmax, n, false)) return rc;
    CU_CHECK(hn, cudaStreamWaitEvent(hn->s_main, ho->ev_comp[0], 0));
    const float a0 = alpha0 + alpha_step * (float)done;
#if defined(PC_EMULATE)
    for (int c = 0; c < Cout; ++c)
      for (size_t i = 0; i < n; ++i) {
        const float al = std::fmin(1.0f, std::fmax(0.0f, a0 + alpha_step * (float)i));
        float* d = hn->dout[0] + (size_t)c * hn->Lmax + i;
        *d = (1.0f - al) * ho->dout[0][(size_t)c * ho->Lmax + i] + al * *d;
      }
#else
    dim3 grid((unsigned)((n + 255) / 256), Cout, 1);
    pc::k_xfade<<<grid, 256, 0, hn->s_main>>>(hn->dout[0], ho->dout[0], hn->dout[0], (long long)hn->Lmax, (long long)n, a0, alpha_step);
    hn->launches++;
    CU_CHECK(hn, cudaGetLastError());
#endif
    for (int c = 0; c < Cout; ++c)
      CU_CHECK(hn, cudaMemcpyAsync(out[c] + done, hn->dout[0] + (size_t)c * hn->Lmax, n * sizeof(float), cudaMemcpyDeviceToHost, hn->s_main));
    CU_CHECK(hn, cudaStreamSynchronize(hn->s_main));
    done += n;
  }
  return B200CONV_OK;
}

// ---- send / wet chain (SURVEY 8f-4 + the rest of 8f-1) ------------------------------------------------------------
namespace {
// Filter::getCoeff (src/dsp/Filter.h:40-44): tan() through the reference's 2048-point lookup table with its cubic
// interpolation (src/dsp/Filter.h:28-36, src/dsp/Utils.h:50-112) — the coefficient has to be the reference's, bit for bit
float chain_coeff(float freq, float srate) {
  static float lut[2048];
  static std::once_flag once;
  std::call_once(once, [] {
    const float pi = 3.14159265358979323846f;
    for (int i = 0; i < 2048; ++i) {
      const float x = (float)i / 2047.0f;
      float mapped = 0.0f + x * (0.5f - 0.0f);
      mapped = std::min(std::max(mapped, 0.0f), 0.5f);
      const float max_rads = 0.499f * pi, scaled = mapped * pi;
      lut[i] = std::tan(std::min(max_rads, scaled));
    }
  });
  freq = std::min(std::max(freq, 20.0f), srate * 0.48f);
  float ratio = std::min(std::max(freq / srate, 0.0f), 0.5f);
  const float scaler = 2047.0f / 0.5f;
  const float index = ratio * scaler + 0.0f;
  const int i = (int)index;
  const float t = index - (float)i;
  const int i0 = std::max(0, i - 1), i1 = i, i2 = std::min(2047, i + 1), i3 = std::min(2047, i + 2);
  const float y0 = lut[i0], y1 = lut[i1], y2 = lut[i2], y3 = lut[i3];
  const float a0 = y3 - y2 - y0 + y1, a1 = y0 - y1 - a0, a2 = y2 - y0, a3 = y1;
  return (a0 * t * t * t) + (a1 * t * t) + (a2 * t) + a3;
}

// samples per channel of the reference's warmer ring, (int)ceil(srate) / 4 (src/PluginProcessor.cpp:610)
size_t chain_warmer_len(double srate) { return (size_t)((long long)std::ceil(srate) / 4); }

// threads of k_chain_send for n samples: two passes of n/T sequential samples (~200 cycles each) + a serial scan of T
// 8x8 matrix-vector steps (~256 cycles each): T ~ sqrt(1.5 n), a power of two in [8, 1024]
int chain_send_threads(size_t n) {
  int T = 8;
  while (T < 1024 && (size_t)T * T < n + n / 2) T *= 2;
  return T;
}

int launch_chain_send(b200conv* h, const pc::ChainSendParams& sp, cudaStream_t st) {
  const int T = chain_send_threads((size_t)sp.n);
#if defined(PC_EMULATE)
  (void)st;
  pc::emu_chain_send(sp, T);
#else
  pc::k_chain_send<<<2, T, 0, st>>>(sp);
  CU_CHECK(h, cudaGetLastError());
#endif
  h->launches++;
  return 0;
}

// Device-pointer pieces of at least this many samples run the whole-GPU send form (kernels_chain.cuh
// k_chain_wide_*), shorter ones k_chain_send exactly as the host entry does.  See DESIGN §4 for the measurement.
constexpr size_t kChainWideMin = 16384;

// the whole-GPU form's scratch inside one allocation of chain_wide_bytes(Lmax): P_j, aggregates, carries, Z_c
size_t chain_wide_bytes(size_t Lmax) {
  const size_t nb = (size_t)pc::chain_wide_ctas((long long)Lmax), S = pc::kChainStates;
  return (pc::kWidePowers * S * S + 4 * nb * S) * sizeof(double) + 2 * nb * pc::kWideT * S * sizeof(float);
}
pc::ChainWideScratch chain_wide_scratch(const b200conv* h) {
  pc::ChainWideScratch w{};
  const long long nb = pc::chain_wide_ctas((long long)h->Lmax), S = pc::kChainStates;
  w.nb_cap = nb;
  w.pw = static_cast<double*>(h->chain.wide);
  w.agg = w.pw + pc::kWidePowers * S * S;
  w.carry = w.agg + 2 * nb * S;
  w.z = reinterpret_cast<float*>(w.carry + 2 * nb * S);
  return w;
}

// the whole-GPU send form of one piece; `powers`: the scratch does not hold the P_j of this piece's filters yet
int launch_chain_wide(b200conv* h, const pc::ChainSendParams& sp, bool powers, cudaStream_t st) {
  const pc::ChainWideScratch w = chain_wide_scratch(h);
#if defined(PC_EMULATE)
  (void)st;
  pc::emu_chain_wide(sp, w, powers);
  h->launches += (sp.lc.on || sp.hc.on) ? 3 + (powers ? 1 : 0) : 1;
#else
  const long long nb = pc::chain_wide_ctas(sp.n);
  const dim3 grid((unsigned)nb, 2);
  if (sp.lc.on || sp.hc.on) {
    if (powers) { pc::k_chain_wide_powers<<<1, 64, 0, st>>>(sp, w.pw); h->launches++; }
    pc::k_chain_wide_pass1<<<grid, pc::kWideT, 0, st>>>(sp, w);
    pc::k_chain_wide_carry<<<2, pc::kWideCarryT, 0, st>>>(sp, w, nb);
    h->launches += 2;
  }
  pc::k_chain_wide_pass2<<<grid, pc::kWideT, 0, st>>>(sp, w);
  CU_CHECK(h, cudaGetLastError());
  h->launches++;
#endif
  return 0;
}

// the segmented form's scratch inside one allocation of chain_seg_bytes(Lmax): P_j and M_b per CTA, T_c per chunk,
// aggregates, carries, Z_c
size_t chain_seg_bytes(size_t Lmax) {
  const size_t nb = (size_t)pc::chain_wide_ctas((long long)Lmax), S = pc::kSegStates, S8 = pc::kChainStates;
  return (nb * pc::kWideLogT * S8 * S8 + nb * S * S + nb * pc::kWideT * S * S + 4 * nb * S) * sizeof(double) +
         2 * nb * pc::kWideT * S * sizeof(float);
}
pc::ChainSegScratch chain_seg_scratch(const b200conv* h) {
  pc::ChainSegScratch w{};
  const long long nb = pc::chain_wide_ctas((long long)h->Lmax), S = pc::kSegStates, S8 = pc::kChainStates;
  w.nb_cap = nb;
  w.pw = static_cast<double*>(h->chain.seg);
  w.mb = w.pw + nb * pc::kWideLogT * S8 * S8;
  w.tc = w.mb + nb * S * S;
  w.agg = w.tc + nb * pc::kWideT * S * S;
  w.carry = w.agg + 2 * nb * S;
  w.z = reinterpret_cast<float*>(w.carry + 2 * nb * S);
  return w;
}

// the segmented whole-GPU send form of one piece that spans several rows of the segment table, and the predelayed
// convolver input read from the ring after it
int launch_chain_seg(b200conv* h, const pc::ChainSendParams& sp, const pc::ChainSegs& S, cudaStream_t st) {
  const pc::ChainSegScratch w = chain_seg_scratch(h);
#if defined(PC_EMULATE)
  (void)st;
  pc::emu_chain_seg(sp, S, w);
  pc::emu_chain_seg_read(sp, S);
#else
  const long long nb = pc::chain_wide_ctas(sp.n);
  const dim3 grid((unsigned)nb, 2);
  pc::k_chain_seg_maps<<<(unsigned)nb, pc::kWideT, 0, st>>>(S, sp.n, w);
  pc::k_chain_seg_pass1<<<grid, pc::kWideT, 0, st>>>(sp, S, w);
  pc::k_chain_seg_carry<<<2, 32, 0, st>>>(sp, w, nb);
  pc::k_chain_seg_pass2<<<grid, pc::kWideT, 0, st>>>(sp, S, w);
  pc::k_chain_seg_read<<<dim3((unsigned)((sp.n + 255) / 256), 2), 256, 0, st>>>(sp, S);
  CU_CHECK(h, cudaGetLastError());
#endif
  h->launches += 5;
  return 0;
}

// Filter::init (src/dsp/Filter.cpp:3-21) with the q the processor passes (src/PluginProcessor.cpp:845-848)
pc::ChainFilter chain_filter(bool on, int slope, int mode, float srate, float freq) {
  pc::ChainFilter f{};
  f.on = on ? 1 : 0; f.slope = slope; f.mode = mode;
  const float q = slope == 2 ? 0.0765f : 0.2929f, q2 = 0.6173f;
  f.g = chain_coeff(freq, srate);
  f.k = 2 - 2 * q;
  f.k2 = 2 - 2 * q2;
  if (slope == 0) {
    f.g = f.g / (1.0f + f.g);
  } else {
    f.a1 = 1.0f / (1.0f + f.g * (f.g + f.k));
    f.a2 = f.g * f.a1;
    f.a3 = f.g * f.a2;
    f.a12 = 1.0f / (1.0f + f.g * (f.g + f.k2));
    f.a22 = f.g * f.a12;
    f.a32 = f.g * f.a22;
  }
  return f;
}

// the low / high cut coefficients of a configuration: Filter::setSlope + Filter::init as onSlider does them
// (src/PluginProcessor.cpp:837-848), switched on or off per block (:1643, :1647)
void chain_filters(const b200conv_chain_config& cfg, pc::ChainFilter* lc, pc::ChainFilter* hc) {
  const float sr = (float)cfg.srate;
  *lc = chain_filter(cfg.lowcut_hz > 20.0f, cfg.lowcut_slope, 2, sr, cfg.lowcut_hz);          // HP, PluginProcessor.h:250
  *hc = chain_filter(cfg.highcut_hz < 20000.0f, cfg.highcut_slope, 0, sr, cfg.highcut_hz);   // LP, :248
}

bool chain_config_ok(const b200conv_chain_config& cfg) {
  return cfg.srate > 0 && cfg.predelay >= 0 && cfg.lowcut_slope >= 0 && cfg.lowcut_slope <= 2 && cfg.highcut_slope >= 0 &&
         cfg.highcut_slope <= 2;
}

// processBlock's growth of the delay line (src/PluginProcessor.cpp:1184-1188): a predelay beyond D makes D = 2 * predelay
long long chain_delay_len(long long D, int predelay) { return predelay > D ? 2 * (long long)predelay : D; }

// the ring holds the delay line and doubles as the warmer of an IR hot swap (W = 0.25 s, src/PluginProcessor.cpp:610):
// a piece of up to Lmax samples reads up to max(D, W) samples behind its end
size_t chain_ring_len(const b200conv* h, long long D) {
  return next_pow2(std::max((size_t)D, chain_warmer_len(h->chain.cfg.srate)) + h->Lmax + 1);
}

// A ring too short for a delay line of D samples is reallocated, the samples it holds carried over to their new
// positions.  The only chain parameter change that allocates and synchronises.
int chain_grow_ring(b200conv* h, long long D) {
  const size_t ring = chain_ring_len(h, D);
  if (ring > h->chain.ring_size) {
    if (int rc = set_device(h)) return rc;
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    if (h->swap_peer) CU_CHECK(h, cudaStreamSynchronize(h->swap_peer->s_main));   // a pending warm-up reads the ring
    float* nr = nullptr;
    CU_CHECK(h, cudaMalloc(&nr, 2 * ring * sizeof(float)));
    const long long osz = (long long)h->chain.ring_size, nsz = (long long)ring, end = h->chain.ring_pos;
    int rc = 0;
    if (cudaMemsetAsync(nr, 0, 2 * ring * sizeof(float), h->s_main) != cudaSuccess) rc = 1;
    for (long long p = std::max(0LL, end - osz); p < end && !rc;) {
      const long long oi = p & (osz - 1), ni = p & (nsz - 1);
      const long long seg = std::min(end - p, std::min(osz - oi, nsz - ni));
      for (int ch = 0; ch < 2 && !rc; ++ch)
        if (cudaMemcpyAsync(nr + ch * nsz + ni, h->chain.ring + ch * osz + oi, (size_t)seg * sizeof(float),
                            cudaMemcpyDeviceToDevice, h->s_main) != cudaSuccess) rc = 1;
      p += seg;
    }
    if (!rc && cudaStreamSynchronize(h->s_main) != cudaSuccess) rc = 1;
    if (rc) { cudaFree(nr); CU_CHECK(h, cudaGetLastError()); return fail(h, B200CONV_ECUDA, "growing the delay line failed"); }
    cudaFree(h->chain.ring);
    h->chain.ring = nr; h->chain.ring_size = ring;
  }
  return 0;
}
// delayBuffer.setSize(2, predelay * 2) + clear() + delaypos = 0 (src/PluginProcessor.cpp:1184-1188): the delay history
// reads zero from here on (delay floor), but the samples stay in the ring, which is also the warmer (a separate buffer
// in the reference that the growth does not touch)
int chain_grow_delay(b200conv* h, long long D) {
  if (int rc = chain_grow_ring(h, D)) return rc;
  h->chain.carry.delay_len = D;
  h->chain.carry.delay_floor = h->chain.ring_pos;
  return 0;
}
}  // namespace

int b200conv_chain_configure(b200conv_t* h, const b200conv_chain_config* cfg) {
  REQUIRE_CUDA(h);
  if (h->swap_peer) return fail(h, B200CONV_ESTATE, "an IR hot swap is pending on this handle");
  if (!cfg) { h->chain.on = false; h->route_in_only = false; return B200CONV_OK; }
  if (h->C != 2 && h->C != 4) return fail(h, B200CONV_ESTATE, "the send / wet chain needs a stereo (C = 2) or quad (C = 4) handle");
  if (h->route_on) return fail(h, B200CONV_ESTATE, "the send / wet chain cannot be combined with b200conv_set_routing");
  if (h->cfg.shard_count != 1) return fail(h, B200CONV_ESTATE, "the send / wet chain needs an unsharded handle");
  if (h->stages.empty()) return fail(h, B200CONV_ESTATE, "load an impulse response first");
  if (!chain_config_ok(*cfg)) return fail(h, B200CONV_EINVAL, "bad chain configuration");
  if (int rc = set_device(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  h->chain.cfg = *cfg;
  chain_filters(*cfg, &h->chain.lc, &h->chain.hc);
  const size_t L = h->Lmax;
  // delayBuffer.setSize(2, int(2.0f * sampleRate)) (src/PluginProcessor.cpp:640), grown by the first block as
  // processBlock grows it (:1184-1188) when the predelay is longer
  h->chain.carry.delay_len = chain_delay_len((long long)(int)(2.0 * cfg->srate), cfg->predelay);
  const size_t ring = chain_ring_len(h, h->chain.carry.delay_len);
  if (!h->chain.io) {
    CU_CHECK(h, cudaMalloc(&h->chain.io, 6 * L * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&h->chain.conv_in, 2 * L * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&h->chain.filt, 3 * L * sizeof(float)));
    CU_CHECK(h, cudaMemsetAsync(h->chain.filt + 2 * L, 0, L * sizeof(float), h->s_main));
    CU_CHECK(h, cudaMalloc(&h->chain.state, 4 * pc::kChainStateStride * sizeof(float)));
    CU_CHECK(h, cudaMalloc(&h->chain.wide, chain_wide_bytes(L)));
    CU_CHECK(h, cudaMallocHost((void**)&h->chain.hpin, 6 * h->hpin_cap * sizeof(float)));
#if defined(PC_EMULATE)
    h->chain.hpin_dev = h->chain.hpin;
#else
    if (cudaHostGetDevicePointer((void**)&h->chain.hpin_dev, h->chain.hpin, 0) != cudaSuccess) { cudaGetLastError(); h->chain.hpin_dev = nullptr; }
#endif
  }
  if (ring != h->chain.ring_size) {
    cudaFree(h->chain.ring); h->chain.ring = nullptr;
    CU_CHECK(h, cudaMalloc(&h->chain.ring, 2 * ring * sizeof(float)));
    h->chain.ring_size = ring;
  }
  // Filter::reset(0) + cleared delay line (src/PluginProcessor.cpp:654-657)
  CU_CHECK(h, cudaMemsetAsync(h->chain.state, 0, 2 * pc::kChainStateStride * sizeof(float), h->s_main));
  CU_CHECK(h, cudaMemsetAsync(h->chain.ring, 0, 2 * ring * sizeof(float), h->s_main));
  h->chain.ring_pos = 0; h->chain.carry.delay_floor = 0;
  h->chain.carry.six[0] = cfg->lowcut_slope == 0; h->chain.carry.six[1] = cfg->highcut_slope == 0;
  for (int c = 0; c < 8; ++c) h->in_map[c] = c & 1;        // LL, RR, LR, RL <- L, R, L, R (StereoConvolver.cpp:35-40)
  // fixed-latency mode: the chain's rings (dry L, dry R, ysend, yrev in; L, R out) start a fresh stream
  if (h->lat_D && !h->chain.lat) {
    if (int rc = lat_alloc(h, &h->chain.lat, 4, 2, h->lat_D, h->stages[0].B, h->hpin_cap)) { lat_free(h->chain.lat); return rc; }
  }
  lat_restart(h->chain.lat);
  h->chain.on = true;
  h->swap_state = 0;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return B200CONV_OK;
}

// onSlider + the per-block parameter reads of processBlock (src/PluginProcessor.cpp:837-848, 1151-1188): new values
// from the next chain call on, with every filter state and the delay history kept.  Host-only (the next call's
// launches take the values) unless the predelay outgrows the delay line.
int b200conv_chain_update(b200conv_t* h, const b200conv_chain_config* cfg) {
  REQUIRE_CUDA(h);
  if (!h->chain.on) return fail(h, B200CONV_ESTATE, "the handle owns no send / wet chain");
  if (!cfg || !chain_config_ok(*cfg)) return fail(h, B200CONV_EINVAL, "bad chain configuration");
  if (cfg->srate != h->chain.cfg.srate)
    return fail(h, B200CONV_EINVAL, "a new sample rate needs b200conv_chain_configure");
  const long long D = chain_delay_len(h->chain.carry.delay_len, cfg->predelay);
  if (D != h->chain.carry.delay_len)
    if (int rc = chain_grow_delay(h, D)) return rc;
  h->chain.cfg = *cfg;
  chain_filters(*cfg, &h->chain.lc, &h->chain.hc);
  return B200CONV_OK;
}

namespace {
// one piece of a chain call through handle x's convolvers: LL, RR[, LR, RL] read rows in_map[c] of `in` (stride
// in_stride); the per-convolver outputs stay in x->dch[0]
int chain_convolve(b200conv* x, const float* in, size_t in_stride, size_t n) {
  x->route_in_only = true;
  int rc = 0;
  if (const int nc = rt_cluster_ctas(x, n)) rc = rt_call(x, nc, in, in_stride, x->dch[0], x->Lmax, n, nullptr, 0);
  else rc = run_group(x, in, in_stride, x->dch[0], x->Lmax, n, false);
  x->route_in_only = false;
  return rc;
}

// The warm-up of an IR hot swap (src/PluginProcessor.cpp:1694-1751), queued on g->s_main behind the send kernel of
// the call's first piece: the replay of numBlocks * host_block samples from the ring, through fresh low / high cut
// filters, into g's staging (LL, RR; zeros for LR / RL), then fed through g in batched launch groups.
int chain_warm_up(b200conv* h, b200conv* g) {
  const long long W = (long long)chain_warmer_len(h->chain.cfg.srate);
  const long long N = W / (long long)h->swap_block * (long long)h->swap_block;
  const size_t L = g->Lmax, chunk = L - g->stages[0].B;
  if (N == 0) return 0;
  float* rstate = h->chain.state + 2 * pc::kChainStateStride;
  CU_CHECK(g, cudaMemsetAsync(rstate, 0, 2 * pc::kChainStateStride * sizeof(float), g->s_main));
  if (g->C > 2) CU_CHECK(g, cudaMemsetAsync(g->din[0] + 2 * L, 0, (size_t)(g->C - 2) * L * sizeof(float), g->s_main));
  for (long long off = 0; off < N;) {
    const long long n = std::min(N - off, (long long)chunk);
    pc::ChainSendParams sp{};
    sp.filt = g->din[0]; sp.filt_stride = (long long)L;
    sp.state = rstate;
    sp.ring = h->chain.ring; sp.ring_stride = (long long)h->chain.ring_size; sp.ring_mask = (long long)h->chain.ring_size - 1;
    sp.ring_pos = h->chain.ring_pos; sp.n = n;
    sp.lc = h->chain.lc; sp.hc = h->chain.hc;
    sp.replay_w = W; sp.replay_off = off;
    if (int rc = launch_chain_send(g, sp, g->s_main)) return rc;
    if (int rc = run_group(g, g->din[0], L, g->dout[0], L, (size_t)n, false)) return rc;
    off += n;
  }
  return 0;
}

// end of the fade: the chain (filter states, predelay / warmer ring, configuration, staging, fixed-latency rings) moves
// to g whole.  h gets g's unused chain in exchange: nothing reads it while h->chain.on is false, and
// b200conv_chain_configure rebuilds it.
void chain_move(b200conv* h, b200conv* g) {
  std::swap(h->chain, g->chain);
  for (int c = 0; c < 8; ++c) g->in_map[c] = c & 1;
  h->swap_peer = g->swap_peer = nullptr;
  h->swap_live = false;
  h->swap_state = 3; g->swap_state = 0;
}

// The row of configuration *cfg from sample `start` of a chain call on h (cfg nullptr: the handle's configuration,
// with its cached filters), as the equivalent b200conv_chain_update would leave the chain: a slope that crossed 6 dB
// <-> 12 / 24 dB since the state was last filtered makes the row exchange slot 0 and the stash at its first sample,
// and a predelay beyond D grows D, with the delay floor at that sample.  *c carries both past the row.
pc::ChainSeg chain_row(const b200conv* h, const b200conv_chain_config* cfg, size_t start, ChainCarry* c) {
  pc::ChainSeg g{};
  g.start = (long long)start;
  if (cfg) {
    chain_filters(*cfg, &g.lc, &g.hc);
  } else {
    cfg = &h->chain.cfg;
    g.lc = h->chain.lc; g.hc = h->chain.hc;
  }
  if (g.lc.on || g.hc.on) {
    g.swap_lc = c->six[0] != (g.lc.slope == 0); g.swap_hc = c->six[1] != (g.hc.slope == 0);
    c->six[0] = g.lc.slope == 0; c->six[1] = g.hc.slope == 0;
  }
  const long long D = chain_delay_len(c->delay_len, cfg->predelay);
  if (D != c->delay_len) { c->delay_len = D; c->delay_floor = h->chain.ring_pos + (long long)start; }
  g.delay_floor = c->delay_floor;
  g.predelay = cfg->predelay;
  g.quad_ts = (h->C == 4 && cfg->true_stereo) ? 1 : 0;
  g.width = cfg->width; g.drygain = cfg->drygain; g.wetgain = cfg->wetgain;
  return g;
}

// The device I/O of a chain piece: dry rows dry_stride apart, out rows out_stride apart (send / rev nullptr:
// envelope 1).  at(a): the same from sample a on.
struct ChainIO {
  const float* dry;
  const float* send;
  const float* rev;
  float* out;
  size_t dry_stride, out_stride;
  ChainIO at(size_t a) const {
    return {dry + a, send ? send + a : nullptr, rev ? rev + a : nullptr, out + a, dry_stride, out_stride};
  }
};

// The send and wet parameters of samples [a, a + n) of a piece of a chain call on h, in row `row`: the piece starts at
// sample `off` of the call, io and h's ring position at its first sample.  The row's slope exchange goes to the
// samples that start the row.  wp may be nullptr.
void chain_params(const b200conv* h, const pc::ChainSeg& row, size_t off, size_t a, size_t n, const ChainIO& io,
                  pc::ChainSendParams* sp, pc::ChainWetParams* wp) {
  const Chain& c = h->chain;
  const ChainIO x = io.at(a);
  const long long L = (long long)h->Lmax;
  *sp = pc::ChainSendParams{};
  sp->dry = x.dry; sp->dry_stride = (long long)x.dry_stride; sp->ysend = x.send;
  sp->conv_in = c.conv_in + a; sp->conv_stride = L;
  sp->filt = c.filt + a; sp->filt_stride = L;
  sp->state = c.state;
  sp->ring = c.ring; sp->ring_stride = (long long)c.ring_size; sp->ring_mask = (long long)c.ring_size - 1;
  sp->ring_pos = c.ring_pos + (long long)a; sp->delay_floor = row.delay_floor; sp->predelay = row.predelay;
  sp->n = (long long)n;
  sp->lc = row.lc; sp->hc = row.hc;
  if ((size_t)row.start == off + a) { sp->swap_lc = row.swap_lc; sp->swap_hc = row.swap_hc; }
  if (!wp) return;
  *wp = pc::ChainWetParams{};
  wp->dry = x.dry; wp->dry_stride = (long long)x.dry_stride;
  wp->conv = h->dch[0] + a; wp->conv_stride = L;
  wp->yrev = x.rev;
  wp->out = x.out; wp->out_stride = (long long)x.out_stride; wp->n = (long long)n;
  wp->quad_ts = row.quad_ts; wp->width = row.width; wp->drygain = row.drygain; wp->wetgain = row.wetgain;
}

// One piece of n samples of a chain call on h, the chain's owner, queued on the handles' streams: the send, the warm-up
// and this piece's send through the incoming handle of a pending swap, the convolvers and the wet kernel.  The piece
// is samples [off, off + n) of the call and overlaps rows [lo, hi) of the call's table (rows: the host copy, d_rows:
// the device copy, nullptr for a call of one row); io points at its first sample.
// The send: k_chain_send once per row, each on the part of the piece in its row, as a call cut at the row's start
// would run it; with `powered` (device calls), pieces of at least kChainWideMin samples run the whole-GPU form over one
// row and the segmented form over several.  *powered: the row whose matrix powers the whole-GPU scratch holds (-1:
// none).  The wet kernel: k_chain_wet; k_chain_wet_xfade while a swap fades, k_chain_wet_seg over several rows.  A
// swap and several rows never meet: the entries refuse parameter events while a swap is pending.
// completing: the fade completes in this call (the wet kernel drops the LR / RL terms).  done_flag (fixed-latency
// steps): the wet kernel raises it to done_val after its last store (ticket: its last-CTA counter).
int chain_piece(b200conv* h, const pc::ChainSeg* rows, const pc::ChainSeg* d_rows, int lo, int hi, size_t off,
                size_t n, const ChainIO& io, bool completing, int* powered, unsigned int* done_flag,
                unsigned int done_val, unsigned int* ticket) {
  const size_t L = h->Lmax;
  b200conv* g = h->swap_live ? h->swap_peer : nullptr;
  const pc::ChainSegs S{d_rows + lo, hi - lo, (long long)off};
  pc::ChainSendParams sp;
  pc::ChainWetParams wp;
  chain_params(h, rows[lo], off, 0, n, io, &sp, &wp);
  if (powered && n >= kChainWideMin) {
    if (!g) sp.filt = nullptr;          // only the incoming convolver of a fading swap reads the undelayed send
    if (hi - lo > 1) {
      if (int rc = launch_chain_seg(h, sp, S, h->s_main)) return rc;
    } else {
      if (int rc = launch_chain_wide(h, sp, *powered != lo, h->s_main)) return rc;
      if (sp.lc.on || sp.hc.on) *powered = lo;
    }
  } else {
    for (int k = lo; k < hi; ++k) {     // one row: sp above is its part
      const size_t a = std::max((size_t)rows[k].start, off) - off;
      const size_t b = (k + 1 < hi ? (size_t)rows[k + 1].start : off + n) - off;
      if (hi - lo > 1) chain_params(h, rows[k], off, a, b - a, io, &sp, nullptr);
      if (int rc = launch_chain_send(h, sp, h->s_main)) return rc;
    }
  }
  h->chain.ring_pos += (long long)n;
  if (g) {
    // the incoming handle runs on its own stream behind the send kernel: warm-up (first piece), then this piece's
    // undelayed send (src/PluginProcessor.cpp:1801-1806)
    CU_CHECK(h, cudaEventRecord(h->ev_h2d[0], h->s_main));
    CU_CHECK(g, cudaStreamWaitEvent(g->s_main, h->ev_h2d[0], 0));
    if (h->swap_state == 1) {
      if (int rc = chain_warm_up(h, g)) return rc;
      h->swap_state = g->swap_state = 2;
    }
    if (int rc = chain_convolve(g, h->chain.filt, L, n)) return rc;
    CU_CHECK(g, cudaEventRecord(g->ev_comp[0], g->s_main));
  }
  // the convolvers: LL, RR[, LR, RL] read the chain's L / R, per-convolver outputs stay on the device
  if (int rc = chain_convolve(h, h->chain.conv_in, L, n)) return rc;
  wp.done_flag = done_flag; wp.done_val = done_val; wp.ticket = ticket;
  if (g) {
    CU_CHECK(h, cudaStreamWaitEvent(h->s_main, g->ev_comp[0], 0));
    wp.conv_in = g->dch[0];
    wp.xfade0 = h->swap_xfade; wp.xfadelen = h->swap_xfadelen;
    if (completing) wp.quad_ts = 0;
    h->swap_xfade -= (long long)n;
  }
#if defined(PC_EMULATE)
  if (g) pc::emu_chain_wet_xfade(wp);
  else if (hi - lo > 1) pc::emu_chain_wet_seg(wp, S);
  else pc::emu_chain_wet(wp);
#else
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (g) pc::k_chain_wet_xfade<<<blocks, 256, 0, h->s_main>>>(wp);
  else if (hi - lo > 1) pc::k_chain_wet_seg<<<blocks, 256, 0, h->s_main>>>(wp, S);
  else pc::k_chain_wet<<<blocks, 256, 0, h->s_main>>>(wp);
  CU_CHECK(h, cudaGetLastError());
#endif
  h->launches++;
  return 0;
}

// Zero-copy staging of a real-time chain call: the dry rows and envelopes into the pinned chain.hpin, and the call's
// device I/O there
ChainIO chain_hpin_in(b200conv* h, const float* const* dry, const float* ysend, const float* yrev, size_t len) {
  const size_t cap = h->hpin_cap;
  float* p = h->chain.hpin;
  std::memcpy(p, dry[0], len * sizeof(float));
  std::memcpy(p + cap, dry[1], len * sizeof(float));
  if (ysend) std::memcpy(p + 2 * cap, ysend, len * sizeof(float));
  if (yrev) std::memcpy(p + 3 * cap, yrev, len * sizeof(float));
  float* d = h->chain.hpin_dev;
  return {d, ysend ? d + 2 * cap : nullptr, yrev ? d + 3 * cap : nullptr, d + 4 * cap, cap, cap};
}

// ... and the mix of its n samples out of it
void chain_hpin_out(const b200conv* h, float* const* out, size_t n) {
  for (int ch = 0; ch < 2; ++ch) std::memcpy(out[ch], h->chain.hpin + (4 + ch) * h->hpin_cap, n * sizeof(float));
}
}  // namespace

// A chain call in fixed-latency mode: one step per head block, each the zero-latency chain piece of B0 samples with the
// dry signal and envelopes read from the chain's input ring and the mix written into its output ring, zero-copy; the
// wet kernel raises the step's sequence value.  A hot swap counts its fade per step; when it completes, the chain (and
// its rings) moves to the incoming handle, whose next step is ordered behind the live handle's last one.
static int chain_process_latency(b200conv_t* h, const float* const* dry, const float* ysend, const float* yrev,
                                 float* const* out, size_t len) {
  LatRing* r = h->chain.lat;
  b200conv* x = h;
  const float* in[4] = {dry[0], dry[1], ysend, yrev};
  if (h->timing) h->ev_used = 0;
  if (h->swap_live && h->swap_peer->timing) h->swap_peer->ev_used = 0;
  return lat_run(h, r, in, 4, out, 2, len, [&](long long k, unsigned int v) -> int {
    const size_t B = r->B, L = r->len, off = (size_t)(k % (long long)r->nslots) * B;
    const float* d = r->in_dev + off;
    b200conv* g = x->swap_live ? x->swap_peer : nullptr;
    const bool completing = g && x->swap_xfade - (long long)B <= 0;
    r->last_st = x->s_main;
    const pc::ChainSeg row = chain_row(x, nullptr, 0, &x->chain.carry);
    const ChainIO io{d, d + 2 * L, d + 3 * L, r->out_dev + off, L, L};
    if (int rc = chain_piece(x, &row, nullptr, 0, 1, 0, B, io, completing, nullptr, r->word_dev, v, r->ticket)) return rc;
    if (g && x->swap_xfade <= 0) {                  // src/PluginProcessor.cpp:1823-1826
      chain_move(x, g);
      CU_CHECK(x, cudaEventRecord(x->ev_h2d[0], x->s_main));
      CU_CHECK(g, cudaStreamWaitEvent(g->s_main, x->ev_h2d[0], 0));
      x = g;
    }
    return 0;
  });
}

int b200conv_chain_process(b200conv_t* h, const float* const* dry, const float* ysend, const float* yrev, float* const* out, size_t len) {
  REQUIRE_CUDA(h);
  if (len == 0) return B200CONV_OK;
  if (!h->chain.on) return fail(h, B200CONV_ESTATE, "b200conv_chain_configure first");
  if (!dry || !out || !dry[0] || !dry[1] || !out[0] || !out[1]) return fail(h, B200CONV_EINVAL, "null buffer");
  if (h->stages.empty()) return fail(h, B200CONV_ESTATE, "no impulse response loaded");
  if (int rc = set_device(h)) return rc;
  if (h->lat_D) {
    if (!h->chain.lat) return fail(h, B200CONV_ESTATE, "the chain has no fixed-latency rings");
    return chain_process_latency(h, dry, ysend, yrev, out, len);
  }
  const size_t L = h->Lmax, B0 = h->stages[0].B;
  b200conv* g = h->swap_live ? h->swap_peer : nullptr;        // incoming handle of a pending IR hot swap
  const size_t chunk = g ? std::min(L - B0, L - (size_t)g->stages[0].B) : L - B0;
  // the call in which the fade completes drops the LR / RL terms (deviation: DESIGN §5)
  const bool completing = g && h->swap_xfade - (long long)len <= 0;
  // real-time calls: the kernels read the dry block + envelopes straight from pinned host memory and write the mix
  // back into it (zero-copy), so a callback is three launches and one synchronise instead of six copies more
  const bool zc = len <= h->hpin_cap && len <= chunk && h->chain.hpin_dev != nullptr && h->opt_rt;
  float* buf = h->chain.io;
  const ChainIO io = zc ? chain_hpin_in(h, dry, ysend, yrev, len)
                        : ChainIO{buf, ysend ? buf + 2 * L : nullptr, yrev ? buf + 3 * L : nullptr, buf + 4 * L, L, L};
  const pc::ChainSeg row = chain_row(h, nullptr, 0, &h->chain.carry);
  for (size_t done = 0; done < len;) {
    const size_t n = std::min(len - done, chunk);
    if (!zc) {
      const size_t b = n * sizeof(float);
      for (int ch = 0; ch < 2; ++ch)
        CU_CHECK(h, cudaMemcpyAsync(buf + ch * L, dry[ch] + done, b, cudaMemcpyHostToDevice, h->s_main));
      if (ysend) CU_CHECK(h, cudaMemcpyAsync(buf + 2 * L, ysend + done, b, cudaMemcpyHostToDevice, h->s_main));
      if (yrev) CU_CHECK(h, cudaMemcpyAsync(buf + 3 * L, yrev + done, b, cudaMemcpyHostToDevice, h->s_main));
    }
    if (int rc = chain_piece(h, &row, nullptr, 0, 1, done, n, io, completing, nullptr, nullptr, 0, nullptr)) return rc;
    if (!zc)
      for (int ch = 0; ch < 2; ++ch)
        CU_CHECK(h, cudaMemcpyAsync(out[ch] + done, buf + (4 + ch) * L, n * sizeof(float), cudaMemcpyDeviceToHost,
                                    h->s_main));
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
    if (zc) chain_hpin_out(h, out, n);
    done += n;
  }
  if (g && h->swap_xfade <= 0) chain_move(h, g);        // src/PluginProcessor.cpp:1823-1826
  return B200CONV_OK;
}

// The chain on the caller's device buffers (b200conv_chain_process_device[_events]): the pieces of
// b200conv_chain_process without staging copies or a synchronise between them.  The parameters are a table of rows,
// one per stretch of samples with one configuration: the handle's configuration up to the first event, then one row
// per event.  A call without events is one row on the host: it uploads no table and allocates nothing.  With events,
// everything is checked first; the delay line grows once to the largest D the events reach; the table goes to the
// device in one copy; the handle ends with the last event's configuration, as after the equivalent
// b200conv_chain_update calls.
static int chain_process_device(b200conv_t* h, const ChainIO& io, size_t len, const b200conv_chain_event* events,
                                size_t n_events, int sync) {
  REQUIRE_CUDA(h);
  if (len == 0 && n_events == 0) return B200CONV_OK;
  if (!h->chain.on) return fail(h, B200CONV_ESTATE, "b200conv_chain_configure first");
  if (h->lat_D) return fail(h, B200CONV_ESTATE, "device-pointer calls are not available in fixed-latency mode");
  if (n_events && h->swap_peer)
    return fail(h, B200CONV_ESTATE, "parameter events are not available while an IR hot swap is pending");
  if (!io.dry || !io.out || (n_events && !events)) return fail(h, B200CONV_EINVAL, "null buffer");
  if (h->stages.empty()) return fail(h, B200CONV_ESTATE, "no impulse response loaded");
  for (size_t i = 0; i < n_events; ++i) {
    const b200conv_chain_event& ev = events[i];
    if (!chain_config_ok(ev.cfg) || ev.cfg.srate != h->chain.cfg.srate)
      return fail(h, B200CONV_EINVAL, "bad chain configuration in an event");
    if (ev.offset >= len || (i > 0 && ev.offset <= events[i - 1].offset))
      return fail(h, B200CONV_EINVAL, "event offsets must increase strictly and stay below len");
  }
  if (int rc = set_device(h)) return rc;
  const size_t L = h->Lmax, B0 = h->stages[0].B;
  b200conv* g = h->swap_live ? h->swap_peer : nullptr;        // never with events
  const size_t chunk = g ? std::min(L - B0, L - (size_t)g->stages[0].B) : L - B0;
  const bool completing = g && h->swap_xfade - (long long)len <= 0;
  ChainCarry carry = h->chain.carry;
  pc::ChainSeg one{};                   // the row of a call without events
  std::vector<pc::ChainSeg> table;      // the rows of a call with events
  if (!n_events) {
    one = chain_row(h, nullptr, 0, &carry);
  } else {
    table.reserve(n_events + 1);
    if (events[0].offset > 0) table.push_back(chain_row(h, nullptr, 0, &carry));
    for (size_t i = 0; i < n_events; ++i) table.push_back(chain_row(h, &events[i].cfg, events[i].offset, &carry));
  }
  const pc::ChainSeg* rows = n_events ? table.data() : &one;
  const int nrows = n_events ? (int)table.size() : 1;
  if (n_events) {
    // allocations, before the first launch: the delay line (synchronising, as b200conv_chain_update does), the
    // segmented form's scratch, the table and its staging (the first call that needs them, or a longer table)
    if (carry.delay_len != h->chain.carry.delay_len)
      if (int rc = chain_grow_ring(h, carry.delay_len)) return rc;
    Chain& c = h->chain;
    bool segmented = false;             // a row starts inside a piece of at least kChainWideMin samples
    for (int k = 1; k < nrows; ++k) {
      const size_t s = (size_t)rows[k].start, p = s / chunk * chunk;     // p: the first sample of s's piece
      segmented |= s > p && std::min(len - p, chunk) >= kChainWideMin;
    }
    if (segmented && !c.seg) CU_CHECK(h, cudaMalloc(&c.seg, chain_seg_bytes(L)));
    if ((size_t)nrows > c.segcap) {
      const size_t cap = std::max((size_t)nrows, 2 * c.segcap);
      cudaFree(c.segtab); c.segtab = nullptr;
      if (c.segpin) cudaFreeHost(c.segpin);
      c.segpin = nullptr; c.segcap = 0; c.segev_live = false;
      CU_CHECK(h, cudaMalloc(&c.segtab, cap * sizeof(pc::ChainSeg)));
      CU_CHECK(h, cudaMallocHost((void**)&c.segpin, cap * sizeof(pc::ChainSeg)));
      c.segcap = cap;
    }
    if (!c.segev) CU_CHECK(h, cudaEventCreateWithFlags(&c.segev, cudaEventDisableTiming));
#if !defined(PC_EMULATE)
    // the staging is rewritten only after the previous events call's copy out of it (the head of that call's work)
    if (c.segev_live) CU_CHECK(h, cudaEventSynchronize(c.segev));
#endif
    std::memcpy(c.segpin, rows, (size_t)nrows * sizeof(pc::ChainSeg));
    CU_CHECK(h, cudaMemcpyAsync(c.segtab, c.segpin, (size_t)nrows * sizeof(pc::ChainSeg), cudaMemcpyHostToDevice,
                                h->s_main));
    CU_CHECK(h, cudaEventRecord(c.segev, h->s_main));
    c.segev_live = true;
  }
  // the pieces: samples [done, done + n) of the call overlap rows [lo, hi)
  int powered = -1, lo = 0;
  for (size_t done = 0; done < len;) {
    const size_t n = std::min(len - done, chunk);
    while (lo + 1 < nrows && (size_t)rows[lo + 1].start <= done) ++lo;
    int hi = lo + 1;
    while (hi < nrows && (size_t)rows[hi].start < done + n) ++hi;
    if (int rc = chain_piece(h, rows, n_events ? h->chain.segtab : nullptr, lo, hi, done, n, io.at(done), completing,
                             &powered, nullptr, 0, nullptr))
      return rc;
    done += n;
  }
  h->chain.carry = carry;
  if (n_events) {
    h->chain.cfg = events[n_events - 1].cfg;
    h->chain.lc = rows[nrows - 1].lc; h->chain.hc = rows[nrows - 1].hc;
  }
  if (g && h->swap_xfade <= 0) {        // the chain moves to g; g's next call runs behind this one
    chain_move(h, g);
    CU_CHECK(h, cudaEventRecord(h->ev_h2d[0], h->s_main));
    CU_CHECK(g, cudaStreamWaitEvent(g->s_main, h->ev_h2d[0], 0));
  }
  if (sync) CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  return B200CONV_OK;
}

int b200conv_chain_process_device(b200conv_t* h, const float* dry_dev, size_t dry_stride, const float* ysend_dev,
                                  const float* yrev_dev, float* out_dev, size_t out_stride, size_t len, int sync) {
  return chain_process_device(h, {dry_dev, ysend_dev, yrev_dev, out_dev, dry_stride, out_stride}, len, nullptr, 0,
                              sync);
}

int b200conv_chain_process_device_events(b200conv_t* h, const float* dry_dev, size_t dry_stride, const float* ysend_dev,
                                         const float* yrev_dev, float* out_dev, size_t out_stride, size_t len,
                                         const b200conv_chain_event* events, size_t n_events, int sync) {
  return chain_process_device(h, {dry_dev, ysend_dev, yrev_dev, out_dev, dry_stride, out_stride}, len, events, n_events,
                              sync);
}

int b200conv_chain_swap(b200conv_t* live, b200conv_t* incoming, size_t host_block) {
  REQUIRE_CUDA(live);
  REQUIRE_CUDA(incoming);
  if (live == incoming) return fail(live, B200CONV_EINVAL, "the IR hot swap needs two different handles");
  if (live->cfg.device != incoming->cfg.device) return fail(live, B200CONV_EINVAL, "the IR hot swap needs both handles on one device");
  if (live->cfg.shard_count > 1 || incoming->cfg.shard_count > 1 || live->route_on || incoming->route_on ||
      live->p2p_on || incoming->p2p_on)
    return fail(live, B200CONV_EINVAL, "the IR hot swap needs unsharded handles without I/O routing");
  if (host_block == 0) return fail(live, B200CONV_EINVAL, "host_block 0");
  if (!live->chain.on) return fail(live, B200CONV_ESTATE, "the live handle has no send / wet chain");
  if (incoming->stages.empty()) return fail(live, B200CONV_ESTATE, "the incoming handle has no impulse response");
  if (incoming->chain.on) return fail(live, B200CONV_ESTATE, "the incoming handle already owns a send / wet chain");
  if (live->swap_peer || incoming->swap_peer) return fail(live, B200CONV_ESTATE, "an IR hot swap is already pending");
  if (incoming->C != 2 && incoming->C != 4)
    return fail(live, B200CONV_ESTATE, "the send / wet chain needs a stereo (C = 2) or quad (C = 4) handle");
  if (live->Lmax != incoming->Lmax || live->hpin_cap != incoming->hpin_cap)
    return fail(live, B200CONV_EINVAL, "the IR hot swap needs equal staging sizes (same head block and batch size)");
  if (live->lat_D != incoming->lat_D) return fail(live, B200CONV_EINVAL, "the IR hot swap needs equal latencies");
  live->swap_peer = incoming; incoming->swap_peer = live;
  live->swap_live = true; incoming->swap_live = false;
  live->swap_state = incoming->swap_state = 1;
  live->swap_block = host_block;
  // src/PluginProcessor.cpp:1754-1755
  live->swap_xfadelen = (long long)std::ceil(live->chain.cfg.srate * 50 / 1000.0);
  live->swap_xfade = live->swap_xfadelen;
  // during the warm-up and the fade only LL and RR get input; LR / RL of a quad handle read chain.filt's zero row
  for (int c = 0; c < 8; ++c) incoming->in_map[c] = c < 2 ? c : 2;
  return B200CONV_OK;
}

int b200conv_chain_swap_state(const b200conv_t* h) { return h ? h->swap_state : 0; }

// ---- groups (b200conv_group_process, b200conv_chain_group_process) --------------------------------------------------
// The real-time calls of the qualifying members run as one k_rt_group launch per shape class on the group's own
// high-priority stream: prepare every member, launch, commit every member.  Event rules:
//  - a member's tail-output waits (rt_prepare) go on the group stream;
//  - a member whose s_main may hold unsynchronised work (main_unsynced) orders the group stream behind it once;
//  - if either happened, or a member completes a tail block, the group records ONE event after its launches: the
//    s_tail of every member that completes a tail block waits on it before run_tail_block, and every prepared member
//    keeps it in grp_ev, so that its next own call orders s_main and s_post behind it (set_device).
// A Stage's job_waited therefore means "ordered before this handle's next head-stage work", through s_main or through
// the group stream and grp_ev.  In steady state (no tail block completes, nothing unsynchronised) a group call makes
// no event operation at all: one launch per shape class, then one spin per member on its completion word.

// A member's part of the step a group call is running
struct GroupSlot {
  pc::RtStepParams R;                // the convolver call (R.p), with its step walk in the step form
  pc::ChainSendParams sp;            // a chain member's send and wet mix
  pc::ChainWetParams wp;
  int nc = 0;                        // cluster width of a member that shares the launches, 0: it runs its own call
  bool prepared = false, launched = false;
  bool shares_latency = false;       // fixed-latency group calls: the member shares the call's steps,
  bool waited = false;               // ... the call waited for its ring
  long long p0 = 0;                  // ... and the ring position its current pass began at
};

struct b200conv_group {
  std::vector<b200conv*> m;
  int device = 0;
  std::string err;
  cudaStream_t st = nullptr;
  cudaEvent_t ev = nullptr;
  unsigned long long launches = 0;
  // per-call scratch, sized by create: a group call allocates nothing
  std::vector<GroupSlot> slot;
  pc::RtGroupParams G;                   // the tables of one launch
  pc::RtStepGroupParams GS;
  pc::ChainSendGroupParams SG;
  pc::ChainWetGroupParams WG;
  // b200conv_chain_group_process: the group's pinned completion word (+ its device-side address) and the wet launch's
  // ticket word on the device
  unsigned int* flag = nullptr;
  unsigned int* flag_dev = nullptr;
  unsigned int epoch = 0;
  unsigned int* ticket = nullptr;
  // fixed-latency group calls (b200conv_group_set_latency): the group's latency (0: none)
  size_t lat_D = 0;
};

static int group_fail(b200conv_group* g, int code, const std::string& msg) { g->err = msg; return code; }
static int group_member_fail(b200conv_group* g, size_t i, int code) {
  g->err = "member " + std::to_string(i) + ": " + g->m[i]->err;
  return code;
}

// cluster width of a member's call when it can share the group's launch, else 0
static int group_ctas(const b200conv* h, size_t len) {
  if (h->cfg.shard_count != 1 || h->lat_D || h->stages.empty() || len > h->hpin_cap || !h->hpin_in_dev ||
      !h->hpin_out_dev || !h->hflag_dev)
    return 0;
  return std::max(rt_cluster_ctas(h, len), 0);
}

// The chain calls of a group (b200conv_chain_group_process).  A member shares the group's launches when
// b200conv_chain_process would run its call as one zero-copy piece through one cluster launch, and it can share a
// k_rt_group launch: a chain, no fixed latency, no pending hot swap, and group_ctas > 0.  Its width, else 0.
static int chain_group_ctas(const b200conv* h, size_t len) {
  if (!h->chain.on || h->lat_D || h->swap_peer || h->stages.empty() || !h->chain.hpin_dev || !h->opt_rt ||
      len > h->Lmax - h->stages[0].B)
    return 0;
  return group_ctas(h, len);
}

// Fixed-latency groups (b200conv_group_set_latency): a member shares the steps of a group call when its latency is the
// group's and each of its steps would be one cluster launch: lat_step's rt_call path, or for the chain
// chain_convolve's, with chain rings and no pending hot swap.  Its cluster width, else 0.
static int group_lat_ctas(const b200conv_group* g, const b200conv* h, bool chain) {
  if (!g->lat_D || h->lat_D != g->lat_D || h->cfg.shard_count != 1 || h->stages.empty()) return 0;
  if (chain ? (!h->chain.on || !h->chain.lat || h->swap_peer || !h->opt_rt) : (!h->lat || !h->hpin_in_dev || !h->hpin_out_dev))
    return 0;
  return std::max(rt_cluster_ctas(h, h->stages[0].B), 0);
}

// Device-buffer group calls (b200conv_group_process_device, b200conv_chain_group_process_device): a member shares the
// group's k_rt_group_steps launches when a one-launch call of it would (group_ctas without the length and host-staging
// rules, not in split mode), its call touches at most kRtMaxSteps head blocks from its fill on, and every later stage
// has a block that is a multiple of the head block, completes at most once in the call, and whose completed block's
// output is first needed after the call (the crossing rule of rt_cluster_ctas for any number of head blocks).  A chain
// member also meets chain_group_ctas' rules and len stays below kChainWideMin, where b200conv_chain_process_device
// runs the serial send.  Its cluster width, else 0.
static int group_step_ctas(const b200conv* h, size_t len, bool chain) {
  if (h->cfg.shard_count != 1 || h->lat_D || h->stages.empty() || len == 0) return 0;
  if (chain && (!h->chain.on || h->swap_peer || !h->opt_rt || len > h->Lmax - h->stages[0].B || len >= kChainWideMin))
    return 0;
  const Stage& s0 = h->stages[0];
  const long long M = s0.B, n = (long long)len;
  const long long len1 = std::min(n, M - s0.fill);
  if (1 + (n - len1 + M - 1) / M > pc::kRtMaxSteps) return 0;
  for (size_t si = 1; si < h->stages.size(); ++si) {
    const Stage& s = h->stages[si];
    const long long d = s.B - s.fill;                 // samples of the call up to the stage's block boundary
    if (s.B % M != 0) return 0;
    if (d <= n && (d < len1 || (d - len1) % M != 0 || n - d >= s.B ||
                   h->abs_pos + n > (s.blocks_done + s.q) * (long long)s.B))
      return 0;
  }
  return std::max(rt_cluster_ctas(h, 1), 0);        // the width of a call inside the open block; -1 (split): 0
}

b200conv_group_t* b200conv_group_create(b200conv_t* const* members, int n) {
  if (!members || n < 1 || n > 64) return nullptr;
  for (int i = 0; i < n; ++i) {
    if (!members[i] || members[i]->cfg.device != members[0]->cfg.device) return nullptr;
    for (int j = 0; j < i; ++j)
      if (members[j] == members[i]) return nullptr;
  }
  b200conv_group* g = new (std::nothrow) b200conv_group();
  if (!g) return nullptr;
  try {
    g->m.assign(members, members + n);
    g->slot.resize(n);
  } catch (...) {
    delete g;
    return nullptr;
  }
  g->device = members[0]->cfg.device;
  int lo = 0, hi = 0;
  bool ok = cudaSetDevice(g->device) == cudaSuccess && cudaDeviceGetStreamPriorityRange(&lo, &hi) == cudaSuccess;
  ok = ok && cudaStreamCreateWithPriority(&g->st, cudaStreamNonBlocking, hi) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&g->ev, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaMallocHost((void**)&g->flag, 64) == cudaSuccess;
  if (ok) *g->flag = 0;
#if defined(PC_EMULATE)
  g->flag_dev = g->flag;
#else
  ok = ok && cudaHostGetDevicePointer((void**)&g->flag_dev, g->flag, 0) == cudaSuccess;
#endif
  ok = ok && cudaMalloc(&g->ticket, sizeof(unsigned int)) == cudaSuccess;
  ok = ok && cudaMemsetAsync(g->ticket, 0, sizeof(unsigned int), g->st) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    b200conv_group_destroy(g);
    return nullptr;
  }
  return g;
}

void b200conv_group_destroy(b200conv_group_t* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  if (g->st) cudaStreamSynchronize(g->st);
  for (b200conv* h : g->m) {
    if (h->grp_ev == g->ev) h->grp_ev = nullptr, h->grp_st = nullptr;   // everything the event covers has completed
    for (LatRing* r : {h->lat, h->chain.lat})          // ... and every step the group stream held
      if (r && r->last_st == g->st) r->last_st = h->s_main;
  }
  if (g->ev) cudaEventDestroy(g->ev);
  if (g->st) cudaStreamDestroy(g->st);
  if (g->flag) cudaFreeHost(g->flag);
  if (g->ticket) cudaFree(g->ticket);
  delete g;
}

const char* b200conv_group_last_error(const b200conv_group_t* g) { return g ? g->err.c_str() : "null group"; }

unsigned long long b200conv_group_launch_count(const b200conv_group_t* g) { return g ? g->launches : 0; }

// A member whose s_main may hold unsynchronised work (main_unsynced) orders the group stream behind it; *waited is set
static int group_order_behind(b200conv_group* g, size_t i, bool* waited) {
  b200conv* h = g->m[i];
  if (!h->main_unsynced) return 0;
  cudaError_t e = cudaEventRecord(h->ev_rt, h->s_main);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(g->st, h->ev_rt, 0);
  if (e != cudaSuccess) return group_member_fail(g, i, cuda_fail(h, e, "group: ordering behind the member's stream"));
  h->main_unsynced = false;
  *waited = true;
  return 0;
}

// Prepares member i's step of len samples on the group stream (its waits and a timeline compaction go there; *waited is
// set if there was a wait); `steps`: the step form of a device-buffer group call (a call of up to kRtMaxSteps head
// blocks, k_rt_group_steps).  in: the input rows, in_stride apart; for a chain member the dry rows, with the send / rev
// envelope rows (nullptr: envelope 1).  out: the output rows, out_stride apart.  flag / val: the step's completion word
// and value, ticket: the wet kernel's ticket word of a chain member (nullptr / 0: none).  A chain member's send and wet
// are those of chain_piece's k_chain_send form with the row of the handle's configuration, and the chain moves past
// the step; its convolvers run from chain.conv_in into dch[0], as chain_convolve runs them.  The member counts as
// prepared even if this fails: waits may have been queued.
static int group_prepare_step(b200conv_group* g, size_t i, bool chain, const float* in, const float* send,
                              const float* rev, size_t in_stride, float* out, size_t out_stride, size_t len,
                              unsigned int* flag, unsigned int val, unsigned int* ticket, bool* waited,
                              bool steps = false) {
  b200conv* h = g->m[i];
  GroupSlot& s = g->slot[i];
  int rc;
  if (chain) {
    const pc::ChainSeg row = chain_row(h, nullptr, 0, &h->chain.carry);
    chain_params(h, row, 0, 0, len, {in, send, rev, out, in_stride, out_stride}, &s.sp, &s.wp);
    h->chain.ring_pos += (long long)len;
    s.wp.done_flag = flag; s.wp.done_val = val; s.wp.ticket = ticket;
    h->route_in_only = true;
    rc = rt_prepare(h, s.nc, h->chain.conv_in, h->Lmax, h->dch[0], h->Lmax, len, g->st, s.R.p, waited,
                    steps ? &s.R : nullptr);
    h->route_in_only = false;
  } else {
    rc = rt_prepare(h, s.nc, in, in_stride, out, out_stride, len, g->st, s.R.p, waited, steps ? &s.R : nullptr);
    s.R.p.done_flag = flag; s.R.p.done_val = val;
  }
  s.prepared = true;
  return rc ? group_member_fail(g, i, rc) : 0;
}

// The prepared members' clusters: one k_rt_group launch (steps: k_rt_group_steps) per shape class (M, C, NC) and
// kRtGroupMax members, in member order within a class, on the group stream
static int group_launch_classes(b200conv_group* g, bool steps) {
  const size_t n = g->m.size();
  for (size_t i = 0; i < n; ++i) {
    if (!g->slot[i].prepared || g->slot[i].launched) continue;
    const pc::RtParams& A = g->slot[i].R.p;
    size_t idx[pc::kRtGroupMax];
    int k = 0;
    for (size_t j = i; j < n && k < pc::kRtGroupMax; ++j) {
      const GroupSlot& s = g->slot[j];
      if (s.prepared && !s.launched && s.R.p.M == A.M && s.R.p.C == A.C && s.R.p.NC == A.NC) {
        if (steps) g->GS.p[k] = s.R;
        else g->G.p[k] = s.R.p;
        idx[k++] = j;
      }
    }
    g->G.n = g->GS.n = k;
#if defined(PC_EMULATE)
    if (steps) pc::emu_rt_group_steps(g->GS);
    else pc::emu_rt_group(g->G);
#else
    if (const cudaError_t e = steps ? rt_launch(g->GS, A.M, A.C, A.NC, g->st) : rt_launch(g->G, A.M, A.C, A.NC, g->st)) {
      cudaGetLastError();
      return group_fail(g, B200CONV_ECUDA, std::string("group launch: ") + cudaGetErrorString(e));
    }
#endif
    g->launches++;
    for (int j = 0; j < k; ++j) g->slot[idx[j]].launched = true;
  }
  return 0;
}

// The sends of the prepared members: one k_chain_send_group per send width and kChainGroupMax members, in member order
static int group_chain_sends(b200conv_group* g) {
  const size_t n = g->m.size();
  bool sent[64] = {};                    // b200conv_group_create admits at most 64 members
  for (size_t i = 0; i < n; ++i) {
    if (!g->slot[i].prepared || sent[i]) continue;
    const int T = chain_send_threads((size_t)g->slot[i].sp.n);
    int k = 0;
    for (size_t j = i; j < n && k < pc::kChainGroupMax; ++j)
      if (g->slot[j].prepared && !sent[j] && chain_send_threads((size_t)g->slot[j].sp.n) == T) {
        g->SG.p[k++] = g->slot[j].sp;
        sent[j] = true;
      }
    g->SG.n = k;
#if defined(PC_EMULATE)
    pc::emu_chain_send_group(g->SG, T);
#else
    pc::k_chain_send_group<<<dim3(2, (unsigned)k), T, 0, g->st>>>(g->SG);
    if (const cudaError_t e = cudaGetLastError())
      return group_fail(g, B200CONV_ECUDA, std::string("group send launch: ") + cudaGetErrorString(e));
#endif
    g->launches++;
  }
  return 0;
}

// The wet mixes of the prepared members: one k_chain_wet_group per kChainGroupMax members, in member order.  The last
// raises `flag` to `want`; with flag nullptr every row raises its own member's word instead (fixed-latency steps).
static int group_chain_wets(b200conv_group* g, unsigned int* flag, unsigned int want) {
  const size_t n = g->m.size();
  size_t left = 0;
  for (size_t i = 0; i < n; ++i) left += g->slot[i].prepared ? 1 : 0;
  for (size_t i = 0, k = 0; i < n; ++i) {
    if (g->slot[i].prepared) { g->WG.p[k++] = g->slot[i].wp; --left; }
    if (k == (size_t)pc::kChainGroupMax || (k && !left)) {
      unsigned blocks = 0;
      for (size_t j = 0; j < k; ++j) blocks = std::max(blocks, (unsigned)((g->WG.p[j].n + 255) / 256));
      g->WG.n = (int)k;
      g->WG.done_flag = left ? nullptr : flag;
      g->WG.done_val = want;
      g->WG.ticket = g->ticket;
#if defined(PC_EMULATE)
      pc::emu_chain_wet_group(g->WG);
#else
      pc::k_chain_wet_group<<<dim3(blocks, (unsigned)k), 256, 0, g->st>>>(g->WG);
      if (const cudaError_t e = cudaGetLastError())
        return group_fail(g, B200CONV_ECUDA, std::string("group wet launch: ") + cudaGetErrorString(e));
#endif
      g->launches++;
      k = 0;
    }
  }
  return 0;
}

// Commit: head bookkeeping and the tail blocks the launched calls complete, behind the group's event (recorded now if
// the prepare queued a wait); every prepared member keeps the event for its next own call.  *rc keeps the first error.
static void group_commit(b200conv_group* g, bool waited, int* rc) {
  const size_t n = g->m.size();
  bool recorded = false;
  if (waited) {
    if (cudaEventRecord(g->ev, g->st) != cudaSuccess) {
      cudaGetLastError();
      if (!*rc) *rc = group_fail(g, B200CONV_ECUDA, "group: event record failed");
    } else {
      recorded = true;
    }
  }
  for (size_t i = 0; i < n; ++i) {
    if (!g->slot[i].launched) continue;
    if (int crc = rt_commit(g->m[i], g->slot[i].R.p.len, g->ev, g->st, &recorded))
      if (!*rc) *rc = group_member_fail(g, i, crc);
  }
  if (recorded)
    for (size_t i = 0; i < n; ++i)
      if (g->slot[i].prepared) g->m[i]->grp_ev = g->ev;
}

// The prepared steps on the group stream: the sends (chain), the convolvers (steps: in the step form), the wet mixes
// (chain: the last raises `flag`, the group's word, to `want`, and g->epoch follows it), then the commit.  Nothing is
// launched once *rc holds an error.
static void group_launch_round(b200conv_group* g, bool chain, unsigned int* flag, unsigned int want, bool waited,
                               int* rc, bool steps = false) {
  if (!*rc && chain) *rc = group_chain_sends(g);
  if (!*rc) *rc = group_launch_classes(g, steps);
  if (!*rc && chain) {
    *rc = group_chain_wets(g, flag, want);
    if (!*rc && flag) g->epoch = want;
  }
  group_commit(g, waited, rc);
}

// wait_word on a word raised by the group stream's work, failing with the group's error
static int group_wait(b200conv_group* g, const volatile unsigned int* f, unsigned int want) {
  cudaError_t e = cudaSuccess;
  if (wait_word(f, want, g->st, &e)) return 0;
  if (!e) return group_fail(g, B200CONV_ECUDA, "group stream: a completion word was not raised");
  cudaGetLastError();
  return group_fail(g, B200CONV_ECUDA, std::string("group stream: ") + cudaGetErrorString(e));
}

// The members that share a group call's fixed-latency steps, walked in passes as lat_run walks one call; a pass is at
// most the smallest ring piece among them.  Per pass: every sharing member's input half; then rounds, round q holding
// the q-th step of every member that completes more than q head blocks in the pass, each prepared as lat_step (or the
// step of chain_process_latency) runs it, with the member's ring word and sequence value, then launched together and
// committed on the group stream, so that each member's steps stay in order; then every sharing member's output half.
// The group stream is ordered behind a member's own steps by main_unsynced, as in a zero-latency group call; a call
// that launched steps records the group's event once, and the members keep it for their next own call (set_device).
// chain: in / ysend / yrev are the chain's dry / ysend / yrev tables.  Sets shares_latency for the callers.
static int group_lat_passes(b200conv_group* g, const float* const* const* in, const float* const* ysend,
                            const float* const* yrev, float* const* const* out, size_t len, bool chain) {
  const size_t n = g->m.size();
  size_t piece = 0;
  for (size_t i = 0; i < n; ++i) {
    b200conv* h = g->m[i];
    GroupSlot& s = g->slot[i];
    s.nc = group_lat_ctas(g, h, chain);
    s.shares_latency = s.nc > 0;
    s.waited = false;
    if (s.shares_latency) {
      const LatRing* r = chain ? h->chain.lat : h->lat;
      piece = piece ? std::min(piece, r->piece) : r->piece;
    }
  }
  int rc = 0;
  bool stepped = false;
  for (size_t done = 0; done < len && piece && !rc;) {
    const long long np = (long long)std::min(len - done, piece);
    long long rounds = 0;
    for (size_t i = 0; i < n && !rc; ++i) {
      GroupSlot& s = g->slot[i];
      if (!s.shares_latency) continue;
      b200conv* h = g->m[i];
      LatRing* r = chain ? h->chain.lat : h->lat;
      const float* rows[4] = {};
      if (chain) { rows[0] = in[i][0]; rows[1] = in[i][1]; rows[2] = ysend ? ysend[i] : nullptr; rows[3] = yrev ? yrev[i] : nullptr; }
      bool w = false;
      s.p0 = r->pos;
      if (int e = lat_in(h, r, chain ? rows : in[i], chain ? 4 : (h->route_on ? h->n_in : h->C), done, np, &w))
        rc = group_member_fail(g, i, e);
      if (w) s.waited = true;
      const long long B = (long long)r->B;
      rounds = std::max(rounds, (s.p0 + np) / B - s.p0 / B);
    }
    for (long long q = 0; q < rounds && !rc; ++q) {
      bool waited = false;
      for (size_t i = 0; i < n; ++i) {
        GroupSlot& s = g->slot[i];
        s.prepared = s.launched = false;
        if (!s.shares_latency || rc) continue;
        b200conv* h = g->m[i];
        LatRing* r = chain ? h->chain.lat : h->lat;
        const long long k = s.p0 / (long long)r->B + q;
        if (k >= (s.p0 + np) / (long long)r->B) continue;
        if ((rc = group_order_behind(g, i, &waited))) continue;
        const size_t B = r->B, L = r->len, off = (size_t)(k % (long long)r->nslots) * B;
        const float* d = r->in_dev + off;
        const unsigned int v = ++r->seq;
        if ((rc = group_prepare_step(g, i, chain, d, chain ? d + 2 * L : nullptr, chain ? d + 3 * L : nullptr, L,
                                     r->out_dev + off, L, B, r->word_dev, v, r->ticket, &waited)))
          continue;
        r->last_st = g->st;                // lat_wait's fallback synchronises the stream that holds the step
      }
      group_launch_round(g, chain, nullptr, 0, waited, &rc);
      for (size_t i = 0; i < n && !rc; ++i) {
        const GroupSlot& s = g->slot[i];
        if (!s.launched) continue;
        LatRing* r = chain ? g->m[i]->chain.lat : g->m[i]->lat;
        const long long k = s.p0 / (long long)r->B + q;
        r->slot_seq[k % (long long)r->nslots] = chain ? s.wp.done_val : s.R.p.done_val;
        stepped = true;
      }
    }
    for (size_t i = 0; i < n && !rc; ++i) {
      GroupSlot& s = g->slot[i];
      if (!s.shares_latency) continue;
      b200conv* h = g->m[i];
      bool w = false;
      if (int e = lat_out(h, chain ? h->chain.lat : h->lat, out[i], chain ? 2 : (h->route_on ? h->n_out : h->C), done,
                          s.p0, np, &w))
        rc = group_member_fail(g, i, e);
      if (w) s.waited = true;
    }
    done += (size_t)np;
  }
  if (stepped) {
    if (cudaEventRecord(g->ev, g->st) != cudaSuccess) {
      cudaGetLastError();
      if (!rc) rc = group_fail(g, B200CONV_ECUDA, "group: event record failed");
    } else {
      for (size_t i = 0; i < n; ++i)
        if (g->slot[i].shares_latency) g->m[i]->grp_ev = g->ev;
    }
  }
  for (size_t i = 0; i < n; ++i)                 // a call that waited counts once in the member's latency_waits
    if (g->slot[i].waited) g->m[i]->lat_waits++;
  return rc;
}

int b200conv_group_process(b200conv_group_t* g, const float* const* const* in, float* const* const* out, size_t len) {
  if (!g) return B200CONV_EINVAL;
  if (len == 0) return B200CONV_OK;
  if (!in || !out) return group_fail(g, B200CONV_EINVAL, "null buffer");
  const size_t n = g->m.size();
  // every member's arguments before anything is enqueued: a refused call advances no member
  for (size_t i = 0; i < n; ++i) {
    const b200conv* h = g->m[i];
    if (h->sticky_cuda_error) return group_member_fail(g, i, B200CONV_ECUDA);
    if (!in[i] || !out[i]) return group_fail(g, B200CONV_EINVAL, "null buffer of member " + std::to_string(i));
    if (h->lat_D)
      for (int c = 0; c < (h->route_on ? h->n_in : h->C); ++c)
        if (!in[i][c]) return group_fail(g, B200CONV_EINVAL, "null buffer of member " + std::to_string(i));
  }
  if (cudaSetDevice(g->device) != cudaSuccess) {
    cudaGetLastError();
    return group_fail(g, B200CONV_ECUDA, "cudaSetDevice failed");
  }
  // the members at the group's fixed latency first, in shared steps
  int rc = group_lat_passes(g, in, nullptr, nullptr, out, len, false);
  bool waited = false;
  // prepare: inputs into the pinned staging, the waits each call needs, its parameters
  for (size_t i = 0; i < n; ++i) {
    b200conv* h = g->m[i];
    GroupSlot& s = g->slot[i];
    s.prepared = s.launched = false;
    s.nc = group_ctas(h, len);
    if (!s.nc || rc) continue;
    if ((rc = group_order_behind(g, i, &waited))) continue;
    const int Cin = h->route_on ? h->n_in : h->C;
    for (int c = 0; c < Cin; ++c) std::memcpy(h->hpin_in + (size_t)c * len, in[i][c], len * sizeof(float));
    if ((rc = group_prepare_step(g, i, false, h->hpin_in_dev, nullptr, nullptr, len, h->hpin_out_dev, len, len,
                                 h->hflag_dev, h->flag_epoch + 1, nullptr, &waited)))
      continue;
    ++h->flag_epoch;
  }
  group_launch_round(g, false, nullptr, 0, waited, &rc);
  // every other member on its own, while the shared launches run
  for (size_t i = 0; i < n && !rc; ++i)
    if (!g->slot[i].nc && !g->slot[i].shares_latency)
      if (int mrc = b200conv_process(g->m[i], in[i], out[i], len)) rc = group_member_fail(g, i, mrc);
  // each launched member's completion word, then its output
  for (size_t i = 0; i < n; ++i) {
    if (!g->slot[i].launched) continue;
    const b200conv* h = g->m[i];
    if (int wrc = group_wait(g, h->hflag, g->slot[i].R.p.done_val)) return wrc;
    const int Cout = h->route_on ? h->n_out : h->C;
    for (int c = 0; c < Cout; ++c) std::memcpy(out[i][c], h->hpin_out + (size_t)c * len, len * sizeof(float));
  }
  return rc;
}

int b200conv_chain_group_process(b200conv_group_t* g, const float* const* const* dry, const float* const* ysend,
                                 const float* const* yrev, float* const* const* out, size_t len) {
  if (!g) return B200CONV_EINVAL;
  if (len == 0) return B200CONV_OK;
  if (!dry || !out) return group_fail(g, B200CONV_EINVAL, "null buffer");
  const size_t n = g->m.size();
  // every member's arguments before anything is enqueued: a refused call advances no member
  for (size_t i = 0; i < n; ++i) {
    const b200conv* h = g->m[i];
    if (h->sticky_cuda_error) return group_member_fail(g, i, B200CONV_ECUDA);
    if (!h->chain.on) return group_fail(g, B200CONV_ESTATE, "member " + std::to_string(i) + " owns no send / wet chain");
    if (h->stages.empty() || (h->lat_D && !h->chain.lat))
      return group_fail(g, B200CONV_ESTATE, "member " + std::to_string(i) + " has no impulse response or chain rings");
    if (!dry[i] || !out[i] || !dry[i][0] || !dry[i][1] || !out[i][0] || !out[i][1])
      return group_fail(g, B200CONV_EINVAL, "null buffer of member " + std::to_string(i));
  }
  if (cudaSetDevice(g->device) != cudaSuccess) {
    cudaGetLastError();
    return group_fail(g, B200CONV_ECUDA, "cudaSetDevice failed");
  }
  int rc = group_lat_passes(g, dry, ysend, yrev, out, len, true);
  bool waited = false;
  size_t shared = 0;
  // prepare: inputs into the chain's pinned staging, the send / wet parameters, the waits the convolver call needs
  // and its parameters
  for (size_t i = 0; i < n; ++i) {
    b200conv* h = g->m[i];
    GroupSlot& s = g->slot[i];
    s.prepared = s.launched = false;
    s.nc = chain_group_ctas(h, len);
    if (!s.nc || rc) continue;
    if ((rc = group_order_behind(g, i, &waited))) continue;
    const ChainIO io = chain_hpin_in(h, dry[i], ysend ? ysend[i] : nullptr, yrev ? yrev[i] : nullptr, len);
    if ((rc = group_prepare_step(g, i, true, io.dry, io.send, io.rev, io.dry_stride, io.out, io.out_stride, len, nullptr,
                                 0, nullptr, &waited)))
      continue;
    ++shared;
  }
  // the last wet launch raises the group's word for every shared member
  const unsigned int want = g->epoch + 1;
  group_launch_round(g, true, shared ? g->flag_dev : nullptr, want, waited, &rc);
  // every other member on its own, while the shared launches run
  for (size_t i = 0; i < n && !rc; ++i)
    if (!g->slot[i].nc && !g->slot[i].shares_latency)
      if (int mrc = b200conv_chain_process(g->m[i], dry[i], ysend ? ysend[i] : nullptr, yrev ? yrev[i] : nullptr, out[i],
                                           len))
        rc = group_member_fail(g, i, mrc);
  if (!shared || g->epoch != want) return rc;
  if (int wrc = group_wait(g, g->flag, want)) return wrc;
  for (size_t i = 0; i < n; ++i)
    if (g->slot[i].launched) chain_hpin_out(g->m[i], out[i], len);
  return rc;
}

// ---- device-buffer group calls --------------------------------------------------------------------------------------
// Every launch goes to the group stream and nothing waits on the host.  The members that share (group_step_ctas) run
// their whole call in the step form: one k_rt_group_steps launch per shape class (chain: the sends before, the wet
// mixes after), with no completion word; their next own call records the group's event lazily (grp_st, set_device).
// Every other member runs its own device call on its own streams, ordered both ways with the group stream: behind one
// event recorded at the start, and the group stream behind each such member's s_main at the end.

// the checks of both entries that need no member's kind: a refused call advances no member
// (tables: every buffer and stride table is there)
static int group_device_check(b200conv_group* g, bool chain, bool tables, const float* const* in_dev,
                              float* const* out_dev, size_t len) {
  if (!tables) return group_fail(g, B200CONV_EINVAL, "null table");
  if (len == 0) return B200CONV_OK;
  if (g->lat_D) return group_fail(g, B200CONV_ESTATE, "device-pointer group calls are not available at a fixed latency");
  for (size_t i = 0; i < g->m.size(); ++i) {
    const b200conv* h = g->m[i];
    const std::string who = "member " + std::to_string(i);
    if (h->sticky_cuda_error) return group_member_fail(g, i, B200CONV_ECUDA);
    if (h->lat_D) return group_fail(g, B200CONV_ESTATE, who + " is in fixed-latency mode");
    if (chain && !h->chain.on) return group_fail(g, B200CONV_ESTATE, who + " owns no send / wet chain");
    if (chain && h->stages.empty()) return group_fail(g, B200CONV_ESTATE, who + " has no impulse response");
    if (!in_dev[i] || !out_dev[i]) return group_fail(g, B200CONV_EINVAL, "null buffer of member " + std::to_string(i));
  }
  if (cudaSetDevice(g->device) != cudaSuccess) {
    cudaGetLastError();
    return group_fail(g, B200CONV_ECUDA, "cudaSetDevice failed");
  }
  return B200CONV_OK;
}

// One device-buffer group call: `own(i)` runs member i's own device call.  The sharing members were chosen and
// prepared by the caller (slot.nc, slot.prepared); this launches them, runs the others and orders the streams.
extern "C++" {
template <class Own>
static int group_device_run(b200conv_group* g, bool chain, bool waited, int rc, int sync, Own own) {
  const size_t n = g->m.size();
  bool any_own = false;
  for (size_t i = 0; i < n; ++i) any_own |= !g->slot[i].nc;
  if (!rc && any_own) {
    cudaError_t e = cudaEventRecord(g->ev, g->st);
    for (size_t i = 0; i < n && e == cudaSuccess; ++i)
      if (!g->slot[i].nc) e = cudaStreamWaitEvent(g->m[i]->s_main, g->ev, 0);
    if (e != cudaSuccess) {
      cudaGetLastError();
      rc = group_fail(g, B200CONV_ECUDA, std::string("group: ordering the members' streams: ") + cudaGetErrorString(e));
    }
  }
  group_launch_round(g, chain, nullptr, 0, waited, &rc, true);
  for (size_t i = 0; i < n; ++i)
    if (g->slot[i].prepared) { g->m[i]->grp_ev = g->ev; g->m[i]->grp_st = g->st; }
  for (size_t i = 0; i < n && !rc; ++i) {
    if (g->slot[i].nc) continue;
    b200conv* h = g->m[i];
    if (int mrc = own(i)) { rc = group_member_fail(g, i, mrc); break; }
    cudaError_t e = cudaEventRecord(h->ev_rt, h->s_main);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(g->st, h->ev_rt, 0);
    if (e != cudaSuccess) rc = group_member_fail(g, i, cuda_fail(h, e, "group: ordering the group stream behind the member"));
  }
  if (!rc && sync) {
    if (const cudaError_t e = cudaStreamSynchronize(g->st)) {
      cudaGetLastError();
      return group_fail(g, B200CONV_ECUDA, std::string("group stream: ") + cudaGetErrorString(e));
    }
  }
  return rc;
}
}  // extern "C++"

int b200conv_group_process_device(b200conv_group_t* g, const float* const* in_dev, const size_t* in_stride,
                                  float* const* out_dev, const size_t* out_stride, size_t len, int sync) {
  if (!g) return B200CONV_EINVAL;
  if (int rc = group_device_check(g, false, in_dev && in_stride && out_dev && out_stride, in_dev, out_dev, len))
    return rc;
  if (len == 0) return B200CONV_OK;
  const size_t n = g->m.size();
  int rc = 0;
  bool waited = false;
  for (size_t i = 0; i < n; ++i) {
    GroupSlot& s = g->slot[i];
    s.prepared = s.launched = false;
    s.nc = group_step_ctas(g->m[i], len, false);
    if (!s.nc || rc) continue;
    if ((rc = group_order_behind(g, i, &waited))) continue;
    rc = group_prepare_step(g, i, false, in_dev[i], nullptr, nullptr, in_stride[i], out_dev[i], out_stride[i], len,
                            nullptr, 0, nullptr, &waited, true);
  }
  return group_device_run(g, false, waited, rc, sync, [&](size_t i) {
    return b200conv_process_device(g->m[i], in_dev[i], in_stride[i], out_dev[i], out_stride[i], len, 0);
  });
}

int b200conv_chain_group_process_device(b200conv_group_t* g, const float* const* dry_dev, const size_t* dry_stride,
                                        const float* const* ysend_dev, const float* const* yrev_dev,
                                        float* const* out_dev, const size_t* out_stride, size_t len, int sync) {
  if (!g) return B200CONV_EINVAL;
  if (int rc = group_device_check(g, true, dry_dev && dry_stride && out_dev && out_stride, dry_dev, out_dev, len))
    return rc;
  if (len == 0) return B200CONV_OK;
  const size_t n = g->m.size();
  int rc = 0;
  bool waited = false;
  for (size_t i = 0; i < n; ++i) {
    GroupSlot& s = g->slot[i];
    s.prepared = s.launched = false;
    s.nc = group_step_ctas(g->m[i], len, true);
    if (!s.nc || rc) continue;
    if ((rc = group_order_behind(g, i, &waited))) continue;
    rc = group_prepare_step(g, i, true, dry_dev[i], ysend_dev ? ysend_dev[i] : nullptr,
                            yrev_dev ? yrev_dev[i] : nullptr, dry_stride[i], out_dev[i], out_stride[i], len, nullptr, 0,
                            nullptr, &waited, true);
  }
  return group_device_run(g, true, waited, rc, sync, [&](size_t i) {
    return b200conv_chain_process_device(g->m[i], dry_dev[i], dry_stride[i], ysend_dev ? ysend_dev[i] : nullptr,
                                         yrev_dev ? yrev_dev[i] : nullptr, out_dev[i], out_stride[i], len, 0);
  });
}

void* b200conv_group_stream(const b200conv_group_t* g) { return g ? (void*)g->st : nullptr; }

// A completed b200conv_chain_swap moves the chain to the incoming handle: the caller puts it in the outgoing one's
// place.  The outgoing handle's next own call must still follow the group's event if it holds it.
int b200conv_group_set_member(b200conv_group_t* g, int index, b200conv_t* h) {
  if (!g) return B200CONV_EINVAL;
  if (index < 0 || (size_t)index >= g->m.size()) return group_fail(g, B200CONV_EINVAL, "member index out of range");
  if (!h) return group_fail(g, B200CONV_EINVAL, "null member");
  if (h->cfg.device != g->device) return group_fail(g, B200CONV_EINVAL, "the member is on another device");
  for (size_t j = 0; j < g->m.size(); ++j)
    if (g->m[j] == h && (int)j != index) return group_fail(g, B200CONV_EINVAL, "the handle is already a member");
  b200conv* old = g->m[index];
  if (old != h && old->grp_ev == g->ev) {
    cudaError_t e = cudaSetDevice(g->device);
    if (e == cudaSuccess && old->grp_st) e = cudaEventRecord(g->ev, g->st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(old->s_main, g->ev, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(old->s_post, g->ev, 0);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return group_fail(g, B200CONV_ECUDA, std::string("set_member: ") + cudaGetErrorString(e));
    }
    old->grp_ev = nullptr;
    old->grp_st = nullptr;
  }
  g->m[index] = h;
  return B200CONV_OK;
}

// Every member is checked against b200conv_set_latency's rules before any changes; then each is switched (and cleared)
// in member order.  samples == 0 switches back only the members in fixed-latency mode.
int b200conv_group_set_latency(b200conv_group_t* g, size_t samples) {
  if (!g) return B200CONV_EINVAL;
  const size_t n = g->m.size();
  for (size_t i = 0; i < n; ++i) {
    const b200conv* h = g->m[i];
    const std::string who = "member " + std::to_string(i) + ": ";
    if (h->sticky_cuda_error) return group_member_fail(g, i, B200CONV_ECUDA);
    if (!samples && !h->lat_D) continue;
    if (h->stages.empty()) return group_fail(g, B200CONV_ESTATE, who + "no impulse response loaded");
    if (h->cfg.shard_count > 1) return group_fail(g, B200CONV_ESTATE, who + "fixed-latency mode needs an unsharded handle");
    if (h->p2p_on || h->p2p_tail) return group_fail(g, B200CONV_ESTATE, who + "the slot exchange is attached");
    if (h->swap_peer) return group_fail(g, B200CONV_ESTATE, who + "an IR hot swap is pending");
    const size_t B0 = (size_t)h->stages[0].B;
    if (samples != 0 && (samples % B0 != 0 || samples > 16 * B0))
      return group_fail(g, B200CONV_EINVAL, who + "the latency must be a multiple of the head block, at most 16 head blocks");
  }
  for (size_t i = 0; i < n; ++i) {
    if (!samples && !g->m[i]->lat_D) continue;
    if (int rc = b200conv_set_latency(g->m[i], samples)) return group_member_fail(g, i, rc);
  }
  g->lat_D = samples;
  return B200CONV_OK;
}

size_t b200conv_group_latency(const b200conv_group_t* g) { return g ? g->lat_D : 0; }

int b200conv_clear(b200conv_t* h) {
  REQUIRE_CUDA(h);
  if (int rc = set_device(h)) return rc;
  if (int rc = clear_state(h)) return rc;
  if (h->chain.on) {            // the chain's own history goes with the convolver's
    CU_CHECK(h, cudaMemsetAsync(h->chain.state, 0, 2 * pc::kChainStateStride * sizeof(float), h->s_main));
    CU_CHECK(h, cudaMemsetAsync(h->chain.ring, 0, 2 * h->chain.ring_size * sizeof(float), h->s_main));
    h->chain.ring_pos = 0; h->chain.carry.delay_floor = 0;   // the delay-line length D stays, as delayBuffer's size does
  }
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  lat_restart(h->lat);          // fixed latency: every enqueued step has completed; the next D samples are zeros
  lat_restart(h->chain.lat);
  return p2p_check(h);
}

int b200conv_set_latency(b200conv_t* h, size_t samples) {
  REQUIRE_CUDA(h);
  if (h->stages.empty()) return fail(h, B200CONV_ESTATE, "load an impulse response first");
  if (h->cfg.shard_count > 1) return fail(h, B200CONV_ESTATE, "fixed-latency mode needs an unsharded handle");
  if (h->p2p_on || h->p2p_tail) return fail(h, B200CONV_ESTATE, "fixed-latency mode is not available with the slot exchange");
  if (h->swap_peer) return fail(h, B200CONV_ESTATE, "an IR hot swap is pending on this handle");
  const size_t B0 = (size_t)h->stages[0].B;
  if (samples != 0 && (samples % B0 != 0 || samples > 16 * B0))
    return fail(h, B200CONV_EINVAL, "the latency must be 0 or a multiple of the head block, at most 16 head blocks");
  if (int rc = set_device(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  if (h->s_tail) CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
  lat_free(h->lat); lat_free(h->chain.lat);
  h->lat_D = 0;
  h->lat_waits = 0;
  if (samples) {
    int rc = lat_alloc(h, &h->lat, h->C, h->C, samples, B0, h->hpin_cap);
    if (!rc && h->chain.on) rc = lat_alloc(h, &h->chain.lat, 4, 2, samples, B0, h->hpin_cap);
    if (rc) { lat_free(h->lat); lat_free(h->chain.lat); return rc; }
    h->lat_D = samples;
  }
  return b200conv_clear(h);
}

size_t b200conv_latency(const b200conv_t* h) { return h ? h->lat_D : 0; }

unsigned long long b200conv_latency_waits(const b200conv_t* h) { return h ? h->lat_waits : 0; }

int b200conv_reset(b200conv_t* h) {
  REQUIRE_CUDA(h);
  if (int rc = set_device(h)) return rc;
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  if (h->s_tail) CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
  swap_cancel(h);
  free_all(h);
  h->swap_state = 0;
  return B200CONV_OK;
}

int b200conv_num_stages(const b200conv_t* h) { return h ? (int)h->stages.size() : 0; }

int b200conv_stage(const b200conv_t* h, int s, b200conv_stage_info* out) {
  if (!h || !out || s < 0 || s >= (int)h->stages.size()) return B200CONV_EINVAL;
  const Stage& st = h->stages[s];
  out->block = st.B; out->partitions = st.P_full; out->tap_offset = st.tap_off;
  out->p_begin = st.p_begin; out->p_end = st.p_end;
  return B200CONV_OK;
}

size_t b200conv_ir_len(const b200conv_t* h, int channel) {
  if (!h || channel < 0 || channel >= h->C) return 0;
  return h->ir_len[channel];
}

unsigned long long b200conv_launch_count(const b200conv_t* h) { return h ? h->launches : 0; }

int b200conv_last_sweep_variant(const b200conv_t* h) { return h ? h->last_variant : 0; }

int b200conv_set_option(b200conv_t* h, const char* name, int value) {
  if (!h || !name) return B200CONV_EINVAL;
  const std::string n(name);
  if (n == "rt") h->opt_rt = value != 0;
  else if (n == "fft512") h->opt_fft512 = value != 0;
  else if (n == "slice_keep_tail") h->opt_slice_tail = value != 0;
  else if (n == "stream_alternate") h->opt_stream_alt = value != 0;
  else if (n == "tc") h->opt_tc = value != 0;
  else if (n == "shard_head") {
    if (!h->stages.empty()) return fail(h, B200CONV_ESTATE, "shard_head is set before the impulse response is loaded");
    h->opt_shard_head = value != 0;
  }
  else return fail(h, B200CONV_EINVAL, "unknown option");
  return B200CONV_OK;
}

int b200conv_set_timing(b200conv_t* h, int enable) {
  if (!h) return B200CONV_EINVAL;
  h->timing = enable != 0;
  return B200CONV_OK;
}

int b200conv_last_timing(const b200conv_t* h, float* cmac_ms, float* fft_ms, float* ifft_ms, int* cmac_launches) {
  if (!h) return B200CONV_EINVAL;
  if (cmac_ms) *cmac_ms = h->t_cmac;
  if (fft_ms) *fft_ms = h->t_fft;
  if (ifft_ms) *ifft_ms = h->t_ifft;
  if (cmac_launches) *cmac_launches = h->n_cmac;
  return B200CONV_OK;
}

void* b200conv_stream(const b200conv_t* h) { return h ? (void*)h->s_main : nullptr; }

int b200conv_set_reduce(b200conv_t* h, b200conv_reduce_fn fn, void* user) {
  if (!h) return B200CONV_EINVAL;
  h->reduce = fn; h->reduce_user = user;
  return B200CONV_OK;
}

int b200conv_set_routing(b200conv_t* h, int n_in, const int* in_map, int n_out, const float* mix) {
  if (!h) return B200CONV_EINVAL;
  if (n_in == 0) { h->route_on = false; return B200CONV_OK; }
  if (h->chain.on) return fail(h, B200CONV_ESTATE, "routing cannot be combined with the send / wet chain");
  const int C = h->C;
  if (C > 8 || n_in < 1 || n_in > C || n_out < 1 || n_out > C || !in_map || !mix)
    return fail(h, B200CONV_EINVAL, "routing needs C <= 8, 1 <= n_in, n_out <= C, in_map[C] and mix[n_out*C]");
  for (int c = 0; c < C; ++c)
    if (in_map[c] < 0 || in_map[c] >= n_in) return fail(h, B200CONV_EINVAL, "in_map entry out of range");
  if (h->s_main) { cudaSetDevice(h->cfg.device); cudaStreamSynchronize(h->s_main); if (h->s_post) cudaStreamSynchronize(h->s_post); }
  h->n_in = n_in; h->n_out = n_out;
  for (int c = 0; c < 8; ++c) h->in_map[c] = c < C ? in_map[c] : 0;
  std::memset(h->mix, 0, sizeof(h->mix));
  for (int i = 0; i < n_out * C; ++i) h->mix[i] = mix[i];
  h->route_on = true;
  return B200CONV_OK;
}

size_t b200conv_p2p_blob_size(const b200conv_t* h) { (void)h; return sizeof(P2PRecord) * kP2PBuffers; }

static int p2p_export_impl(b200conv_t* h, void* blob, int mode);
static int p2p_import_impl(b200conv_t* h, const void* all_blobs);

// A failed export / import (CUDA IPC not permitted in this container, out of memory for the exchange
// buffers, ...) releases whatever was set up and leaves the handle usable on the reduce-hook path.
int b200conv_p2p_export(b200conv_t* h, void* blob, int mode) {
  REQUIRE_CUDA(h);
  const int rc = p2p_export_impl(h, blob, mode);
  if (rc != B200CONV_OK && rc != B200CONV_EINVAL && !h->sticky_cuda_error) { const std::string keep = h->err; p2p_release(h); h->err = keep; }
  return rc;
}

int b200conv_p2p_import(b200conv_t* h, const void* all_blobs) {
  REQUIRE_CUDA(h);
  const int rc = p2p_import_impl(h, all_blobs);
  if (rc != B200CONV_OK && !h->sticky_cuda_error) { const std::string keep = h->err; p2p_release(h); h->err = keep; }
  return rc;
}

static int p2p_export_impl(b200conv_t* h, void* blob, int mode) {
  if (!blob) return fail(h, B200CONV_EINVAL, "null blob");
  if (h->cfg.shard_count < 2 || h->cfg.shard_count > 8) return fail(h, B200CONV_ESTATE, "slot exchange needs 2..8 shards");
  const bool tails = tail_layout(h);
  if (tails) {
    if (h->stages.empty()) return fail(h, B200CONV_ESTATE, "load an impulse response first");
    for (size_t si = 1; si < h->stages.size(); ++si)
      if (h->stages[si].B < 64) return fail(h, B200CONV_ESTATE, "the tail slot exchange needs tail blocks of at least 64 samples");
  } else if (h->stages.size() != 1) {
    return fail(h, B200CONV_ESTATE, "slot exchange supports uniform (single-stage) handles, or staged handles with shard_head = 0");
  }
  if (int rc = set_device(h)) return rc;
  if (int rc = tails ? p2p_alloc_tail(h) : p2p_alloc(h)) return rc;
  h->p2p_mode = mode;
  // tail layout: records 0..2 = Tx of stages 1..3 (rank 0 only), 5 = flags; the others stay empty
  void* bufs[kP2PBuffers] = {h->Yx[0], h->Yx[1], h->Hh, h->xout[0], h->xout[1], h->xflags, h->din[0], h->din[1]};
  if (tails) for (int i = 0; i < kP2PBuffers; ++i) bufs[i] = i < 3 ? (void*)h->Tx[i + 1] : (i == 5 ? (void*)h->xflags : nullptr);
  P2PRecord* rec = static_cast<P2PRecord*>(blob);
  for (int i = 0; i < kP2PBuffers; ++i) {
    std::memset(&rec[i], 0, sizeof(P2PRecord));
    rec[i].ptr = (unsigned long long)(uintptr_t)bufs[i];
#if defined(PC_EMULATE)
    rec[i].kind = 1;
#else
    if (mode == 1 || !bufs[i]) {
      rec[i].kind = 1;
    } else {
      rec[i].kind = 2;
      cudaIpcMemHandle_t hd;
      CU_CHECK(h, cudaIpcGetMemHandle(&hd, bufs[i]));
      static_assert(sizeof(hd) == 64, "IPC handle size");
      std::memcpy(rec[i].ipc, &hd, 64);
    }
#endif
  }
  return B200CONV_OK;
}

static int p2p_import_tail(b200conv_t* h, const void* all_blobs) {
  const int G = h->cfg.shard_count, me = h->cfg.shard_rank;
  const P2PRecord* rec = static_cast<const P2PRecord*>(all_blobs);
  for (int r = 0; r < G; ++r)
    for (int i = 0; i < kP2PBuffers; ++i) {
      const P2PRecord& x = rec[r * kP2PBuffers + i];
      // every rank's flags (rank 0 publishes into them), rank 0's Tx (every rank stores its slots there)
      if (!(i == 5 || (r == 0 && i < 3))) continue;
      void* p = (void*)(uintptr_t)x.ptr;
      if (r != me && x.kind != 1) {
#if defined(PC_EMULATE)
        return fail(h, B200CONV_EINVAL, "IPC records in the emulation build");
#else
        cudaIpcMemHandle_t hd;
        std::memcpy(&hd, x.ipc, 64);
        CU_CHECK(h, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
        h->ipc_opened.push_back(p);
#endif
      }
      if (i == 5) h->peer_flags[r] = static_cast<unsigned int*>(p);
      else h->peerTx0[i + 1] = static_cast<float2*>(p);
    }
  // rank 0 keeps the overlap state of every tail stage in its Tx from now on (the reduce-hook path kept it in Y row 0)
  CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
  CU_CHECK(h, cudaStreamSynchronize(h->s_post));
  for (size_t si = 1; si < h->stages.size() && me == 0; ++si) {
    const Stage& s = h->stages[si];
    const size_t row = (size_t)h->C * s.B;
    CU_CHECK(h, cudaMemcpyAsync(h->Tx[si] + (size_t)((h->tx_blocks[si] + 1) & 1) * G * 2 * row, s.Y[s.ybuf],
                                row * sizeof(float2), cudaMemcpyDeviceToDevice, h->s_main));
  }
  CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  h->p2p_tail = true;
  return B200CONV_OK;
}

static int p2p_import_impl(b200conv_t* h, const void* all_blobs) {
  if (all_blobs && h->ttick) {
    if (int rc = set_device(h)) return rc;
    return p2p_import_tail(h, all_blobs);
  }
  if (!all_blobs || !h->Yx[0]) return fail(h, B200CONV_ESTATE, "export before import");
  if (int rc = set_device(h)) return rc;
  const int G = h->cfg.shard_count, me = h->cfg.shard_rank;
  const P2PRecord* rec = static_cast<const P2PRecord*>(all_blobs);
  for (int r = 0; r < G; ++r) {
    void* ptrs[kP2PBuffers];
    for (int i = 0; i < kP2PBuffers; ++i) {
      const P2PRecord& x = rec[r * kP2PBuffers + i];
      if (r == me || x.kind == 1) {
        ptrs[i] = (void*)(uintptr_t)x.ptr;
      } else {
#if defined(PC_EMULATE)
        return fail(h, B200CONV_EINVAL, "IPC records in the emulation build");
#else
        // only the buffers this shard touches are mapped: every peer's Yx + flags, shard 0's Hh + xout
        // (the din records, i >= 6, are only opened if the input broadcast gets enabled)
        const bool needed = (i <= 1) || (i == 5) || (r == 0 && i <= 4);
        ptrs[i] = nullptr;
        if (needed) {
          cudaIpcMemHandle_t hd;
          std::memcpy(&hd, x.ipc, 64);
          void* p = nullptr;
          CU_CHECK(h, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
          h->ipc_opened.push_back(p);
          ptrs[i] = p;
        }
#endif
      }
    }
    h->peerYx[r][0] = static_cast<float2*>(ptrs[0]);
    h->peerYx[r][1] = static_cast<float2*>(ptrs[1]);
    h->peer_flags[r] = static_cast<unsigned int*>(ptrs[5]);
    h->peer_din[r][0] = (r == me || rec[r * kP2PBuffers + 6].kind == 1) ? static_cast<float*>(ptrs[6]) : nullptr;
    h->peer_din[r][1] = (r == me || rec[r * kP2PBuffers + 7].kind == 1) ? static_cast<float*>(ptrs[7]) : nullptr;
    if (r == 0) {
      h->peerHh0 = static_cast<float2*>(ptrs[2]);
      h->peer_xout0[0] = static_cast<float*>(ptrs[3]);
      h->peer_xout0[1] = static_cast<float*>(ptrs[4]);
    }
  }
  h->din_records.assign(reinterpret_cast<const unsigned char*>(all_blobs),
                        reinterpret_cast<const unsigned char*>(all_blobs) + (size_t)G * kP2PBuffers * sizeof(P2PRecord));
  h->p2p_on = true;
  return B200CONV_OK;
}

int b200conv_p2p_set_input_broadcast(b200conv_t* h, int enable) {
  if (!h) return B200CONV_EINVAL;
  if (enable && !h->p2p_on) return fail(h, B200CONV_ESTATE, "input broadcast needs an attached slot exchange");
#if !defined(PC_EMULATE)
  if (enable && h->cfg.shard_rank == 0) {      // map the peers' staging buffers now (cross-process: CUDA IPC)
    if (int rc = set_device(h)) return rc;
    const P2PRecord* rec = reinterpret_cast<const P2PRecord*>(h->din_records.data());
    for (int r = 1; r < h->cfg.shard_count; ++r)
      for (int i = 0; i < 2; ++i) {
        if (h->peer_din[r][i]) continue;
        const P2PRecord& x = rec[r * kP2PBuffers + 6 + i];
        cudaIpcMemHandle_t hd;
        std::memcpy(&hd, x.ipc, 64);
        void* p = nullptr;
        CU_CHECK(h, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
        h->ipc_opened.push_back(p);
        h->peer_din[r][i] = static_cast<float*>(p);
      }
  }
#endif
  h->bcast_in = enable != 0;
  return B200CONV_OK;
}

int b200conv_p2p_detach(b200conv_t* h) {
  if (!h) return B200CONV_EINVAL;
  if (h->s_main) { cudaSetDevice(h->cfg.device); cudaStreamSynchronize(h->s_main); if (h->s_post) cudaStreamSynchronize(h->s_post); }
  if (h->p2p_tail && !h->sticky_cuda_error && h->cfg.shard_rank == 0) {
    // the reduce-hook path takes the overlap state of every tail stage back into Y row 0
    CU_CHECK(h, cudaStreamSynchronize(h->s_tail));
    for (size_t si = 1; si < h->stages.size(); ++si) {
      const Stage& s = h->stages[si];
      const size_t row = (size_t)h->C * s.B;
      CU_CHECK(h, cudaMemcpyAsync(s.Y[s.ybuf], h->Tx[si] + (size_t)((h->tx_blocks[si] + 1) & 1) * h->cfg.shard_count * 2 * row,
                                  row * sizeof(float2), cudaMemcpyDeviceToDevice, h->s_main));
    }
    CU_CHECK(h, cudaStreamSynchronize(h->s_main));
  }
  const int rc = h->sticky_cuda_error ? B200CONV_OK : p2p_check(h);   // a barrier that gave up is reported here at the latest
  h->p2p_on = false;
  h->p2p_tail = false;
  h->bcast_in = false;
  return rc;
}

int b200conv_p2p_set_host_barrier(b200conv_t* h, b200conv_barrier_fn fn, void* user) {
  if (!h) return B200CONV_EINVAL;
  h->host_barrier = fn; h->host_barrier_user = user;
  return B200CONV_OK;
}

#if defined(PC_EMULATE)
// tests/emu only: make the (n+1)-th device allocation from now fail once
void pc_emu_fail_malloc_after(int n) { g_emu_fail_malloc_in = n; }
#endif

void* b200conv_alloc_host(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}
void b200conv_free_host(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
