/*
 * b200conv.h — C ABI of the H100-native partitioned-convolution engine.
 *
 * Drop-in boundary for the hot path of tiagolr/reevr (REEV-R): everything behind
 *   fftconvolver::FFTConvolver::{init,process,clear,reset}          libs/FFTConvolver/FFTConvolver.h:62-80
 *   fftconvolver::TwoStageFFTConvolver::{init,process,reset,clear}  libs/FFTConvolver/TwoStageFFTConvolver.h:65-83
 *   StereoConvolver::{loadImpulse,process,reset,clear}              src/dsp/StereoConvolver.h:20-25
 * i.e. AudioFFT::fft/ifft (AudioFFT.h:135-158), ComplexMultiplyAccumulate / Sum (Utilities.h:319-344)
 * and the frequency-domain delay line they operate on.  Plain C: opaque handle, raw pointers
 * and sizes only, no C++/torch types, never throws.  One handle = C independent mono
 * convolvers ("channels", each with its own impulse response) that share the block schedule
 * and are processed by the same kernel launches (C = 1 reproduces one reference object;
 * C = 2 / 4 reproduces one StereoConvolver in stereo / quad mode).
 *
 * Status codes: 0 = ok, negative = error (message via b200conv_last_error).  There is NO CPU
 * fall-back: if CUDA is unavailable every call fails loudly with B200CONV_ECUDA.
 *
 * Threading contract = the reference's (FFTConvolver.h:44-47): one caller at a time per
 * handle; different handles are fully independent (own streams, own device arena).
 */
#ifndef B200CONV_H
#define B200CONV_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200CONV_OK        0
#define B200CONV_EINVAL   -1   /* bad argument (e.g. block size 0 — the reference's init()==false) */
#define B200CONV_ECUDA    -2   /* CUDA runtime error / no device */
#define B200CONV_ESTATE   -3   /* call not valid in this state */
#define B200CONV_ENOMEM   -4

typedef struct b200conv b200conv_t;

typedef struct b200conv_config {
  int n_channels;        /* C >= 1 mono convolvers in this handle                                  */
  int device;            /* CUDA device ordinal                                                     */
  int max_batch_blocks;  /* head-stage blocks processed per internal launch group (0 = default 4224) */
  int shard_rank;        /* partition-range shard owned by this handle (multi-GPU), 0 <= rank < n   */
  int shard_count;       /* number of shards (1 = unsharded)                                        */
  int cmac_variant;      /* 0 = auto; >0 selects a specific CMAC kernel variant (tuning/bench):     */
                         /* 22 packed-FMA batched, 40 tensor cores (wgmma),   100..108 streaming,   */
                         /* 41 line FFTs along the block index (overlap-save, FP32),                */
                         /* 42 four-step 2^21-point FFTs of the samples (overlap-save, FP32)        */
} b200conv_config;

/* Lifetime ------------------------------------------------------------------------------- */
b200conv_t* b200conv_create(const b200conv_config* cfg);     /* NULL only if cfg is invalid/OOM */
void        b200conv_destroy(b200conv_t* h);
const char* b200conv_last_error(const b200conv_t* h);         /* "" if none                      */

/* IR load (replaces FFTConvolver::init FFTConvolver.cpp:93-152 and
 * TwoStageFFTConvolver::init TwoStageFFTConvolver.cpp:87-148).  ir[c] points to ir_len[c]
 * float32 taps of channel c (host memory, copied during the call).  Same semantics as the
 * reference: trailing taps with |h| < 1e-6 are trimmed, block sizes are rounded up to a power
 * of two, an empty IR is legal (process() then writes zeros), block size 0 -> B200CONV_EINVAL. */
int b200conv_init_uniform(b200conv_t* h, size_t block, const float* const* ir, const size_t* ir_len);
int b200conv_init_twostage(b200conv_t* h, size_t head_block, size_t tail_block,
                           const float* const* ir, const size_t* ir_len);
/* Non-uniform schedule (beyond the reference): stage s uses block size blocks[s] for the taps
 * [offsets[s], offsets[s+1]) (offsets[0] = 0, last stage runs to the end of the IR).  Stage 0
 * is the zero-latency head; for s >= 1 offsets[s] must be a multiple of blocks[s] and >= blocks[s]. */
int b200conv_init_stages(b200conv_t* h, int n_stages, const size_t* blocks, const size_t* offsets,
                         const float* const* ir, const size_t* ir_len);

/* Streaming convolution (replaces FFTConvolver::process FFTConvolver.cpp:155-212 and
 * TwoStageFFTConvolver::process TwoStageFFTConvolver.cpp:151-233): in[c] / out[c] are HOST
 * pointers to `len` float32 samples per channel; any len >= 0, zero added latency, output is
 * complete on return.  in/out may not alias (same rule as the reference, SURVEY §8a-2).
 * A call of at most one head block (len <= head block size, whether or not it crosses a head-block
 * boundary, so any host block size a REEV-R host uses) is one cluster-kernel launch with zero-copy
 * I/O, plus the tail blocks it completes, on handles whose later stages' blocks are multiples of the
 * head block; uniform handles whose head stage is too large for one cluster run such a call as
 * three launches if it stays inside the open block and on the multi-kernel path if it crosses.
 * Long calls are internally cut into block batches and pipelined over PCIe. */
int b200conv_process(b200conv_t* h, const float* const* in, float* const* out, size_t len);

/* Same, with DEVICE-resident buffers: channel c at in_dev + c*in_stride (floats).  Asynchronous
 * on the handle's stream unless sync != 0.  This is the throughput path bench.py times; a call of
 * at most one head block takes the same one-launch path as b200conv_process. */
int b200conv_process_device(b200conv_t* h, const float* in_dev, size_t in_stride,
                            float* out_dev, size_t out_stride, size_t len, int sync);

/* Time-slice sharding of an offline / batch call over several GPUs — no collective, no exchange.  Every GPU holds
 * the WHOLE convolver (a handle with the same IR and the same history, shard_count = 1); for one call of `len`
 * samples GPU `slice_rank` of `slice_count` produces only the output blocks [a, b) of its contiguous time slice
 * (ceil(T / slice_count) blocks each) and writes out[c][a*B .. b*B) — the rest of `out` is left untouched for the
 * other GPUs (which are given the same `in` / `out` arrays, e.g. one shared, pinned host buffer, or run in other
 * threads of the same process).  The sum over partitions of FFTConvolver.cpp:179-187 needs the spectra of the P
 * blocks in front of a slice: the GPU uploads and forward-transforms that history (FFT only, no sweep), convolves its
 * slice, then transforms the last P blocks of the call, so that after the call EVERY handle is in the state the
 * whole call would have left (the next call — sliced or not — continues the stream).  Per GPU: T/G + P blocks
 * of H2D and forward FFT, T/G blocks of sweep, inverse FFT and D2H.  Pays off when T/G >> P (batch jobs); for
 * streaming calls and IRs longer than the batch use the partition-range shards below.
 * Needs: uniform (single-stage) handle, no routing, no open block, len a multiple of the block size
 * (else B200CONV_ESTATE, nothing processed). */
int b200conv_process_sliced(b200conv_t* h, const float* const* in, float* const* out, size_t len,
                            int slice_rank, int slice_count);
int b200conv_process_device_sliced(b200conv_t* h, const float* in_dev, size_t in_stride, float* out_dev, size_t out_stride,
                                   size_t len, int slice_rank, int slice_count, int sync);

/* FFTConvolver::clear (FFTConvolver.cpp:80-90) / TwoStageFFTConvolver::clear (:69-84): forget
 * all audio history, keep the IR.  Implemented as a TRUE clear (also mid-block), see DESIGN.md. */
int b200conv_clear(b200conv_t* h);
/* FFTConvolver::reset (FFTConvolver.cpp:56-78): drop the IR and all device memory. */
int b200conv_reset(b200conv_t* h);

/* Fixed-latency mode (beyond the reference; a plugin reports it to its host, e.g. JUCE setLatencySamples).
 * samples = 0: zero latency (default).  Otherwise a multiple of the head block B0 with B0 <= samples <= 16 * B0.
 * With latency D, b200conv_process writes out[c][i] = y[c][n0 + i - D], y = what the same handle returns at zero
 * latency fed head-block calls, n0 = the call's first absolute sample; samples before 0 are exact zeros.  Any call
 * length and the routing work as usual.  b200conv_chain_process delays the whole mix the same way (dry and wet stay
 * aligned); b200conv_chain_update takes effect at the next head-block step; b200conv_chain_swap needs equal latencies
 * on both handles (else B200CONV_EINVAL) and counts its warm-up and fade in head-block steps.
 * The call only copies the samples into a pinned ring, enqueues one step per head block the samples complete (one
 * launch on the real-time shapes) and copies out the output of blocks earlier calls completed: it waits for the device
 * only if a needed block has not finished yet.
 * Call after the IR is loaded; it clears the handle (b200conv_clear).  init_* and b200conv_reset return the handle to
 * zero latency.  b200conv_clear waits for the enqueued steps; the next D samples are zeros again.
 * B200CONV_EINVAL: not a multiple / out of range.  B200CONV_ESTATE: no IR, a sharded handle, an attached slot exchange,
 * a pending IR hot swap.  On a latency handle b200conv_process_device*, b200conv_process_sliced*, b200conv_prime and
 * b200conv_process_xfade fail with B200CONV_ESTATE.  A latency handle is driven through either b200conv_process or
 * b200conv_chain_process, not both. */
int    b200conv_set_latency(b200conv_t* h, size_t samples);
size_t b200conv_latency(const b200conv_t* h);
/* calls in fixed-latency mode that had to wait for device work (the host's underrun indicator); reset by set_latency */
unsigned long long b200conv_latency_waits(const b200conv_t* h);

/* Groups of handles (beyond the reference): the real-time calls of several handles in one launch, for hosts that drive
 * several instances from one audio callback (a session with several reverbs, one handle per zone of a game engine).
 * Semantics: b200conv_group_process(g, in, out, len) is exactly b200conv_process(members[i], in[i], out[i], len) for
 * every i, in member order; outputs and handle states are what those calls would leave, within float rounding.
 * A member QUALIFIES for a call when b200conv_process would run it as one cluster launch (a call of at most one head
 * block on a head stage that fits one cluster) and it is unsharded, not in fixed-latency mode or in fixed-latency mode
 * at the group's latency (b200conv_group_set_latency, below), timing is off and it has zero-copy staging and a
 * completion word.  Qualifying members with the same head block, channel count and cluster
 * width form one shape class: one launch per class (per 32 members), one cluster per member; routing / mixdown, the
 * stages and whether the call crosses a head-block boundary may differ inside a class.  Every other member (split-mode
 * uniform long IRs, C > 8, len above the head block, a latency handle, timing on, a tail shard, no IR, ...) runs its
 * ordinary b200conv_process inside the group call, after the shared launches are enqueued.  The host waits once per
 * call for all shared launches.
 * Errors: b200conv_group_create returns NULL for n < 1, n > 64, a NULL or repeated member, members on different
 * devices, or when it runs out of memory or CUDA resources.  b200conv_group_process checks every member's arguments
 * (in / out / in[i] / out[i] NULL with len > 0, as b200conv_process does) before it enqueues anything: B200CONV_EINVAL
 * (B200CONV_ECUDA for a member whose CUDA context failed) and no member advances.  len == 0 does nothing.  A CUDA error
 * inside the call returns the first error; members already processed stay processed.
 * Lifetime / threading: members must outlive the group; while a group call runs no other thread may call a member.
 * Between group calls the members stay fully usable on their own (device calls, clear, reset, init_* included).
 * Steady state: a group call allocates nothing, never synchronises, makes one driver launch per shape class and no
 * event operation unless a member completes a tail block or has unsynchronised work queued on its own stream. */
typedef struct b200conv_group b200conv_group_t;
b200conv_group_t*  b200conv_group_create(b200conv_t* const* members, int n);
void               b200conv_group_destroy(b200conv_group_t* g);
const char*        b200conv_group_last_error(const b200conv_group_t* g);
/* in[i] / out[i]: what b200conv_process(members[i], in[i], out[i], len) takes */
int                b200conv_group_process(b200conv_group_t* g, const float* const* const* in,
                                          float* const* const* out, size_t len);
/* launches of the group's shared calls, chain calls included (members count only the tail blocks they enqueue) */
unsigned long long b200conv_group_launch_count(const b200conv_group_t* g);
/* Send / wet chain calls of the group: b200conv_chain_group_process(g, dry, ysend, yrev, out, len) is exactly
 * b200conv_chain_process(members[i], dry[i], ysend ? ysend[i] : NULL, yrev ? yrev[i] : NULL, out[i], len) for every i,
 * in member order; outputs, filter states, predelay rings and convolver stages are what those calls would leave,
 * within float rounding.  dry[i] / out[i]: the member's L / R buffers.  A member shares the group's launches when
 * b200conv_chain_process would run its call as one zero-copy piece through one cluster launch: it has a chain, no fixed
 * latency or fixed latency at the group's latency (then the conditions of b200conv_group_set_latency apply instead of
 * the length ones) and no pending hot swap, len <= the staging size and <= Lmax - head block, the "rt" option on, a head stage
 * that fits one cluster, and the conditions of b200conv_group_process.  The shared members take one send launch per
 * 32 members, one cluster launch per shape class and one wet launch per 32 members, and the host waits once, on one
 * completion word of the group.  Every other member runs its own b200conv_chain_process inside the call.
 * Errors, checked for every member before anything is enqueued (no member advances): B200CONV_ESTATE for a member
 * without a chain or without an impulse response, B200CONV_EINVAL for a NULL dry / out table or entry with len > 0,
 * B200CONV_ECUDA for a member whose CUDA context failed.  len == 0 does nothing. */
int                b200conv_chain_group_process(b200conv_group_t* g, const float* const* const* dry,
                                                const float* const* ysend, const float* const* yrev,
                                                float* const* const* out, size_t len);
/* Replace member `index` by h, e.g. by the incoming handle of a completed b200conv_chain_swap (state 3), which then
 * owns the chain.  B200CONV_EINVAL for an index out of range, h NULL, h already a member at another index or on
 * another device.  Allocates nothing; the outgoing handle stays usable on its own. */
int                b200conv_group_set_member(b200conv_group_t* g, int index, b200conv_t* h);
/* Fixed latency for the whole group (the host reports one latency for its set of instances).  samples != 0: every
 * member is checked against b200conv_set_latency's rules first (IR loaded, unsharded, no slot exchange, no pending hot
 * swap, samples a multiple of its head block and at most 16 of them); a refusal returns B200CONV_ESTATE / B200CONV_EINVAL
 * with the member's index in b200conv_group_last_error and changes no member.  Then b200conv_set_latency(member,
 * samples) runs on every member in member order (each is cleared) and the group records `samples`.  If that fails
 * part-way with a CUDA or memory error, the members before the failing one are switched, the failing one is at zero
 * latency, the later ones are unchanged, and the group keeps its previous latency.  samples == 0: the members in
 * fixed-latency mode go back to zero latency (and are cleared), and group calls are those above again.
 * A member SHARES the steps of a group call when b200conv_latency(member) equals the group's non-zero latency and each
 * of its head-block steps would be one cluster launch: unsharded, timing off, zero-copy rings, a head stage that fits
 * one cluster, and for b200conv_chain_group_process chain rings, the "rt" option on and no pending hot swap.  Any call
 * length works.  Every other member (a latency set later on its own by b200conv_set_latency, init_* or b200conv_reset;
 * a split-mode uniform long IR; C > 8; ...) runs its own call inside the group call, as above.
 * Semantics stay those of the group calls: outputs, filter states, rings and b200conv_latency_waits are what the
 * members' own fixed-latency calls would leave, within float rounding (output D samples late, zeros before).
 * Steady state of the sharing members: a call whose samples complete no head block of any of them makes no launch, no
 * event operation and no wait unless an output block is still pending on the device.  A call that completes steps
 * makes, per round (the r-th step of every member completing more than r head blocks in the call), one k_rt_group
 * launch per shape class and 32 members, plus for the chain one send launch per send width (one for equal head blocks)
 * and one wet launch per 32 members, and records one event.  The group call allocates nothing. */
int                b200conv_group_set_latency(b200conv_group_t* g, size_t samples);
size_t             b200conv_group_latency(const b200conv_group_t* g);
/* Group calls on device buffers.  b200conv_group_process_device(g, in_dev, in_stride, out_dev, out_stride, len, sync)
 * gives member i exactly what b200conv_process_device(members[i], in_dev[i], in_stride[i], out_dev[i], out_stride[i],
 * len, 0) would; b200conv_chain_group_process_device what b200conv_chain_process_device(members[i], dry_dev[i],
 * dry_stride[i], ysend_dev ? ysend_dev[i] : NULL, yrev_dev ? yrev_dev[i] : NULL, out_dev[i], out_stride[i], len, 0)
 * would (ysend_dev / yrev_dev and their entries may be NULL: envelope 1).  Outputs, stage states, filter states and
 * predelay rings are those calls', in member order, within float rounding; in-place and aliasing rules are theirs.
 * A member SHARES the group's launches when a one-launch call of it would qualify for b200conv_group_process (length
 * and staging aside) and its head stage fits one cluster, its call touches at most 16 head blocks counting from its
 * current fill, and every later stage's block is a multiple of the head block, completes at most once in the call and
 * its completed block's output is first needed after the call (REEV-R's head 64..1024 / tail 8192 shapes: calls up to
 * min(16 head blocks, 8192) samples).  A chain member also needs what b200conv_chain_group_process asks, no pending
 * hot swap, and len < 16384.  Sharing members cost one cluster launch per shape class and 32 members for the whole
 * call, which walks each member's head blocks inside its cluster (chain: one send launch per send width before, one
 * wet launch per 32 members after).  Every other member runs its own device call inside the group call.
 * Stream contract, on the group's stream b200conv_group_stream(g):
 *  - work the caller enqueued on it before the call happens before the call reads any member's input;
 *  - work enqueued on it after the call returns sees every member's output;
 *  - members that run their own call are ordered both ways with it (one event at the start, one per such member at
 *    the end); sharing members need no event;
 *  - sync != 0 returns only after the call has completed; the call never spins on a completion word and allocates
 *    nothing; each member's next own call is ordered behind it.
 * Errors, checked for every member before anything is enqueued (no member advances): B200CONV_EINVAL for a NULL
 * table, or a NULL entry with len > 0; B200CONV_ESTATE when the group has a non-zero latency, a member is in
 * fixed-latency mode, or (chain) a member has no chain or no impulse response; B200CONV_ECUDA for a member whose CUDA
 * context failed.  len == 0 does nothing.  b200conv_group_launch_count counts the shared launches. */
int                b200conv_group_process_device(b200conv_group_t* g, const float* const* in_dev,
                                                 const size_t* in_stride, float* const* out_dev,
                                                 const size_t* out_stride, size_t len, int sync);
int                b200conv_chain_group_process_device(b200conv_group_t* g, const float* const* dry_dev,
                                                       const size_t* dry_stride, const float* const* ysend_dev,
                                                       const float* const* yrev_dev, float* const* out_dev,
                                                       const size_t* out_stride, size_t len, int sync);
/* the cudaStream_t of the group's calls */
void*              b200conv_group_stream(const b200conv_group_t* g);

/* Introspection --------------------------------------------------------------------------- */
typedef struct b200conv_stage_info {
  size_t block;        /* B_s                                  */
  size_t partitions;   /* P_s (max over channels, post-trim)    */
  size_t tap_offset;   /* first IR tap handled by this stage     */
  size_t p_begin;      /* partition range owned by this shard    */
  size_t p_end;
} b200conv_stage_info;
int    b200conv_num_stages(const b200conv_t* h);
int    b200conv_stage(const b200conv_t* h, int s, b200conv_stage_info* out);
size_t b200conv_ir_len(const b200conv_t* h, int channel);    /* post-trim tap count            */
/* Kernel launches issued by this handle since creation (bench.py's gpu_launches). */
unsigned long long b200conv_launch_count(const b200conv_t* h);
/* Form of the FDL sweep (FFTConvolver.cpp:176-187) the last launch resolved to: 22 / 26 = packed-FMA batched sweep,
 * 40 = tensor-core sweep (wgmma f16, 3xFP16 with power-of-two scales), 41 = line-FFT sweep (4096-point FP32 overlap-save along
 * the block index, kernels_lfft.cuh), 42 = four-step sweep (2^21-point FP32 overlap-save of the samples themselves, in place
 * of the group's forward FFT, sweep and inverse FFT, kernels_fourstep.cuh; whole-block, block-aligned B = 512 groups of an
 * unsharded single-stage handle with at most 961 partitions; a forced 42 on any other shape is B200CONV_EINVAL),
 * 100..108 = streaming forms.  For benchmarks and tests. */
int b200conv_last_sweep_variant(const b200conv_t* h);
/* Tuning / A-B switches: "rt" (1 = real-time calls of at most one head block run as ONE cluster-kernel launch
 * with zero-copy I/O, see b200conv_process; 0 = multi-kernel path), "fft512" (1 = register-resident FFT kernels for block size 512),
 * "slice_keep_tail" (default 1; 0 = b200conv_process_sliced does not upload / transform the last P blocks of the call:
 * the handle then only supports a following sliced call whose slice starts >= P blocks into the call — every rank
 * but 0 of a steady batch job — until the next b200conv_clear), "stream_alternate" (default 1: the streaming sweep
 * walks its partition slices in alternating directions from launch to launch, see kernels_stream.cuh), "tc" (default 1:
 * launch groups of >= 4096 blocks with <= 961 partitions run the sweep on the tensor cores, kernels_tc.cuh, and groups of
 * >= 16384 such blocks as FFT convolutions along the block index, kernels_lfft.cuh, and B = 512 groups of >= 32768 blocks
 * that qualify for it (see b200conv_last_sweep_variant) as four-step FFT convolutions of the samples, kernels_fourstep.cuh;
 * 0 = always the packed-FMA sweep).
 * "shard_head" (sharded handles; set before b200conv_init_*, B200CONV_ESTATE once an IR is loaded; default 1 = every
 * stage partition-range sharded): 0 = tail layout — shard 0 holds the head stage (stage 0) whole and keeps the one-launch
 * real-time call, the other shards hold none of it (no head FFT, sweep or output, only the input buffering of the
 * later stages), and only the stages >= 1 are partition-range sharded.  Their partial spectra are summed on shard 0 by
 * the reduce hook, called once per completed tail block (one row of C*B complex bins) and never for the head, or by the
 * tail slot exchange (b200conv_p2p_export / import below).  Applies to every init, up to 4 stages. */
int    b200conv_set_option(b200conv_t* h, const char* name, int value);
/* Device time (ms) spent in the dominant CMAC kernel / all kernels during the last
 * b200conv_process_device call, measured with CUDA events on the handle's stream
 * (enabled by b200conv_set_timing(h, 1); adds two event records per kernel). */
int    b200conv_set_timing(b200conv_t* h, int enable);
int    b200conv_last_timing(const b200conv_t* h, float* cmac_ms, float* fft_ms, float* ifft_ms,
                            int* cmac_launches);
void*  b200conv_stream(const b200conv_t* h);                  /* cudaStream_t of the head path  */

/* Multi-GPU partition-range sharding (SURVEY §8e): with shard_count > 1 every handle computes
 * the partial spectrum sum over its own partition range; between the CMAC sweep and the
 * inverse FFT the engine calls `reduce(user, dev_ptr, n_floats, stream)` which must sum the
 * buffer over all shards into shard 0 (ncclReduce on that stream).  Only shard 0 produces output;
 * the other shards do not write their `out` buffers. */
typedef int (*b200conv_reduce_fn)(void* user, float* dev_buf, size_t n_floats, void* cuda_stream);
int b200conv_set_reduce(b200conv_t* h, b200conv_reduce_fn fn, void* user);

/* Optional I/O routing of a multi-convolver handle (SURVEY 8f-1: StereoConvolver as ONE call incl.
 * the true-stereo mixdown of src/PluginProcessor.cpp:1833-1838).  Convolver c reads input buffer
 * in_map[c] (0 <= in_map[c] < n_in) and output o = sum_c mix[o*C + c] * y_c, computed on the device.
 * Afterwards b200conv_process / b200conv_process_device take n_in input and n_out output buffers
 * (e.g. quad reverb: in = {L, R}, convolvers {LL, RR, LR, RL} <- {0, 1, 0, 1}, out L = LL + RL,
 * out R = RR + LR: 2 buffers each way over PCIe instead of 4).  n_in = 0 removes the routing.
 * Limits: C <= 8, n_in <= 8, n_out <= 8; not combinable with the slot exchange. */
int b200conv_set_routing(b200conv_t* h, int n_in, const int* in_map, int n_out, const float* mix);

/* The per-sample chain REEV-R runs on the host around the convolver (SURVEY 8f-4 and the rest of 8f-1), on the device:
 *   send: dry * ysend -> low cut (HP) if lowcut_hz > 20 -> high cut (LP) if highcut_hz < 20000 -> predelay ring
 *         (src/PluginProcessor.cpp:1639-1653, 1766-1790; filters = src/dsp/Filter.cpp state-variable sections, slope
 *         0/1/2 = 6/12/24 dB, coefficients as Filter::init / getCoeff compute them);
 *   convolvers LL, RR[, LR, RL] on the chain's L / R (a C = 2 or C = 4 handle);
 *   wet:  L = LL (+ RL), R = RR (+ LR when true_stereo) ; * yrev ; mid/side width ; out = drygain * dry + wetgain * wet
 *         (src/PluginProcessor.cpp:1832-1876).
 * dry[2] / out[2]: host L, R; ysend / yrev: per-sample send and reverb envelopes (NULL = 1).  One H2D of the dry
 * signal + envelopes and one D2H of the final mix per call, whatever the number of convolvers.
 * b200conv_chain_configure(h, cfg) after the IR is loaded (resets filter states and the delay line; NULL disables);
 * b200conv_chain_update(h, cfg) for parameter changes while playing. */
typedef struct b200conv_chain_config {
  double srate;
  float lowcut_hz;  int lowcut_slope;
  float highcut_hz; int highcut_slope;
  int predelay;                 /* samples */
  float width, drygain, wetgain;
  int true_stereo;              /* quad handles: add RL to the left and LR to the right */
} b200conv_chain_config;
int b200conv_chain_configure(b200conv_t* h, const b200conv_chain_config* cfg);
/* New chain parameters without a reset: what REEV-R's onSlider and the per-block parameter reads of processBlock do
 * (src/PluginProcessor.cpp:837-848, 1151-1188).  b200conv_chain_configure is prepareToPlay: it clears the filters and
 * the delay line.  b200conv_chain_update takes the same struct and applies it from the start of the next
 * b200conv_chain_process call (once per call, however the call is cut into pieces):
 *   - cut frequencies / slopes: new coefficients, filter state continues; a filter switched off keeps its state; each
 *     filter keeps the reference's separate 6 dB and 12 / 24 dB state variables across slope switches;
 *   - predelay: the delay history is kept and read at the new delay.  The delay line has the reference's length
 *     D = (int)(2 * srate); a predelay beyond D sets D = 2 * predelay and the delay history reads zero from there
 *     (the reference clears its delay line), while the send history an IR hot swap replays is kept;
 *   - width, drygain, wetgain, true_stereo: from the next call, including the crossfade of a pending swap.
 * It applies to the handle that owns the chain, including the live handle while a swap is pending (an update before
 * the warm-up call changes the filters the warm-up replays through); at the end of the fade the configuration moves to
 * the incoming handle with the chain.
 * Real-time safe: no CUDA call, allocation, synchronise or launch.  The one exception is a predelay that grows the
 * delay line past what the device ring holds: the ring is then reallocated (synchronising the handle's streams).
 * B200CONV_ESTATE: the handle owns no chain (never configured, the incoming handle of a pending swap, or a handle that
 * gave its chain away).  B200CONV_EINVAL: cfg == NULL, a slope outside 0..2, predelay < 0, or an srate different from
 * the configured one (a new rate needs b200conv_chain_configure).  On any error nothing changes. */
int b200conv_chain_update(b200conv_t* h, const b200conv_chain_config* cfg);
int b200conv_chain_process(b200conv_t* h, const float* const* dry, const float* ysend, const float* yrev,
                           float* const* out, size_t len);

/* The same chain on DEVICE-resident buffers, for batch work from device memory (a PyTorch pipeline, an offline render):
 * dry L at dry_dev, R at dry_dev + dry_stride; the mix at out_dev / out_dev + out_stride (floats); ysend_dev / yrev_dev
 * one row each (NULL = 1).  out_dev == dry_dev with out_stride == dry_stride runs in place; any other overlap is
 * undefined.  Asynchronous on b200conv_stream(h) unless sync != 0, like b200conv_process_device: no staging copy and no
 * synchronise between the pieces (at most Lmax - B0 samples each) the call is cut into.
 * Semantics are b200conv_chain_process's for the same samples and call lengths, and the two entries can be mixed on one
 * handle: b200conv_chain_update takes effect at the next call; a pending b200conv_chain_swap warms up in the first call,
 * fades, and hands the chain over at the end of the completing call, after which the incoming handle's stream is ordered
 * behind this call's work.
 * Pieces shorter than 16 384 samples run the send filters exactly as b200conv_chain_process does, so a call made of such
 * pieces is bit for bit the host call.  Longer pieces run the send filters as a chunked scan spread over the whole GPU
 * (same FP32 chunk arithmetic, FP64 scan, different chunking): within float rounding of the host call, not bit-identical.
 * B200CONV_ESTATE: no chain, or a fixed-latency handle.  B200CONV_EINVAL: dry_dev or out_dev NULL.  len == 0 does
 * nothing. */
int b200conv_chain_process_device(b200conv_t* h, const float* dry_dev, size_t dry_stride, const float* ysend_dev,
                                  const float* yrev_dev, float* out_dev, size_t out_stride, size_t len, int sync);

/* b200conv_chain_process_device with parameter changes at sample offsets inside the call, for renders with automation
 * of the low / high cut, predelay, width, dry / wet gain or true stereo (the envelopes already vary per sample).
 * events[i].cfg takes effect at sample events[i].offset of the call.  The output equals, within float rounding, the
 * call cut at every event offset into consecutive b200conv_chain_process_device calls with
 * b200conv_chain_update(h, &events[i].cfg) made just before the call that starts at events[i].offset; everything
 * b200conv_chain_update documents holds per event, at that sample (filter states continue, the 6 dB and 12 / 24 dB
 * state variables are kept across slope switches, a filter switched off keeps its state, the delay line is read at
 * the new predelay, and a predelay beyond D sets D = 2 * predelay with the delay history reading zero from that
 * sample on).  Afterwards the handle's configuration is the last event's.
 * events: host memory, read during the call; offsets strictly increasing and below len.  n_events == 0 is
 * b200conv_chain_process_device exactly (events may then be NULL).  Every event is checked before anything is
 * enqueued; on any error nothing changes.  Asynchronous like b200conv_chain_process_device, except that a predelay
 * whose D outgrows the device ring reallocates the ring once, before the first launch (synchronising the handle's
 * stream, as b200conv_chain_update does).  The first call that needs them allocates the segmented send form's
 * scratch (sized for the handle's batch) and a table of one row per event; a call with more events than any before
 * grows the table; both happen before the call's first launch.  A call waits for the previous events call's table
 * copy (the start of that call's work on the stream) before it rewrites the table's staging.
 * The convolvers run the pieces of b200conv_chain_process_device unchanged; the send filters of a long piece over
 * several events run a segmented form of the whole-GPU scan.
 * B200CONV_ESTATE: no chain, a fixed-latency handle, or an IR hot swap pending (b200conv_chain_swap_state 1 or 2).
 * B200CONV_EINVAL: dry_dev or out_dev NULL, events NULL with n_events > 0, or a bad event (b200conv_chain_update's
 * rules, an srate other than the configured one, offsets out of order or not below len). */
typedef struct b200conv_chain_event {
  size_t offset;                /* sample of the call at which cfg takes effect, 0 <= offset < len */
  b200conv_chain_config cfg;    /* the struct b200conv_chain_update takes */
} b200conv_chain_event;
int b200conv_chain_process_device_events(b200conv_t* h, const float* dry_dev, size_t dry_stride,
                                         const float* ysend_dev, const float* yrev_dev, float* out_dev,
                                         size_t out_stride, size_t len, const b200conv_chain_event* events,
                                         size_t n_events, int sync);

/* IR hot-swap inside the device chain (src/PluginProcessor.cpp:1655-1668, 1694-1756, 1799-1830).
 * `live` has the chain configured; `incoming` holds the new IR (e.g. b200conv_init_twostage_recalc).
 * The next b200conv_chain_process(live, ...) does the warm-up (0.25 s of send history, replayed on the device in
 * ONE batched call, host_block = the host's samplesPerBlock), then the calls crossfade for ceil(srate * 0.05)
 * samples. At the end of the call where the fade completes, the chain (filter states, predelay / warmer ring,
 * configuration, staging) moves to `incoming`, and `live` no longer has a chain. The caller then swaps its
 * pointers, exactly like std::swap(loadConvolver, convolver).
 * The handles may differ in channel count (stereo <-> quad).  B200CONV_ESTATE: `live` has no chain, `incoming` has no
 * IR or already owns a chain, or a swap is pending on either; while a swap is pending, b200conv_chain_configure on
 * either handle and any init on either handle fail with B200CONV_ESTATE too.  B200CONV_EINVAL: the same handle twice,
 * different devices, sharded or routed handles, unequal staging sizes, host_block == 0.  b200conv_reset /
 * b200conv_destroy of either handle cancels the swap (the live handle continues alone); b200conv_clear(live) clears
 * the chain's history as usual and leaves `incoming` as it is. */
int b200conv_chain_swap(b200conv_t* live, b200conv_t* incoming, size_t host_block);
/* 0 = no swap pending, 1 = armed (warm-up at the next chain call), 2 = fading,
 * 3 = completed: this handle gave its chain away.                  */
int b200conv_chain_swap_state(const b200conv_t* h);

/* IR hot-swap helpers (SURVEY 8f-2; the reference replays a 0.25 s "warmer" ring through the freshly
 * loaded convolver call by call and crossfades two convolvers on the host for 50 ms,
 * src/PluginProcessor.cpp:1695-1750,1800-1830).
 * b200conv_prime: feeds `len` samples of history through the handle in ONE batched call, no output.
 * b200conv_process_xfade: runs both handles on the same input and returns
 *   out[c][i] = (1 - a_i) * old[c][i] + a_i * new[c][i],  a_i = clamp(alpha0 + i*alpha_step, 0, 1),
 *   blended on the device (one D2H).  Both handles: same device, same channel count / routing, unsharded. */
int b200conv_prime(b200conv_t* h, const float* const* in, size_t len);
int b200conv_process_xfade(b200conv_t* h_old, b200conv_t* h_new, const float* const* in, float* const* out,
                           size_t len, float alpha0, float alpha_step);

/* Fused multi-GPU path ("slot exchange", uniform single-stage handles with shard_count > 1):
 * the sweep kernel's epilogue stores each partial spectrum row straight into the exchange buffer of
 * the GPU that owns the row's time slice (peer memory over NVLink), a flag barrier follows, every
 * GPU runs the inverse FFT on its own slice (summing the shard_count partial slots while loading)
 * and writes the audio directly into shard 0's output exchange buffer.  No NCCL call on the data
 * path.  Set-up: every shard exports a blob, the caller all-gathers the blobs (rank order) and
 * every shard imports the concatenation.  mode 0 = CUDA IPC handles (one process per GPU),
 * mode 1 = raw pointers (all shards in one process on one device; tests).
 * Handles with shard_head = 0 (any stage schedule) attach the TAIL slot exchange instead: the single-block sweep of
 * every tail block stores this shard's partial spectrum into its slot on shard 0 and raises its flag; shard 0 waits for
 * the flags on its lowest-priority stream and runs the inverse FFT over the summed slots into the look-ahead ring, off
 * the path of the real-time call.  Tail blocks need B >= 64.  Every shard gets the same input and call lengths (no input
 * broadcast).  Staged handles with a sharded head (shard_head = 1) are refused: the fused exchange of those is for
 * uniform (single-stage) handles only. */
size_t b200conv_p2p_blob_size(const b200conv_t* h);
int    b200conv_p2p_export(b200conv_t* h, void* blob, int mode);
int    b200conv_p2p_import(b200conv_t* h, const void* all_blobs /* shard_count * blob_size bytes */);
/* Back to the reduce-hook path (e.g. when the import failed on some other shard: all shards must agree). */
int    b200conv_p2p_detach(b200conv_t* h);
/* Host-pointer calls (b200conv_process) on a slot-exchange handle: with the input broadcast enabled only
 * shard 0 reads its `in` buffers and crosses PCIe; it stores every launch group into the peers' staging
 * buffers over NVLink (the other shards' `in` arguments are ignored).  Off by default (round 1: implemented and
 * covered by the in-process tests, not yet timed on a multi-GPU box). */
int    b200conv_p2p_set_input_broadcast(b200conv_t* h, int enable);
/* Host-side barrier used instead of the flag kernel by the CPU emulation build (tests only). */
typedef int (*b200conv_barrier_fn)(void* user);
int    b200conv_p2p_set_host_barrier(b200conv_t* h, b200conv_barrier_fn fn, void* user);

/* SURVEY 8f-3 (a "next" row, not part of the hot path): the STFT decay-EQ of the IR shaping,
 * Impulse::applyDecay (src/dsp/Impulse.cpp:602-648), on the device: `ir` (host, n float32 taps) is
 * processed in place; lut = 2049 per-bin decay factors per STFT block (Impulse.cpp:566-590 builds them
 * on the host from the EQ bands); srate as in the reference (sets the early-reflection blocks that are
 * left untouched).  Stand-alone call: no handle, own temporary device buffers. */
int b200conv_ir_decay_eq(int device, float* ir, size_t n, const double* lut, double srate);

/* SURVEY 8f-3, the pipeline: the device-resident subset of Impulse::recalcImpulse (src/dsp/Impulse.cpp:297-360) in the
 * reference's order — auto gain (:313-320, :703-720), reverse (:322-330), trim (:437-470), gain (:472-486), decay EQ
 * (:602-648), clip (:488-501), attack / decay envelope (:651-680) — on the raw taps of all 2 / 4 channels with ONE upload.
 * (No resampling, stretch or parametric EQ, and a ready-made decay table: b200conv_ir_recalc below adds those.)
 *   b200conv_ir_shape            shaped taps back to the host (out[c] needs room for n floats, *out_len taps written);
 *   b200conv_init_*_shaped       shape on the device and build the partition spectra straight from the device-resident
 *                                taps — the IR never returns to the host between shaping and FFTConvolver::init. */
typedef struct b200conv_ir_shape_params {
  int autogain, reverse;
  float trim_left, trim_right;      /* fractions of the length removed at either end */
  float gain;
  const double* decay_lut;          /* 2049 per-bin decay factors (Impulse.cpp:566-590), NULL = no decay EQ */
  double srate;
  int clip;
  float attack, decay;              /* fractions of the (trimmed) length */
} b200conv_ir_shape_params;
int b200conv_ir_shape(int device, const float* const* raw, int n_channels, size_t n, const b200conv_ir_shape_params* sp,
                      float* const* out, size_t* out_len);
int b200conv_init_uniform_shaped(b200conv_t* h, size_t block, const float* const* raw, size_t n,
                                 const b200conv_ir_shape_params* sp);
int b200conv_init_twostage_shaped(b200conv_t* h, size_t head_block, size_t tail_block, const float* const* raw, size_t n,
                                  const b200conv_ir_shape_params* sp);

/* SURVEY 8f-3, the whole of Impulse::recalcImpulse (src/dsp/Impulse.cpp:299-360) on the device, in the reference's order:
 * auto gain -> reverse -> resampling to the project rate (:362-389) -> stretch (:391-434) -> trim -> gain -> parametric EQ
 * (:503-537) -> decay EQ (:539-599, the 2049-entry table is built from the bands inside) -> clip -> envelope.
 * Resampling and stretch follow JUCE's ResamplingAudioSource (linear interpolation, second-order low pass in double
 * precision before down-sampling / after up-sampling); the EQ bands are REEV-R's SVF sections (src/dsp/SVF.cpp), with
 * Off and unknown modes run as a peak band, as Impulse.cpp:511-519 does.  Channel order {LL, RR[, LR, RL]}; one upload.
 *   b200conv_ir_recalc_len     output taps per channel (host arithmetic only; 0 if p is NULL); can exceed n
 *                              (up-sampling and positive stretch);
 *   b200conv_ir_recalc         taps back to the host: out[c] has room for out_cap >= b200conv_ir_recalc_len(n, p) floats;
 *   b200conv_init_*_recalc     recalculate and build the partition spectra from the device-resident taps (no download).
 * B200CONV_EINVAL: a NULL pointer, srate or ir_srate <= 0, more than 8 bands or a mode outside 0..9, out_cap too small. */
typedef struct b200conv_eq_band {
  int mode;                         /* SVF::Mode: 0 LP, 1 BP, 2 HP, 3 LS, 4 HS, 5 PK, 6 BS, 7 HP6, 8 LP6, 9 Off */
  float freq, q, gain;
} b200conv_eq_band;
typedef struct b200conv_ir_recalc_params {
  double ir_srate, srate;           /* rate of the IR file / of the session (Impulse::irsrate / srate)               */
  float stretch;                    /* Impulse::stretch (-1..1 in REEV-R): rate factor 2^stretch                       */
  int autogain, reverse;
  float trim_left, trim_right, gain;
  int n_param_eq; const b200conv_eq_band* param_eq;   /* applyParamEQ, <= 8 bands (0: off)                        */
  int n_decay_eq; const b200conv_eq_band* decay_eq;   /* applyDecayEQ, <= 8 bands (0: off)                        */
  float decay_rate;                 /* Impulse::decayRate                                                              */
  int clip;
  float attack, decay;              /* fractions of the (trimmed) length                                               */
} b200conv_ir_recalc_params;
size_t b200conv_ir_recalc_len(size_t n, const b200conv_ir_recalc_params* p);
int b200conv_ir_recalc(int device, const float* const* raw, int n_channels, size_t n, const b200conv_ir_recalc_params* p,
                       float* const* out, size_t out_cap, size_t* out_len);
int b200conv_init_uniform_recalc(b200conv_t* h, size_t block, const float* const* raw, size_t n,
                                 const b200conv_ir_recalc_params* p);
int b200conv_init_twostage_recalc(b200conv_t* h, size_t head_block, size_t tail_block, const float* const* raw, size_t n,
                                  const b200conv_ir_recalc_params* p);

/* Pinned host memory helpers (staging buffers for the e2e path).  register/unregister page-lock memory the caller
 * owns (e.g. a shared-memory region several per-GPU processes write their output slices into). */
void* b200conv_alloc_host(size_t bytes);
void  b200conv_free_host(void* p);
int   b200conv_register_host(void* p, size_t bytes);
int   b200conv_unregister_host(void* p);

/* Version / build info string ("b200conv x.y sm_90a ..."). */
const char* b200conv_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200CONV_H */
