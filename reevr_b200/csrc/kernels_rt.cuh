// kernels_rt.cuh — K0 k_rt_block: ONE launch per real-time call.
//
// A plugin calls process() with one host block (64..1024 samples) at a time (src/PluginProcessor.cpp:1793 ->
// StereoConvolver::process -> TwoStageFFTConvolver::process -> FFTConvolver::process, FFTConvolver.cpp:155-212).  On the
// multi-kernel path such a call is launch-bound: H2D copy, forward FFT, memset, streaming sweep, inverse FFT, mixdown,
// D2H copy, each a separate stream operation (56 us per call in round 1 for 7 us of work).  This kernel does the
// whole head-stage step of a call of at most one head block in one launch of one thread-block CLUSTER.  A call that
// completes the open block and starts the next one runs phases A-E twice in the launch, once per SEGMENT (the samples
// up to the block boundary, then the rest at the next timeline row), as the reference runs two iterations of its loop
// (FFTConvolver.cpp:164-208):
//
//   cluster = C convolvers x NC CTAs (<= 16 CTAs), 256 threads each
//   A  every CTA of convolver c assembles the open block [samples of earlier calls ; this call's samples ; 0] in shared
//      memory — the new samples are read straight from the caller's pinned host buffer (zero-copy) — and (q = 0)
//      appends them to the open blocks of all stages on the device
//   B  forward real FFT of the open block by the whole CTA (the NC CTAs of a convolver compute it redundantly: 1-2 us,
//      cheaper than a cluster exchange) -> spectrum row Xnew in shared memory; q = 0 also stores it as timeline row `head`
//   C  FDL sweep of the CTA's bin tile [q M/NC, (q+1) M/NC): partition 0 from Xnew in shared memory, partitions >= 1
//      from the timeline (FFTConvolver.cpp:176-187), partition groups reduced through shared memory
//   D  the tile of Y goes into the q = 0 CTA's shared memory through DSMEM (and, if the block completes, to the
//      overlap row of the next block) — cluster barrier
//   E  q = 0: frequency-domain overlap-add with the previous block's spectrum, inverse FFT, look-ahead rings of the
//      tail stages added, the segment's samples written to the caller's pinned host buffer (or, with routing, to CTA
//      0's mix buffer through DSMEM — after the last segment: cluster barrier, CTA 0 applies the mixdown matrix,
//      src/PluginProcessor.cpp:1833-1838)
// The second segment takes partition 1 of its sweep (the first segment's spectrum) from the CTA's own xnew of the first
// segment and its overlap spectrum from the q = 0 CTA's yfull of the first segment, so nothing the launch writes to
// global memory is read back inside it; the cluster barrier of phase D separates the segments.
//
// k_rt_group_steps generalises the crossing call to a walk of up to kRtMaxSteps head blocks (device-buffer group
// calls, RtStepParams).
//
// The host keeps the bookkeeping (fill, head, buffer parity); tail stages whose block completes in the call are
// enqueued on a low-priority stream and consumed one tail period later (TwoStageFFTConvolver.cpp:213-222).
#pragma once

#include "kernels.cuh"

namespace pc {

// The samples of a call that fall into one head block.  A crossing call has two segments; the second starts its block
// and never completes it (a call takes at most one head block).
struct RtSeg {
  int fill, len, complete;   // samples of the block before the segment, samples it takes, it completes the block
  int off;                   // first sample of the segment in the call's input and output
  long long head;            // timeline row of the block
  long long abs0;            // stream position of the block's first sample (look-ahead rings)
  // open blocks of the later stages: the segment's samples are appended at later_fill[s] of later_inbuf[s]
  float* later_inbuf[3]; int later_fill[3];
};

struct RtParams {
  int M, C, NC, P;
  int len;                   // samples of the call
  int nseg; RtSeg seg[2];
  // input: routed input i at in + i * in_stride (pinned host memory, device-accessible, or device memory)
  const float* in; long long in_stride; int in_map[8];
  // stage 0
  float* inbuf0; long long inbuf0_stride;
  const float2* H; long long h_cstride;
  float2* X; long long x_cstride;
  // Yprev: spectrum of the block before seg[0]'s; Ynext: seg[0]'s, stored when seg[0] completes its block
  const float2* Yprev; float2* Ynext; long long y_cstride;
  const float2* tw;
  int n_later; long long later_stride[3];
  // look-ahead rings added on top of the head output
  int n_add; const float* add[3]; long long add_cstride[3]; long long add_mask[3];
  // output: n_out mixed channels (mix_on) or C channels at out + o * out_stride
  float* out; long long out_stride;
  int mix_on, n_out; float mix[64];
  // completion word in pinned host memory (nullptr: none): set to done_val once every output sample is written, so
  // that the caller can spin on it instead of paying the driver's stream-synchronise latency
  unsigned int* done_flag; unsigned int done_val;
  // mode 0: the whole step in this launch.  Head stages too large for one cluster (uniform long IRs) split a call of
  // one segment:
  // mode 1 = FRONT (phases A, B: assemble, forward FFT, timeline row) -> the all-SM TMA sweep (K2t) writes Yt ->
  // mode 2 = BACK (phase E from the global row Yt: overlap-add, inverse FFT, output, overlap row of the next block)
  int mode; const float2* Yt;
};

// The calls of one shape class of a group, one cluster each (k_rt_group), passed by value: about 23 KB, inside the
// 32 764-byte kernel-parameter limit of CUDA >= 12.1 on sm_90
constexpr int kRtGroupMax = 32;
struct RtGroupParams {
  int n;
  RtParams p[kRtGroupMax];
};
static_assert(sizeof(RtGroupParams) <= 32764, "k_rt_group's parameter table exceeds the kernel-parameter limit");

// The step form (k_rt_group_steps, the device-buffer group calls): one member's call of up to kRtMaxSteps head blocks,
// walked in one cluster as consecutive segments (the rest of the open block, whole head blocks, a final partial
// block), each running phases A-E as the reference runs its FFTConvolver::process loop.  `p` carries everything but
// the segments (p.nseg = 0); the kernel derives them from the call's start (rt_step_seg), so the record stays the same
// size for any call length.
constexpr int kRtMaxSteps = 16;
struct RtStepParams {
  RtParams p;
  int fill;                  // samples of the open head block before the call
  long long head;            // its timeline row
  long long abs_pos;         // stream position of the call's first sample
  // later stage s: open block later_inbuf[s] holds later_fill[s] of its later_B[s] samples; the samples after the one
  // boundary where its block completes go to the front of later_alt[s]
  float* later_inbuf[3]; float* later_alt[3]; int later_fill[3]; int later_B[3];
};
struct RtStepGroupParams {
  int n;
  RtStepParams p[kRtGroupMax];
};
static_assert(sizeof(RtStepGroupParams) <= 32764, "k_rt_group_steps' parameter table exceeds the kernel-parameter limit");

// segments of a step-form call
PC_HD int rt_step_count(const RtStepParams& T) {
  const int M = T.p.M, len1 = T.p.len < M - T.fill ? T.p.len : M - T.fill;
  return 1 + (T.p.len - len1 + M - 1) / M;
}
// Segment g of a step-form call.  `complete` marks only the LAST block the call completes: that step alone stores
// the overlap spectrum Ynext, which the host picked with the parity the equivalent one-launch calls would leave (with
// an even number of completed blocks it is Yprev, read by step 0 before any later step stores).
PC_HD RtSeg rt_step_seg(const RtStepParams& T, int g) {
  const int M = T.p.M, len1 = T.p.len < M - T.fill ? T.p.len : M - T.fill;
  RtSeg S;
  S.fill = g ? 0 : T.fill;
  S.off = g ? len1 + (g - 1) * M : 0;
  S.len = T.p.len - S.off < M - S.fill ? T.p.len - S.off : M - S.fill;
  S.complete = (g == (T.fill + T.p.len) / M - 1) ? 1 : 0;
  S.head = T.head + g;
  S.abs0 = T.abs_pos + S.off - S.fill;
  for (int s = 0; s < T.p.n_later; ++s) {
    const int f = T.later_fill[s] + S.off;
    const bool alt = f >= T.later_B[s];
    S.later_inbuf[s] = alt ? T.later_alt[s] : T.later_inbuf[s];
    S.later_fill[s] = alt ? f - T.later_B[s] : f;
  }
  return S;
}

// shared-memory layout of one CTA (float2 units unless noted); xnew and yfull hold one row per segment, MB apart
struct RtSmem {
  int tw, bufA, bufB, xnew, yfull;       // float2 offsets
  int xs, ys, red, mixbuf;               // byte offsets of float / float4 regions
  int bytes;
};
PC_HD int rt_row(int M) { return M < 16 ? 16 : M; }
PC_HD RtSmem rt_smem_layout(int M, int C) {
  RtSmem L;
  const int MB = rt_row(M);
  int o = 0;
  L.tw = o; o += (tw_table_len(M) + 15) & ~15;
  L.bufA = o; o += MB;
  L.bufB = o; o += MB;
  L.xnew = o; o += 2 * MB;
  L.yfull = o; o += 2 * MB;
  int b = o * 8;
  L.xs = b; b += M * 4;
  L.ys = b; b += M * 4;
  L.red = b; b += 256 * 16;
  L.mixbuf = b; b += C * M * 4;
  L.bytes = (b + 15) & ~15;
  return L;
}

// sweep geometry of a CTA: tile of TB = M / NC bins = TB / 2 bin pairs, PG partition groups
PC_HD int rt_pairs(int M, int NC) { return M / NC / 2; }

// first forward pass reads the assembled time block from shared memory
struct RtSmemIn {
  const float* xs; int nv;
  PC_HD int prep(int base) const { return base; }
  PC_HD float2 at(int tok, int off) const {
    const int i0 = 2 * (tok + off), i1 = i0 + 1;
    return make_float2(i0 < nv ? xs[i0] : 0.0f, i1 < nv ? xs[i1] : 0.0f);
  }
};
// last inverse pass writes the scaled time samples of the block to shared memory
struct RtSmemOut {
  float* ys; float scale; int half;
  PC_HD int prep(int base) const { return base; }
  PC_HD void put(int tok, int off, float2 v) const {
    const int n = tok + off;
    if (n >= half) return;
    ys[2 * n] = v.x * scale;
    ys[2 * n + 1] = v.y * scale;
  }
};

// ---- per-thread phase bodies (shared with the CPU emulation) ---------------------------------------------
// A: sample i of the segment's block
PC_HD void rt_assemble(const RtParams& P, const RtSeg& S, int c, int q, int i, float* xs) {
  float v = 0.0f;
  if (i < S.fill) {
    v = P.inbuf0[(long long)c * P.inbuf0_stride + i];
  } else if (i < S.fill + S.len) {
    v = P.in[(long long)P.in_map[c] * P.in_stride + S.off + (i - S.fill)];
    if (q == 0) {
      P.inbuf0[(long long)c * P.inbuf0_stride + i] = v;
      for (int s = 0; s < P.n_later; ++s)
        S.later_inbuf[s][(long long)c * P.later_stride[s] + S.later_fill[s] + (i - S.fill)] = v;
    }
  }
  xs[i] = v;
}

// a timeline pair the same launch may have stored (step form): a coherent load, never the read-only path
PC_HD float4c ld_pair_live(const float2* p) {
#if defined(__CUDA_ARCH__)
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  float4c r; r.a = make_float2(v.x, v.y); r.b = make_float2(v.z, v.w); return r;
#else
  float4c r; r.a = p[0]; r.b = p[1]; return r;
#endif
}

// C: partial sum of one thread: bin pair at k, partitions pg, pg + PG, ...; partition 0 from xnew, partition 1 from
// xprev unless it is nullptr (then from the timeline like the rest).  kLive: timeline rows may have been stored earlier
// in the same launch (step form), read them coherently.
template <bool kLive = false>
PC_HD float4c rt_sweep_thread(const RtParams& P, long long head, int c, int k, int pg, int PG, const float2* xnew,
                              const float2* xprev) {
  const float2* Hk = P.H + (long long)c * P.h_cstride + k;
  const float2* Xk = P.X + (long long)c * P.x_cstride + head * (long long)P.M + k;
  const bool packed_first = (k == 0);
  const float m = packed_first ? 0.0f : 1.0f;
  float2 a0 = make_float2(0.f, 0.f), a1 = make_float2(0.f, 0.f);
  // batches of 8 partitions: 16 independent 16-byte loads in flight per thread before any arithmetic (one SM only
  // reaches its share of the L2 bandwidth with deep memory-level parallelism); the ragged last batch is predicated,
  // partition 0 takes the spectrum of the open block from shared memory
  for (int p = pg; p < P.P; p += 8 * PG) {
    float4c h[8], x[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int pp = p + u * PG;
      if (pp < P.P) {
        h[u] = ld_pair(Hk + (long long)pp * P.M);
        if (pp == 0) { x[u].a = xnew[k]; x[u].b = xnew[k + 1]; }
        else if (pp == 1 && xprev) { x[u].a = xprev[k]; x[u].b = xprev[k + 1]; }
        else x[u] = kLive ? ld_pair_live(Xk - (long long)pp * P.M) : ld_pair(Xk - (long long)pp * P.M);
      } else {
        h[u].a = h[u].b = x[u].a = x[u].b = make_float2(0.f, 0.f);
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      float re = fmaf(h[u].a.x, x[u].a.x, a0.x);
      re = fmaf(-m * h[u].a.y, x[u].a.y, re);
      const float im = packed_first ? fmaf(h[u].a.y, x[u].a.y, a0.y) : fmaf(h[u].a.y, x[u].a.x, fmaf(h[u].a.x, x[u].a.y, a0.y));
      a0 = make_float2(re, im);
      a1.x = fmaf(-h[u].b.y, x[u].b.y, fmaf(h[u].b.x, x[u].b.x, a1.x));
      a1.y = fmaf(h[u].b.y, x[u].b.x, fmaf(h[u].b.x, x[u].b.y, a1.y));
    }
  }
  float4c r; r.a = a0; r.b = a1;
  return r;
}

// E: sample s of the block after the inverse transform: look-ahead rings added
PC_HD float rt_out_sample(const RtParams& P, const RtSeg& S, int c, const float* ys, int s) {
  float r = ys[s];
  for (int a = 0; a < P.n_add; ++a)
    r += P.add[a][(long long)c * P.add_cstride[a] + ((S.abs0 + s) & P.add_mask[a])];
  return r;
}

#if defined(__CUDACC__)
PC_D void rt_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// A CTA may only be written through DSMEM once it is known to have STARTED (its shared memory exists): every CTA
// arrives on the cluster barrier first thing and waits on it right before its first remote store (split barrier, so
// the wait is free by then).
PC_D void rt_cluster_arrive() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
PC_D void rt_cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// step form: a CTA done with a step's shared rows and timeline stores arrives; the next step's phase D waits
PC_D void rt_cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
// generic address of `p` (own shared memory) in CTA `rank` of the cluster
template <class T>
PC_D T* rt_map_rank(T* p, unsigned rank) {
  unsigned long long out;
  asm volatile("mapa.u64 %0, %1, %2;" : "=l"(out) : "l"(reinterpret_cast<unsigned long long>(p)), "r"(rank));
  return reinterpret_cast<T*>(out);
}

// all passes of the forward transform by the whole CTA (256 threads), first pass from the assembled block
template <int M, int PASS>
__device__ __forceinline__ float2* rt_fwd_passes(float2* in, float2* out, const float2* tw, int tid) {
  if constexpr (PASS >= M) {
    return in;
  } else {
    constexpr int R = pass_radix(M, PASS);
    for (int i = tid; i < M / R; i += 256)
      stockham_butterfly<false>(SmemIn{in}, SmemOut{out}, tw + tw_pass_offset(M, PASS), M, PASS, R, i);
    __syncthreads();
    return rt_fwd_passes<M, PASS * R>(out, in, tw, tid);
  }
}
template <int M, int PASS>
__device__ __forceinline__ void rt_inv_passes(float2* in, float2* out, const float2* tw, int tid, float* ys, float scale) {
  constexpr int R = pass_radix(M, PASS);
  if constexpr (PASS * R == M) {       // last pass: scaled samples to shared memory (first half of the transform only)
    for (int i = tid; i < M / R; i += 256)
      stockham_butterfly<true>(SmemIn{in}, RtSmemOut{ys, scale, M / 2}, tw + tw_pass_offset(M, PASS), M, PASS, R, i);
    __syncthreads();
  } else {
    for (int i = tid; i < M / R; i += 256)
      stockham_butterfly<true>(SmemIn{in}, SmemOut{out}, tw + tw_pass_offset(M, PASS), M, PASS, R, i);
    __syncthreads();
    rt_inv_passes<M, PASS * R>(out, in, tw, tid, ys, scale);
  }
}

// one real-time call: launched with cluster dimension (C * NC, 1, 1) = the whole grid
template <int M>
__global__ void __launch_bounds__(256) k_rt_block(RtParams P) {
  const int rank = blockIdx.x;
#include "kernels_rt_step.inc"
}

// The real-time calls of up to kRtGroupMax handles of one shape class (same M, C, NC) in one launch
// (b200conv_group_process): grid n * C * NC, cluster (C * NC, 1, 1); cluster i runs G.p[i] and raises its own member's
// completion word.  The clusters share nothing and never wait for each other, so a grid with more clusters than the
// GPU keeps resident runs them in waves.  The table stays in the kernel-parameter space (__grid_constant__: read in
// place, no local copy), which saves the driver operation of copying it to the device.
template <int M>
__global__ void __launch_bounds__(256) k_rt_group(const __grid_constant__ RtGroupParams G) {
  const int cs = G.p[0].C * G.p[0].NC;
  const RtParams& P = G.p[blockIdx.x / cs];
  const int rank = blockIdx.x % cs;
#include "kernels_rt_step.inc"
}

// The device-buffer group calls (b200conv_group_process_device, b200conv_chain_group_process_device): cluster i walks
// member G.p[i]'s whole call of up to kRtMaxSteps head blocks (step form, RtStepParams); grid and cluster as k_rt_group.
// No completion word: the caller orders its work on the stream.
template <int M>
__global__ void __launch_bounds__(256) k_rt_group_steps(const __grid_constant__ RtStepGroupParams G) {
  const int cs = G.p[0].p.C * G.p[0].p.NC;
  const RtStepParams& T = G.p[blockIdx.x / cs];
  const RtParams& P = T.p;
  const int rank = blockIdx.x % cs;
#define PC_RT_STEPS
#include "kernels_rt_step.inc"
#undef PC_RT_STEPS
}
#else
// CPU emulation (tests/emu): the CTAs of the cluster run phase by phase; a DSMEM store is a store into the other
// CTA's arrays
// T (step form): the call's segments are its step walk, the rows of xnew / yfull alternate, and every step is mixed
// down before the next one
inline void emu_rt_walk(const RtParams& P, const RtStepParams* T) {
  const int M = P.M, n = P.C * P.NC;
  const int MB = rt_row(M);
  struct Cta { float2 *bufA, *bufB, *xnew, *yfull; float *xs, *ys, *mix; float4* red; };
  Cta* ct = new Cta[n];
  for (int r = 0; r < n; ++r) {
    ct[r].bufA = new float2[MB]; ct[r].bufB = new float2[MB]; ct[r].xnew = new float2[2 * MB]; ct[r].yfull = new float2[2 * MB];
    ct[r].xs = new float[M]; ct[r].ys = new float[M]; ct[r].mix = new float[(size_t)P.C * M]; ct[r].red = new float4[256];
  }
  const int nseg = T ? rt_step_count(*T) : P.nseg;
  for (int g = 0; g < nseg; ++g) {
    const RtSeg S = T ? rt_step_seg(*T, g) : P.seg[g];
    const int row = g & 1, prev = (g + 1) & 1;
    // A + B (each phase runs over every CTA before the next, so the second segment's stores into the open block
    // follow every CTA's reads of the first)
    for (int r = 0; r < n && P.mode != 2; ++r) {
      const int c = r / P.NC, q = r % P.NC;
      Cta& t = ct[r];
      float2* xnew = t.xnew + row * MB;
      for (int i = 0; i < M; ++i) rt_assemble(P, S, c, q, i, t.xs);
      float2* res = t.bufA;
      if (M == 1) {
        t.bufA[0] = make_float2(t.xs[0], 0.0f);
      } else {
        const int R0 = pass_radix(M, 1);
        for (int i = 0; i < M / R0; ++i)
          stockham_butterfly<false>(RtSmemIn{t.xs, S.fill + S.len}, SmemOut{t.bufA}, P.tw + tw_pass_offset(M, 1), M, 1, R0, i);
        float2* in = t.bufA; float2* out = t.bufB;
        for (int p = R0; p < M;) {
          const int R = pass_radix(M, p);
          for (int i = 0; i < M / R; ++i) stockham_butterfly<false>(SmemIn{in}, SmemOut{out}, P.tw + tw_pass_offset(M, p), M, p, R, i);
          float2* x = in; in = out; out = x;
          p *= R;
        }
        res = in;
      }
      for (int k = 0; k <= M / 2; ++k) fwd_split(res, xnew, P.tw, M, k);
      if (q == 0) {
        float2* row = P.X + (long long)c * P.x_cstride + S.head * (long long)M;
        for (int k = 0; k < M; ++k) row[k] = xnew[k];
      }
    }
    // C + D  (q = 0 wrote the timeline row before any CTA reads older rows: rows < head only)
    for (int r = 0; r < n && P.mode == 0; ++r) {
      const int c = r / P.NC, q = r % P.NC;
      Cta& t = ct[r];
      const int pairs = rt_pairs(M, P.NC), PG = 256 / pairs;
      for (int tid = 0; tid < 256; ++tid) {
        const int pi = tid % pairs, pg = tid / pairs, k = q * (M / P.NC) + 2 * pi;
        if (pg < PG) {
          const float4c v = rt_sweep_thread(P, S.head, c, k, pg, PG, t.xnew + row * MB, g ? t.xnew + prev * MB : nullptr);
          t.red[tid].x = v.a.x; t.red[tid].y = v.a.y; t.red[tid].z = v.b.x; t.red[tid].w = v.b.y;
        }
      }
      for (int tid = 0; tid < pairs; ++tid) {
        float4 v = t.red[tid];
        for (int gg = 1; gg < PG; ++gg) { const float4 u = t.red[tid + gg * pairs]; v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w; }
        const int k = q * (M / P.NC) + 2 * tid;
        float2* dst = ct[c * P.NC].yfull + row * MB;
        dst[k] = make_float2(v.x, v.y); dst[k + 1] = make_float2(v.z, v.w);
        if (S.complete) {
          float2* yn = P.Ynext + (long long)c * P.y_cstride + k;
          yn[0] = make_float2(v.x, v.y); yn[1] = make_float2(v.z, v.w);
        }
      }
    }
    // E
    for (int c = 0; c < P.C && P.mode != 1; ++c) {
      Cta& t = ct[c * P.NC];
      const float2* Yp = g ? t.yfull + prev * MB : P.Yprev + (long long)c * P.y_cstride;
      const float2* Yt_src = t.yfull + row * MB;
      if (P.mode == 2) {
        Yt_src = P.Yt + (long long)c * P.y_cstride;
        if (S.complete) for (int k = 0; k < M; ++k) P.Ynext[(long long)c * P.y_cstride + k] = Yt_src[k];
      }
      for (int kk = 0; kk <= M / 2; ++kk) inv_pre(Yt_src, Yp, t.bufA, P.tw, M, kk, 1, 0);
      const float scale = 1.0f / (float)M;
      if (M == 1) {
        t.ys[0] = t.bufA[0].x * scale;
      } else {
        float2* in = t.bufA; float2* out = t.bufB;
        for (int p = 1; p < M;) {
          const int R = pass_radix(M, p);
          if (p * R == M) {
            for (int i = 0; i < M / R; ++i)
              stockham_butterfly<true>(SmemIn{in}, RtSmemOut{t.ys, scale, M / 2}, P.tw + tw_pass_offset(M, p), M, p, R, i);
          } else {
            for (int i = 0; i < M / R; ++i) stockham_butterfly<true>(SmemIn{in}, SmemOut{out}, P.tw + tw_pass_offset(M, p), M, p, R, i);
            float2* x = in; in = out; out = x;
          }
          p *= R;
        }
      }
      for (int i = 0; i < S.len; ++i) {
        const float v = rt_out_sample(P, S, c, t.ys, S.fill + i);
        const int at = T ? i : S.off + i;
        if (P.mix_on) ct[0].mix[(size_t)c * M + at] = v; else P.out[(long long)c * P.out_stride + S.off + i] = v;
      }
    }
    // the mixdown: after every step of the step form, after the last segment otherwise
    const int mlen = T ? S.len : P.len, moff = T ? S.off : 0;
    if (P.mix_on && P.mode != 1 && (T || g + 1 == nseg))
      for (int o = 0; o < P.n_out; ++o)
        for (int i = 0; i < mlen; ++i) {
          float acc = 0.0f;
          for (int cc = 0; cc < P.C; ++cc) {
            const float mm = P.mix[o * P.C + cc];
            if (mm != 0.0f) acc = fmaf(mm, ct[0].mix[(size_t)cc * M + i], acc);
          }
          P.out[(long long)o * P.out_stride + moff + i] = acc;
        }
  }
  if (P.done_flag && P.mode != 1) *P.done_flag = P.done_val;
  for (int r = 0; r < n; ++r) {
    delete[] ct[r].bufA; delete[] ct[r].bufB; delete[] ct[r].xnew; delete[] ct[r].yfull;
    delete[] ct[r].xs; delete[] ct[r].ys; delete[] ct[r].mix; delete[] ct[r].red;
  }
  delete[] ct;
}

inline void emu_rt_block(const RtParams& P) { emu_rt_walk(P, nullptr); }

// the clusters of a group launch one after the other
inline void emu_rt_group(const RtGroupParams& G) {
  for (int i = 0; i < G.n; ++i) emu_rt_block(G.p[i]);
}
inline void emu_rt_group_steps(const RtStepGroupParams& G) {
  for (int i = 0; i < G.n; ++i) emu_rt_walk(G.p[i].p, &G.p[i]);
}
#endif

// Completion word of a fixed-latency step that ran as several launches and copies (b200conv_set_latency): one thread,
// queued behind the step's last operation on the same stream, makes everything before it visible system-wide and
// raises the sequence value.
#if defined(__CUDACC__)
static __global__ void k_seq_flag(unsigned int* flag, unsigned int val) {
  __threadfence_system();
  *reinterpret_cast<volatile unsigned int*>(flag) = val;
  __threadfence_system();
}
#else
inline void emu_seq_flag(unsigned int* flag, unsigned int val) { *flag = val; }
#endif

}  // namespace pc
