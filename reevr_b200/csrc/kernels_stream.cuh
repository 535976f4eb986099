// kernels_stream.cuh — K2t k_cmac_stream_tma: the memory-bound FDL sweep of a real-time call (ONE block per
// launch) fed by the TMA engine.
//
//   Y[k] = sum_p H[p][k] * X[xrow0 - p][k]            (FFTConvolver.cpp:176-187, Utilities.cpp:62-111)
//
// Every H and FDL row is read exactly once per block step (algorithmic bytes = actual bytes), so the only thing
// that matters is keeping enough bytes in flight per SM, all the time.  k_cmac_stream_rows did that with batches
// of register loads — load 16 x 16 B per thread, wait, multiply, repeat — which leaves the memory pipe idle
// during every multiply phase and capped at 0.69 of the measured HBM peak on the 120 s IR.  Here a producer
// warp streams whole row segments into a ring of shared-memory stages with 1-D bulk copies
// (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes — SASS UBLKCP) and the 8 consumer warps only
// ever touch shared memory:
//
//   CTA tile      W = min(B, 512) bins x a contiguous slice of the partition range
//   stage         PP partitions: PP H-row segments + PP FDL-row segments of W*8 bytes each, 16 KB per stage for
//                 every B — two 8 KB bulk copies when a tile spans whole rows (B <= 512: consecutive rows are
//                 contiguous), 2*PP copies of 4 KB otherwise; completion counted in bytes on the stage's `full` mbarrier
//   ring          S stages (S*16 KB in flight per CTA, up to 3 CTAs per SM = 192 KB per SM), `empty` mbarriers
//                 (one arrival per consumer warp) hand a stage back to the producer
//   consumers     thread = one bin pair (16 B) x one partition group; RG = 512 / W partition groups per stage
//                 (1 at B >= 512); partial sums go to Y with RED.ADD like the register version
//
// The index arithmetic lives in plain inline functions shared with the CPU emulation (tests/emu), where a memcpy
// stands in for the bulk copy.
#pragma once

#include "kernels.cuh"

namespace pc {

constexpr int kStreamStageBytes = 16384;

constexpr PC_HD int stream_tma_w(int B) { return B < 512 ? B : 512; }                       // bins per CTA tile
constexpr PC_HD int stream_tma_pp(int B) { return kStreamStageBytes / (2 * 8 * stream_tma_w(B)); }   // partitions per stage
constexpr PC_HD int stream_tma_rg(int B) { return 512 / stream_tma_w(B); }                  // partition groups of the 256 consumers

// partition slice of CTA y out of nsplit (same rule as k_cmac_stream_rows)
PC_HD void stream_slice(int P, int nsplit, int y, int* p_lo, int* p_hi) {
  const int per = (P + nsplit - 1) / nsplit;
  *p_lo = y * per;
  *p_hi = (*p_lo + per < P) ? *p_lo + per : P;
}

// skewed slices: weight of slice y = 1 + skew * (1 - 2 y / (nsplit - 1)); boundaries are multiples of `align` partitions
PC_HD int stream_skew_bound(int P, int nsplit, int y, float skew, int align) {
  if (y <= 0) return 0;
  if (y >= nsplit) return P;
  const double f = (double)y * (1.0 + (double)skew) - (nsplit > 1 ? (double)skew * (double)y * (double)(y - 1) / (double)(nsplit - 1) : 0.0);
  long long b = (long long)((double)P * f / (double)nsplit + 0.5);
  b = (b + align / 2) / align * align;
  if (b < 0) b = 0;
  if (b > P) b = P;
  return (int)b;
}
PC_HD void stream_slice_skewed(int P, int nsplit, int y, float skew, int align, int* p_lo, int* p_hi) {
  *p_lo = stream_skew_bound(P, nsplit, y, skew, align);
  *p_hi = stream_skew_bound(P, nsplit, y + 1, skew, align);
}

// stage i of a slice [p_lo, p_hi): first partition and partition count, ascending or descending walk
PC_HD void stream_stage_range(int p_lo, int p_hi, int PP, int i, int descending, int* p0, int* np) {
  if (!descending) {
    *p0 = p_lo + i * PP;
    *np = (p_hi - *p0 < PP) ? p_hi - *p0 : PP;
  } else {
    const int hi = p_hi - i * PP;
    *p0 = (hi - PP > p_lo) ? hi - PP : p_lo;
    *np = hi - *p0;
  }
}

// sources of the j-th partition of the stage that starts at partition p0 (W-bin segments of one row each)
PC_HD const float2* stream_src_h(const StreamParams& P, int c, int k0, int p) {
  return P.H + (long long)c * P.h_cstride + (long long)p * P.B + k0;
}
PC_HD const float2* stream_src_x(const StreamParams& P, int c, int k0, int p) {
  return P.X + (long long)c * P.x_cstride + (P.xrow0 - p) * (long long)P.B + k0;
}

// one consumer thread, one stage: stage memory = [PP][W] H segments followed by [PP][W] FDL segments.
// xrev: the FDL segments were fetched as ONE contiguous run of rows (W == B), i.e. in ascending row = descending
// partition order, so partition j of the stage sits at segment np-1-j.
PC_HD void stream_consume_stage(const float2* stage, int W, int PP, int np, int col, int rg, int RG, bool packed_first,
                                bool xrev, float2* acc /*[2]*/) {
  const float m = packed_first ? 0.0f : 1.0f;
  for (int j = rg; j < np; j += RG) {
    const float2* hp = stage + (long long)j * W + 2 * col;
    const float2* xp = stage + (long long)(PP + (xrev ? np - 1 - j : j)) * W + 2 * col;
    const float2 ha = hp[0], hb = hp[1], xa = xp[0], xb = xp[1];
    float re = fmaf(ha.x, xa.x, acc[0].x);
    re = fmaf(-m * ha.y, xa.y, re);
    const float im = packed_first ? fmaf(ha.y, xa.y, acc[0].y) : fmaf(ha.y, xa.x, fmaf(ha.x, xa.y, acc[0].y));
    acc[0] = make_float2(re, im);
    acc[1].x = fmaf(-hb.y, xb.y, fmaf(hb.x, xb.x, acc[1].x));
    acc[1].y = fmaf(hb.y, xb.x, fmaf(hb.x, xb.y, acc[1].y));
  }
}

#if defined(__CUDACC__)
// ---- mbarrier / bulk-copy primitives (PTX ISA 8.x, sm_90+) -----------------------------------------------
PC_D unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
PC_D void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
PC_D void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
PC_D void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
PC_D void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
// global -> shared bulk copy (bytes % 16 == 0, both addresses 16-byte aligned), completes on `bar`
PC_D void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// grid (B / W, nsplit, C), block 288 = 8 consumer warps + 1 producer warp; dynamic smem = S*16 KB + 16*S bytes.
// With a StreamXchParams argument (Xch = StreamXchParams): the tail slot exchange epilogue.  A tile's value is final
// only once the last of its nsplit CTAs has added its share, so every CTA (empty slices included) takes a ticket of its
// (channel, bin tile) after a release fence; the CTA drawing the last one reads the summed tile back from L2 and stores
// it into this rank's slot on rank 0, then counts the tile; the last tile raises this rank's flag with a system-scope
// release.  Without it (empty pack) the kernel and its parameter block are exactly the plain sweep's.
template <class T> PC_D const T& stream_xch_arg(const T& x) { return x; }

template <int S, class... Xch>
__global__ void __launch_bounds__(288) k_cmac_stream_tma(StreamParams P, Xch... xch) {
  constexpr bool XCH = sizeof...(Xch) > 0;
  extern __shared__ __align__(128) unsigned char pc_stream_smem[];
  float2* ring = reinterpret_cast<float2*>(pc_stream_smem);
  unsigned long long* full = reinterpret_cast<unsigned long long*>(pc_stream_smem + (size_t)S * kStreamStageBytes);
  unsigned long long* empty = full + S;
  const int W = stream_tma_w(P.B), PP = stream_tma_pp(P.B), RG = stream_tma_rg(P.B);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int k0 = blockIdx.x * W;
  int c = blockIdx.z, p_lo, p_hi;
  if (P.interleave) {                                        // launch order = slice-major, channels interleaved
    const int C = gridDim.y / P.nsplit;
    c = blockIdx.y % C;
    stream_slice_skewed(P.P, P.nsplit, blockIdx.y / C, P.skew, PP, &p_lo, &p_hi);
  } else {
    stream_slice(P.P, P.nsplit, blockIdx.y, &p_lo, &p_hi);
  }
  if (p_lo >= p_hi) {                                        // whole CTA (uniform)
    if constexpr (!XCH) return;
    else p_hi = p_lo;                                        // no stage, but the CTA still takes its ticket
  }
  const int nst = (p_hi - p_lo + PP - 1) / PP;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  constexpr int kStageElems = kStreamStageBytes / 8;
  if (warp == 8) {                                           // ---- producer: one elected lane drives the TMA engine
    if (lane == 0) {
      for (int i = 0; i < nst; ++i) {
        const int s = i % S;
        if (i >= S) mbar_wait(&empty[s], ((i / S) - 1) & 1); // the consumers are done with this stage's previous content
        int p0, np;
        stream_stage_range(p_lo, p_hi, PP, i, P.descending, &p0, &np);
        mbar_expect_tx(&full[s], (unsigned)(np * 2 * W * 8));
        float2* st = ring + (size_t)s * kStageElems;
        if (W == P.B) {          // whole rows: the np rows of H (and of the FDL) are one contiguous run -> 2 copies per stage
          bulk_g2s(st, stream_src_h(P, c, k0, p0), (unsigned)(np * W * 8), &full[s]);
          bulk_g2s(st + (size_t)PP * W, stream_src_x(P, c, k0, p0 + np - 1), (unsigned)(np * W * 8), &full[s]);
        } else {
          for (int j = 0; j < np; ++j) {
            bulk_g2s(st + (size_t)j * W, stream_src_h(P, c, k0, p0 + j), (unsigned)(W * 8), &full[s]);
            bulk_g2s(st + (size_t)(PP + j) * W, stream_src_x(P, c, k0, p0 + j), (unsigned)(W * 8), &full[s]);
          }
        }
      }
    }
    return;
  }
  // ---- consumers
  const int col = tid % (W / 2), rg = tid / (W / 2);
  const bool packed_first = (k0 + 2 * col) == 0;
  float2 acc[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
  for (int i = 0; i < nst; ++i) {
    const int s = i % S;
    int p0, np;
    stream_stage_range(p_lo, p_hi, PP, i, P.descending, &p0, &np);
    (void)p0;
    mbar_wait(&full[s], (i / S) & 1);                        // the stage's bytes have landed
    stream_consume_stage(ring + (size_t)s * kStageElems, W, PP, np, col, rg, RG, packed_first, W == P.B, acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + P.yrow0 * P.y_rstride + k0 + 2 * col);
  if (P.nsplit == 1 && RG == 1) {
    *reinterpret_cast<float4*>(y) = make_float4(acc[0].x, acc[0].y, acc[1].x, acc[1].y);
  } else {
    atomicAdd(y + 0, acc[0].x); atomicAdd(y + 1, acc[0].y);
    atomicAdd(y + 2, acc[1].x); atomicAdd(y + 3, acc[1].y);
  }
  if constexpr (XCH) {
    const StreamXchParams& X = stream_xch_arg(xch...);
    // the 256 consumer threads only (named barrier 1): the producer warp has left
    int* last = reinterpret_cast<int*>(pc_stream_smem);       // stage 0 is free: every stage has been consumed
    __threadfence();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (tid == 0) {
      __threadfence();
      unsigned int* tick = X.xtick + (size_t)c * gridDim.x + blockIdx.x;
      const bool is_last = atomicAdd(tick, 1u) == gridDim.y - 1;
      if (is_last) { *tick = 0; __threadfence(); }
      *last = is_last ? 1 : 0;
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (*last) {
      if (rg == 0) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(y));
        *reinterpret_cast<float4*>(X.xdst + (long long)c * P.y_cstride + k0 + 2 * col) = v;
      }
      __threadfence_system();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid == 0) {
        unsigned int* tiles = X.xtick + (size_t)gridDim.x * gridDim.z;
        __threadfence_system();
        if (atomicAdd(tiles, 1u) == gridDim.x * gridDim.z - 1) {
          *tiles = 0;
          __threadfence_system();
          asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(X.xflag), "r"(X.xepoch) : "memory");
        }
      }
    }
  }
}
#else
// CPU emulation (tests/emu): same slices, stages and consumer arithmetic; memcpy stands in for the bulk copies
inline void emu_cmac_stream_tma(EmuDim grid, const StreamParams& P, const StreamXchParams* X = nullptr) {
  const int W = stream_tma_w(P.B), PP = stream_tma_pp(P.B), RG = stream_tma_rg(P.B);
  float2* stage = new float2[kStreamStageBytes / 8];
  for (int cz = 0; cz < grid.z; ++cz)
    for (int by = 0; by < grid.y; ++by)
      for (int bx = 0; bx < grid.x; ++bx) {
        const int k0 = bx * W;
        int c = cz, p_lo, p_hi;
        if (P.interleave) {
          const int C = grid.y / P.nsplit;
          c = by % C;
          stream_slice_skewed(P.P, P.nsplit, by / C, P.skew, PP, &p_lo, &p_hi);
        } else {
          stream_slice(P.P, P.nsplit, by, &p_lo, &p_hi);
        }
        if (p_lo >= p_hi) continue;
        const int nst = (p_hi - p_lo + PP - 1) / PP;
        float2* accs = new float2[2 * 256];
        for (int t = 0; t < 512; ++t) accs[t] = make_float2(0.f, 0.f);
        for (int i = 0; i < nst; ++i) {
          int p0, np;
          stream_stage_range(p_lo, p_hi, PP, i, P.descending, &p0, &np);
          if (W == P.B) {
            std::memcpy(stage, stream_src_h(P, c, k0, p0), (size_t)np * W * 8);
            std::memcpy(stage + (size_t)PP * W, stream_src_x(P, c, k0, p0 + np - 1), (size_t)np * W * 8);
          } else {
            for (int j = 0; j < np; ++j) {
              std::memcpy(stage + (size_t)j * W, stream_src_h(P, c, k0, p0 + j), (size_t)W * 8);
              std::memcpy(stage + (size_t)(PP + j) * W, stream_src_x(P, c, k0, p0 + j), (size_t)W * 8);
            }
          }
          for (int tid = 0; tid < 256; ++tid) {
            const int col = tid % (W / 2), rg = tid / (W / 2);
            stream_consume_stage(stage, W, PP, np, col, rg, RG, (k0 + 2 * col) == 0, W == P.B, accs + 2 * tid);
          }
        }
        for (int tid = 0; tid < 256; ++tid) {
          const int col = tid % (W / 2);
          float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + P.yrow0 * P.y_rstride + k0 + 2 * col);
          const float2* a = accs + 2 * tid;
          if (P.nsplit == 1 && RG == 1) { y[0] = a[0].x; y[1] = a[0].y; y[2] = a[1].x; y[3] = a[1].y; }
          else { y[0] += a[0].x; y[1] += a[0].y; y[2] += a[1].x; y[3] += a[1].y; }
        }
        delete[] accs;
      }
  delete[] stage;
  if (X) {                      // tail slot exchange epilogue: every tile is final here
    for (int c = 0; c < grid.z; ++c)
      std::memcpy(X->xdst + (long long)c * P.y_cstride, P.Y + (long long)c * P.y_cstride + P.yrow0 * P.y_rstride,
                  (size_t)P.B * sizeof(float2));
    *X->xflag = X->xepoch;
  }
}
#endif

// ---------------------------------------------------------------------------------------------------------
// Dynamic variant: the partition range is cut into chunks of `chunk_stages` ring stages and the CTAs of a (channel,
// bin tile) column draw chunk tickets from a global counter instead of owning a fixed slice.  A 35 us kernel whose
// CTAs all stream the same number of bytes still ends ragged (DRAM channel / L2 slice contention differs per SM): with
// tickets the fast CTAs take more chunks and the tail of the kernel shrinks to one chunk.  The producer draws the
// next ticket while it issues the copies of the current chunk (the atomic's round trip hides behind the ring), tells the
// consumers each stage's partition range through shared memory (written before the arrive that opens the stage) and
// closes with an empty stage.  Every CTA draws exactly one ticket beyond the last chunk, so a launch always consumes
// nchunks + nsplit tickets per counter and the host can advance `ticket_base` without ever resetting the counters.
// ---------------------------------------------------------------------------------------------------------
PC_HD int stream_dyn_chunks(int P, int PP, int KS) { return (P + PP * KS - 1) / (PP * KS); }

#if defined(__CUDACC__)
// grid (B / W, nsplit, C), block 288; dynamic smem = S*16 KB + 16*S (barriers) + 8*S (stage descriptors)
template <int S>
__global__ void __launch_bounds__(288) k_cmac_stream_tma_dyn(StreamParams P) {
  extern __shared__ __align__(128) unsigned char pc_stream_smem[];
  float2* ring = reinterpret_cast<float2*>(pc_stream_smem);
  unsigned long long* full = reinterpret_cast<unsigned long long*>(pc_stream_smem + (size_t)S * kStreamStageBytes);
  unsigned long long* empty = full + S;
  int* stage_p0 = reinterpret_cast<int*>(empty + S);      // first partition of the stage
  int* stage_np = stage_p0 + S;                            // partitions in the stage, 0 = no more work
  const int W = stream_tma_w(P.B), PP = stream_tma_pp(P.B), RG = stream_tma_rg(P.B);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int k0 = blockIdx.x * W, c = blockIdx.z;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  constexpr int kStageElems = kStreamStageBytes / 8;
  if (warp == 8) {                                           // ---- producer
    if (lane == 0) {
      unsigned long long* ctr = P.ticket + (size_t)c * gridDim.x + blockIdx.x;
      const int KS = P.chunk_stages, nchunks = stream_dyn_chunks(P.P, PP, KS);
      long long t = (long long)(atomicAdd(ctr, 1ull) - P.ticket_base);
      int i = 0;
      while (t < nchunks) {
        const long long tn = (long long)(atomicAdd(ctr, 1ull) - P.ticket_base);   // next ticket, in flight during this chunk
        const int c_lo = (int)t * PP * KS;
        const int c_hi = (c_lo + PP * KS < P.P) ? c_lo + PP * KS : P.P;
        for (int p0 = c_lo; p0 < c_hi; p0 += PP, ++i) {
          const int s = i % S;
          if (i >= S) mbar_wait(&empty[s], ((i / S) - 1) & 1);
          const int np = (c_hi - p0 < PP) ? c_hi - p0 : PP;
          stage_p0[s] = p0; stage_np[s] = np;
          mbar_expect_tx(&full[s], (unsigned)(np * 2 * W * 8));
          float2* st = ring + (size_t)s * kStageElems;
          if (W == P.B) {
            bulk_g2s(st, stream_src_h(P, c, k0, p0), (unsigned)(np * W * 8), &full[s]);
            bulk_g2s(st + (size_t)PP * W, stream_src_x(P, c, k0, p0 + np - 1), (unsigned)(np * W * 8), &full[s]);
          } else {
            for (int j = 0; j < np; ++j) {
              bulk_g2s(st + (size_t)j * W, stream_src_h(P, c, k0, p0 + j), (unsigned)(W * 8), &full[s]);
              bulk_g2s(st + (size_t)(PP + j) * W, stream_src_x(P, c, k0, p0 + j), (unsigned)(W * 8), &full[s]);
            }
          }
        }
        t = tn;
      }
      const int s = i % S;                                   // closing stage: np = 0
      if (i >= S) mbar_wait(&empty[s], ((i / S) - 1) & 1);
      stage_np[s] = 0;
      mbar_arrive(&full[s]);
    }
    return;
  }
  // ---- consumers
  const int col = tid % (W / 2), rg = tid / (W / 2);
  const bool packed_first = (k0 + 2 * col) == 0;
  float2 acc[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
  bool any = false;
  for (int i = 0;; ++i) {
    const int s = i % S;
    mbar_wait(&full[s], (i / S) & 1);
    const int np = stage_np[s];
    if (np == 0) break;
    any = true;
    stream_consume_stage(ring + (size_t)s * kStageElems, W, PP, np, col, rg, RG, packed_first, W == P.B, acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  if (any) {
    float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + P.yrow0 * P.y_rstride + k0 + 2 * col);
    atomicAdd(y + 0, acc[0].x); atomicAdd(y + 1, acc[0].y);
    atomicAdd(y + 2, acc[1].x); atomicAdd(y + 3, acc[1].y);
  }
}
#else
// CPU emulation: tickets are drawn in CTA order (the first CTA of a column takes every chunk); same stage arithmetic
inline void emu_cmac_stream_tma_dyn(EmuDim grid, const StreamParams& P) {
  const int W = stream_tma_w(P.B), PP = stream_tma_pp(P.B), RG = stream_tma_rg(P.B);
  float2* stage = new float2[kStreamStageBytes / 8];
  const int KS = P.chunk_stages, nchunks = stream_dyn_chunks(P.P, PP, KS);
  for (int c = 0; c < grid.z; ++c)
    for (int bx = 0; bx < grid.x; ++bx) {
      unsigned long long* ctr = P.ticket + (size_t)c * grid.x + bx;
      for (int by = 0; by < grid.y; ++by) {
        const int k0 = bx * W;
        float2* accs = new float2[2 * 256];
        for (int t = 0; t < 512; ++t) accs[t] = make_float2(0.f, 0.f);
        bool any = false;
        for (;;) {
          const long long t = (long long)((*ctr)++ - P.ticket_base);
          if (t >= nchunks) break;
          const int c_lo = (int)t * PP * KS;
          const int c_hi = (c_lo + PP * KS < P.P) ? c_lo + PP * KS : P.P;
          for (int p0 = c_lo; p0 < c_hi; p0 += PP) {
            const int np = (c_hi - p0 < PP) ? c_hi - p0 : PP;
            if (W == P.B) {
              std::memcpy(stage, stream_src_h(P, c, k0, p0), (size_t)np * W * 8);
              std::memcpy(stage + (size_t)PP * W, stream_src_x(P, c, k0, p0 + np - 1), (size_t)np * W * 8);
            } else {
              for (int j = 0; j < np; ++j) {
                std::memcpy(stage + (size_t)j * W, stream_src_h(P, c, k0, p0 + j), (size_t)W * 8);
                std::memcpy(stage + (size_t)(PP + j) * W, stream_src_x(P, c, k0, p0 + j), (size_t)W * 8);
              }
            }
            any = true;
            for (int tid = 0; tid < 256; ++tid) {
              const int col = tid % (W / 2), rg = tid / (W / 2);
              stream_consume_stage(stage, W, PP, np, col, rg, RG, (k0 + 2 * col) == 0, W == P.B, accs + 2 * tid);
            }
          }
        }
        if (any)
          for (int tid = 0; tid < 256; ++tid) {
            const int col = tid % (W / 2);
            float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + P.yrow0 * P.y_rstride + k0 + 2 * col);
            const float2* a = accs + 2 * tid;
            y[0] += a[0].x; y[1] += a[0].y; y[2] += a[1].x; y[3] += a[1].y;
          }
        delete[] accs;
      }
    }
  delete[] stage;
}
#endif

}  // namespace pc
