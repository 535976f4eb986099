// kernels.cuh — sm_90a kernels of the partitioned-convolution hot path.
//
//   K1 k_fwd_fft      X[t]  = RFFT_2B([x_t ; 0_B])        replaces CopyAndPad + AudioFFT::fft
//                                                         (FFTConvolver.cpp:172-173, AudioFFT.cpp:114-137);
//                                                         the same kernel builds the IR spectra H[p]
//                                                         (FFTConvolver::init, FFTConvolver.cpp:129-137)
//   K2 k_cmac_batch2  Y[t]  = sum_p H[p] (.) X[t-p]       replaces the ComplexMultiplyAccumulate sweep over
//      (batched, float2-pair FMA; k_cmac_batch = scalar A/B variant)   the frequency-domain delay line
//   K2s k_cmac_stream_rows  same sum, one block per launch,  (FFTConvolver.cpp:176-187, Utilities.cpp:62-111)
//      memory-bound (k_cmac_stream: generic fallback, B < 64)
//   K3 k_inv_fft_ola  y_t   = IRFFT_2B(Y[t] + (-1)^k Y[t-1])[0:B] (+ look-ahead stage outputs)
//                                                         replaces AudioFFT::ifft + Sum + overlap save
//                                                         (FFTConvolver.cpp:190-204, AudioFFT.cpp:139-159,
//                                                         Utilities.cpp:34-51) and the tail sums of
//                                                         TwoStageFFTConvolver::process (:166-193)
//
// Spectrum layout (private to the engine, as in the reference where spectra never cross the API,
// FFTConvolver.h:83-96): interleaved float2, exactly B entries per 2B-point real transform;
// entry 0 packs the two purely real bins as (DC, Nyquist), entries 1..B-1 are bins 1..B-1.
// Rows are therefore B*8 bytes — a power of two, 32-byte-sector aligned for every B >= 4.
//
// Also here: the multi-GPU slot-exchange pieces (cmac_store epilogue, sum_partials, k_p2p_barrier), the
// device mixdown / crossfade / row-copy helpers (k_mix, k_xfade, k_copy_rows).
//
// The per-thread / per-phase bodies are plain inline functions so that tests/emu (g++) can run
// the identical index arithmetic on the CPU; the __global__ wrappers only add the thread
// geometry and the barriers between phases.
#pragma once

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#define PC_HD __host__ __device__ __forceinline__
#define PC_D __device__ __forceinline__
#else
#include <cmath>
#define PC_HD inline
struct float2 { float x, y; };
static inline float2 make_float2(float a, float b) { float2 r; r.x = a; r.y = b; return r; }
struct float4 { float x, y, z, w; };
static inline float4 make_float4(float a, float b, float c, float d) { float4 r; r.x = a; r.y = b; r.z = c; r.w = d; return r; }
#endif

namespace pc {

// ------------------------------------------------------------------------------------------
// complex helpers
// ------------------------------------------------------------------------------------------
PC_HD float2 c_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
PC_HD float2 c_sub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
PC_HD float2 c_mul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
PC_HD float2 c_conj(float2 a) { return make_float2(a.x, -a.y); }

constexpr PC_HD int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// radix of the Stockham pass that starts with sub-transform length p (M total):
// radix-8 wherever possible, the remainder as 4*4 / 4 / 2  (M = 512 -> 8,8,8; 128 -> 8,4,4; 8192 -> 8,8,8,4,4)
constexpr PC_HD int pass_radix(int M, int p) {
  const int l = ilog2(M / p);
  return l == 1 ? 2 : ((l == 2 || l == 4) ? 4 : 8);
}

// threads per transform of the FFT kernels: one warp up to M = 1024, the whole CTA above
constexpr PC_HD int fft_threads(int M) { return M <= 1024 ? 32 : (M / 8 < 512 ? M / 8 : 512); }
constexpr PC_HD bool fft_warp_mode(int M) { return M <= 1024; }

// 4-point DFT in place (forward: e^{-2*pi*i/4}; INV: conjugate)
template <bool INV>
PC_HD void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 b0 = c_add(a0, a2), b1 = c_sub(a0, a2), b2 = c_add(a1, a3);
  const float2 d = c_sub(a1, a3);
  const float2 b3 = INV ? make_float2(-d.y, d.x) : make_float2(d.y, -d.x);   // -/+ i * d
  a0 = c_add(b0, b2);
  a1 = c_add(b1, b3);
  a2 = c_sub(b0, b2);
  a3 = c_sub(b1, b3);
}

// ------------------------------------------------------------------------------------------
// Shared-memory addressing and twiddle-table layout of the FFT kernels.
//
// swz(): bank swizzle of the M-element work buffers.  Every index keeps its aligned 16-element
// group (so contiguous accesses stay conflict-free); the low 4 bits are XOR-ed with bits 4..6 so
// that the strided Stockham stores of the radix-8 passes (stride 8 in pass 1, 8 contiguous
// elements every 64 in pass 2) hit 16 distinct 8-byte banks per half-warp.
//
// Twiddle table (device array `tw`, 3M/2 float2, built in double on the host):
//   [0, M/2]                          split twiddles  exp(-2*pi*i*k/(2M))
//   [tw_pass_offset(M,p) + (r-1)*p+k] pass twiddles   exp(-2*pi*i*r*k/(p*R)), k < p, r = 1..R-1
// i.e. for a given pass and r the k-index is contiguous, which makes the reads of consecutive
// lanes consecutive words (the sum of (R-1)*p over the earlier passes telescopes to p-1).
// ------------------------------------------------------------------------------------------
PC_HD int swz(int a) { return a ^ ((a >> 4) & 7) ^ (((a >> 6) & 1) << 3); }
constexpr PC_HD int tw_pass_offset(int M, int p) { return M / 2 + 1 + (p - 1); }
constexpr PC_HD int tw_table_len(int M) { return M / 2 + 1 + (M - 1); }

// Accessors used by the butterflies.  swz() is linear over GF(2) (XOR of shifted copies of the
// index), and inside a butterfly the base index (i resp. j) and the per-leg offsets (r*stride resp.
// m*p) occupy disjoint bit ranges, hence swz(base + off) = swz(base) ^ swz(off): the base is
// swizzled once per butterfly and every leg costs one XOR with a compile-time constant.
struct SmemIn {
  const float2* buf;
  PC_HD int prep(int base) const { return swz(base); }
  PC_HD float2 at(int tok, int off) const { return buf[tok ^ swz(off)]; }
};
struct SmemOut {
  float2* buf;
  PC_HD int prep(int base) const { return swz(base); }
  PC_HD void put(int tok, int off, float2 v) const { buf[tok ^ swz(off)] = v; }
};
// forward first pass reads the time-domain block straight from global memory:
// z[n] = x[2n] + i*x[2n+1], zero beyond the nv valid samples (the [x ; 0] padding is never stored)
struct FwdGlobalIn {
  const float* src; int nv;
  PC_HD int prep(int base) const { return base; }
  PC_HD float2 at(int tok, int off) const {
    const int i0 = 2 * (tok + off), i1 = i0 + 1;
    return make_float2(i0 < nv ? src[i0] : 0.0f, i1 < nv ? src[i1] : 0.0f);
  }
};

// ------------------------------------------------------------------------------------------
// One Stockham autosort pass (radix R, sub-transform length p -> p*R), butterfly i in [0, M/R):
//   k = i mod p ; inputs in(i + r*M/R) * w^(r*k) ; outputs out((i-k)*R + k + m*p) = DFT_R[m]
// `in` / `out` are accessor functors so the first / last pass can touch global memory directly.
// ------------------------------------------------------------------------------------------
template <bool INV, class In, class Out>
PC_HD void stockham_butterfly(In in, Out out, const float2* twp, int M, int p, int R, int i) {
  const int k = i & (p - 1);
  const int j = (i - k) * R + k;
  const int stride = M / R;
  const int ti = in.prep(i);
  const int to = out.prep(j);
  if (R == 8) {
    float2 a[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) a[r] = in.at(ti, r * stride);
    if (k != 0) {
#pragma unroll
      for (int r = 1; r < 8; ++r) {
        float2 w = twp[(r - 1) * p + k];
        if (INV) w.y = -w.y;
        a[r] = c_mul(a[r], w);
      }
    }
    // radix-2 stage on (r, r+4), W8 twiddles on the odd half, then two DFT4
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float2 s = c_add(a[r], a[r + 4]), d = c_sub(a[r], a[r + 4]);
      a[r] = s; a[r + 4] = d;
    }
    const float h = 0.70710678118654752440f;
    if (!INV) {   // W8 = e^{-i*pi/4}
      a[5] = make_float2(h * (a[5].x + a[5].y), h * (a[5].y - a[5].x));
      a[6] = make_float2(a[6].y, -a[6].x);
      a[7] = make_float2(h * (a[7].y - a[7].x), -h * (a[7].x + a[7].y));
    } else {
      a[5] = make_float2(h * (a[5].x - a[5].y), h * (a[5].x + a[5].y));
      a[6] = make_float2(-a[6].y, a[6].x);
      a[7] = make_float2(-h * (a[7].x + a[7].y), h * (a[7].x - a[7].y));
    }
    dft4<INV>(a[0], a[1], a[2], a[3]);     // even outputs X[0], X[2], X[4], X[6]
    dft4<INV>(a[4], a[5], a[6], a[7]);     // odd outputs  X[1], X[3], X[5], X[7]
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      out.put(to, (2 * m) * p, a[m]);
      out.put(to, (2 * m + 1) * p, a[4 + m]);
    }
  } else if (R == 4) {
    float2 a0 = in.at(ti, 0), a1 = in.at(ti, stride), a2 = in.at(ti, 2 * stride), a3 = in.at(ti, 3 * stride);
    if (k != 0) {
      float2 w1 = twp[k], w2 = twp[p + k], w3 = twp[2 * p + k];
      if (INV) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
      a1 = c_mul(a1, w1); a2 = c_mul(a2, w2); a3 = c_mul(a3, w3);
    }
    dft4<INV>(a0, a1, a2, a3);
    out.put(to, 0, a0); out.put(to, p, a1); out.put(to, 2 * p, a2); out.put(to, 3 * p, a3);
  } else {
    float2 a0 = in.at(ti, 0), a1 = in.at(ti, stride);
    if (k != 0) {
      float2 w1 = twp[k];
      if (INV) w1.y = -w1.y;
      a1 = c_mul(a1, w1);
    }
    out.put(to, 0, c_add(a0, a1));
    out.put(to, p, c_sub(a0, a1));
  }
}

// ------------------------------------------------------------------------------------------
// K1 phases.  Real transform of size N = 2M computed as an M-point complex transform of
// z[n] = x[2n] + i*x[2n+1] followed by the even/odd split.
// ------------------------------------------------------------------------------------------
// load (only used when M == 1, i.e. no pass exists): z -> work buffer
PC_HD void fwd_load(const float* src, int nv, float2* z, int M, int n) {
  z[swz(n)] = FwdGlobalIn{src, nv}.at(n, 0);
}

// split: Z = FFT_M(z) (swizzled work buffer) -> packed spectrum row X (B = M entries), k in [0, M/2]
PC_HD void fwd_split(const float2* Z, float2* X, const float2* tw, int M, int k) {
  if (k == 0) {
    const float2 z0 = Z[swz(0)];
    X[0] = make_float2(z0.x + z0.y, z0.x - z0.y);      // (DC, Nyquist)
    return;
  }
  const float2 a = Z[swz(k)];
  const float2 b = c_conj(Z[swz(M - k)]);
  const float2 E = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
  const float2 D = make_float2(0.5f * (a.x - b.x), 0.5f * (a.y - b.y));
  const float2 O = make_float2(D.y, -D.x);              // -i * D
  const float2 wO = c_mul(tw[k], O);
  X[k] = c_add(E, wO);
  X[M - k] = c_conj(c_sub(E, wO));
}

// ------------------------------------------------------------------------------------------
// K3 phases.
// ------------------------------------------------------------------------------------------
// merge + pre-twist: W = Yt + (-1)^k Yp  (overlap-add done in the frequency domain: the second
// half of IRFFT(Yp) equals the first half of IRFFT((-1)^k Yp)), then Z such that
// IFFT_M(Z)[n] = x[2n] + i*x[2n+1].   k in [0, M/2].
// np > 1 (multi-GPU slot exchange): row k of the spectrum is the sum of np partial rows that lie
// `ps` float2 apart (one slot per contributing GPU)
PC_HD float2 sum_partials(const float2* Y, int k, int np, long long ps) {
  float2 a = Y[k];
  if (np > 1) {
    float2 v[7];
#pragma unroll
    for (int g = 1; g < 8; ++g) v[g - 1] = g < np ? Y[(long long)g * ps + k] : make_float2(0.f, 0.f);   // loads first
#pragma unroll
    for (int g = 0; g < 7; ++g) { a.x += v[g].x; a.y += v[g].y; }
  }
  return a;
}

PC_HD float2 ola_merge(const float2* Yt, const float2* Yp, int M, int k, int np, long long ps) {
  const float2 a = sum_partials(Yt, k, np, ps), b = sum_partials(Yp, k, np, ps);
  if (k == 0) {
    const float s = (M & 1) ? -1.0f : 1.0f;             // Nyquist index M: (-1)^M
    return make_float2(a.x + b.x, a.y + s * b.y);
  }
  return (k & 1) ? c_sub(a, b) : c_add(a, b);
}

PC_HD void inv_pre(const float2* Yt, const float2* Yp, float2* Z, const float2* tw, int M, int k, int np, long long ps) {
  if (k == 0) {
    const float2 w0 = ola_merge(Yt, Yp, M, 0, np, ps);
    Z[swz(0)] = make_float2(0.5f * (w0.x + w0.y), 0.5f * (w0.x - w0.y));
    return;
  }
  const float2 a = ola_merge(Yt, Yp, M, k, np, ps);
  const float2 b = c_conj(ola_merge(Yt, Yp, M, M - k, np, ps));
  const float2 E = make_float2(0.5f * (a.x + b.x), 0.5f * (a.y + b.y));
  const float2 D = make_float2(0.5f * (a.x - b.x), 0.5f * (a.y - b.y));
  const float2 O = c_mul(c_conj(tw[k]), D);
  Z[swz(k)] = make_float2(E.x - O.y, E.y + O.x);
  Z[swz(M - k)] = make_float2(E.x + O.y, O.x - E.y);
}

// where the B output samples of one block go
struct OutSpec {
  float* dst;            // channel base
  long long index0;      // dst index of sample 0 of this block (before masking)
  long long lo, hi;      // valid dst index range [lo, hi) (head: this call's samples)
  long long mask;        // index & mask (ring destination) ; -1 = linear
  // look-ahead stage rings added on top (head stage only)
  int n_add;
  const float* add[3];
  long long add_mask[3];
  long long abs0;        // absolute stream position of sample 0 (ring read position)
};

PC_HD void inv_store_sample(float val, float scale, const OutSpec& o, int s) {
  const long long idx = o.index0 + s;
  if (idx < o.lo || idx >= o.hi) return;
  float r = val * scale;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (a < o.n_add) r += o.add[a][(o.abs0 + s) & o.add_mask[a]];
  o.dst[idx & o.mask] = r;
}

// sample s of the block from the (swizzled) work buffer; used when M == 1 (no pass)
PC_HD void inv_store(const float2* z, int M, float scale, const OutSpec& o, int s) {
  const float2 v = z[swz(s >> 1)];
  inv_store_sample((s & 1) ? v.y : v.x, scale, o, s);
}

// last inverse pass writes z[n] = (x[2n], x[2n+1]) straight to the destination; only the first
// B = M output samples (n < M/2) of the 2M-point inverse transform are needed
struct InvGlobalOut {
  const OutSpec* o; float scale; int half;
  PC_HD int prep(int base) const { return base; }
  PC_HD void put(int tok, int off, float2 v) const {
    const int n = tok + off;
    if (n >= half) return;
    inv_store_sample(v.x, scale, *o, 2 * n);
    inv_store_sample(v.y, scale, *o, 2 * n + 1);
  }
};

// ------------------------------------------------------------------------------------------
// K2: per-thread body of the batched FDL sweep.
//   thread owns bin k and TT consecutive output blocks t0..t0+TT-1 of one channel:
//     acc[j] = sum_{p=0}^{Ppad-1} H[p][k] * X[xrow0 + t0 + j - p][k]
//   H rows beyond P are zero; X rows exist (finite values) for every index touched.
//   The X window slides by one row per partition and lives in registers: per partition the
//   thread loads one H value and one X value (16 B) and issues 4*TT FFMAs.
//   D = software prefetch distance (partitions); TT % D == 0; H/X are readable D rows past the end.
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#define PC_LD(p) __ldg(p)
#else
#define PC_LD(p) (*(p))
#endif

//   BS > 0: row pitch known at compile time (B = BS) so that all row offsets inside the unrolled
//   body become immediate operands of the loads (no per-step 64-bit pointer arithmetic).
template <int TT, int D, int BS = 0>
PC_HD void cmac_thread(const float2* __restrict__ Hk,   // &H[c][0][k]
                       const float2* __restrict__ Xk,   // &X[c][xrow0 + t0][k]  (row of output t0, p = 0)
                       long long rowstride_rt,          // B (float2 elements per row)
                       int Ppad, bool packed_bin,
                       float2* acc) {
  const long long rowstride = BS > 0 ? (long long)BS : rowstride_rt;
  float2 win[TT];
#pragma unroll
  for (int j = 0; j < TT; ++j) {
    win[j] = PC_LD(Xk + (long long)j * rowstride);
    acc[j] = make_float2(0.0f, 0.0f);
  }
  float2 hq[D], xq[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    hq[d] = PC_LD(Hk + (long long)d * rowstride);
    xq[d] = PC_LD(Xk - (long long)(d + 1) * rowstride);
  }
  const float2* hp = Hk + (long long)D * rowstride;       // next H row to prefetch
  const float2* xp = Xk - (long long)(D + 1) * rowstride; // next X row to prefetch
  for (int p0 = 0; p0 < Ppad; p0 += TT, hp += (long long)TT * rowstride, xp -= (long long)TT * rowstride) {
#pragma unroll
    for (int u = 0; u < TT; ++u) {
      const float2 h = hq[u % D];
      const float2 xn = xq[u % D];
      hq[u % D] = PC_LD(hp + (long long)u * rowstride);
      xq[u % D] = PC_LD(xp - (long long)u * rowstride);
      // logical window entry j lives in win[(j - u) mod TT]
      if (!packed_bin) {
#pragma unroll
        for (int j = 0; j < TT; ++j) {
          const float2 x = win[(j - u + TT) % TT];
          acc[j].x = fmaf(h.x, x.x, acc[j].x);
          acc[j].x = fmaf(-h.y, x.y, acc[j].x);
          acc[j].y = fmaf(h.x, x.y, acc[j].y);
          acc[j].y = fmaf(h.y, x.x, acc[j].y);
        }
      } else {   // entry 0: two independent real bins (DC, Nyquist)
#pragma unroll
        for (int j = 0; j < TT; ++j) {
          const float2 x = win[(j - u + TT) % TT];
          acc[j].x = fmaf(h.x, x.x, acc[j].x);
          acc[j].y = fmaf(h.y, x.y, acc[j].y);
        }
      }
      // slide: logical j of the next step is logical j-1 now; new logical 0 replaces old TT-1
      win[(TT - 1 - u + TT) % TT] = xn;
    }
  }
}

// ------------------------------------------------------------------------------------------
// K2 (packed-FMA form): same tiling as cmac_thread, arithmetic on float2 pairs (two independent FP32 FMAs per
// pair).  Per output block two float2 accumulators:
//     A += (h.re, h.re) * (x.re, x.im)        B += (h.im, h.im) * (x.re, x.im)
//   => re = A.re - B.im ,  im = A.im + B.re          (complex bins)
//      re = A.re        ,  im = B.im                 (entry 0 = the two real bins DC / Nyquist)
// so the inner loop is identical for every bin (no divergence on the packed entry).
// ------------------------------------------------------------------------------------------
PC_HD float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <int TT, int D, int BS = 0>
PC_HD void cmac_thread2(const float2* __restrict__ Hk, const float2* __restrict__ Xk, long long rowstride_rt,
                        int Ppad, bool packed_bin, float2* out) {
  const long long rowstride = BS > 0 ? (long long)BS : rowstride_rt;
  float2 win[TT], accA[TT], accB[TT];
#pragma unroll
  for (int j = 0; j < TT; ++j) {
    win[j] = PC_LD(Xk + (long long)j * rowstride);
    accA[j] = make_float2(0.0f, 0.0f);
    accB[j] = make_float2(0.0f, 0.0f);
  }
  float2 hq[D], xq[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    hq[d] = PC_LD(Hk + (long long)d * rowstride);
    xq[d] = PC_LD(Xk - (long long)(d + 1) * rowstride);
  }
  const float2* hp = Hk + (long long)D * rowstride;
  const float2* xp = Xk - (long long)(D + 1) * rowstride;
  for (int p0 = 0; p0 < Ppad; p0 += TT, hp += (long long)TT * rowstride, xp -= (long long)TT * rowstride) {
#pragma unroll
    for (int u = 0; u < TT; ++u) {
      const float2 h = hq[u % D];
      const float2 xn = xq[u % D];
      hq[u % D] = PC_LD(hp + (long long)u * rowstride);
      xq[u % D] = PC_LD(xp - (long long)u * rowstride);
      const float2 hr = make_float2(h.x, h.x), hi = make_float2(h.y, h.y);
#pragma unroll
      for (int j = 0; j < TT; ++j) {
        const float2 x = win[(j - u + TT) % TT];
        accA[j] = ffma2(hr, x, accA[j]);
        accB[j] = ffma2(hi, x, accB[j]);
      }
      win[(TT - 1 - u + TT) % TT] = xn;
    }
  }
#pragma unroll
  for (int j = 0; j < TT; ++j)
    out[j] = packed_bin ? make_float2(accA[j].x, accB[j].y)
                        : make_float2(accA[j].x - accB[j].y, accA[j].y + accB[j].x);
}

// ------------------------------------------------------------------------------------------
// K2s: per-thread body of the STREAMING FDL sweep (real-time calls: 1..NBS blocks per launch).
//   This is the memory-bound form of the reference loop (FFTConvolver.cpp:179-187): every H[p]
//   and FDL row is read exactly once per block step; a thread owns two adjacent bins (one
//   16-byte load per operand), a warp strides over the partitions of its CTA's slice
//   p = p_lo + warp, p_lo + warp + PW, ... and keeps NBS accumulators per bin.
// ------------------------------------------------------------------------------------------
struct float4c { float2 a, b; };   // two adjacent bins

PC_HD float4c ld_pair(const float2* p) {
#if defined(__CUDA_ARCH__)
  // volatile asm keeps the loads of one batch back to back (issued before any dependent math):
  // the streaming sweep lives on memory-level parallelism
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  float4c r; r.a = make_float2(v.x, v.y); r.b = make_float2(v.z, v.w); return r;
#else
  float4c r; r.a = p[0]; r.b = p[1]; return r;
#endif
}

template <int NBS>
PC_HD void cmac_stream_thread(const float2* __restrict__ Hk,   // &H[c][0][k2]
                              const float2* __restrict__ Xk,   // &X[c][xrow0][k2] (output 0, partition 0)
                              long long rowstride, int p_lo, int p_hi, int p_step, int nblocks,
                              bool packed_first, float2* acc /*[NBS][2]*/) {
#pragma unroll
  for (int t = 0; t < NBS; ++t) { acc[2 * t] = make_float2(0.f, 0.f); acc[2 * t + 1] = make_float2(0.f, 0.f); }
  const float m = packed_first ? 0.0f : 1.0f;
#pragma unroll 4
  for (int p = p_lo; p < p_hi; p += p_step) {
    const float4c h = ld_pair(Hk + (long long)p * rowstride);
#pragma unroll
    for (int t = 0; t < NBS; ++t) {
      if (t < nblocks) {
        const float4c x = ld_pair(Xk + (long long)(t - p) * rowstride);
        // first bin: complex, or (DC, Nyquist) as two real products when packed_first
        float re = fmaf(h.a.x, x.a.x, acc[2 * t].x);
        re = fmaf(-m * h.a.y, x.a.y, re);
        float im = packed_first ? fmaf(h.a.y, x.a.y, acc[2 * t].y)
                                : fmaf(h.a.y, x.a.x, fmaf(h.a.x, x.a.y, acc[2 * t].y));
        acc[2 * t] = make_float2(re, im);
        acc[2 * t + 1].x = fmaf(-h.b.y, x.b.y, fmaf(h.b.x, x.b.x, acc[2 * t + 1].x));
        acc[2 * t + 1].y = fmaf(h.b.y, x.b.x, fmaf(h.b.x, x.b.y, acc[2 * t + 1].y));
      }
    }
  }
}


// ------------------------------------------------------------------------------------------
// K2s (row form): streaming sweep where a CTA walks whole spectrum rows.  Thread = two adjacent
// bins (one 16-byte load per operand), CTA = `threads` consecutive bin pairs of ONE row, CTAs
// split the partition range [0, P) in contiguous slices; no cross-warp reduction, each thread adds
// its NB results to Y with RED.ADD (or stores them when the slice is the whole range).
// U partitions are loaded back to back before any arithmetic: U*(1+NB) independent 16-byte loads
// in flight per thread — this is what makes the kernel bandwidth- instead of latency-bound.
// ------------------------------------------------------------------------------------------
template <int NB, int U>
PC_HD void cmac_stream_rows(const float2* __restrict__ Hk, const float2* __restrict__ Xk, long long rowstride,
                            int p_lo, int p_hi, bool packed_first, float2* acc /*[NB][2]*/) {
#pragma unroll
  for (int i = 0; i < 2 * NB; ++i) acc[i] = make_float2(0.f, 0.f);
  const float m = packed_first ? 0.0f : 1.0f;
  int p = p_lo;
  for (; p + U <= p_hi; p += U) {
    float4c h[U], x[U][NB];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      h[u] = ld_pair(Hk + (long long)(p + u) * rowstride);
#pragma unroll
      for (int t = 0; t < NB; ++t) x[u][t] = ld_pair(Xk + (long long)(t - p - u) * rowstride);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int t = 0; t < NB; ++t) {
        float re = fmaf(h[u].a.x, x[u][t].a.x, acc[2 * t].x);
        re = fmaf(-m * h[u].a.y, x[u][t].a.y, re);
        const float im = packed_first ? fmaf(h[u].a.y, x[u][t].a.y, acc[2 * t].y)
                                      : fmaf(h[u].a.y, x[u][t].a.x, fmaf(h[u].a.x, x[u][t].a.y, acc[2 * t].y));
        acc[2 * t] = make_float2(re, im);
        acc[2 * t + 1].x = fmaf(-h[u].b.y, x[u][t].b.y, fmaf(h[u].b.x, x[u][t].b.x, acc[2 * t + 1].x));
        acc[2 * t + 1].y = fmaf(h[u].b.y, x[u][t].b.x, fmaf(h[u].b.x, x[u][t].b.y, acc[2 * t + 1].y));
      }
    }
  }
  for (; p < p_hi; ++p) {
    const float4c h = ld_pair(Hk + (long long)p * rowstride);
#pragma unroll
    for (int t = 0; t < NB; ++t) {
      const float4c x = ld_pair(Xk + (long long)(t - p) * rowstride);
      float re = fmaf(h.a.x, x.a.x, acc[2 * t].x);
      re = fmaf(-m * h.a.y, x.a.y, re);
      const float im = packed_first ? fmaf(h.a.y, x.a.y, acc[2 * t].y)
                                    : fmaf(h.a.y, x.a.x, fmaf(h.a.x, x.a.y, acc[2 * t].y));
      acc[2 * t] = make_float2(re, im);
      acc[2 * t + 1].x = fmaf(-h.b.y, x.b.y, fmaf(h.b.x, x.b.x, acc[2 * t + 1].x));
      acc[2 * t + 1].y = fmaf(h.b.y, x.b.x, fmaf(h.b.x, x.b.y, acc[2 * t + 1].y));
    }
  }
}

// ------------------------------------------------------------------------------------------
// launch parameter blocks (shared by the CUDA kernels and the CPU emulation drivers)
// ------------------------------------------------------------------------------------------
struct FwdParams {
  const float* src;          // time-domain samples, channel c at src + c*src_cstride
  long long src_cstride;
  const int* nvalid_c;       // optional per-channel valid sample count (IR build), else nvalid
  long long nvalid;          // samples available from src (blocks past it read zeros)
  float2* dst;               // spectra, channel c at dst + c*dst_cstride, row r at + r*M
  long long dst_cstride;
  long long dst_row0;        // row of block 0
  const float2* tw;
  int M;                     // = B
  int nblocks;
  int use_cmap;              // routing: channel c reads source channel cmap[c] (StereoConvolver: LL,RR,LR,RL <- L,R,L,R)
  int cmap[8];
  const float2* tab512;      // tables of the register-resident B = 512 kernels (kernels_fft512.cuh), else nullptr
  // time-line output (k_fwd_fft512_lines, B = 512 groups on the tensor-core sweep): block b of channel c is sample
  // line_tau0 + b of the FP32 time lines of lines c * M ... c * M + M - 1 (tc::xf_index, line_rows rows of 64 samples);
  // its X row is written only for b >= xrow_from.  lines == nullptr: X rows only
  float* lines;
  long long line_tau0;
  int line_rows;
  int xrow_from;
};

struct CmacParams {
  const float2* H;           // [C][Prows][B]
  long long h_cstride;
  const float2* X;           // [C][R][B]
  long long x_cstride;
  long long xrow0;           // X row of output block 0 at partition 0
  float2* Y;                 // output block t of channel c -> Y + c*y_cstride + (yrow0+t)*y_rstride
  long long y_cstride;
  long long y_rstride;
  long long yrow0;
  int B;
  int Ppad;                  // multiple of TT
  int nblocks;
  // multi-GPU slot exchange (xg > 0): instead of Y, output block j is stored into the exchange
  // buffer of the GPU that owns its time slice, in this GPU's slot:
  //   owner o = min(xg-1, j / xper), row 1 + j - o*xper of xbase[o] + xrank*xslot   (row pitch y_rstride)
  // the last block of slice o is also stored as row 0 (halo) of owner o+1, and block xhalo_block
  // (last completed block of the group) into xhalo (owner 0's halo for the next group).
  int xg, xrank, xper, xhalo_block;
  long long xslot;
  float2* xbase[8];
  float2* xhalo;
};


// output store of the batched sweeps: plain Y row, or the multi-GPU slot exchange (CmacParams::xg > 0)
PC_HD void cmac_store(const CmacParams& P, int c, int k, int j, float2 v) {
  if (P.xg <= 0) {
    P.Y[(long long)c * P.y_cstride + (P.yrow0 + j) * P.y_rstride + k] = v;
    return;
  }
  int o = j / P.xper;
  if (o > P.xg - 1) o = P.xg - 1;
  const long long col = (long long)c * P.y_cstride + k;
  const long long slot = (long long)P.xrank * P.xslot;
  P.xbase[o][slot + (long long)(1 + j - o * P.xper) * P.y_rstride + col] = v;
  if (o + 1 < P.xg && j == (o + 1) * P.xper - 1) P.xbase[o + 1][slot + col] = v;     // halo row of the next slice
  if (j == P.xhalo_block) P.xhalo[(long long)P.xrank * P.y_rstride + col] = v;       // halo of the next group
}

struct InvParams {
  const float2* Y;           // block t of channel c: Y + c*y_cstride + (yrow0+t)*y_rstride; previous = one row before
  long long y_cstride;
  long long y_rstride;
  long long yrow0;
  const float2* tw;
  int M;
  int nblocks;
  float scale;               // 1/M
  int n_partials;            // >= 1: every row is the sum of n_partials rows partial_stride apart (slot exchange)
  long long partial_stride;
  // output
  float* dst; long long dst_cstride;
  long long index0;          // dst index of sample 0 of block 0
  long long lo, hi, mask;
  int n_add;
  const float* add[3]; long long add_cstride[3]; long long add_mask[3];
  long long abs0;            // absolute stream position of sample 0 of block 0
  const float2* tab512;      // tables of the register-resident B = 512 kernels (kernels_fft512.cuh), else nullptr
  // bin-major input (k_inv_fft512 only; the tensor-core sweep's result): block t of line c * M + k at
  // yc[line * yc_stride + yc_slot0 + t], its predecessor one slot before.  yc_prev_row: block 0's predecessor is Y row
  // yrow0 - 1 instead.  yc == nullptr: rows of Y
  const float2* yc;
  long long yc_stride, yc_slot0;
  int yc_prev_row;
};

struct StreamParams {
  const float2* H; long long h_cstride;
  const float2* X; long long x_cstride; long long xrow0;
  float2* Y; long long y_cstride, y_rstride, yrow0;   // rows must be zero before the launch when nsplit > 1
  int B, P, nblocks, nsplit;
  // dynamic variant (k_cmac_stream_tma_dyn): one ticket counter per (channel, bin tile); counters only grow, launch k
  // starts at ticket_base (every launch takes nchunks + nsplit tickets per counter)
  unsigned long long* ticket; unsigned long long ticket_base; int chunk_stages;
  // skewed static slices (k_cmac_stream_tma with interleave = 1): grid.y = nsplit * C, launch index li = blockIdx.y,
  // channel = li % C, slice = li / C; slice sizes fall linearly with the slice index by +-skew around the mean, because
  // CTAs are dispatched in launch order over a few microseconds and equal slices would end equally staggered
  int interleave; float skew;
  // descending = 1: every CTA walks its slice from the last partition to the first.  The host alternates the direction
  // from launch to launch: what the previous block step touched last is still in L2 and is what this one touches first
  // (a working set moderately above the L2 capacity then hits for a large part instead of thrashing an LRU cache).
  int descending;
};

// tail slot exchange epilogue of k_cmac_stream_tma (its optional second parameter): the last CTA of every (bin tile,
// channel) stores the summed tile into xdst (this rank's slot on rank 0, peer memory, channel pitch y_cstride); the last
// tile of the launch raises *xflag = xepoch.  xtick: one ticket word per (channel, bin tile) + one tile counter, zero
// between launches.
struct StreamXchParams {
  float2* xdst;
  unsigned int* xtick;
  unsigned int* xflag;
  unsigned int xepoch;
};

#if defined(__CUDACC__)
// ==========================================================================================
// __global__ wrappers
// ==========================================================================================


// FFT kernels, templated on the transform size M (= B) so that every index, radix, stride and
// trip count is a compile-time constant (the passes unroll completely; no integer division).
//   block (NT, ty): NT = fft_threads(M) threads per transform, ty transforms per CTA, grid (ceil(nblocks/ty), C)
//   M <= 1024 : NT = 32, one WARP owns one transform -> passes separated by __syncwarp() only
//   M >  1024 : NT = min(512, M/8), the CTA owns one transform (ty = 1), __syncthreads()
//   TWS       : the twiddle table (3M/2 float2) is staged in shared memory once per CTA
// dynamic smem = (TWS ? roundup16(3M/2) : 0) + ty * 2 * max(M,16) float2.

template <bool WARP>
__device__ __forceinline__ void fft_sync() {
  if (WARP) __syncwarp(); else __syncthreads();
}

// passes P, P*R, ... of an M-point transform between two work buffers; returns the buffer holding the result
template <bool INV, int M, int P>
__device__ __forceinline__ float2* fft_mid_passes(float2* in, float2* out, const float2* tw, int tx, bool active) {
  if constexpr (P >= M) {
    return in;
  } else {
    constexpr int R = pass_radix(M, P);
    constexpr int NT = fft_threads(M);
    if constexpr (INV && P * R == M) {
      return in;                                    // the inverse kernel runs its last pass itself
    } else {
      if (active) {
#pragma unroll
        for (int i0 = 0; i0 < M / R; i0 += NT) {
          const int i = i0 + tx;
          if (M / R >= NT || i < M / R)
            stockham_butterfly<INV>(SmemIn{in}, SmemOut{out}, tw + tw_pass_offset(M, P), M, P, R, i);
        }
      }
      fft_sync<fft_warp_mode(M)>();
      return fft_mid_passes<INV, M, P * R>(out, in, tw, tx, active);
    }
  }
}


// runs the LAST pass of the M-point inverse transform (the pass whose output length reaches M)
template <int M, int P>
__device__ __forceinline__ void last_inverse_pass(const float2* in, const float2* tw, int tx, const OutSpec& o, float scale) {
  constexpr int R = pass_radix(M, P);
  if constexpr (P * R == M) {
    constexpr int NT = fft_threads(M);
#pragma unroll
    for (int i0 = 0; i0 < M / R; i0 += NT) {
      const int i = i0 + tx;
      if (M / R >= NT || i < M / R)
        stockham_butterfly<true>(SmemIn{in}, InvGlobalOut{&o, scale, M / 2}, tw + tw_pass_offset(M, P), M, P, R, i);
    }
  } else {
    last_inverse_pass<M, P * R>(in, tw, tx, o, scale);
  }
}

template <int M, bool TWS>
__global__ void __launch_bounds__(512) k_fwd_fft(FwdParams P) {
  extern __shared__ float2 pc_smem[];
  constexpr bool WARP = fft_warp_mode(M);
  constexpr int NT = fft_threads(M);
  const int tx = threadIdx.x;
  const int blk = blockIdx.x * blockDim.y + threadIdx.y;
  const int c = blockIdx.y;
  const bool active = blk < P.nblocks;
  const float2* tw = P.tw;
  float2* data = pc_smem;
  if (TWS) {
    constexpr int tl = tw_table_len(M);
    const int tid = threadIdx.y * blockDim.x + tx, nthr = blockDim.x * blockDim.y;
    for (int j = tid; j < tl; j += nthr) pc_smem[j] = P.tw[j];
    tw = pc_smem;
    data = pc_smem + ((tl + 15) & ~15);
    __syncthreads();
  }
  constexpr int MB = M < 16 ? 16 : M;
  float2* bufA = data + (size_t)threadIdx.y * 2 * MB;
  float2* bufB = bufA + MB;
  int nv = 0;
  const float* src = nullptr;
  if (active) {
    const long long nv_total = P.nvalid_c ? (long long)P.nvalid_c[c] : P.nvalid;
    long long rem = nv_total - (long long)blk * M;
    nv = rem <= 0 ? 0 : (rem > M ? M : (int)rem);
    src = P.src + (long long)(P.use_cmap ? P.cmap[c] : c) * P.src_cstride + (long long)blk * M;
  }
  float2* res = bufA;
  if constexpr (M == 1) {
    if (active && tx == 0) fwd_load(src, nv, bufA, M, 0);
  } else {
    // first pass straight from global memory (zero padding applied in the accessor)
    constexpr int R0 = pass_radix(M, 1);
    if (active) {
#pragma unroll
      for (int i0 = 0; i0 < M / R0; i0 += NT) {
        const int i = i0 + tx;
        if (M / R0 >= NT || i < M / R0)
          stockham_butterfly<false>(FwdGlobalIn{src, nv}, SmemOut{bufA}, tw + tw_pass_offset(M, 1), M, 1, R0, i);
      }
    }
    fft_sync<WARP>();
    res = fft_mid_passes<false, M, R0>(bufA, bufB, tw, tx, active);
  }
  if (active) {
    float2* X = P.dst + (long long)c * P.dst_cstride + (P.dst_row0 + blk) * (long long)M;
#pragma unroll 4
    for (int k = tx; k <= M / 2; k += NT) fwd_split(res, X, tw, M, k);
  }
}


// grid (ceil(B/32), ceil(nblocks/(TT*TW)), C), block (32, TW)
template <int TT, int D, int TW, int BS = 0>
__global__ void __launch_bounds__(32 * TW) k_cmac_batch(CmacParams P) {
  const int k = blockIdx.x * 32 + threadIdx.x;
  const int t0 = (blockIdx.y * TW + threadIdx.y) * TT;
  const int c = blockIdx.z;
  if (k >= P.B || t0 >= P.nblocks) return;
  const float2* Hk = P.H + (long long)c * P.h_cstride + k;
  const float2* Xk = P.X + (long long)c * P.x_cstride + (P.xrow0 + t0) * (long long)P.B + k;
  float2 acc[TT];
  if (k == 0) cmac_thread<TT, D, BS>(Hk, Xk, P.B, P.Ppad, true, acc);
  else        cmac_thread<TT, D, BS>(Hk, Xk, P.B, P.Ppad, false, acc);
  float2* Yk = P.Y + (long long)c * P.y_cstride + (P.yrow0 + t0) * P.y_rstride + k;
#pragma unroll
  for (int j = 0; j < TT; ++j)
    if (t0 + j < P.nblocks) Yk[(long long)j * P.y_rstride] = acc[j];
}


// same geometry as k_fwd_fft
template <int M, bool TWS, bool PART>
__global__ void __launch_bounds__(512) k_inv_fft_ola(InvParams P) {
  extern __shared__ float2 pc_smem[];
  constexpr bool WARP = fft_warp_mode(M);
  constexpr int NT = fft_threads(M);
  const int tx = threadIdx.x;
  const int blk = blockIdx.x * blockDim.y + threadIdx.y;
  const int c = blockIdx.y;
  const bool active = blk < P.nblocks;
  const float2* tw = P.tw;
  float2* data = pc_smem;
  if (TWS) {
    constexpr int tl = tw_table_len(M);
    const int tid = threadIdx.y * blockDim.x + tx, nthr = blockDim.x * blockDim.y;
    for (int j = tid; j < tl; j += nthr) pc_smem[j] = P.tw[j];
    tw = pc_smem;
    data = pc_smem + ((tl + 15) & ~15);
    __syncthreads();                    // inv_pre already needs the table
  }
  constexpr int MB = M < 16 ? 16 : M;
  float2* bufA = data + (size_t)threadIdx.y * 2 * MB;
  float2* bufB = bufA + MB;
  OutSpec o;
  if (active) {
    o.dst = P.dst + (long long)c * P.dst_cstride;
    o.index0 = P.index0 + (long long)blk * M;
    o.lo = P.lo; o.hi = P.hi; o.mask = P.mask;
    o.n_add = P.n_add;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      o.add[a] = a < P.n_add ? P.add[a] + (long long)c * P.add_cstride[a] : nullptr;
      o.add_mask[a] = P.add_mask[a];
    }
    o.abs0 = P.abs0 + (long long)blk * M;
    const float2* Yt = P.Y + (long long)c * P.y_cstride + (P.yrow0 + blk) * P.y_rstride;
    const float2* Yp = Yt - P.y_rstride;
    const int np = PART ? P.n_partials : 1;      // PART = false: single-GPU path without the partial-slot sums
#pragma unroll 4
    for (int k = tx; k <= M / 2; k += NT) inv_pre(Yt, Yp, bufA, tw, M, k, np, P.partial_stride);
  }
  fft_sync<WARP>();
  if constexpr (M == 1) {
    if (active && tx == 0) inv_store(bufA, M, P.scale, o, 0);
  } else {
    float2* in = fft_mid_passes<true, M, 1>(bufA, bufB, tw, tx, active);   // all passes but the last
    // last pass: scaled samples straight to the destination (first half of the transform only)
    if (active) last_inverse_pass<M, 1>(in, tw, tx, o, P.scale);
  }
}

// packed-FMA variant; MINB = CTAs per SM the register allocation must allow
template <int TT, int D, int TW, int BS, int MINB>
__global__ void __launch_bounds__(32 * TW, MINB) k_cmac_batch2(CmacParams P) {
  const int k = blockIdx.x * 32 + threadIdx.x;
  const int t0 = (blockIdx.y * TW + threadIdx.y) * TT;
  const int c = blockIdx.z;
  if (k >= P.B || t0 >= P.nblocks) return;
  const float2* Hk = P.H + (long long)c * P.h_cstride + k;
  const float2* Xk = P.X + (long long)c * P.x_cstride + (P.xrow0 + t0) * (long long)P.B + k;
  float2 acc[TT];
  cmac_thread2<TT, D, BS>(Hk, Xk, P.B, P.Ppad, k == 0, acc);
#pragma unroll
  for (int j = 0; j < TT; ++j)
    if (t0 + j < P.nblocks) cmac_store(P, c, k, t0 + j, acc[j]);
}

// grid (ceil(B/2/threads), nsplit, C), block (threads) with threads = min(256, B/2)
template <int NB, int U>
__global__ void __launch_bounds__(256) k_cmac_stream_rows(StreamParams P) {
  const int k2 = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  const int c = blockIdx.z;
  if (k2 >= P.B) return;
  const int per = (P.P + P.nsplit - 1) / P.nsplit;
  const int p_lo = blockIdx.y * per;
  const int p_hi = min(P.P, p_lo + per);
  if (p_lo >= p_hi && P.nsplit > 1) return;
  const float2* Hk = P.H + (long long)c * P.h_cstride + k2;
  const float2* Xk = P.X + (long long)c * P.x_cstride + P.xrow0 * (long long)P.B + k2;
  float2 acc[2 * NB];
  cmac_stream_rows<NB, U>(Hk, Xk, P.B, p_lo, p_hi, k2 == 0, acc);
#pragma unroll
  for (int t = 0; t < NB; ++t) {
    if (t < P.nblocks) {
      float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + (P.yrow0 + t) * P.y_rstride + k2);
      if (P.nsplit == 1) {
        *reinterpret_cast<float4*>(y) = make_float4(acc[2 * t].x, acc[2 * t].y, acc[2 * t + 1].x, acc[2 * t + 1].y);
      } else {
        atomicAdd(y + 0, acc[2 * t].x); atomicAdd(y + 1, acc[2 * t].y);
        atomicAdd(y + 2, acc[2 * t + 1].x); atomicAdd(y + 3, acc[2 * t + 1].y);
      }
    }
  }
}

// grid (B/64 or 1, nsplit, C), block (32, PW); smem: PW * NBS * 32 * 4 floats (static)
template <int NBS, int PW>
__global__ void __launch_bounds__(32 * PW) k_cmac_stream(StreamParams P) {
  __shared__ float4 red[PW][NBS][32];
  const int lane = threadIdx.x, w = threadIdx.y;
  const int k2 = (blockIdx.x * 32 + lane) * 2;
  const int c = blockIdx.z;
  const bool live = k2 < P.B;
  const int per = (P.P + P.nsplit - 1) / P.nsplit;
  const int p_lo = blockIdx.y * per;
  const int p_hi = min(P.P, p_lo + per);
  float2 acc[2 * NBS];
  if (live) {
    const float2* Hk = P.H + (long long)c * P.h_cstride + k2;
    const float2* Xk = P.X + (long long)c * P.x_cstride + P.xrow0 * (long long)P.B + k2;
    cmac_stream_thread<NBS>(Hk, Xk, P.B, p_lo + w, p_hi, PW, P.nblocks, k2 == 0, acc);
  } else {
#pragma unroll
    for (int i = 0; i < 2 * NBS; ++i) acc[i] = make_float2(0.f, 0.f);
  }
#pragma unroll
  for (int t = 0; t < NBS; ++t) red[w][t][lane] = make_float4(acc[2 * t].x, acc[2 * t].y, acc[2 * t + 1].x, acc[2 * t + 1].y);
  __syncthreads();
  // warp w reduces output block t = w, w + PW, ...
  for (int t = w; t < P.nblocks; t += PW) {
    float4 v = red[0][t][lane];
#pragma unroll
    for (int q = 1; q < PW; ++q) {
      const float4 u = red[q][t][lane];
      v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
    }
    if (live) {
      float* y = reinterpret_cast<float*>(P.Y + (long long)c * P.y_cstride + (P.yrow0 + t) * P.y_rstride + k2);
      if (P.nsplit == 1) {
        *reinterpret_cast<float4*>(y) = v;
      } else {
        atomicAdd(y + 0, v.x); atomicAdd(y + 1, v.y); atomicAdd(y + 2, v.z); atomicAdd(y + 3, v.w);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Cross-GPU barrier over peer-mapped flag words (slot exchange).  One CTA, thread t < G:
// publishes `epoch` in peer t's flag array at index `rank`, then waits until peer t has published
// the same epoch here.  Flags only grow, so no reset is needed.  A spin bounded in wall-clock time
// (BarrierParams::timeout_ns) turns a lost peer into an error word instead of a hung GPU.
// ------------------------------------------------------------------------------------------
struct BarrierParams {
  unsigned int* peer_flags[8];   // flag array (8 words) of every rank, peer-mapped
  unsigned int* my_flags;
  unsigned int* error_word;      // set to epoch on timeout
  int rank, G;
  unsigned int epoch;
  unsigned long long timeout_ns;   // wall-clock bound of the spin (%globaltimer)
};

static __global__ void k_p2p_barrier(BarrierParams P) {
  const int t = threadIdx.x;
  if (t >= P.G) return;
  __threadfence_system();                      // everything this GPU wrote before the barrier is visible first
  volatile unsigned int* out = P.peer_flags[t] + P.rank;
  *out = P.epoch;
  __threadfence_system();
  volatile unsigned int* in = P.my_flags + t;
  unsigned long long t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while ((int)(*in - P.epoch) < 0) {
    __nanosleep(64);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > P.timeout_ns) { *P.error_word = P.epoch; break; }
  }
  __threadfence_system();
}

// out[o][i] = sum_c mix[o*C + c] * in[c][i]   (true-stereo mixdown of the per-convolver outputs,
// src/PluginProcessor.cpp:1833-1838: wet L = LL + RL, wet R = RR + LR); grid (ceil(n/256), n_out)
struct MixParams {
  const float* in; long long in_stride;
  float* out; long long out_stride;
  long long n;
  int C, n_out;
  float mix[64];
};

static __global__ void k_mix(MixParams P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int o = blockIdx.y;
  if (i >= P.n) return;
  float acc = 0.0f;
  for (int c = 0; c < P.C; ++c) {
    const float m = P.mix[o * P.C + c];
    if (m != 0.0f) acc = fmaf(m, P.in[(long long)c * P.in_stride + i], acc);
  }
  P.out[(long long)o * P.out_stride + i] = acc;
}

// crossfade of two convolver outputs on the device (IR hot-swap, src/PluginProcessor.cpp:1800-1830):
// dst[c][i] = (1 - a_i) * a[c][i] + a_i * b[c][i],  a_i = clamp(alpha0 + i*step, 0, 1); grid (ceil(n/256), C)
static __global__ void k_xfade(float* dst, const float* a, const float* b, long long stride, long long n, float alpha0, float step) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long o = (long long)blockIdx.y * stride + i;
  const float al = fminf(1.0f, fmaxf(0.0f, alpha0 + step * (float)i));
  dst[o] = (1.0f - al) * a[o] + al * b[o];
}

// strided row copy on the SMs (rows x width floats); used where a copy-engine copy queued behind a spinning
// flag barrier would block the H2D copies of the following launch groups (slot-exchange path)
static __global__ void k_copy_rows(float* dst, long long dpitch, const float* src, long long spitch, long long width, int rows) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (i < width && r < rows) dst[(long long)r * dpitch + i] = src[(long long)r * spitch + i];
}

// dst[i] = sum over np slots of src[g*ps + i] (tail slot exchange: the summed spectrum of a tail block becomes the
// overlap row of the next one); same summation order as the inverse FFT's sum_partials
static __global__ void k_sum_slots(float2* dst, const float2* src, long long n, int np, long long ps) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = sum_partials(src + i, 0, np, ps);
}
#endif  // __CUDACC__


#if !defined(__CUDACC__)
// ==========================================================================================
// CPU emulation drivers (tests/emu only): same phase functions, the CTA's threads replaced by
// loops, __syncthreads() by the loop boundaries.  Geometry arguments mirror the launches.
// ==========================================================================================
struct EmuDim { int x, y, z; };

inline void emu_fwd_fft(EmuDim grid, EmuDim block, const FwdParams& P) {
  const int M = P.M;
  const int Mp = M < 16 ? 16 : M;
  float2* bufA = new float2[(size_t)Mp];
  float2* bufB = new float2[(size_t)Mp];
  for (int c = 0; c < grid.y; ++c)
    for (int bx = 0; bx < grid.x; ++bx)
      for (int ty = 0; ty < block.y; ++ty) {
        const int blk = bx * block.y + ty;
        if (blk >= P.nblocks) continue;
        const long long nv_total = P.nvalid_c ? (long long)P.nvalid_c[c] : P.nvalid;
        long long rem = nv_total - (long long)blk * M;
        const int nv = rem <= 0 ? 0 : (rem > M ? M : (int)rem);
        const float* src = P.src + (long long)(P.use_cmap ? P.cmap[c] : c) * P.src_cstride + (long long)blk * M;
        float2* in = bufA; float2* out = bufB;
        if (M == 1) {
          fwd_load(src, nv, in, M, 0);
        } else {
          const int R0 = pass_radix(M, 1);
          for (int i = 0; i < M / R0; ++i)
            stockham_butterfly<false>(FwdGlobalIn{src, nv}, SmemOut{in}, P.tw + tw_pass_offset(M, 1), M, 1, R0, i);
          for (int p = R0; p < M;) {
            const int R = pass_radix(M, p);
            for (int i = 0; i < M / R; ++i)
              stockham_butterfly<false>(SmemIn{in}, SmemOut{out}, P.tw + tw_pass_offset(M, p), M, p, R, i);
            float2* t = in; in = out; out = t;
            p *= R;
          }
        }
        float2* X = P.dst + (long long)c * P.dst_cstride + (P.dst_row0 + blk) * (long long)M;
        for (int k = 0; k <= M / 2; ++k) fwd_split(in, X, P.tw, M, k);
      }
  delete[] bufA; delete[] bufB;
}

template <int TT, int D, int TW>
inline void emu_cmac_batch(EmuDim grid, const CmacParams& P) {
  for (int c = 0; c < grid.z; ++c)
    for (int by = 0; by < grid.y; ++by)
      for (int bx = 0; bx < grid.x; ++bx)
        for (int w = 0; w < TW; ++w)
          for (int lane = 0; lane < 32; ++lane) {
            const int k = bx * 32 + lane;
            const int t0 = (by * TW + w) * TT;
            if (k >= P.B || t0 >= P.nblocks) continue;
            const float2* Hk = P.H + (long long)c * P.h_cstride + k;
            const float2* Xk = P.X + (long long)c * P.x_cstride + (P.xrow0 + t0) * (long long)P.B + k;
            float2 acc[TT];
            cmac_thread<TT, D>(Hk, Xk, P.B, P.Ppad, k == 0, acc);
            float2* Yk = P.Y + (long long)c * P.y_cstride + (P.yrow0 + t0) * P.y_rstride + k;
            for (int j = 0; j < TT; ++j)
              if (t0 + j < P.nblocks) Yk[(long long)j * P.y_rstride] = acc[j];
          }
}

template <int TT, int D, int TW>
inline void emu_cmac_batch2(EmuDim grid, const CmacParams& P) {
  for (int c = 0; c < grid.z; ++c)
    for (int by = 0; by < grid.y; ++by)
      for (int bx = 0; bx < grid.x; ++bx)
        for (int w = 0; w < TW; ++w)
          for (int lane = 0; lane < 32; ++lane) {
            const int k = bx * 32 + lane;
            const int t0 = (by * TW + w) * TT;
            if (k >= P.B || t0 >= P.nblocks) continue;
            const float2* Hk = P.H + (long long)c * P.h_cstride + k;
            const float2* Xk = P.X + (long long)c * P.x_cstride + (P.xrow0 + t0) * (long long)P.B + k;
            float2 acc[TT];
            cmac_thread2<TT, D>(Hk, Xk, P.B, P.Ppad, k == 0, acc);
            for (int j = 0; j < TT; ++j)
              if (t0 + j < P.nblocks) cmac_store(P, c, k, t0 + j, acc[j]);
          }
}

inline void emu_inv_fft_ola(EmuDim grid, EmuDim block, const InvParams& P) {
  const int M = P.M;
  const int Mp = M < 16 ? 16 : M;
  float2* bufA = new float2[(size_t)Mp];
  float2* bufB = new float2[(size_t)Mp];
  for (int c = 0; c < grid.y; ++c)
    for (int bx = 0; bx < grid.x; ++bx)
      for (int ty = 0; ty < block.y; ++ty) {
        const int blk = bx * block.y + ty;
        if (blk >= P.nblocks) continue;
        OutSpec o;
        o.dst = P.dst + (long long)c * P.dst_cstride;
        o.index0 = P.index0 + (long long)blk * M;
        o.lo = P.lo; o.hi = P.hi; o.mask = P.mask;
        o.n_add = P.n_add;
        for (int a = 0; a < 3; ++a) {
          o.add[a] = a < P.n_add ? P.add[a] + (long long)c * P.add_cstride[a] : nullptr;
          o.add_mask[a] = P.add_mask[a];
        }
        o.abs0 = P.abs0 + (long long)blk * M;
        const float2* Yt = P.Y + (long long)c * P.y_cstride + (P.yrow0 + blk) * P.y_rstride;
        const float2* Yp = Yt - P.y_rstride;
        for (int k = 0; k <= M / 2; ++k) inv_pre(Yt, Yp, bufA, P.tw, M, k, P.n_partials, P.partial_stride);
        float2* in = bufA; float2* out = bufB;
        if (M == 1) {
          inv_store(in, M, P.scale, o, 0);
        } else {
          for (int p = 1; p < M;) {
            const int R = pass_radix(M, p);
            const bool last = p * R == M;
            for (int i = 0; i < M / R; ++i) {
              if (!last) stockham_butterfly<true>(SmemIn{in}, SmemOut{out}, P.tw + tw_pass_offset(M, p), M, p, R, i);
              else stockham_butterfly<true>(SmemIn{in}, InvGlobalOut{&o, P.scale, M / 2}, P.tw + tw_pass_offset(M, p), M, p, R, i);
            }
            float2* t = in; in = out; out = t;
            p *= R;
          }
        }
      }
  delete[] bufA; delete[] bufB;
}

template <int NBS, int PW>
inline void emu_cmac_stream(EmuDim grid, const StreamParams& P) {
  for (int c = 0; c < grid.z; ++c)
    for (int by = 0; by < grid.y; ++by)
      for (int bx = 0; bx < grid.x; ++bx) {
        const int per = (P.P + P.nsplit - 1) / P.nsplit;
        const int p_lo = by * per;
        const int p_hi = P.P < p_lo + per ? P.P : p_lo + per;
        for (int lane = 0; lane < 32; ++lane) {
          const int k2 = (bx * 32 + lane) * 2;
          if (k2 >= P.B) continue;
          float2 sum[2 * NBS];
          for (int i = 0; i < 2 * NBS; ++i) sum[i] = make_float2(0.f, 0.f);
          for (int w = 0; w < PW; ++w) {
            float2 acc[2 * NBS];
            const float2* Hk = P.H + (long long)c * P.h_cstride + k2;
            const float2* Xk = P.X + (long long)c * P.x_cstride + P.xrow0 * (long long)P.B + k2;
            cmac_stream_thread<NBS>(Hk, Xk, P.B, p_lo + w, p_hi, PW, P.nblocks, k2 == 0, acc);
            for (int i = 0; i < 2 * NBS; ++i) { sum[i].x += acc[i].x; sum[i].y += acc[i].y; }
          }
          for (int t = 0; t < P.nblocks; ++t) {
            float2* y = P.Y + (long long)c * P.y_cstride + (P.yrow0 + t) * P.y_rstride + k2;
            if (P.nsplit == 1) { y[0] = sum[2 * t]; y[1] = sum[2 * t + 1]; }
            else { y[0].x += sum[2 * t].x; y[0].y += sum[2 * t].y; y[1].x += sum[2 * t + 1].x; y[1].y += sum[2 * t + 1].y; }
          }
        }
      }
}

template <int NB, int U>
inline void emu_cmac_stream_rows(EmuDim grid, int threads, const StreamParams& P) {
  for (int c = 0; c < grid.z; ++c)
    for (int by = 0; by < grid.y; ++by)
      for (int bx = 0; bx < grid.x; ++bx)
        for (int tid = 0; tid < threads; ++tid) {
          const int k2 = (bx * threads + tid) * 2;
          if (k2 >= P.B) continue;
          const int per = (P.P + P.nsplit - 1) / P.nsplit;
          const int p_lo = by * per;
          const int p_hi = P.P < p_lo + per ? P.P : p_lo + per;
          if (p_lo >= p_hi && P.nsplit > 1) continue;
          const float2* Hk = P.H + (long long)c * P.h_cstride + k2;
          const float2* Xk = P.X + (long long)c * P.x_cstride + P.xrow0 * (long long)P.B + k2;
          float2 acc[2 * NB];
          cmac_stream_rows<NB, U>(Hk, Xk, P.B, p_lo, p_hi, k2 == 0, acc);
          for (int t = 0; t < NB && t < P.nblocks; ++t) {
            float2* y = P.Y + (long long)c * P.y_cstride + (P.yrow0 + t) * P.y_rstride + k2;
            if (P.nsplit == 1) { y[0] = acc[2 * t]; y[1] = acc[2 * t + 1]; }
            else { y[0].x += acc[2 * t].x; y[0].y += acc[2 * t].y; y[1].x += acc[2 * t + 1].x; y[1].y += acc[2 * t + 1].y; }
          }
        }
}
#endif  // !__CUDACC__

}  // namespace pc
