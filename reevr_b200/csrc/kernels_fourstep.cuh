// kernels_fourstep.cuh — K2s: long B = 512 launch groups of a single-stage handle as overlap-save of the samples with
// M = 2^21-point FFTs, each computed as a four-step factorisation (cmac_variant 42).
//
// Each channel's output is y[t] = sum_j h[j] x[t - j] over the Lh = P B taps of the IR (the partition padding is
// zeros).  Segment q of the group produces the outputs [q L, q L + L), L = M - (Lh - 1), from the window of samples
// [q L - (Lh - 1), q L - (Lh - 1) + M): negative positions are the history in front of the group, positions past the
// group's end read zeros, the last segment is partial.  With n = N2 n1 + n2, k = k1 + N1 k2 (N1 = 512, N2 = 4096):
//
//   pass 1  k_fs_cols      per column n2: A[k1][n2] = W_M^{n2 k1} sum_n1 x[N2 n1 + n2] W_512^{n1 k1}, k1 = 0 ... 256
//   pass 2  k_fs_rows      per row k1:    X[k1 + N1 k2] = sum_n2 A[k1][n2] W_4096^{n2 k2}; times S = H / M; inverse
//                          4096-point DFT over k2, in place
//   pass 3  k_fs_cols_inv  per column n2: y[N2 n1 + n2] = sum_k1 W_512^{-n1 k1} W_M^{-n2 k1} C[k1][n2], the rows
//                          k1 > 256 being conj(rows 512 - k1) (the output is real); only the L valid outputs are stored
//
// The samples are real, so the spectrum is Hermitian: X[M - k] = conj X[k] puts rows 257 ... 511 of A (and of C after
// the twiddle) on the conjugates of rows 255 ... 1, and only the 257 rows k1 = 0 ... 256 are kept.  The intermediate
// is then the size of the samples (257 / 256 of it), where the block FFTs of K2f produce twice as many complex values
// as there are samples.  Rows 0 and 256 are ordinary complex rows between the passes; their columns' values are real
// before the pass-1 twiddle and after the pass-3 one.
//
// Column passes: one CTA per 32 adjacent columns, one warp per pair of real columns packed as one complex column
// (z = x_a + i x_b) through kernels_fft512.cuh's three-step 512-point DFT.  The lane that holds bin k1 also holds
// 512 - k1, so (Z[k1] + conj Z[-k1]) / 2 and (Z[k1] - conj Z[-k1]) / 2i separate the two columns without data
// movement.  Samples come in as 128-byte rows of 32 columns and column spectra leave as 256-byte rows: a shared-memory
// tile transposes both ways, and doubles as the warps' exchange buffers.  Twiddles W_M^e: e = n2 k1 < 2^20, so
// sincospif(e / 2^20) has an exact argument.
// Row pass: kernels_lfft.cuh's 4096-point transform, pointwise product and conjugate inverse, 1 / M folded into S,
// in persistent CTAs that walk contiguous ranges of the rows with the next row and the spectrum row bulk-copied into
// shared memory.  Column spectra are [C][kRows][nseg][kN2]: the segments of a row are one contiguous run.
//
// k_fs_taps turns packed 1024-point spectrum rows back into their first 512 samples: the taps from the partition
// spectra H (for the IR spectrum: taps, pass 1, pass 2 without the product), and the history in front of a group
// from the X rows, which are all that is kept of the samples before it.
#pragma once

#include "kernels_lfft.cuh"
#if defined(__CUDACC__)
#include "kernels_fft512.cuh"
#endif

namespace pc {
namespace fs {

constexpr int kN1 = 512, kN2 = 4096;
constexpr long long kM = (long long)kN1 * kN2;     // 2^21
constexpr int kRows = kN1 / 2 + 1;                  // the Hermitian half of every column spectrum
constexpr int kMaxP = 961;                          // Lh - 1 < M / 4: at least 3/4 of each segment are outputs
constexpr int kCols = 32;                           // columns per CTA of the column passes
constexpr int kColThreads = 512;                    // one warp per column pair
constexpr int kStage4 = 17;                         // float4 per staged row (16 column pairs + 1 pad)

// Segment plan of a group of n samples with P partitions of B = 512
struct Plan {
  int P, nseg;
  long long Lh, L, n;
};

PC_TC_HD Plan make_plan(int P, long long n) {
  Plan p;
  p.P = P;
  p.Lh = (long long)P * kN1;
  p.L = kM - (p.Lh - 1);
  p.n = n;
  p.nseg = (int)((n + p.L - 1) / p.L);
  return p;
}
PC_TC_HD bool plan_ok(int P) { return P >= 1 && P <= kMaxP; }
// the items [begin, end) of CTA b of the persistent row pass: ctas contiguous ranges of items whose lengths differ by at
// most one, so no range is longer than ceil(items / ctas)
struct ItemRange {
  unsigned begin, end;
};
PC_TC_HD ItemRange item_range(unsigned items, unsigned ctas, unsigned b) {
  return ItemRange{(unsigned)((unsigned long long)items * b / ctas), (unsigned)((unsigned long long)items * (b + 1) / ctas)};
}
// first window sample (relative to the group's first sample) of segment q
PC_TC_HD long long window_start(const Plan& p, int q) { return (long long)q * p.L - (p.Lh - 1); }
// group output of window position m of segment q, or -1 (m < Lh - 1: the wrapped part; or past the group's end)
PC_TC_HD long long output_of(const Plan& p, int q, long long m) {
  if (m < p.Lh - 1) return -1;
  const long long t = (long long)q * p.L + m - (p.Lh - 1);
  return t < p.n ? t : -1;
}
// the column spectra of every segment and channel, [C][kRows][nseg][kN2] complex: the nseg segments of a row are one
// contiguous run
PC_TC_HD size_t work_bytes(const Plan& p, int C) { return (size_t)C * p.nseg * kRows * kN2 * 8; }
// the IR spectrum in pass-2 layout, [C][kRows][kN2] complex
PC_TC_HD size_t spectrum_bytes(int C) { return (size_t)C * kRows * kN2 * 8; }
// the taps / the history in front of a group, [C][P * 512] floats
PC_TC_HD size_t hist_bytes(int P, int C) { return (size_t)C * P * kN1 * 4; }

#if defined(__CUDACC__)

// dynamic shared memory of the column passes: the 512-point tables and the tile (257 staged rows of 32 columns)
constexpr size_t kColSmem = (size_t)(kF512_TabLen + 2 * kStage4 * kRows) * sizeof(float2);

// W_M^{e} (INV: W_M^{-e}), 0 <= e < 2^20
__device__ __forceinline__ float2 wM(int e, bool inv) {
  float s, c;
  sincospif((inv ? 1.0f : -1.0f) * (float)e * (1.0f / 1048576.0f), &s, &c);
  return make_float2(c, s);
}

// ---- packed spectrum rows -> their first 512 samples ---------------------------------------------------------
struct TapsParams {
  const float2* rows;       // channel c, row r: rows + c * row_cstride + r * 512 (packed 1024-point spectra)
  long long row_cstride;
  int nrows;
  float* dst;               // channel c, row r: dst + c * dst_cstride + r * 512
  long long dst_cstride;
};

// grid (ceil(nrows / 8), C), block (32, 8), dynamic smem kF512Smem: one warp per row, k_inv_fft512's arithmetic
// without the overlap-add merge
__global__ void __launch_bounds__(256, 3) k_fs_taps(TapsParams p, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem512[];
  float2* tab = pc_smem512;
  float2* S = pc_smem512 + kF512_TabLen + threadIdx.y * kF512_Xch;
  const int lane = threadIdx.x, tid = threadIdx.y * 32 + lane;
  for (int j = tid; j < kF512_TabLen; j += 256) tab[j] = tab512[j];
  __syncthreads();
  const int c = blockIdx.y, r = blockIdx.x * 8 + threadIdx.y;
  if (r >= p.nrows) return;
  const float2* Y = p.rows + (long long)c * p.row_cstride + (long long)r * kN1;
  const int la = f512_la(lane), lb = f512_lb(lane);
  float2 A[8], B[8];
#pragma unroll
  for (int q1 = 0; q1 < 8; ++q1) { A[q1] = __ldg(Y + la + 64 * q1); B[q1] = __ldg(Y + lb + 64 * q1); }
  f512_inv_p1_core(lane, A, B, S, tab);
  __syncwarp();
  f512_mid_load<true>(lane, S, tab, A, B);
  __syncwarp();
  f512_mid_store<true>(lane, S, A, B);
  __syncwarp();
  OutSpec o{};
  o.dst = p.dst + (long long)c * p.dst_cstride;
  o.index0 = (long long)r * kN1;
  o.lo = 0; o.hi = (long long)1 << 62; o.mask = -1;
  f512_inv_p3<true>(lane, S, 1.0f / (float)kN1, o);
}

// ---- pass 1 ---------------------------------------------------------------------------------------------------
struct ColsParams {
  const float* src;         // channel c: src + (use_cmap ? cmap[c] : c) * src_cstride, position 0 = the group's first sample
  long long src_cstride;
  int use_cmap;
  int cmap[8];
  long long nsrc;           // positions >= nsrc read zeros
  const float* hist;        // [C][hist_len]: the samples at positions -hist_len ... -1 (nullptr: no negative positions)
  long long hist_len;
  long long w0, L;          // segment q's window starts at position w0 + q L
  int nseg;
  float2* dst;              // [C][kRows][nseg][kN2]
};

// grid (kN2 / kCols, nseg, C), block kColThreads, dynamic smem kColSmem
__global__ void __launch_bounds__(kColThreads, 2) k_fs_cols(ColsParams p, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem_fs[];
  float2* tab = pc_smem_fs;
  float2* buf = pc_smem_fs + kF512_TabLen;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int n2_0 = blockIdx.x * kCols, q = blockIdx.y, c = blockIdx.z;
  const long long w0 = p.w0 + (long long)q * p.L;
  int ch = c;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (p.use_cmap && i == c) ch = p.cmap[i];
  const float* src = p.src + (long long)ch * p.src_cstride;
  const float* hist = p.hist ? p.hist + (long long)c * p.hist_len + p.hist_len : nullptr;
  for (int j = tid; j < kF512_TabLen; j += kColThreads) tab[j] = tab512[j];
  // the tile: row n1 = w + 16 i of the 32 columns, one 128-byte run per warp and row.  Column pair u = lane / 2 as one
  // complex column: z[n1] at buf[u * 512 + (n1 ^ u)] (the XOR spreads the 16 pairs of a store over the banks), i.e.
  // in the exchange buffer of warp u
  float* tile = reinterpret_cast<float*>(buf);
  const int u = lane >> 1;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const long long pos = w0 + (long long)(w + 16 * (i + 16 * half)) * kN2 + n2_0 + lane;
      float x = 0.0f;
      if (pos >= 0) { if (pos < p.nsrc) x = __ldg(src + pos); }
      else if (hist) x = __ldg(hist + pos);
      v[i] = x;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) tile[u * 2 * kF512_Xch + 2 * ((w + 16 * (i + 16 * half)) ^ u) + (lane & 1)] = v[i];
  }
  __syncthreads();
  float2* S = buf + w * kF512_Xch;
  float2 a[16];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int n2 = 0; n2 < 8; ++n2) a[8 * h + n2] = S[(64 * n2 + lane + 32 * h) ^ w];
  __syncwarp();
  // step 1 of the 512-point DFT on all eight points of the columns m = lane, lane + 32 (f512_fwd_p1 without the zero half)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = lane + 32 * h;
    float2* x = a + 8 * h;
    f512_dft8<false>(x);
    S[f512_s1(0, m)] = x[0];
#pragma unroll
    for (int k2 = 1; k2 < 8; ++k2) S[f512_s1(k2, m)] = f2_cmul<false>(x[k2], tab[kF512_T1 + k2 * 64 + m]);
  }
  __syncwarp();
  float2 A[8], B[8];
  f512_mid_load<false>(lane, S, tab, A, B);
  __syncwarp();
  f512_mid_store<false>(lane, S, A, B);
  __syncwarp();
  const int la = f512_la(lane), lb = f512_lb(lane);
#pragma unroll
  for (int n0 = 0; n0 < 8; ++n0) {
    A[n0] = S[f512_s2(la & 7, la >> 3, n0)];
    B[n0] = S[f512_s2(lb & 7, lb >> 3, n0)];
  }
  f512_dft8<false>(A);      // A[q1] = Z[la + 64 q1]
  f512_dft8<false>(B);      // B[q1] = Z[lb + 64 q1]
  __syncthreads();          // every exchange buffer is done: buf becomes the staged rows [k1][pair]
  float4* st = reinterpret_cast<float4*>(buf);
  // bin k of the two columns from Z[k] and zm = Z[512 - k]
  auto put = [&](int k, float2 zk, float2 zm) {
    const float2 e = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));     // (Z[k] + conj Z[-k]) / 2
    const float2 d = make_float2(0.5f * (zk.x - zm.x), 0.5f * (zk.y + zm.y));     // (Z[k] - conj Z[-k]) / 2
    st[k * kStage4 + w] = make_float4(e.x, e.y, d.y, -d.x);                        // second column: d / i
  };
  if (lane != 0) {          // the mirror of la + 64 q1 is lb + 64 (7 - q1)
#pragma unroll
    for (int q1 = 0; q1 < 4; ++q1) {
      put(la + 64 * q1, A[q1], B[7 - q1]);
      put(lb + 64 * q1, B[q1], A[7 - q1]);
    }
  } else {                  // residues 0 and 32: bins 0, 64, ..., 256 and 32, 96, 160, 224
#pragma unroll
    for (int q1 = 0; q1 < 5; ++q1) put(64 * q1, A[q1], A[(8 - q1) & 7]);
#pragma unroll
    for (int q1 = 0; q1 < 4; ++q1) put(32 + 64 * q1, B[q1], B[7 - q1]);
  }
  __syncthreads();
  float4* dst = reinterpret_cast<float4*>(p.dst + ((long long)c * kRows * p.nseg + q) * kN2 + n2_0);
  const long long rs4 = (long long)p.nseg * (kN2 / 2);       // row stride in float4
#pragma unroll 3
  for (int e = tid; e < kRows * 16; e += kColThreads) {
    const int k1 = e >> 4, pr = e & 15, n2 = n2_0 + 2 * pr;
    const float4 s = st[k1 * kStage4 + pr];
    const float2 x0 = lfft::cmul(make_float2(s.x, s.y), wM(n2 * k1, false));
    const float2 x1 = lfft::cmul(make_float2(s.z, s.w), wM((n2 + 1) * k1, false));
    dst[k1 * rs4 + pr] = make_float4(x0.x, x0.y, x1.x, x1.y);
  }
}

// ---- pass 2 ---------------------------------------------------------------------------------------------------
struct RowsParams {
  float2* X;                // [C][kRows][nseg][kN2], in place
  const float2* S;          // [C][kRows][kN2] (MUL)
  int nseg;
  unsigned items;           // C * kRows * nseg: item i is row i of X, spectrum row i / nseg
};

// dynamic shared memory of the row pass: every thread's twiddle bases, the stage (the next item's row) and, for MUL,
// the spectrum row
template <bool MUL>
constexpr size_t rows_smem() { return (size_t)(2 * lfft::kThreads + (MUL ? 2 : 1) * kN2) * sizeof(float2); }

// lfft::fft4096 with thread j's twiddle bases read from tw[2 j], tw[2 j + 1] where each pass needs them: held in
// registers across the loop of k_fs_rows, they would not fit its register budget
__device__ __forceinline__ void fft4096_tw(float2 (&a)[16], float* sre, float* sim, int j, const float2* tw) {
  lfft::dft16(a);
  lfft::exchange<1>(a, sre, sim, j);
  lfft::twiddle(a, tw[2 * j]);
  lfft::dft16(a);
  lfft::exchange<16>(a, sre, sim, j);
  lfft::twiddle(a, tw[2 * j + 1]);
  lfft::dft16(a);
}

// Persistent: grid = the resident CTAs (at most items), block lfft::kThreads, dynamic smem rows_smem<MUL>().  CTA b
// walks item_range(items, gridDim.x, b) in order, so the resident CTAs move through one contiguous region of X and a
// CTA's items share a spectrum row nseg at a time.  While item i is transformed, item i + 1's row is already on its way
// into the stage by a bulk copy (`full` mbarrier); the spectrum row is bulk-copied into shared memory only when the
// item's row k1 changes (`spec` mbarrier).  Each stage and spectrum copy is issued by thread 0 after a barrier that
// follows every thread's last read of the previous content.  Results are stored from registers.  MUL = false (the IR
// spectrum): the forward transform only, stored times 1 / M
template <bool MUL>
__global__ void __launch_bounds__(lfft::kThreads, 2) k_fs_rows(RowsParams p) {
  __shared__ float sre[lfft::kSmemFloats], sim[lfft::kSmemFloats];
  __shared__ unsigned long long bar[2];             // full, spec
  extern __shared__ __align__(128) float2 pc_smem_fs_rows[];
  float2* tw = pc_smem_fs_rows;
  float2* stage = pc_smem_fs_rows + 2 * lfft::kThreads;
  float2* spec = stage + kN2;
  constexpr unsigned kRowBytes = kN2 * sizeof(float2);
  const int j = threadIdx.x;
  const ItemRange rg = item_range(p.items, gridDim.x, blockIdx.x);
  if (rg.begin >= rg.end) return;
  if (j == 0) {
    tc::mbar_init(&bar[0], 1);
    tc::mbar_init(&bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tc::mbar_expect(&bar[0], kRowBytes);
    tc::bulk_load(stage, p.X + (size_t)rg.begin * kN2, kRowBytes, &bar[0]);
  }
  lfft::twiddle_bases(j, tw[2 * j], tw[2 * j + 1]);
  __syncthreads();
  unsigned srow = ~0u, nspec = 0;
  for (unsigned i = rg.begin; i < rg.end; ++i) {
    float2 a[16];
    (void)tc::mbar_wait(&bar[0], (i - rg.begin) & 1u);
#pragma unroll
    for (int r = 0; r < 16; ++r) a[r] = stage[j + 256 * r];
    __syncthreads();                                // the stage and the previous item's spectrum row are read
    const unsigned row = MUL ? i / (unsigned)p.nseg : 0u;
    if (j == 0) {
      if (i + 1 < rg.end) {
        tc::mbar_expect(&bar[0], kRowBytes);
        tc::bulk_load(stage, p.X + (size_t)(i + 1) * kN2, kRowBytes, &bar[0]);
      }
      if (MUL && row != srow) {
        tc::mbar_expect(&bar[1], kRowBytes);
        tc::bulk_load(spec, p.S + (size_t)row * kN2, kRowBytes, &bar[1]);
      }
    }
    if (MUL && row != srow) { srow = row; ++nspec; }
    fft4096_tw(a, sre, sim, j, tw);
    float2* y = p.X + (size_t)i * kN2;
    if (MUL) {
      (void)tc::mbar_wait(&bar[1], (nspec - 1) & 1u);
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const float2 v = lfft::cmul(a[r], spec[j + 256 * r]);
        a[r] = make_float2(v.x, -v.y);               // conj: the inverse as a forward transform
      }
      fft4096_tw(a, sre, sim, j, tw);
#pragma unroll
      for (int r = 0; r < 16; ++r) y[j + 256 * r] = make_float2(a[r].x, -a[r].y);
    } else {
      constexpr float inv_m = 1.0f / (float)kM;     // exact
#pragma unroll
      for (int r = 0; r < 16; ++r) y[j + 256 * r] = make_float2(a[r].x * inv_m, a[r].y * inv_m);
    }
  }
}

// ---- pass 3 ---------------------------------------------------------------------------------------------------
struct ColsInvParams {
  const float2* X;          // [C][kRows][nseg][kN2] (pass 2)
  int nseg;
  Plan plan;
  float* dst;               // channel c: dst + c * dst_cstride, index t = group output t
  long long dst_cstride;
};

// grid (kN2 / kCols, nseg, C), block kColThreads, dynamic smem kColSmem
__global__ void __launch_bounds__(kColThreads, 2) k_fs_cols_inv(ColsInvParams p, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem_fs[];
  float2* tab = pc_smem_fs;
  float2* buf = pc_smem_fs + kF512_TabLen;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int n2_0 = blockIdx.x * kCols, q = blockIdx.y, c = blockIdx.z;
  const float4* src = reinterpret_cast<const float4*>(p.X + ((long long)c * kRows * p.nseg + q) * kN2 + n2_0);
  const unsigned rs4 = (unsigned)p.nseg * (kN2 / 2);         // row stride in float4
  float4* st = reinterpret_cast<float4*>(buf);
  constexpr int kIt = (kRows * 16 + kColThreads - 1) / kColThreads;
  float4 v[kIt];
#pragma unroll
  for (int i = 0; i < kIt; ++i) {
    const int e = tid + i * kColThreads;
    if (e < kRows * 16) v[i] = __ldg(src + (size_t)((e >> 4) * rs4) + (e & 15));
  }
  for (int j = tid; j < kF512_TabLen; j += kColThreads) tab[j] = tab512[j];
#pragma unroll
  for (int i = 0; i < kIt; ++i) {
    const int e = tid + i * kColThreads;
    if (e >= kRows * 16) break;
    const int k1 = e >> 4, pr = e & 15, n2 = n2_0 + 2 * pr;
    float2 x0 = lfft::cmul(make_float2(v[i].x, v[i].y), wM(n2 * k1, true));
    float2 x1 = lfft::cmul(make_float2(v[i].z, v[i].w), wM((n2 + 1) * k1, true));
    if (k1 == 0 || k1 == kN1 / 2) { x0.y = 0.0f; x1.y = 0.0f; }   // real bins of a real column
    st[k1 * kStage4 + pr] = make_float4(x0.x, x0.y, x1.x, x1.y);
  }
  __syncthreads();
  // the packed column pair's full spectrum, Z[k] = Da[k] + i Db[k] with D[512 - k] = conj D[k]
  auto z_at = [&](int k) {
    const int kk = k <= kN1 / 2 ? k : kN1 - k;
    const float4 s = st[kk * kStage4 + w];
    const float sg = k <= kN1 / 2 ? 1.0f : -1.0f;
    return make_float2(s.x - sg * s.w, sg * s.y + s.z);
  };
  const int la = f512_la(lane), lb = f512_lb(lane);
  float2 ZA[8], ZB[8];
#pragma unroll
  for (int q1 = 0; q1 < 8; ++q1) { ZA[q1] = z_at(la + 64 * q1); ZB[q1] = z_at(lb + 64 * q1); }
  __syncthreads();          // the staged rows are read: buf becomes the warps' exchange buffers
  float2* S = buf + w * kF512_Xch;
  // the rest of f512_inv_p1_core (the column spectrum needs no un-split)
  f512_dft8<true>(ZA);
  f512_dft8<true>(ZB);
#pragma unroll
  for (int n0 = 0; n0 < 8; ++n0) {
    S[f512_s2(la & 7, la >> 3, n0)] = n0 ? f2_cmul<true>(ZA[n0], tab[kF512_T1 + n0 * 64 + la]) : ZA[0];
    S[f512_s2(lb & 7, lb >> 3, n0)] = n0 ? f2_cmul<true>(ZB[n0], tab[kF512_T1 + n0 * 64 + lb]) : ZB[0];
  }
  __syncwarp();
  float2 A[8], B[8];
  f512_mid_load<true>(lane, S, tab, A, B);
  __syncwarp();
  f512_mid_store<true>(lane, S, A, B);
  __syncwarp();
  // last step (f512_inv_p3 over all eight output rows): A / B = the columns m = lane / lane + 32
#pragma unroll
  for (int k2 = 0; k2 < 8; ++k2) { A[k2] = S[f512_s1(k2, lane)]; B[k2] = S[f512_s1(k2, lane + 32)]; }
  f512_dft8<true>(A);       // A[j] = output row n1 = 64 j + lane of the pair
  f512_dft8<true>(B);
  __syncthreads();          // buf becomes the output tile [n1][2 * kStage4 floats]
  float2* ot = buf;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    ot[(64 * j + lane) * kStage4 + w] = A[j];
    ot[(64 * j + lane + 32) * kStage4 + w] = B[j];
  }
  __syncthreads();
  const float* of = reinterpret_cast<const float*>(buf);
  float* dst = p.dst + (long long)c * p.dst_cstride;
#pragma unroll 4
  for (int i = 0; i < 32; ++i) {
    const int n1 = w + 16 * i;
    const long long t = output_of(p.plan, q, (long long)n1 * kN2 + n2_0 + lane);
    if (t >= 0) dst[t] = of[n1 * 2 * kStage4 + lane];
  }
}

#endif  // __CUDACC__

}  // namespace fs
}  // namespace pc
