// kernels_tc.cuh — K2x: the batched sweep on the Hopper tensor cores (wgmma.mma_async f16 with FP32 accumulate,
// 3xFP16 split of power-of-two scaled operands).
//
//   Y[t][k] = sum_p H[p][k] * X[t - p][k]          (FFTConvolver.cpp:176-187, Utilities.cpp:62-111)
//
// For a long launch group the sweep is, per frequency bin k, a 1-D convolution ALONG THE BLOCK INDEX t of the
// bin's time line x_k[t] with the bin's P partition values H[.][k].  Cut t into segments of R = 64 steps: the
// outputs of segment n are a Toeplitz matrix of H applied to a window of x,
//
//   D[i][n] = sum_j A[i][j] * B[j][n],   A[i][j] = H[i + Q - j],   B[j][n] = x[64 n - Q + j],   0 <= j < K = Q + 64
//
// (Q = P - 1 rounded up to 64) — a GEMM with M = 64 outputs per segment, N = segments, K = Q + 64, one per bin
// and channel.  The complex product takes three real GEMMs (Gauss), with the images [Hr ; Hi ; Hr + Hi] stacked into
// 192 rows and three time lines xr, xi, xr + xi:
//   D1 = Hr xr,  D2 = Hi xi,  D3 = (Hr + Hi)(xr + xi);   y.re = D1 - D2,  y.im = D3 - (D1 + D2)
//   (entry 0 = DC / Nyquist: y = (D1, D2))
// The sweep issues the transposed products D^T[n][i] = sum_j B[j][n] * A[i][j]: the wgmma A operand is a time-line
// window (M = 64 segments), the wgmma B operand the 64-row slice of the image that goes with it (N = 64).  Work items
// are pairs of tiles of one line: MMA warpgroup w takes tile 2m + w, and both read the same image stream.
//
// FP32 accuracy comes from the 3xFP16 split: a = a_hi + a_lo, b = b_hi + b_lo (each FP16-exact, round to nearest),
// and a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi accumulated in FP32 (dropped term ~2^-22 relative).  FP16 has tf32's
// 11-bit significand, and its MMAs issue at twice the tf32 rate; what it lacks is exponent range, which exact
// power-of-two scales restore: 2^eh per line (channel, bin) for H, chosen once per IR from the bin's P values, and
// 2^ex per tile and time line (re / im / re + im) for x, chosen from the 80 x 64 samples the tile reads; Hr + Hi has
// its own 2^eh'.  Each puts the window's largest magnitude into [2^14, 2^15) (scale_exp); the epilogue multiplies each
// product by its own 2^-(ex + eh).  A sample keeps the full ~2^-22 relative precision while it lies within ~2^-17 of
// its window's peak; below that its lo part is an FP16 subnormal and the error is absolute, at most ~2^-39 of the
// window's peak (DESIGN.md §5).
//
// The time-line operand of chunk c (64 values of j) is a ROW-SHIFTED WINDOW of one shared-memory strip.  The bin's
// time line is stored as rows of 64 samples; B[64c + jj][n] = x[64 (n + c) + jj - Q] is row n + c of the strip, i.e.
// the same SWIZZLE_128B K-major strip (rows of 64 halves = 128 B) with the descriptor start address advanced by
// c * 128 bytes: the 128-byte swizzle is a function of the absolute shared-memory address, so a start address inside
// the 1024-byte swizzle atom reads the rows it names.  One 80-row strip per time line and hi / lo part feeds all K
// chunks of a 64-segment tile.  Each MMA warpgroup owns six strips (60 KB); between pairs it reads its next tile's FP32
// rows from global memory (asked into L2 while the previous pair ran), picks ex and writes the strips itself.  The
// Toeplitz images of H (24 KB per chunk and hi / lo part, pre-swizzled, 1-D bulk copies) stream through a 3-stage ring.
//
// Kernels: k_tc_build_a (H -> FP16 hi/lo Toeplitz tile images and eh, once per IR), k_tc_split_x (timeline rows ->
// per-bin FP32 time lines), k_tc_sweep (a producer warp streams the image ring / two MMA warpgroups convert their
// strips and accumulate in registers; the epilogue combines the complex product into bin-major float2 lines), k_tc_merge_y
// (bin-major lines -> Y rows, for the groups whose inverse FFT reads rows).
#pragma once

#if defined(PC_EMULATE)                             // tests/emu: only the host-side geometry and layout functions
#define PC_TC_HD inline
#else
#include <cuda_runtime.h>
#define PC_TC_HD inline __host__ __device__
#endif
#include <cstdint>
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif

namespace pc {
namespace tc {

constexpr int kR = 64;                              // block steps per segment
constexpr int kN = 64;                              // segments per tile (MMA M of the transposed product)
constexpr int kStripRows = kN + 16;                 // a tile's rows plus the largest row shift (15) and padding
constexpr int kStripBytes = kStripRows * 128;       // 10240: 80 rows of 128 B (a multiple of the 1024-byte swizzle atom)
constexpr int kATileBytes = 128 * 128;              // one Toeplitz tile image: 128 rows of 128 B
constexpr int kAStages = 4;
constexpr int kThreads = 384;                       // two MMA warpgroups + a producer warpgroup
constexpr int kMmaRegs = 232, kProducerRegs = 40;   // setmaxnreg split of the register file: 256 x 232 + 128 x 40 <= 64 K

// Geometry.  Q, nseg, ntile, rows (64-sample rows per time line) and Lty are those of the FP16 sweep; `nchunk`
// (K chunks of 32), kMaxChunks, kFlush and kSmemBytes describe the earlier tf32 form and are only read by
// tests/test_tc_layout.py (as are sw128 and xt_index below).  geom_ok's limit (Q <= 960, P <= 961) is the same in both.
constexpr int kMaxChunks = 32;
constexpr int kSmemBytes = 8 * kStripBytes + kAStages * kATileBytes + 1024;
constexpr int kFlush = 4;

struct Geom {
  int P, Q, nchunk, nb, nseg, ntile, rows;
  long long Lt, Lty;
};

PC_TC_HD Geom make_geom(int P, int nb) {
  Geom g;
  g.P = P;
  g.Q = ((P > 1 ? P - 1 : 0) + 63) / 64 * 64;
  g.nchunk = g.Q / 32 + 2;
  g.nb = nb;
  g.nseg = (nb + kR - 1) / kR;
  g.ntile = (g.nseg + kN - 1) / kN;
  g.rows = g.ntile * kN + 16;
  g.Lt = (long long)g.rows * 64;
  g.Lty = (long long)g.ntile * kN * 64;
  return g;
}
PC_TC_HD bool geom_ok(const Geom& g, int B) { return g.nchunk <= kMaxChunks && B % 32 == 0 && g.nb > 0; }

// byte offset of element (row r, float e < 32) in a SWIZZLE_128B K-major image with a 1024-byte aligned base
PC_TC_HD uint32_t sw128(uint32_t r, uint32_t e) { return r * 128u + ((((e >> 2) ^ (r & 7u)) & 7u) << 4) + (e & 3u) * 4u; }

// tf32 time-line layout: [line][re_hi, re_lo, im_hi, im_lo][e][row R][32 floats], pre-swizzled
PC_TC_HD size_t xt_index(long long line, int pl, int e, long long R, int jj, int rows) {
  return ((((size_t)line * 4 + pl) * 2 + e) * (size_t)rows + (size_t)R) * 32 + (size_t)(((((jj >> 2) ^ (int)(R & 7)) & 7) << 2) | (jj & 3));
}

// ---- FP16 form ---------------------------------------------------------------------------------------------------
constexpr int kChunkK = 64;                         // K values per chunk: one 128-byte row of halves
constexpr int kMaxChunksF16 = 16;                   // row shifts 0..15 stay inside the 80-row strip
constexpr int kStageBytes = 2 * kStripRows * 64 * 4;  // FP32 re / im rows of one tile (40 KB)
constexpr int kSmemBytesF16 = 8 * kStripBytes + kAStages * kATileBytes + kStageBytes + 1024;
constexpr int kStripThreads = 96;                   // producer warps 9-11 convert the strips (warp 8 feeds the ring)
// K chunks accumulated by the tensor core before the FP32 register add: 2 x 64 = the same K per chain as 4 x 32 tf32
constexpr int kFlushF16 = 2;

PC_TC_HD int nchunk_f16(int Q) { return Q / kChunkK + 1; }

// byte offset of element (row r, half e < 64) in a SWIZZLE_128B K-major image with a 1024-byte aligned base
PC_TC_HD uint32_t sw128_h(uint32_t r, uint32_t e) { return r * 128u + ((((e >> 3) ^ (r & 7u)) & 7u) << 4) + (e & 7u) * 2u; }

// FP32 time lines: [line][re, im][rows * 64 samples]; sample tau sits in row tau / 64, so the 80 rows of tile nt's
// strip are the contiguous samples 64 * 64 nt ... + 80 * 64
PC_TC_HD size_t xf_index(long long line, int comp, long long tau, int rows) {
  return ((size_t)line * 2 + comp) * (size_t)rows * 64 + (size_t)tau;
}

// complex result: [line][ystride] float2, sweep output tau at slot kYLead + tau.  The lead slots in front of output 0
// hold the block before it where the inverse FFT wants it there (its overlap-add reads every block's predecessor)
constexpr int kYLead = 8;
PC_TC_HD long long yc_stride(const Geom& g) { return g.Lty + 2 * kYLead; }

// Toeplitz images of the four-product form: [line][chunk][hi, lo][128 rows x 64 halves]
PC_TC_HD size_t a_image_bytes(size_t lines, int nchunk) { return lines * (size_t)nchunk * 2 * kATileBytes; }

// ---- three-product (Gauss) form: what k_tc_sweep runs ------------------------------------------------------------
// kATileBytes, kAStages, kStageBytes, kSmemBytesF16, kStripThreads and a_image_bytes above describe the four-product
// form it replaced; tests/test_tc_f16_layout.py reads them.
constexpr int kGRows = 192;                         // image rows: [Hr ; Hi ; Hr + Hi], 64 output steps each
constexpr int kGSliceBytes = 64 * 128;              // one 64-row slice (8 KB, a multiple of the 1024-byte swizzle atom)
constexpr int kGImageBytes = kGRows * 128;          // 24 KB: one chunk's hi or lo image, one ring stage
constexpr int kGStages = 3;
constexpr int kGStripBytes = 6 * kStripBytes;       // per MMA warpgroup: re, im, re + im lines x hi, lo strips (60 KB)
constexpr int kSmemBytesGauss = 2 * kGStripBytes + kGStages * kGImageBytes + 1024;
constexpr int kGProducts = 3;

// Toeplitz images: [line][chunk][hi, lo][192 rows x 64 halves], then eh of every line ([line][Hr / Hi, Hr + Hi] int)
PC_TC_HD size_t a_image_bytes_gauss(size_t lines, int nchunk) { return lines * (size_t)nchunk * 2 * kGImageBytes; }
// work items: pairs of consecutive 64-segment tiles of one line (the last pair of an odd tile count has one)
PC_TC_HD int npair(const Geom& g) { return (g.ntile + 1) / 2; }
// 64-sample rows of the FP32 time lines that pair m reads (tiles 2m and 2m + 1 overlap in 16 rows)
PC_TC_HD int pair_rows(int ntile, int m) { return (2 * m + 1 < ntile ? kN : 0) + kStripRows; }

// power-of-two exponent that puts a window's largest magnitude into [2^14, 2^15).  m = bit pattern of that magnitude
// (sign cleared).  Zero and non-finite windows use 0: zeros stay exact zeros, NaN / Inf propagate unscaled.
PC_TC_HD int scale_exp(uint32_t m) {
  if (m == 0u || m >= 0x7f800000u) return 0;
  int E = (int)(m >> 23);                           // biased exponent: m in [2^(E-127), 2^(E-126))
  if (E == 0) {                                     // subnormal: the exponent of its leading bit
    E = 1;
    while (m < 0x00800000u) { m <<= 1; --E; }
  }
  return 141 - E;
}

#if defined(__CUDACC__)

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t abs_bits(float v) { return __float_as_uint(v) & 0x7fffffffu; }
__device__ __forceinline__ float pow2f(int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }   // k in [-126, 127]

// ---- H -> Toeplitz tile images ---------------------------------------------------------------------------------
struct BuildAParams {
  const float2* H;          // [C][Prows][B]
  long long h_cstride;
  int B, P, Q, nchunk;
  __half* A;                // [C*B lines][nchunk][hi, lo][192 x 64]: SWIZZLE_128B images of 2^eh Hr, 2^eh Hi, 2^eh' (Hr + Hi)
  int* eh;                  // [C*B lines][eh, eh']
};

// grid (nchunk, B, C), block 256.  Every chunk's CTA finds the same eh / eh' from the bin's P values (a few KB, once
// per IR).  Hr + Hi is rounded to FP32 before it is scaled and split.
__global__ void __launch_bounds__(256) k_tc_build_a(BuildAParams p) {
  __shared__ uint32_t red[8][2];
  const int c = blockIdx.x, k = blockIdx.y, ch = blockIdx.z;
  const long long line = (long long)ch * p.B + k;
  const float2* Hk = p.H + (long long)ch * p.h_cstride + k;
  uint32_t m = 0, ms = 0;
  for (int pp = threadIdx.x; pp < p.P; pp += 256) {
    const float2 h = Hk[(long long)pp * p.B];
    m = max(m, max(abs_bits(h.x), abs_bits(h.y)));
    ms = max(ms, abs_bits(__fadd_rn(h.x, h.y)));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  ms = __reduce_max_sync(0xffffffffu, ms);
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = m; red[threadIdx.x >> 5][1] = ms; }
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 8; ++w) { m = max(m, red[w][0]); ms = max(ms, red[w][1]); }
  const int eh = scale_exp(m), ehs = scale_exp(ms);
  if (c == 0 && threadIdx.x == 0) { p.eh[2 * line] = eh; p.eh[2 * line + 1] = ehs; }
  __half* hi = p.A + (line * p.nchunk + c) * 2 * (kGImageBytes / 2);
  __half* lo = hi + kGImageBytes / 2;
  for (int idx = threadIdx.x; idx < kGImageBytes / 2; idx += 256) {
    const int mr = idx >> 6, jj = idx & 63;
    const int part = mr >> 6, i = mr & 63;
    const int pp = i + p.Q - (kChunkK * c + jj);
    float v = 0.0f;
    if (pp >= 0 && pp < p.P) {
      const float2 h = Hk[(long long)pp * p.B];
      v = part == 0 ? ldexpf(h.x, eh) : part == 1 ? ldexpf(h.y, eh) : ldexpf(__fadd_rn(h.x, h.y), ehs);
    }
    const __half vh = __float2half_rn(v);
    const uint32_t off = sw128_h((uint32_t)mr, (uint32_t)jj) >> 1;
    hi[off] = vh;
    lo[off] = __float2half_rn(v - __half2float(vh));
  }
}

// ---- timeline rows -> per-bin FP32 time lines ------------------------------------------------------------------
struct SplitXParams {
  const float2* X;          // [C][R][B]
  long long x_cstride;
  long long row_base;       // timeline row of tau = 0 (= row of output block 0 minus Q); may be negative
  long long row_lo, row_hi; // rows outside [row_lo, row_hi) read as zero
  int B;
  int rows;                 // 64-sample rows per time line
  float* Xt;
  // samples in [skip_lo, skip_hi) are left alone (the B = 512 forward FFT wrote them: k_fwd_fft512_lines).  The grid
  // covers the 32-sample chunks 0 ... nchunk_lo - 1 and chunk_hi ... rows * 2 - 1 (split_x_chunks)
  long long skip_lo, skip_hi;
  int nchunk_lo, chunk_hi;
};

// the chunks of 32 samples a split has to visit: [0, *nlo) and [*hi, rows * 2)
PC_TC_HD void split_x_chunks(int rows, long long skip_lo, long long skip_hi, int* nlo, int* hi) {
  *nlo = (int)((skip_lo + 31) / 32);
  *hi = (int)(skip_hi / 32) > *nlo ? (int)(skip_hi / 32) : *nlo;
  if (*hi > rows * 2) *hi = rows * 2;
}

// grid (nchunk_lo + rows * 2 - chunk_hi, B / 32, C), block (32, 8)
__global__ void __launch_bounds__(256) k_tc_split_x(SplitXParams p) {
  __shared__ float2 tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int chunk = (int)blockIdx.x < p.nchunk_lo ? (int)blockIdx.x : p.chunk_hi + ((int)blockIdx.x - p.nchunk_lo);
  const long long tau0 = (long long)chunk * 32;
  const int k0 = blockIdx.y * 32, ch = blockIdx.z;
  for (int r = ty; r < 32; r += 8) {
    const long long row = p.row_base + tau0 + r;
    const bool skip = tau0 + r >= p.skip_lo && tau0 + r < p.skip_hi;
    float2 v = make_float2(0.0f, 0.0f);
    if (!skip && row >= p.row_lo && row < p.row_hi) v = p.X[(long long)ch * p.x_cstride + row * p.B + k0 + tx];
    tile[r][tx] = v;
  }
  __syncthreads();
  if (tau0 + tx >= p.skip_lo && tau0 + tx < p.skip_hi) return;
  for (int kk = ty; kk < 32; kk += 8) {
    const float2 v = tile[tx][kk];
    const long long line = (long long)ch * p.B + k0 + kk;
    p.Xt[xf_index(line, 0, tau0 + tx, p.rows)] = v.x;
    p.Xt[xf_index(line, 1, tau0 + tx, p.rows)] = v.y;
  }
}

// ---- bin-major complex lines -> Y rows -------------------------------------------------------------------------
struct MergeYParams {
  const float2* Yc;         // [C*B lines][ystride], output t at slot kYLead + t
  long long ystride;
  int B, nb;
  float2* Y;
  long long y_cstride, y_rstride, yrow0;
};

// grid (ceil(nb / 32), B / 32, C), block (32, 8)
__global__ void __launch_bounds__(256) k_tc_merge_y(MergeYParams p) {
  __shared__ float2 tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long long t0 = (long long)blockIdx.x * 32;
  const int k0 = blockIdx.y * 32, ch = blockIdx.z;
  for (int kk = ty; kk < 32; kk += 8) {
    const long long line = (long long)ch * p.B + k0 + kk;
    tile[tx][kk] = t0 + tx < p.nb ? p.Yc[line * p.ystride + kYLead + t0 + tx] : make_float2(0.0f, 0.0f);
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const long long t = t0 + r;
    if (t < p.nb) p.Y[(long long)ch * p.y_cstride + (p.yrow0 + t) * p.y_rstride + k0 + tx] = tile[r][tx];
  }
}

// ---- the sweep -------------------------------------------------------------------------------------------------
struct SweepParams {
  const __half* A;
  const int* eh;            // [lines][eh, eh']
  const float* Xt;
  float2* Yc;               // [lines][ystride] complex result, bin-major (kYLead)
  long long ystride;
  int lines, ntile, npair, nchunk, rows, B;
  int* err;                // (mapped host word) set non-zero when a barrier wait gave up — a bug, not a data condition
};

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive1(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_wait(unsigned long long* bar, unsigned parity) {
  const long long t0 = clock64();
  unsigned ok = 0;
  while (true) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    if (ok) return true;
    if (clock64() - t0 > 4000000000LL) return false;
  }
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
// orders this thread's generic-proxy shared-memory accesses before later async-proxy ones (bulk copies, wgmma)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// asks L2 for `bytes` (a multiple of 16) of global memory at a 16-byte aligned address; no completion to wait for
__device__ __forceinline__ void prefetch_l2(const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(src), "r"(bytes) : "memory");
}
// wgmma shared-memory descriptor of a SWIZZLE_128B K-major operand (rows of 128 bytes, 8-row groups 1024 bytes
// apart, base offset 0), split in two words: only the low word (start address in 16-byte units | leading-offset
// field, unused by swizzled K-major layouts) changes between MMAs
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// keeps the compiler from moving or copying accumulator registers across the wgmma issue / wait points
__device__ __forceinline__ void fence_operands(float (&d)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) asm volatile("" : "+f"(d[j]) :: "memory");
}
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// d[64 x 64] (+)= A[64 x 16] * B[16 x 64], f16 operands (both K-major) from shared memory, FP32 accumulators in 32
// registers per thread
__device__ __forceinline__ void mma_f16(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t accumulate) {
  const uint64_t da = ((uint64_t)kDescHi << 32) | a_lo, db = ((uint64_t)kDescHi << 32) | b_lo;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
               "%32, %33, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                 "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
                 "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
                 "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
// two FP32 values -> their FP16 hi parts and the FP16 rounding of the residuals, packed in pairs
__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ void bar_sync_n(uint32_t id, uint32_t count) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(count) : "memory"); }

// One MMA warpgroup's strips of tile nt: FP32 rows of the re and im time lines -> re + im (one FP32 add) -> max |x| per
// line -> ex -> FP16 hi / lo SWIZZLE_128B strips [re, im, re + im][hi, lo].  Called once the warpgroup's MMAs on its
// previous strips are complete; the 80 x 64 samples of each line are read from global memory straight into registers
// (5 units of 8 samples per thread and line; the ring producer asked L2 for them while the previous pair ran).
__device__ __forceinline__ void tc_convert_strips(const SweepParams& P, int line, int nt, unsigned char* strips, uint32_t (*red)[kGProducts],
                                                  int wq, int lane, int t128, uint32_t bar, int (&ex)[kGProducts]) {
  constexpr int kU = kStripRows * 8 / 128;                // 16-byte units of 8 halves per thread and line
  const float4* xr = reinterpret_cast<const float4*>(P.Xt + xf_index(line, 0, (long long)nt * kN * 64, P.rows));
  const float4* xi = reinterpret_cast<const float4*>(P.Xt + xf_index(line, 1, (long long)nt * kN * 64, P.rows));
  float4 v[kU][2][2];
#pragma unroll
  for (int k = 0; k < kU; ++k) {
    const int u = t128 + 128 * k;
    v[k][0][0] = __ldg(xr + 2 * u); v[k][0][1] = __ldg(xr + 2 * u + 1);
    v[k][1][0] = __ldg(xi + 2 * u); v[k][1][1] = __ldg(xi + 2 * u + 1);
  }
  uint32_t mx[kGProducts] = {0u, 0u, 0u};
#pragma unroll
  for (int k = 0; k < kU; ++k)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 a = v[k][0][h], b = v[k][1][h];
      mx[0] = max(mx[0], max(max(abs_bits(a.x), abs_bits(a.y)), max(abs_bits(a.z), abs_bits(a.w))));
      mx[1] = max(mx[1], max(max(abs_bits(b.x), abs_bits(b.y)), max(abs_bits(b.z), abs_bits(b.w))));
      mx[2] = max(mx[2], max(max(abs_bits(__fadd_rn(a.x, b.x)), abs_bits(__fadd_rn(a.y, b.y))),
                             max(abs_bits(__fadd_rn(a.z, b.z)), abs_bits(__fadd_rn(a.w, b.w)))));
    }
#pragma unroll
  for (int p = 0; p < kGProducts; ++p) {
    mx[p] = __reduce_max_sync(0xffffffffu, mx[p]);
    if (lane == 0) red[wq][p] = mx[p];
  }
  bar_sync_n(bar, 128);
#pragma unroll
  for (int p = 0; p < kGProducts; ++p) ex[p] = scale_exp(max(max(red[0][p], red[1][p]), max(red[2][p], red[3][p])));
#pragma unroll
  for (int p = 0; p < kGProducts; ++p) {
    // 2^ex as two factors: each is a normal float for every ex scale_exp returns, and x * s1 * s2 is exact wherever
    // the FP16 result can hold it
    const float s1 = pow2f(ex[p] >> 1), s2 = pow2f(ex[p] - (ex[p] >> 1));
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      const int u = t128 + 128 * k, r = u >> 3, q = u & 7;
      float f[8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float4 a = v[k][0][h], b = v[k][1][h];
        const float4 w = p == 0 ? a : p == 1 ? b : make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
        f[4 * h] = w.x * s1 * s2; f[4 * h + 1] = w.y * s1 * s2; f[4 * h + 2] = w.z * s1 * s2; f[4 * h + 3] = w.w * s1 * s2;
      }
      uint4 hi, lo;
      split_pair(f[0], f[1], hi.x, lo.x);
      split_pair(f[2], f[3], hi.y, lo.y);
      split_pair(f[4], f[5], hi.z, lo.z);
      split_pair(f[6], f[7], hi.w, lo.w);
      const uint32_t off = sw128_h((uint32_t)r, (uint32_t)(8 * q));
      *reinterpret_cast<uint4*>(strips + (p * 2 + 0) * kStripBytes + off) = hi;
      *reinterpret_cast<uint4*>(strips + (p * 2 + 1) * kStripBytes + off) = lo;
    }
  }
  fence_async_smem();                                     // the strips are read by wgmma (async proxy)
  bar_sync_n(bar, 128);                                   // ... and `red` is free again
}

// grid: any (persistent, tile pairs walked round-robin); block 384 = MMA warpgroups 0 and 1 (warps 0-7), producer
// warpgroup 2 (warp 8 lane 0 streams the Toeplitz images; warps 9-11 only give their registers to the MMA warps).
// Gauss's three-multiplication form of the complex product:
//   D1 = Hr xr,  D2 = Hi xi,  D3 = (Hr + Hi)(xr + xi);   y.re = D1 - D2,  y.im = D3 - (D1 + D2)
//   (entry 0 = DC / Nyquist: y = (D1, D2))
// Warpgroup w takes tile 2m + w of pair m; both read the same image stream, so every image row meets two time-line
// tiles.  Each product p is an m64n64k16 chain: A = the warpgroup's strip of line p (re, im, re + im) shifted by
// chunk c, B = slice p of the stage's 192-row image.  Each product accumulates kFlushF16 chunks in its wgmma
// registers and is added to FP32 registers (round-to-nearest) between chains: the tensor core's accumulate truncates,
// so short chains keep the error at the level of the FFMA sweep (tools/tc_accuracy_model.py).  Every product's MMAs
// of a stage are one commit group, and a warpgroup keeps two groups in flight: a product's finished chain is folded
// while the other two products' groups run.  The strips are single-buffered (60 KB per warpgroup): between pairs each
// warpgroup stores its results and converts its next strips while the tensor core idles for it.
__global__ void __launch_bounds__(kThreads, 1) k_tc_sweep(SweepParams P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* strips = base;                           // [warpgroup][line re, im, re + im][hi, lo] x kStripBytes
  unsigned char* ring = base + 2 * kGStripBytes;          // kGStages x [192 rows x 64 halves]
  __shared__ unsigned long long bar_a_full[kGStages], bar_a_empty[kGStages];
  __shared__ uint32_t strip_max[2][4][kGProducts];        // [warpgroup][warp][line]
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  if (tid == 0) {
    for (int i = 0; i < kGStages; ++i) { mbar_init(&bar_a_full[i], 1); mbar_init(&bar_a_empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = P.lines * P.npair;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kProducerRegs));
    if (warp == 8 && lane == 0) {                         // ---- image ring
      unsigned it_a = 0;
      for (int item = blockIdx.x; item < total; item += gridDim.x) {
        const int line = item / P.npair, m = item - line * P.npair;
        // the pair's FP32 time-line rows: the MMA warpgroups read them once this pair's first stages are loaded
        const unsigned xbytes = (unsigned)pair_rows(P.ntile, m) * 256u;
        prefetch_l2(P.Xt + xf_index(line, 0, (long long)m * 2 * kN * 64, P.rows), xbytes);
        prefetch_l2(P.Xt + xf_index(line, 1, (long long)m * 2 * kN * 64, P.rows), xbytes);
        const __half* Aline = P.A + (size_t)line * P.nchunk * 2 * (kGImageBytes / 2);
        for (int s = 0; s < P.nchunk * 2; ++s, ++it_a) {
          const unsigned st = it_a % kGStages, use = it_a / kGStages;
          if (use > 0 && !mbar_wait(&bar_a_empty[st], (use - 1) & 1u)) { *reinterpret_cast<volatile int*>(P.err) = 2; return; }
          mbar_expect(&bar_a_full[st], kGImageBytes);
          bulk_load(ring + st * kGImageBytes, Aline + (size_t)s * (kGImageBytes / 2), kGImageBytes, &bar_a_full[st]);
        }
      }
    }
    return;
  }

  // ---- MMA warpgroup wg: tile 2m + wg of every pair m, all three products
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kMmaRegs));   // 3 chain accumulators + 3 FP32 sums
  const int wg = warp >> 2, wq = warp & 3, t128 = tid & 127;
  const bool leader = t128 == 0;
  unsigned char* my_strips = strips + wg * kGStripBytes;
  const uint32_t strip_lo = desc_lo(smem_addr(my_strips)), ring_lo = desc_lo(smem_addr(ring));
  unsigned it_a = 0;
  float d[kGProducts][32], acc[kGProducts][32];
  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    const int line = item / P.npair, nt = 2 * (item - line * P.npair) + wg;
    const bool live = nt < P.ntile;                       // false: warpgroup 1 on the last pair of an odd tile count
    int ex[kGProducts] = {0, 0, 0};
    if (live) tc_convert_strips(P, line, nt, my_strips, strip_max[wg], wq, lane, t128, 2 + wg, ex);
#pragma unroll
    for (int p = 0; p < kGProducts; ++p)
#pragma unroll
      for (int j = 0; j < 32; ++j) { d[p][j] = 0.0f; acc[p][j] = 0.0f; }   // each chain's first MMA overwrites d
    int pending = -1;                                     // ring stage whose MMAs may still be in flight
    for (int c = 0; c < P.nchunk; ++c) {
      const bool chain0 = c % kFlushF16 == 0;             // first chunk of an accumulation chain
#pragma unroll
      for (int hl = 0; hl < 2; ++hl, ++it_a) {
        const unsigned stage = it_a % kGStages, use = it_a / kGStages;
        if (!mbar_wait(&bar_a_full[stage], use & 1u)) { if (leader) *reinterpret_cast<volatile int*>(P.err) = 5; wg_wait<0>(); return; }
        if (!live) {                                      // nothing reads the stage: hand it straight back
          __syncwarp();
          if (leader) mbar_arrive1(&bar_a_empty[stage]);
          continue;
        }
        const uint32_t img = ring_lo + stage * (kGImageBytes >> 4);
#pragma unroll
        for (int p = 0; p < kGProducts; ++p) {
          __syncwarp();                                   // wgmma is .aligned: the warp issues it converged
          fence_operands(d[p]);
          wg_fence();
          const uint32_t xhi = strip_lo + ((p * 2 * kStripBytes) >> 4) + c * 8, xlo = xhi + (kStripBytes >> 4);   // row shift c
          const uint32_t b = img + p * (kGSliceBytes >> 4);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            if (hl == 0) {
              mma_f16(d[p], xhi + kk * 2, b + kk * 2, (chain0 && kk == 0) ? 0u : 1u);
              mma_f16(d[p], xlo + kk * 2, b + kk * 2, 1u);
            } else {
              mma_f16(d[p], xhi + kk * 2, b + kk * 2, 1u);
            }
          }
          wg_commit();
          fence_operands(d[p]);
          wg_wait<2>();                                   // every group before the last two is done
          if (p == 1 && pending >= 0) {                   // ... so the previous stage's three groups are
            if (leader) mbar_arrive1(&bar_a_empty[pending]);
            pending = -1;
          }
          // ... and so is the last group of product q = p + 1: fold its chain if the next MMAs of q start a new one
          const int q = (p + 1) % kGProducts;
          if (p < 2 ? chain0 && hl == 0 && c > 0 : hl == 1 && (c + 1) % kFlushF16 == 0 && c + 1 < P.nchunk) {
            fence_operands(d[q]);
#pragma unroll
            for (int j = 0; j < 32; ++j) acc[q][j] += d[q][j];
          }
        }
        pending = (int)stage;
      }
    }
    wg_wait<0>();                                         // the last chains are complete: fold them, hand back the stage
    if (!live) continue;
#pragma unroll
    for (int p = 0; p < kGProducts; ++p) {
      fence_operands(d[p]);
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[p][j] += d[p][j];
    }
    if (leader) mbar_arrive1(&bar_a_empty[pending]);
    // undo the operand scales, per product: one exact multiply when 2^-(ex + eh) is a normal float, ldexpf beyond that
    const int eh = __ldg(P.eh + 2 * line), ehs = __ldg(P.eh + 2 * line + 1);
#pragma unroll
    for (int p = 0; p < kGProducts; ++p) {
      const int e = ex[p] + (p == 2 ? ehs : eh);
      if (e >= -127 && e <= 126) {
        const float s = pow2f(-e);
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[p][j] *= s;
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[p][j] = ldexpf(acc[p][j], -e);
      }
    }
    // register 4 j + r of lane l in warp wq: segment 16 wq + l / 4 + 8 (r / 2), step i = 8 j + 2 (l % 4) + (r % 2)
    float2* dst = P.Yc + (size_t)line * P.ystride + kYLead + (size_t)nt * kN * 64;
    const bool dc = line % P.B == 0;
    const int n0 = 16 * wq + (lane >> 2), i0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float y[4];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = 4 * j + 2 * h + e;
          const float d1 = acc[0][r], d2 = acc[1][r], d3 = acc[2][r];
          y[2 * e] = dc ? d1 : __fsub_rn(d1, d2);
          y[2 * e + 1] = dc ? d2 : __fsub_rn(d3, __fadd_rn(d1, d2));
        }
        *reinterpret_cast<float4*>(dst + (size_t)(n0 + 8 * h) * 64 + 8 * j + i0) = make_float4(y[0], y[1], y[2], y[3]);
      }
  }
  wg_wait<0>();
}

#endif  // __CUDACC__

}  // namespace tc
}  // namespace pc
