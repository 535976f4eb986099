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
// and channel.  The complex product becomes real GEMMs by stacking [Hr ; Hi] into M = 128 rows and running the
// same A against the real and the imaginary time line (two accumulators D, D2):
//   y.re = D[0:64] - D2[64:128],  y.im = D[64:128] + D2[0:64]        (entry 0 = DC / Nyquist: y = (D[0:64], D2[64:128]))
// The sweep issues the transposed product D^T[n][i] = sum_j B[j][n] * A[i][j]: the wgmma A operand is the time-line
// window (M = 64 segments), the wgmma B operand the whole 128 x 64 Toeplitz image (N = 128).  Consumer warpgroup w
// owns time line w (re, im), i.e. accumulator D (w = 0) or D2 (w = 1), all 128 rows.
//
// FP32 accuracy comes from the 3xFP16 split: a = a_hi + a_lo, b = b_hi + b_lo (each FP16-exact, round to nearest),
// and a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi accumulated in FP32 (dropped term ~2^-22 relative).  FP16 has tf32's
// 11-bit significand, and its MMAs issue at twice the tf32 rate; what it lacks is exponent range, which exact
// power-of-two scales restore: 2^eh per line (channel, bin) for H, chosen once per IR from the bin's P values, and
// 2^ex per tile and time line (re / im) for x, chosen from the 80 x 64 samples the tile reads.  Each puts the
// window's largest magnitude into [2^14, 2^15) (scale_exp); the epilogue multiplies by 2^-(ex + eh).  A sample keeps
// the full ~2^-22 relative precision while it lies within ~2^-17 of its window's peak; below that its lo part is an
// FP16 subnormal and the error is absolute, at most ~2^-39 of the window's peak (DESIGN.md §5).
//
// The time-line operand of chunk c (64 values of j) is a ROW-SHIFTED WINDOW of one shared-memory strip.  The bin's
// time line is stored as rows of 64 samples; B[64c + jj][n] = x[64 (n + c) + jj - Q] is row n + c of the strip, i.e.
// the same SWIZZLE_128B K-major strip (rows of 64 halves = 128 B) with the descriptor start address advanced by
// c * 128 bytes: the 128-byte swizzle is a function of the absolute shared-memory address, so a start address inside
// the 1024-byte swizzle atom reads the rows it names.  One 80-row strip per time line and hi / lo part feeds all K
// chunks of a 64-segment tile: the producer warpgroup bulk-copies the tile's FP32 rows (one contiguous 20 KB piece per
// time line), picks ex and writes the FP16 hi / lo strips into one of two buffers while the MMA warpgroups work on the
// previous tile.  The Toeplitz images of H (16 KB, pre-swizzled, 1-D bulk copies) stream through a 4-stage ring.
//
// Kernels: k_tc_build_a (H -> FP16 hi/lo Toeplitz tile images and eh, once per IR), k_tc_split_x (timeline rows ->
// per-bin FP32 time lines), k_tc_sweep (producer warpgroup: image ring + strip conversion / two MMA warpgroups
// accumulating in registers; the epilogue combines the complex product into bin-major float2 lines), k_tc_merge_y
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

// Toeplitz images: [line][chunk][hi, lo][128 rows x 64 halves], then eh of every line (int)
PC_TC_HD size_t a_image_bytes(size_t lines, int nchunk) { return lines * (size_t)nchunk * 2 * kATileBytes; }

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
  __half* A;                // [C*B lines][nchunk][hi, lo][128 x 64]: SWIZZLE_128B images of 2^eh H
  int* eh;                  // [C*B lines]
};

// grid (nchunk, B, C), block 256.  Every chunk's CTA finds the same eh from the bin's P values (a few KB, once per IR).
__global__ void __launch_bounds__(256) k_tc_build_a(BuildAParams p) {
  __shared__ uint32_t red[8];
  const int c = blockIdx.x, k = blockIdx.y, ch = blockIdx.z;
  const long long line = (long long)ch * p.B + k;
  const float2* Hk = p.H + (long long)ch * p.h_cstride + k;
  uint32_t m = 0;
  for (int pp = threadIdx.x; pp < p.P; pp += 256) {
    const float2 h = Hk[(long long)pp * p.B];
    m = max(m, max(abs_bits(h.x), abs_bits(h.y)));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 8; ++w) m = max(m, red[w]);
  const int eh = scale_exp(m);
  if (c == 0 && threadIdx.x == 0) p.eh[line] = eh;
  __half* hi = p.A + (line * p.nchunk + c) * 2 * (kATileBytes / 2);
  __half* lo = hi + kATileBytes / 2;
  for (int idx = threadIdx.x; idx < kATileBytes / 2; idx += 256) {
    const int mr = idx >> 6, jj = idx & 63;
    const int part = mr >> 6, i = mr & 63;
    const int pp = i + p.Q - (kChunkK * c + jj);
    float v = 0.0f;
    if (pp >= 0 && pp < p.P) { const float2 h = Hk[(long long)pp * p.B]; v = ldexpf(part ? h.y : h.x, eh); }
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
  const int* eh;
  const float* Xt;
  float2* Yc;               // [lines][ystride] complex result, bin-major (kYLead)
  long long ystride;
  int lines, ntile, nchunk, rows, B;
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
// named barrier 1 over the kStripThreads strip converters; true when every one of them passes `ok`
__device__ __forceinline__ bool strip_sync(bool ok) {
  uint32_t r;
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %1, 0;\n\tbar.red.and.pred q, 1, %2, p;\n\tselp.u32 %0, 1, 0, q;\n\t}"
               : "=r"(r) : "r"((uint32_t)ok), "n"(kStripThreads) : "memory");
  return r != 0;
}
// wgmma shared-memory descriptor of a SWIZZLE_128B K-major operand (rows of 128 bytes, 8-row groups 1024 bytes
// apart, base offset 0), split in two words: only the low word (start address in 16-byte units | leading-offset
// field, unused by swizzled K-major layouts) changes between MMAs
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// keeps the compiler from moving or copying accumulator registers across the wgmma issue / wait points
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
  for (int j = 0; j < 64; ++j) asm volatile("" : "+f"(d[j]) :: "memory");
}
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// d[64 x 128] (+)= A[64 x 16] * B[16 x 128], f16 operands (both K-major) from shared memory, FP32 accumulators in 64
// registers per thread
__device__ __forceinline__ void mma_f16(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t accumulate) {
  const uint64_t da = ((uint64_t)kDescHi << 32) | a_lo, db = ((uint64_t)kDescHi << 32) | b_lo;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
               "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
               "%64, %65, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                 "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
                 "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
                 "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
                 "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
                 "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
                 "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
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

// Epilogue of MMA warpgroup CP (0: D = x_re [Hr ; Hi], 1: D2 = x_im [Hr ; Hi]) for one tile, acc scaled:
//   y.re = D[i] - D2[64 + i],  y.im = D[64 + i] + D2[i]     (entry 0 = DC / Nyquist: y = (D[i], D2[64 + i]))
// Warpgroup CP stores the output steps i in [32 CP, 32 CP + 32): fragment registers 4 j + r with j in KEEP = {4 CP ..
// 4 CP + 3} (rows m = i) and 8 + KEEP (rows m = 64 + i).  It hands its other registers (j in GIVE and 8 + GIVE) to the
// partner through `xch` (this tile's strip buffer; per warpgroup [32 registers][128 threads] floats over its own hi / lo
// strips, which it stopped reading at its wg_wait<0>) and takes the partner's registers of its own positions into them.
// The leader releases the buffer (`strip_empty`) once its warpgroup has read the partner's half.  The FP32 operations are one
// __fsub_rn / __fadd_rn per component on the same operands as everywhere else this product is combined.
template <int CP>
__device__ __forceinline__ void tc_store_complex(float (&acc)[64], float* xch, unsigned long long* strip_empty, bool leader,
                                                 bool dc, float2* dst, int wq, int lane, int t128) {
  constexpr int KEEP = 4 * CP, GIVE = 4 - KEEP;
  constexpr int kHalf = 2 * kStripBytes / 4;          // a warpgroup's own hi / lo strips: the partner may still read the other's
  float* mine = xch + CP * kHalf;
  const float* theirs = xch + (1 - CP) * kHalf;
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      mine[(q * 4 + r) * 128 + t128] = acc[4 * (GIVE + q) + r];
      mine[((4 + q) * 4 + r) * 128 + t128] = acc[4 * (8 + GIVE + q) + r];
    }
  bar_sync_n(2, 256);
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      acc[4 * (GIVE + q) + r] = theirs[(q * 4 + r) * 128 + t128];
      acc[4 * (8 + GIVE + q) + r] = theirs[((4 + q) * 4 + r) * 128 + t128];
    }
  bar_sync_n(3 + CP, 128);
  if (leader) mbar_arrive1(strip_empty);
  // register 4 j + r of lane l in warp wq: segment 16 wq + l / 4 + 8 (r / 2), row m = 8 j + 2 (l % 4) + (r % 2)
  const int n0 = 16 * wq + (lane >> 2), i0 = 2 * (lane & 3);
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float y[4];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = 2 * h + e;
        const float own_lo = acc[4 * (KEEP + q) + r], own_hi = acc[4 * (8 + KEEP + q) + r];
        const float oth_lo = acc[4 * (GIVE + q) + r], oth_hi = acc[4 * (8 + GIVE + q) + r];
        const float d0 = CP ? oth_lo : own_lo, d1 = CP ? oth_hi : own_hi;     // D[i], D[64 + i]
        const float e0 = CP ? own_lo : oth_lo, e1 = CP ? own_hi : oth_hi;     // D2[i], D2[64 + i]
        y[2 * e] = dc ? d0 : __fsub_rn(d0, e1);
        y[2 * e + 1] = dc ? e1 : __fadd_rn(d1, e0);
      }
      *reinterpret_cast<float4*>(dst + (size_t)(n0 + 8 * h) * 64 + 8 * (KEEP + q) + i0) = make_float4(y[0], y[1], y[2], y[3]);
    }
}

// grid: any (persistent, tiles walked round-robin); block 384 = MMA warpgroups 0 and 1 (warps 0-7), producer
// warpgroup 2 (warp 8 lane 0 streams the Toeplitz images, warps 9-11 stage and convert the time-line strips).
// Each MMA warpgroup accumulates the products of kFlushF16 chunks in its wgmma registers and adds them to FP32
// registers (round-to-nearest) between groups: the tensor core's accumulate truncates, so short accumulation chains
// keep the error at the level of the FFMA sweep (tools/tc_accuracy_model.py).
__global__ void __launch_bounds__(kThreads, 1) k_tc_sweep(SweepParams P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* strips = base;                           // [buf][comp][hi, lo] x kStripBytes, FP16 SWIZZLE_128B
  unsigned char* ring = base + 8 * kStripBytes;
  float* stage = reinterpret_cast<float*>(ring + kAStages * kATileBytes);   // [comp][kStripRows][64] FP32
  __shared__ unsigned long long bar_strip_full[2], bar_strip_empty[2], bar_stage, bar_a_full[kAStages], bar_a_empty[kAStages];
  __shared__ int strip_ex[2][2];                          // [buf][comp]
  __shared__ uint32_t strip_max[kStripThreads / 32][2];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  if (tid == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(&bar_strip_full[b], kStripThreads); mbar_init(&bar_strip_empty[b], 2); }
    mbar_init(&bar_stage, 1);
    for (int i = 0; i < kAStages; ++i) { mbar_init(&bar_a_full[i], 1); mbar_init(&bar_a_empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = P.lines * P.ntile;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kProducerRegs));
    if (warp == 8) {
      if (lane == 0) {                                    // ---- image ring
        unsigned it_a = 0;
        bool ok = true;
        for (int tile = blockIdx.x; tile < total && ok; tile += gridDim.x) {
          const __half* Aline = P.A + (size_t)(tile / P.ntile) * P.nchunk * 2 * (kATileBytes / 2);
          for (int s = 0; s < P.nchunk * 2; ++s, ++it_a) {
            const unsigned st = it_a % kAStages, use = it_a / kAStages;
            if (use > 0 && !mbar_wait(&bar_a_empty[st], (use - 1) & 1u)) { *reinterpret_cast<volatile int*>(P.err) = 2; ok = false; break; }
            mbar_expect(&bar_a_full[st], kATileBytes);
            bulk_load(ring + st * kATileBytes, Aline + (size_t)s * (kATileBytes / 2), kATileBytes, &bar_a_full[st]);
          }
        }
      }
      return;
    }
    // ---- strips: FP32 rows -> max |x| -> ex -> FP16 hi / lo SWIZZLE_128B strips, double-buffered
    const int sid = tid - 9 * 32;
    const float4* stage4 = reinterpret_cast<const float4*>(stage);
    int n = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++n) {
      const int line = tile / P.ntile, nt = tile - line * P.ntile;
      const int buf = n & 1;
      if (sid == 0) {
        fence_async_smem();                               // the previous tile's reads of the staging rows come first
        mbar_expect(&bar_stage, kStageBytes);
        for (int comp = 0; comp < 2; ++comp)
          bulk_load(stage + comp * kStripRows * 64, P.Xt + xf_index(line, comp, (long long)nt * kN * 64, P.rows), kStageBytes / 2, &bar_stage);
      }
      bool ok = mbar_wait(&bar_stage, (unsigned)n & 1u);
      uint32_t mx[2] = {0u, 0u};
#pragma unroll
      for (int comp = 0; comp < 2; ++comp)
        for (int u = sid; u < kStripRows * 16 && ok; u += kStripThreads) {
          const float4 v = stage4[comp * kStripRows * 16 + u];
          mx[comp] = max(mx[comp], max(max(abs_bits(v.x), abs_bits(v.y)), max(abs_bits(v.z), abs_bits(v.w))));
        }
#pragma unroll
      for (int comp = 0; comp < 2; ++comp) {
        mx[comp] = __reduce_max_sync(0xffffffffu, mx[comp]);
        if (lane == 0) strip_max[warp - 9][comp] = mx[comp];
      }
      if (!strip_sync(ok)) { if (sid == 0) *reinterpret_cast<volatile int*>(P.err) = 4; break; }
      int ex[2];
#pragma unroll
      for (int comp = 0; comp < 2; ++comp) {
        uint32_t m = strip_max[0][comp];
#pragma unroll
        for (int w = 1; w < kStripThreads / 32; ++w) m = max(m, strip_max[w][comp]);
        ex[comp] = scale_exp(m);
      }
      if (n >= 2) ok = mbar_wait(&bar_strip_empty[buf], (unsigned)((n >> 1) - 1) & 1u);   // tile n - 2's MMAs are done
      if (ok) {
        unsigned char* dst = strips + buf * 4 * kStripBytes;
#pragma unroll
        for (int comp = 0; comp < 2; ++comp) {
          // 2^ex as two factors: each is a normal float for every ex scale_exp returns, and x * s1 * s2 is exact
          // wherever the FP16 result can hold it
          const float s1 = pow2f(ex[comp] >> 1), s2 = pow2f(ex[comp] - (ex[comp] >> 1));
          for (int u = sid; u < kStripRows * 8; u += kStripThreads) {      // 16-byte units of 8 halves
            const int r = u >> 3, q = u & 7;
            const float4 a = stage4[(comp * kStripRows + r) * 16 + 2 * q];
            const float4 b = stage4[(comp * kStripRows + r) * 16 + 2 * q + 1];
            uint4 hi, lo;
            split_pair(a.x * s1 * s2, a.y * s1 * s2, hi.x, lo.x);
            split_pair(a.z * s1 * s2, a.w * s1 * s2, hi.y, lo.y);
            split_pair(b.x * s1 * s2, b.y * s1 * s2, hi.z, lo.z);
            split_pair(b.z * s1 * s2, b.w * s1 * s2, hi.w, lo.w);
            const uint32_t off = sw128_h((uint32_t)r, (uint32_t)(8 * q));
            *reinterpret_cast<uint4*>(dst + (comp * 2 + 0) * kStripBytes + off) = hi;
            *reinterpret_cast<uint4*>(dst + (comp * 2 + 1) * kStripBytes + off) = lo;
          }
        }
        if (sid == 0) { strip_ex[buf][0] = ex[0]; strip_ex[buf][1] = ex[1]; }
        fence_async_smem();                               // the strips are read by wgmma (async proxy)
        mbar_arrive1(&bar_strip_full[buf]);
      }
      if (!strip_sync(ok)) { if (sid == 0) *reinterpret_cast<volatile int*>(P.err) = 4; break; }   // staging rows free
    }
    return;
  }

  // ---- MMA warpgroup `comp` (time line re / im against all 128 rows of the stacked [Hr ; Hi] Toeplitz tile)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kMmaRegs));   // two accumulator sets + the FP32 sums
  const int comp = warp >> 2, wq = warp & 3;
  const bool leader = (tid & 127) == 0;
  const uint32_t strip_lo = desc_lo(smem_addr(strips)), ring_lo = desc_lo(smem_addr(ring));
  unsigned it_a = 0;
  int n = 0;
  int ex = 0;
  // Accumulation chains alternate between d0 and d1: the chain of group g is folded into acc once the first stage of
  // group g + 1 has been committed, so the tensor core keeps working on g + 1 while g drains and is added (same chains,
  // same order of the FP32 adds as draining each chain before the next one starts).
  float d0[64], d1[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) { d0[j] = 0.0f; d1[j] = 0.0f; }
  float acc[64];
  int pending = -1;                                       // ring stage whose MMAs may still be in flight
  // issues chunks [g0, min(g0 + kFlushF16, nchunk)) into d; folds `prev` (the previous chain, if g0 > 0) into acc as
  // soon as it is complete.  false: a barrier wait gave up
  auto chain = [&](float (&d)[64], float (&prev)[64], int g0) -> bool {
    const int gend = min(g0 + kFlushF16, P.nchunk);
    const int buf = n & 1;
    const uint32_t xs = strip_lo + (((buf * 2 + comp) * 2) * kStripBytes >> 4);   // hi strip; lo strip kStripBytes on
    for (int c = g0; c < gend; ++c) {
      if (c == 0) {
        if (!mbar_wait(&bar_strip_full[buf], (unsigned)(n >> 1) & 1u)) { if (leader) *reinterpret_cast<volatile int*>(P.err) = 3; return false; }
        ex = strip_ex[buf][comp];
      }
#pragma unroll
      for (int hl = 0; hl < 2; ++hl, ++it_a) {
        const unsigned stage = it_a % kAStages, use = it_a / kAStages;
        if (!mbar_wait(&bar_a_full[stage], use & 1u)) { if (leader) *reinterpret_cast<volatile int*>(P.err) = 5; return false; }
        __syncwarp();                                     // wgmma is .aligned: the warp issues it converged
        fence_operands(d);
        wg_fence();
        const uint32_t img = ring_lo + stage * (kATileBytes >> 4);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint32_t xhi = xs + c * 8 + kk * 2, xlo = xhi + (kStripBytes >> 4);   // row shift c, k16 step kk
          if (hl == 0) {
            mma_f16(d, xhi, img + kk * 2, (c > g0 || kk > 0) ? 1u : 0u);
            mma_f16(d, xlo, img + kk * 2, 1u);
          } else {
            mma_f16(d, xhi, img + kk * 2, 1u);
          }
        }
        wg_commit();
        fence_operands(d);
        wg_wait<1>();                                     // everything before this stage's MMAs is done
        fence_operands(d);
        if (leader && pending >= 0) mbar_arrive1(&bar_a_empty[pending]);
        pending = (int)stage;
        if (c == g0 && hl == 0 && g0 > 0) {               // the previous chain is complete: fold it
          fence_operands(prev);
#pragma unroll
          for (int j = 0; j < 64; ++j) acc[j] += prev[j];
        }
      }
    }
    return true;
  };
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++n) {
    const int line = tile / P.ntile, nt = tile - line * P.ntile;
    const int eh = __ldg(P.eh + line);
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.0f;
    for (int g0 = 0; g0 < P.nchunk; g0 += 2 * kFlushF16) {  // one accumulation chain per group of kFlushF16 chunks
      if (!chain(d0, d1, g0)) { wg_wait<0>(); return; }
      if (g0 + kFlushF16 >= P.nchunk) break;
      if (!chain(d1, d0, g0 + kFlushF16)) { wg_wait<0>(); return; }
    }
    wg_wait<0>();                                         // the last chain is complete: fold it, hand back the strips
    fence_operands(d0);
    fence_operands(d1);
    if (leader) mbar_arrive1(&bar_a_empty[pending]);
    pending = -1;
    if ((P.nchunk + kFlushF16 - 1) / kFlushF16 & 1) {     // an odd number of chains ends in d0
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += d0[j];
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += d1[j];
    }
    // undo the operand scales: one exact multiply when 2^-(ex + eh) is a normal float, ldexpf beyond that
    const int e = ex + eh;
    if (e >= -127 && e <= 126) {
      const float s = pow2f(-e);
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] *= s;
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = ldexpf(acc[j], -e);
    }
    float* xch = reinterpret_cast<float*>(strips + (n & 1) * 4 * kStripBytes);
    float2* dst = P.Yc + (size_t)line * P.ystride + kYLead + (size_t)nt * kN * 64;
    const bool dc = line % P.B == 0;
    if (comp == 0) tc_store_complex<0>(acc, xch, &bar_strip_empty[n & 1], leader, dc, dst, wq, lane, tid & 127);
    else tc_store_complex<1>(acc, xch, &bar_strip_empty[n & 1], leader, dc, dst, wq, lane, tid & 127);
  }
}

#endif  // __CUDACC__

}  // namespace tc
}  // namespace pc
