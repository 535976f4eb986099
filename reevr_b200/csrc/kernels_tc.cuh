// kernels_tc.cuh — K2x: the batched sweep on the Hopper tensor cores (wgmma.mma_async tf32, 3xTF32).
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
// window (M = 64 segments), the wgmma B operand the whole 128 x 32 Toeplitz image (N = 128), so every m64n128k8 reads
// 2 KB + 4 KB of shared memory for 64 K FMA (an m64n64k8 reads 4 KB for 32 K FMA, which at the tf32 rate is the whole
// shared-memory port).  Consumer warpgroup w owns time line w (re, im), i.e. accumulator D (w = 0) or D2 (w = 1), all
// 128 rows.
// FP32 accuracy comes from the 3xTF32 split: a = a_hi + a_lo, b = b_hi + b_lo (each tf32-exact), and
// a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi accumulated in FP32 (dropped term ~2^-22 relative).
//
// The time-line operand of chunk c (32 values of j) is a ROW-SHIFTED WINDOW of one shared-memory strip.  The bin's time
// line is stored as rows of 64 samples; plane e in {0, 1} holds the 32-sample half rows (128 B, SWIZZLE_128B
// K-major).  B[32c + jj][n] = x[64 (n + c/2) + 32 (c%2) + jj - Q] is row n + c/2 of plane c%2, i.e. the same strip
// with the descriptor start address advanced by (c/2) * 128 bytes: the 128-byte swizzle is a function of the
// absolute shared-memory address, so a start address inside the 1024-byte swizzle atom reads the rows it names.
// One 80-row strip per plane (8 planes: re/im x hi/lo x e, 80 KB, one 1-D bulk copy each: the global time lines are
// stored as pre-swizzled strip images) feeds all K chunks of a 64-segment tile: every x sample enters shared
// memory once, and only the Toeplitz tiles of H (16 KB, pre-swizzled images, 1-D bulk copies through a 4-stage
// ring) stream during the tile.
//
// Kernels: k_tc_build_a (H -> tf32 hi/lo Toeplitz tile images, once per IR), k_tc_split_x (timeline rows -> per-bin
// hi/lo time lines), k_tc_sweep (bulk-copy producer warpgroup / two MMA warpgroups accumulating in registers),
// k_tc_merge_y (partial planes -> Y rows, combines the complex product).
#pragma once

#include <cuda_runtime.h>
#include <cstdint>

namespace pc {
namespace tc {

constexpr int kR = 64;                              // block steps per segment
constexpr int kN = 64;                              // segments per tile (MMA N)
constexpr int kMaxChunks = 32;                      // K chunks of 32 -> K <= 1024, row shifts 0..15
constexpr int kStripRows = kN + 16;
constexpr int kStripBytes = kStripRows * 128;       // 10240 (a multiple of the 1024-byte swizzle atom)
constexpr int kATileBytes = 128 * 128;              // one 128 x 32 tf32 Toeplitz tile image
constexpr int kAStages = 4;
constexpr int kSmemBytes = 8 * kStripBytes + kAStages * kATileBytes + 1024;
constexpr int kThreads = 384;                       // two MMA warpgroups + a producer warpgroup (one thread issues the copies)
constexpr int kMmaRegs = 232, kProducerRegs = 40;   // setmaxnreg split of the register file: 256 x 232 + 128 x 40 <= 64 K
constexpr int kFlush = 4;                           // K chunks accumulated by the tensor core before the FP32 register add

struct Geom {
  int P, Q, nchunk, nb, nseg, ntile, rows;
  long long Lt, Lty;
};

inline __host__ __device__ Geom make_geom(int P, int nb) {
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
inline __host__ __device__ bool geom_ok(const Geom& g, int B) { return g.nchunk <= kMaxChunks && B % 32 == 0 && g.nb > 0; }

// byte offset of element (row r, float e < 32) in a SWIZZLE_128B K-major image with a 1024-byte aligned base
inline __host__ __device__ uint32_t sw128(uint32_t r, uint32_t e) { return r * 128u + ((((e >> 2) ^ (r & 7u)) & 7u) << 4) + (e & 3u) * 4u; }

// Xt layout: [line][re_hi, re_lo, im_hi, im_lo][e][row R][32 floats], the sample tau = 64 R + 32 e + jj stored at
// 16-byte chunk (jj / 4) ^ (R % 8) of its 128-byte row: a strip (kStripRows consecutive rows of one plane, first row a
// multiple of 8) is ONE contiguous 10 KB piece of global memory that is already the SWIZZLE_128B shared-memory image,
// so the sweep fetches it with a single 1-D bulk copy (no tensor map, no per-row TMA requests).
inline __host__ __device__ size_t xt_index(long long line, int pl, int e, long long R, int jj, int rows) {
  return ((((size_t)line * 4 + pl) * 2 + e) * (size_t)rows + (size_t)R) * 32 + (size_t)(((((jj >> 2) ^ (int)(R & 7)) & 7) << 2) | (jj & 3));
}

#if defined(__CUDACC__)

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// ---- H -> Toeplitz tile images ---------------------------------------------------------------------------------
struct BuildAParams {
  const float2* H;          // [C][Prows][B]
  long long h_cstride;
  int B, P, Q, nchunk;
  float* A;                 // [C*B lines][nchunk][hi, lo][4096]
};

// grid (nchunk, B, C), block 256
__global__ void __launch_bounds__(256) k_tc_build_a(BuildAParams p) {
  const int c = blockIdx.x, k = blockIdx.y, ch = blockIdx.z;
  const long long line = (long long)ch * p.B + k;
  float* hi = p.A + ((line * p.nchunk + c) * 2) * 4096;
  float* lo = hi + 4096;
  const float2* Hk = p.H + (long long)ch * p.h_cstride + k;
  for (int idx = threadIdx.x; idx < 4096; idx += 256) {
    const int m = idx >> 5, jj = idx & 31;
    const int part = m >> 6, i = m & 63;
    const int pp = i + p.Q - (32 * c + jj);
    float v = 0.0f;
    if (pp >= 0 && pp < p.P) { const float2 h = Hk[(long long)pp * p.B]; v = part ? h.y : h.x; }
    const float vh = tf32_rn(v), vl = tf32_rn(v - vh);
    const uint32_t off = sw128((uint32_t)m, (uint32_t)jj) >> 2;
    hi[off] = vh;
    lo[off] = vl;
  }
}

// ---- timeline rows -> per-bin hi / lo time lines ---------------------------------------------------------------
struct SplitXParams {
  const float2* X;          // [C][R][B]
  long long x_cstride;
  long long row_base;       // timeline row of tau = 0 (= row of output block 0 minus Q); may be negative
  long long row_lo, row_hi; // rows outside [row_lo, row_hi) read as zero
  int B;
  int rows;                 // 64-sample rows per plane
  float* Xt;
};

// grid (rows * 2, B / 32, C), block (32, 8)
__global__ void __launch_bounds__(256) k_tc_split_x(SplitXParams p) {
  __shared__ float2 tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long long tau0 = (long long)blockIdx.x * 32;
  const int k0 = blockIdx.y * 32, ch = blockIdx.z;
  for (int r = ty; r < 32; r += 8) {
    const long long row = p.row_base + tau0 + r;
    float2 v = make_float2(0.0f, 0.0f);
    if (row >= p.row_lo && row < p.row_hi) v = p.X[(long long)ch * p.x_cstride + row * p.B + k0 + tx];
    tile[r][tx] = v;
  }
  __syncthreads();
  const long long R = tau0 >> 6;
  const int e = (int)((tau0 >> 5) & 1);
  for (int kk = ty; kk < 32; kk += 8) {
    const float2 v = tile[tx][kk];
    const long long line = (long long)ch * p.B + k0 + kk;
    const float rh = tf32_rn(v.x), ih = tf32_rn(v.y);
    p.Xt[xt_index(line, 0, e, R, tx, p.rows)] = rh;
    p.Xt[xt_index(line, 1, e, R, tx, p.rows)] = tf32_rn(v.x - rh);
    p.Xt[xt_index(line, 2, e, R, tx, p.rows)] = ih;
    p.Xt[xt_index(line, 3, e, R, tx, p.rows)] = tf32_rn(v.y - ih);
  }
}

// ---- partial planes -> Y rows ----------------------------------------------------------------------------------
struct MergeYParams {
  const float* Yt;          // [C*B lines][D part0, D part1, D2 part0, D2 part1][Lty]
  long long Lty;
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
    const float* src = p.Yt + line * 4 * p.Lty + t0 + tx;
    float2 y = make_float2(0.0f, 0.0f);
    if (t0 + tx < p.nb) {
      const float d0 = src[0], d1 = src[p.Lty], e0 = src[2 * p.Lty], e1 = src[3 * p.Lty];
      y = (k0 + kk == 0) ? make_float2(d0, e1) : make_float2(d0 - e1, d1 + e0);
    }
    tile[tx][kk] = y;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const long long t = t0 + r;
    if (t < p.nb) p.Y[(long long)ch * p.y_cstride + (p.yrow0 + t) * p.y_rstride + k0 + tx] = tile[r][tx];
  }
}

// ---- the sweep -------------------------------------------------------------------------------------------------
struct SweepParams {
  const float* A;
  const float* Xt;
  float* Yt;
  int lines, ntile, nchunk, rows;
  long long Lty;
  int* err;                 // (mapped host word) set non-zero when a barrier wait gave up — a bug, not a data condition
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
// d[64 x 128] (+)= A[64 x 8] * B[8 x 128], tf32 operands from shared memory, FP32 accumulators in 64 registers per thread
__device__ __forceinline__ void mma_tf32(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t accumulate) {
  const uint64_t da = ((uint64_t)kDescHi << 32) | a_lo, db = ((uint64_t)kDescHi << 32) | b_lo;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
               "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
               "%64, %65, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                 "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
                 "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
                 "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
                 "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
                 "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
                 "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// grid: any (persistent, tiles walked round-robin); block 384 = MMA warpgroups 0 and 1 (warps 0-7), producer
// warpgroup 2 (warp 8 lane 0 issues the copies; the warpgroup exists so that setmaxnreg can hand its registers over).
// Each MMA warpgroup accumulates the products of kFlush chunks in its wgmma registers and adds them to FP32
// registers (round-to-nearest) between groups: the tensor core's accumulate truncates, so short accumulation chains
// keep the error at the level of the FFMA sweep (tools/tc_accuracy_model.py).
__global__ void __launch_bounds__(kThreads, 1) k_tc_sweep(SweepParams P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* strips = base;                           // [comp][hi, lo][e] x kStripBytes
  unsigned char* ring = base + 8 * kStripBytes;
  __shared__ unsigned long long bar_strip_full[2], bar_strip_empty, bar_a_full[kAStages], bar_a_empty[kAStages];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  if (tid == 0) {
    mbar_init(&bar_strip_full[0], 1); mbar_init(&bar_strip_full[1], 1); mbar_init(&bar_strip_empty, 2);
    for (int i = 0; i < kAStages; ++i) { mbar_init(&bar_a_full[i], 1); mbar_init(&bar_a_empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = P.lines * P.ntile;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kProducerRegs));
    if (warp == 8 && lane == 0) {                         // ---- producer
      unsigned it_a = 0;
      int n = 0;
      bool ok = true;
      for (int tile = blockIdx.x; tile < total && ok; tile += gridDim.x, ++n) {
        const int line = tile / P.ntile, nt = tile - line * P.ntile;
        if (n > 0 && !mbar_wait(&bar_strip_empty, (unsigned)(n - 1) & 1u)) { *reinterpret_cast<volatile int*>(P.err) = 1; break; }
        for (int e = 0; e < 2; ++e) {                     // plane e = 0 first: chunk 0 needs only that one
          mbar_expect(&bar_strip_full[e], 4 * kStripBytes);
          for (int pl = 0; pl < 4; ++pl)
            bulk_load(strips + (pl * 2 + e) * kStripBytes, P.Xt + ((((size_t)line * 4 + pl) * 2 + e) * (size_t)P.rows + (size_t)nt * kN) * 32, kStripBytes,
                      &bar_strip_full[e]);
        }
        const float* Aline = P.A + (size_t)line * P.nchunk * 2 * 4096;
        for (int s = 0; s < P.nchunk * 2; ++s, ++it_a) {
          const unsigned stage = it_a % kAStages, use = it_a / kAStages;
          if (use > 0 && !mbar_wait(&bar_a_empty[stage], (use - 1) & 1u)) { *reinterpret_cast<volatile int*>(P.err) = 2; ok = false; break; }
          mbar_expect(&bar_a_full[stage], kATileBytes);
          bulk_load(ring + stage * kATileBytes, Aline + (size_t)s * 4096, kATileBytes, &bar_a_full[stage]);
        }
      }
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
  // Accumulation chains alternate between d0 and d1: the chain of group g is folded into acc once the first stage of
  // group g + 1 has been committed, so the tensor core keeps working on g + 1 while g drains and is added (same chains,
  // same order of the FP32 adds as draining each chain before the next one starts).
  float d0[64], d1[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) { d0[j] = 0.0f; d1[j] = 0.0f; }
  float acc[64];
  int pending = -1;                                       // ring stage whose MMAs may still be in flight
  // issues chunks [g0, min(g0 + kFlush, nchunk)) into d; folds `prev` (the previous chain, if g0 > 0) into acc as soon
  // as it is complete.  false: a barrier wait gave up
  auto chain = [&](float (&d)[64], float (&prev)[64], int g0) -> bool {
    const int gend = min(g0 + kFlush, P.nchunk);
    for (int c = g0; c < gend; ++c) {
      if (c < 2 && !mbar_wait(&bar_strip_full[c], (unsigned)n & 1u)) { if (leader) *reinterpret_cast<volatile int*>(P.err) = 3; return false; }
      const uint32_t e = (uint32_t)c & 1u, q = (uint32_t)c >> 1;
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
          const uint32_t xhi = strip_lo + (((comp * 2 + 0) * 2 + e) * kStripBytes >> 4) + q * 8 + kk * 2;
          const uint32_t xlo = strip_lo + (((comp * 2 + 1) * 2 + e) * kStripBytes >> 4) + q * 8 + kk * 2;
          if (hl == 0) {
            mma_tf32(d, xhi, img + kk * 2, (c > g0 || kk > 0) ? 1u : 0u);
            mma_tf32(d, xlo, img + kk * 2, 1u);
          } else {
            mma_tf32(d, xhi, img + kk * 2, 1u);
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
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.0f;
    for (int g0 = 0; g0 < P.nchunk; g0 += 2 * kFlush) {  // one accumulation chain per group of kFlush chunks
      if (!chain(d0, d1, g0)) { wg_wait<0>(); return; }
      if (g0 + kFlush >= P.nchunk) break;
      if (!chain(d1, d0, g0 + kFlush)) { wg_wait<0>(); return; }
    }
    wg_wait<0>();                                         // the last chain is complete: fold it, hand back the strips
    fence_operands(d0);
    fence_operands(d1);
    if (leader) {
      mbar_arrive1(&bar_a_empty[pending]);
      mbar_arrive1(&bar_strip_empty);
    }
    pending = -1;
    if ((P.nchunk + kFlush - 1) / kFlush & 1) {           // an odd number of chains ends in d0
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += d0[j];
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += d1[j];
    }
    // accumulator fragment of m64n128: register 4 j + r of lane l in warp wq holds segment 16 wq + l / 4 + 8 (r / 2) and
    // Toeplitz row m = 8 j + 2 (l % 4) + (r % 2), i.e. output step m % 64 of plane comp * 2 + m / 64; registers 4 j + r
    // and 4 j + r + 1 (r even) are consecutive steps
    const int n0 = 16 * wq + (lane >> 2), i0 = 2 * (lane & 3);
#pragma unroll
    for (int part = 0; part < 2; ++part) {
      float* dst = P.Yt + ((size_t)line * 4 + comp * 2 + part) * P.Lty + (size_t)nt * kN * 64;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 4 * (8 * part + j) + 2 * h;
          *reinterpret_cast<float2*>(dst + (size_t)(n0 + 8 * h) * 64 + 8 * j + i0) = make_float2(acc[r], acc[r + 1]);
        }
    }
  }
}

#endif  // __CUDACC__

}  // namespace tc
}  // namespace pc
