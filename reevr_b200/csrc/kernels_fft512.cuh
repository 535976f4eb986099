// kernels_fft512.cuh — K1r / K3r: register-resident real FFTs for the block size of the headline shapes
// (B = 512: 1024-point real transform = 512-point complex transform + even/odd split).
//
// Replaces, for B = 512, the shared-memory Stockham kernels of kernels.cuh (CopyAndPad + AudioFFT::fft,
// FFTConvolver.cpp:172-173 / AudioFFT.cpp:114-137;  AudioFFT::ifft + Sum + overlap save, FFTConvolver.cpp:190-204 /
// AudioFFT.cpp:139-159).  Those spend ~2300 warp-instructions per transform, half of them index arithmetic
// and shared-memory traffic of three out-of-place radix-8 passes, at 33 % occupancy (two 4 KB ping-pong buffers per
// transform): the round-1 captures show them issue-bound at ~50 % of the issue slots.  Here one WARP owns one
// transform and keeps its 16 complex points per lane in registers through a three-step 8 x 8 x 8 decomposition
//
//   n = 64 n2 + 8 n1 + n0        k = k2 + 8 q0 + 64 q1                (all digits in [0, 8))
//   W512^{nk} = W8^{n2 k2} . W512^{(8 n1 + n0) k2} . W8^{n1 q0} . W64^{n0 q0} . W8^{n0 q1}
//
//   step 1  DFT8 over n2 for the two columns m = 8 n1 + n0 in {lane, lane + 32}   -> twiddle W512^{m k2}
//   step 2  DFT8 over n1 for the two pairs (k2, n0) = (pid / 8, pid % 8), pid in {lane, lane + 32} -> twiddle W64^{n0 q0}
//   step 3  DFT8 over n0 for the two residues l = k2 + 8 q0 in {lane, 64 - lane}  (lane 0: {0, 32})
//
// with two exchanges through ONE 4 KB shared buffer per warp (XOR-swizzled so that both the writing and the reading
// side of each exchange are bank-conflict free: every half-warp of a 64-bit access touches 16 distinct bank pairs)
// and __syncwarp() only.  Everything that touches global memory is coalesced: for a fixed
// register index consecutive lanes hold consecutive points (first step: consecutive columns; last step: consecutive /
// mirrored residues).  The lane that owns residue l also owns 64 - l, i.e. bins k and M - k of every mirror pair, so
// the even/odd split of the real transform (and its inverse, merged with the frequency-domain overlap-add) needs no
// data movement at all.  The forward transform exploits the zero half of [x ; 0] (n2 >= 4 is zero), the inverse
// computes only the first half of its output (n2 < 4) — the other half is what the overlap-add merge replaced.
// The inverse runs the same three steps backwards with conjugated twiddles.
//
// Tables (device array `tab512`, 1088 float2, built in double on the host, staged in shared memory once per CTA):
//   T1[k2 * 64 + m] = exp(-2 pi i m k2 / 512)     T2[a * 8 + b] = exp(-2 pi i a b / 64)     TS[k] = exp(-2 pi i k / 1024), k < 512
//
// The per-lane phase bodies are plain inline functions so that tests/emu runs the identical arithmetic on the CPU.
#pragma once

#include "kernels.cuh"
#include "kernels_tc.cuh"

namespace pc {

constexpr int kF512_M = 512;
constexpr int kF512_T1 = 0, kF512_T2 = 512, kF512_TS = 576, kF512_TabLen = 1088;
constexpr int kF512_Xch = 512;          // float2 per warp exchange buffer

// complex add / sub / scale on float2: on the device the _rn intrinsics keep the compiler from contracting them
// into FMAs with a neighbouring product (the results are those of one IEEE add / multiply per component)
PC_HD float2 f2_add(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#else
  return make_float2(a.x + b.x, a.y + b.y);
#endif
}
PC_HD float2 f2_sub(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
#else
  return make_float2(a.x - b.x, a.y - b.y);
#endif
}
PC_HD float2 f2_scale(float2 a, float s) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s));
#else
  return make_float2(a.x * s, a.y * s);
#endif
}
// a * w (INV: a * conj(w))
template <bool INV>
PC_HD float2 f2_cmul(float2 a, float2 w) {
  if (INV) w.y = -w.y;
  // (a.x w.x - a.y w.y, a.x w.y + a.y w.x) = (a.x, a.x) * w + (-a.y w.y, a.y w.x)
  const float2 t = make_float2(-a.y * w.y, a.y * w.x);
  return make_float2(fmaf(a.x, w.x, t.x), fmaf(a.x, w.y, t.y));
}

// 8-point DFT, natural order in and out (forward: e^{-2 pi i / 8}; INV: conjugate), unscaled
template <bool INV>
PC_HD void f512_dft8(float2* a) {
  float2 s[8];
#pragma unroll
  for (int r = 0; r < 4; ++r) { s[r] = f2_add(a[r], a[r + 4]); s[r + 4] = f2_sub(a[r], a[r + 4]); }
  const float h = 0.70710678118654752440f;
  if (!INV) {   // W8^1, W8^2, W8^3 on the odd half
    s[5] = make_float2(h * (s[5].x + s[5].y), h * (s[5].y - s[5].x));
    s[6] = make_float2(s[6].y, -s[6].x);
    s[7] = make_float2(h * (s[7].y - s[7].x), -h * (s[7].x + s[7].y));
  } else {
    s[5] = make_float2(h * (s[5].x - s[5].y), h * (s[5].x + s[5].y));
    s[6] = make_float2(-s[6].y, s[6].x);
    s[7] = make_float2(-h * (s[7].x + s[7].y), h * (s[7].x - s[7].y));
  }
#pragma unroll
  for (int g = 0; g < 2; ++g) {     // 4-point DFTs: g = 0 -> even outputs 0,2,4,6 ; g = 1 -> odd outputs 1,3,5,7
    const float2 b0 = f2_add(s[4 * g], s[4 * g + 2]), b1 = f2_sub(s[4 * g], s[4 * g + 2]);
    const float2 b2 = f2_add(s[4 * g + 1], s[4 * g + 3]), d = f2_sub(s[4 * g + 1], s[4 * g + 3]);
    const float2 b3 = INV ? make_float2(-d.y, d.x) : make_float2(d.y, -d.x);
    a[g] = f2_add(b0, b2);
    a[g + 2] = f2_add(b1, b3);
    a[g + 4] = f2_sub(b0, b2);
    a[g + 6] = f2_sub(b1, b3);
  }
}

// residues owned by a lane in step 3 (and, mirrored, in the first inverse step)
PC_HD int f512_la(int lane) { return lane; }
PC_HD int f512_lb(int lane) { return lane == 0 ? 32 : 64 - lane; }
// exchange-buffer layouts (float2 index; 16 consecutive float2 = the 32 banks).
// s1 [k2][m = 8 n1 + n0]: written with consecutive m per k2, read with (k2, k2 + 1) x n0 = 0..7 per half-warp at a
//    fixed n1 -> bit 3 of m is flipped for odd k2 so that the two k2 land in different halves of the bank set.
// s2 [k2][q0][n0]: written with (k2, k2 + 1) x n0 = 0..7 at a fixed q0, read with k2 = 0..7 x (q0, q0 + 1) at a fixed
//    n0 -> n0 ^ k2 spreads the eight k2 over eight bank pairs, bit 0 of q0 ^ k2 picks the half.
PC_HD int f512_s1(int k2, int m) { return k2 * 64 + (m ^ ((k2 & 1) << 3)); }
PC_HD int f512_s2(int k2, int q0, int n0) { return k2 * 64 + ((q0 ^ (k2 & 1)) << 3) + (n0 ^ k2); }

// ---------------------------------------------------------------------------------------------------------
// forward: z[n] = (x[2n], x[2n+1]), n < 256 valid (the upper half of [x ; 0] is zero)
// ---------------------------------------------------------------------------------------------------------
// loads of step 1: the 8 non-zero points of the lane's two columns (z[64 n2 + m], n2 < 4), a[4 h + n2]
PC_HD void f512_fwd_load(int lane, const float* src, int nv, bool vec, float2* a) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = lane + 32 * h;
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      const int n = 64 * n2 + m;
      if (vec) {
        a[4 * h + n2] = *reinterpret_cast<const float2*>(src + 2 * n);
      } else {
        const int i0 = 2 * n, i1 = i0 + 1;
        a[4 * h + n2] = make_float2(i0 < nv ? src[i0] : 0.0f, i1 < nv ? src[i1] : 0.0f);
      }
    }
  }
}

// step 1: DFT8 over n2 (upper half of the input is the zero padding) + twiddle, result into the exchange buffer (layout s1)
PC_HD void f512_fwd_p1(int lane, const float2* in, float2* S, const float2* tab) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = lane + 32 * h;
    float2 a[8];
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) a[n2] = in[4 * h + n2];
#pragma unroll
    for (int n2 = 4; n2 < 8; ++n2) a[n2] = make_float2(0.0f, 0.0f);
    f512_dft8<false>(a);
    S[f512_s1(0, m)] = a[0];
#pragma unroll
    for (int k2 = 1; k2 < 8; ++k2) S[f512_s1(k2, m)] = f2_cmul<false>(a[k2], tab[kF512_T1 + k2 * 64 + m]);
  }
}

// step 2 (both directions): the two (k2, n0) pairs of the lane; forward reads layout s1 over n1, inverse layout s2 over q0
template <bool INV>
PC_HD void f512_mid_load(int lane, const float2* S, const float2* tab, float2* A, float2* B) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float2* a = h ? B : A;
    const int pid = lane + 32 * h, k2 = pid >> 3, n0 = pid & 7;
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = INV ? S[f512_s2(k2, j, n0)] : S[f512_s1(k2, 8 * j + n0)];
    f512_dft8<INV>(a);
    // forward: C[q0] *= W64^{n0 q0} ; inverse: E[n1] *= conj(W64^{n1 k2})
#pragma unroll
    // (T2 is symmetric, W64^{ab} = W64^{ba}: index it row-major in the loop variable so that the 8 distinct
    //  addresses of an instruction are consecutive words)
#pragma unroll
    for (int j = 1; j < 8; ++j) a[j] = f2_cmul<INV>(a[j], tab[kF512_T2 + j * 8 + (INV ? k2 : n0)]);
  }
}
template <bool INV>
PC_HD void f512_mid_store(int lane, float2* S, const float2* A, const float2* B) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float2* a = h ? B : A;
    const int pid = lane + 32 * h, k2 = pid >> 3, n0 = pid & 7;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (INV) S[f512_s1(k2, 8 * j + n0)] = a[j];     // E[n1 = j] at [k2][8 n1 + n0]
      else S[f512_s2(k2, j, n0)] = a[j];              // C[q0 = j] at [k2][q0][n0]
    }
  }
}

// even/odd split of one mirror pair: a = Z[k], bm = Z[M-k]  ->  X[k], X[M-k]   (fwd_split of kernels.cuh)
PC_HD void f512_split_pair(float2 a, float2 bm, float2 w, float2* xk, float2* xmk) {
  const float2 b = make_float2(bm.x, -bm.y);
  const float2 E = f2_scale(f2_add(a, b), 0.5f), D = f2_scale(f2_sub(a, b), 0.5f);
  const float2 O = make_float2(D.y, -D.x);              // -i * D
  const float2 wO = f2_cmul<false>(O, w);
  *xk = f2_add(E, wO);
  const float2 t = f2_sub(E, wO);
  *xmk = make_float2(t.x, -t.y);
}

// step 3: DFT8 over n0 for both residues and split: XA[q1] = X[la + 64 q1], XB[q1] = X[lb + 64 q1] of the packed spectrum
PC_HD void f512_fwd_p3_core(int lane, const float2* S, const float2* tab, float2* XA, float2* XB) {
  const int la = f512_la(lane), lb = f512_lb(lane);
  float2 A[8], B[8];
#pragma unroll
  for (int n0 = 0; n0 < 8; ++n0) {
    A[n0] = S[f512_s2(la & 7, la >> 3, n0)];
    B[n0] = S[f512_s2(lb & 7, lb >> 3, n0)];
  }
  f512_dft8<false>(A);      // A[q1] = Z[la + 64 q1]
  f512_dft8<false>(B);      // B[q1] = Z[lb + 64 q1]
  if (lane != 0) {          // mirror of la + 64 q1 is lb + 64 (7 - q1)
#pragma unroll
    for (int q1 = 0; q1 < 8; ++q1)
      f512_split_pair(A[q1], B[7 - q1], tab[kF512_TS + la + 64 * q1], &XA[q1], &XB[7 - q1]);
  } else {                  // lane 0 owns the two self-mirrored residues 0 and 32
    XA[0] = make_float2(A[0].x + A[0].y, A[0].x - A[0].y);          // (DC, Nyquist)
    XA[4] = make_float2(A[4].x, -A[4].y);                            // k = M/2
#pragma unroll
    for (int q1 = 1; q1 < 4; ++q1) f512_split_pair(A[q1], A[8 - q1], tab[kF512_TS + 64 * q1], &XA[q1], &XA[8 - q1]);
#pragma unroll
    for (int q1 = 0; q1 < 4; ++q1) f512_split_pair(B[q1], B[7 - q1], tab[kF512_TS + 32 + 64 * q1], &XB[q1], &XB[7 - q1]);
  }
}

// packed spectrum row to global memory
PC_HD void f512_fwd_store(int lane, const float2* XA, const float2* XB, float2* X) {
  const int la = f512_la(lane), lb = f512_lb(lane);
#pragma unroll
  for (int q1 = 0; q1 < 8; ++q1) {
    X[la + 64 * q1] = XA[q1];
    X[lb + 64 * q1] = XB[q1];
  }
}

// step 3 with the row store
PC_HD void f512_fwd_p3(int lane, const float2* S, const float2* tab, float2* X) {
  float2 XA[8], XB[8];
  f512_fwd_p3_core(lane, S, tab, XA, XB);
  f512_fwd_store(lane, XA, XB, X);
}

// Time-line tiles of the forward transform (k_fwd_fft512_lines): 16 consecutive blocks, one aligned 64-byte run of
// every line component.  Tile [re / im][512 bins][16 samples]: a bin's 16 samples are one 64-byte row, XOR-swizzled by
// bits 1-4 of the bin so that step 3's stores (32 consecutive bins at one sample) and the run reads (16 samples of two
// adjacent bins) are both free of bank conflicts
constexpr int kF512_LineR = 16;
PC_HD int f512_lt(int k, int t) { return k * kF512_LineR + (t ^ ((k >> 1) & 15)); }

// ---------------------------------------------------------------------------------------------------------
// inverse: W[k] = Yt[k] + (-1)^k Yp[k]  (frequency-domain overlap-add), un-split, inverse steps, first half of the output
// ---------------------------------------------------------------------------------------------------------
PC_HD void f512_unsplit_pair(float2 a, float2 bm, float2 w, float2* zk, float2* zmk) {
  const float2 b = make_float2(bm.x, -bm.y);
  const float2 E = f2_scale(f2_add(a, b), 0.5f), D = f2_scale(f2_sub(a, b), 0.5f);
  const float2 O = f2_cmul<true>(D, w);                 // conj(w) * D
  *zk = make_float2(E.x - O.y, E.y + O.x);
  *zmk = make_float2(E.x + O.y, O.x - E.y);
}

// overlap-add merge of one bin k: W = Y[t] + (-1)^k Y[t - 1]
PC_HD float2 f512_ola(float2 yt, float2 yp, float sg) { return make_float2(fmaf(yp.x, sg, yt.x), fmaf(yp.y, sg, yt.y)); }

// first inverse step after the merge (A[q1] = W[la + 64 q1], B[q1] = W[lb + 64 q1]): un-split + inverse DFT8 over q1
// + twiddle -> exchange buffer (layout s2)
PC_HD void f512_inv_p1_core(int lane, float2* A, float2* B, float2* S, const float2* tab) {
  const int la = f512_la(lane), lb = f512_lb(lane);
  float2 ZA[8], ZB[8];
  if (lane != 0) {
#pragma unroll
    for (int q1 = 0; q1 < 8; ++q1)
      f512_unsplit_pair(A[q1], B[7 - q1], tab[kF512_TS + la + 64 * q1], &ZA[q1], &ZB[7 - q1]);
  } else {
    // entry 0 packs (DC, Nyquist); the Nyquist index M is even, so its overlap sign is + (ola_merge)
    ZA[0] = make_float2(0.5f * (A[0].x + A[0].y), 0.5f * (A[0].x - A[0].y));
    ZA[4] = make_float2(A[4].x, -A[4].y);
#pragma unroll
    for (int q1 = 1; q1 < 4; ++q1) f512_unsplit_pair(A[q1], A[8 - q1], tab[kF512_TS + 64 * q1], &ZA[q1], &ZA[8 - q1]);
#pragma unroll
    for (int q1 = 0; q1 < 4; ++q1) f512_unsplit_pair(B[q1], B[7 - q1], tab[kF512_TS + 32 + 64 * q1], &ZB[q1], &ZB[7 - q1]);
  }
  f512_dft8<true>(ZA);      // ZA[n0] = sum_q1 Z[la + 64 q1] W8^{-n0 q1}
  f512_dft8<true>(ZB);
#pragma unroll
  for (int n0 = 0; n0 < 8; ++n0) {
    const float2 da = n0 ? f2_cmul<true>(ZA[n0], tab[kF512_T1 + n0 * 64 + la]) : ZA[0];
    const float2 db = n0 ? f2_cmul<true>(ZB[n0], tab[kF512_T1 + n0 * 64 + lb]) : ZB[0];
    S[f512_s2(la & 7, la >> 3, n0)] = da;
    S[f512_s2(lb & 7, lb >> 3, n0)] = db;
  }
}

// first inverse step from rows: loads of Y[t] (Yt) and Y[t - 1] (Yp) + merge + the rest of the step
PC_HD void f512_inv_p1(int lane, const float2* Yt, const float2* Yp, float2* S, const float2* tab) {
  const int la = f512_la(lane), lb = f512_lb(lane);
  float2 A[8], B[8], PA[8], PB[8];
#pragma unroll
  for (int q1 = 0; q1 < 8; ++q1) {       // all 32 loads first
    A[q1] = PC_LD(Yt + la + 64 * q1); B[q1] = PC_LD(Yt + lb + 64 * q1);
    PA[q1] = PC_LD(Yp + la + 64 * q1); PB[q1] = PC_LD(Yp + lb + 64 * q1);
  }
  const float sg = (lane & 1) ? -1.0f : 1.0f;          // (-1)^k: k has the parity of the lane for both residues
#pragma unroll
  for (int q1 = 0; q1 < 8; ++q1) {
    A[q1] = f512_ola(A[q1], PA[q1], sg);
    B[q1] = f512_ola(B[q1], PB[q1], sg);
  }
  f512_inv_p1_core(lane, A, B, S, tab);
}

// last inverse step: inverse DFT8 over k2 for the two columns; only n2 < 4 (the first B of the 2B output samples)
// FAST: the whole block is inside the destination, no look-ahead rings, linear, 8-byte aligned -> float2 stores
template <bool FAST>
PC_HD void f512_inv_p3(int lane, const float2* S, float scale, const OutSpec& o) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = lane + 32 * h;
    float2 e[8];
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) e[k2] = S[f512_s1(k2, m)];
    f512_dft8<true>(e);
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      const int n = 64 * n2 + m;
      if (FAST) {
        *reinterpret_cast<float2*>(o.dst + o.index0 + 2 * n) = f2_scale(e[n2], scale);
      } else {
        inv_store_sample(e[n2].x, scale, o, 2 * n);
        inv_store_sample(e[n2].y, scale, o, 2 * n + 1);
      }
    }
  }
}

#if defined(__CUDACC__)
// grid (ceil(nblocks / 8) capped, C), block (32, 8): warp = one transform, looping over blocks with stride 8 * gridDim.x
// dynamic smem = (1088 + 8 * 512) float2 = 41472 bytes
__global__ void __launch_bounds__(256, 4) k_fwd_fft512(FwdParams P, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem512[];
  float2* tab = pc_smem512;
  float2* S = pc_smem512 + kF512_TabLen + threadIdx.y * kF512_Xch;
  const int lane = threadIdx.x, tid = threadIdx.y * 32 + lane;
  for (int j = tid; j < kF512_TabLen; j += 256) tab[j] = tab512[j];
  __syncthreads();
  const int c = blockIdx.y;
  const long long nv_total = P.nvalid_c ? (long long)P.nvalid_c[c] : P.nvalid;
  const float* src_c = P.src + (long long)(P.use_cmap ? P.cmap[c] : c) * P.src_cstride;
  // software pipeline: the loads of the warp's NEXT block are issued before the current one is transformed
  auto issue = [&](int blk, float2* a) {
    const long long rem = nv_total - (long long)blk * kF512_M;
    const int nv = rem <= 0 ? 0 : (rem > kF512_M ? kF512_M : (int)rem);
    const float* src = src_c + (long long)blk * kF512_M;
    const bool vec = nv == kF512_M && (reinterpret_cast<size_t>(src) & 7) == 0;
    f512_fwd_load(lane, src, nv, vec, a);
  };
  const int stride = gridDim.x * 8;
  int blk = blockIdx.x * 8 + threadIdx.y;
  float2 nxt[8];
  if (blk < P.nblocks) issue(blk, nxt);
  for (; blk < P.nblocks; blk += stride) {
    float2 cur[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cur[j] = nxt[j];
    if (blk + stride < P.nblocks) issue(blk + stride, nxt);
    f512_fwd_p1(lane, cur, S, tab);
    __syncwarp();
    float2 A[8], B[8];
    f512_mid_load<false>(lane, S, tab, A, B);
    __syncwarp();
    f512_mid_store<false>(lane, S, A, B);
    __syncwarp();
    f512_fwd_p3(lane, S, tab, P.dst + (long long)c * P.dst_cstride + (P.dst_row0 + blk) * (long long)kF512_M);
    __syncwarp();
  }
}

// Time-line mode (P.lines): block b goes to sample tau = line_tau0 + b of the 2 x 512 FP32 time lines of its channel,
// which the tensor-core sweep reads, instead of through an X row and k_tc_split_x.  The CTA owns tiles of 16 samples
// aligned to 16 in tau (the first and the last tile of the group partial): warp w transforms the blocks at samples
// w and w + 8 of the tile with k_fwd_fft512's arithmetic, leaves the spectra in the tile (f512_lt), and the CTA then
// stores every (line, component) run of the tile as one 64-byte piece, two runs per warp instruction.
// grid (min(tiles, 2 * SMs / C), C), block (32, 8); dynamic smem = (1088 + 8 * 512 + 8192) float2 = 107008 bytes
__global__ void __launch_bounds__(256, 2) k_fwd_fft512_lines(FwdParams P, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem512[];
  float2* tab = pc_smem512;
  float2* S = pc_smem512 + kF512_TabLen + threadIdx.y * kF512_Xch;
  float* Tre = reinterpret_cast<float*>(pc_smem512 + kF512_TabLen + 8 * kF512_Xch);
  float* Tim = Tre + kF512_M * kF512_LineR;
  const int lane = threadIdx.x, wid = threadIdx.y, tid = wid * 32 + lane;
  for (int j = tid; j < kF512_TabLen; j += 256) tab[j] = tab512[j];
  __syncthreads();
  const int c = blockIdx.y;
  const long long nv_total = P.nvalid_c ? (long long)P.nvalid_c[c] : P.nvalid;
  const float* src_c = P.src + (long long)(P.use_cmap ? P.cmap[c] : c) * P.src_cstride;
  const long long tile0 = P.line_tau0 / kF512_LineR;
  const int ntiles = (int)((P.line_tau0 + P.nblocks - 1) / kF512_LineR - tile0 + 1);
  // block at sample w + 8 h of tile ti (outside [0, nblocks) in the partial tiles)
  auto block_of = [&](int ti, int h) { return (int)((tile0 + ti) * kF512_LineR - P.line_tau0) + wid + 8 * h; };
  auto issue = [&](int blk, float2* a) {
    if (blk < 0 || blk >= P.nblocks) return;
    const long long rem = nv_total - (long long)blk * kF512_M;
    const int nv = rem <= 0 ? 0 : (rem > kF512_M ? kF512_M : (int)rem);
    const float* src = src_c + (long long)blk * kF512_M;
    const bool vec = nv == kF512_M && (reinterpret_cast<size_t>(src) & 7) == 0;
    f512_fwd_load(lane, src, nv, vec, a);
  };
  float2 nxt[8];
  if ((int)blockIdx.x < ntiles) issue(block_of(blockIdx.x, 0), nxt);
  for (int ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      const int blk = block_of(ti, h);
      float2 cur[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) cur[j] = nxt[j];
      // software pipeline as in k_fwd_fft512: the warp's next block, in this tile or the next one
      if (h == 0) issue(block_of(ti, 1), nxt);
      else if (ti + (int)gridDim.x < ntiles) issue(block_of(ti + gridDim.x, 0), nxt);
      if (blk < 0 || blk >= P.nblocks) continue;
      f512_fwd_p1(lane, cur, S, tab);
      __syncwarp();
      float2 A[8], B[8];
      f512_mid_load<false>(lane, S, tab, A, B);
      __syncwarp();
      f512_mid_store<false>(lane, S, A, B);
      __syncwarp();
      f512_fwd_p3_core(lane, S, tab, A, B);
      const int t = wid + 8 * h, la = f512_la(lane), lb = f512_lb(lane);
#pragma unroll
      for (int q1 = 0; q1 < 8; ++q1) {
        Tre[f512_lt(la + 64 * q1, t)] = A[q1].x; Tim[f512_lt(la + 64 * q1, t)] = A[q1].y;
        Tre[f512_lt(lb + 64 * q1, t)] = B[q1].x; Tim[f512_lt(lb + 64 * q1, t)] = B[q1].y;
      }
      if (blk >= P.xrow_from)
        f512_fwd_store(lane, A, B, P.dst + (long long)c * P.dst_cstride + (P.dst_row0 + blk) * (long long)kF512_M);
      __syncwarp();
    }
    __syncthreads();                    // the tile is complete
    const int t = lane & 15;
    const long long tau = (tile0 + ti) * kF512_LineR + t;
    if (tau >= P.line_tau0 && tau < P.line_tau0 + P.nblocks) {
      const long long line0 = (long long)c * kF512_M;
#pragma unroll 4
      for (int k = 2 * wid + (lane >> 4); k < kF512_M; k += 16) {
        P.lines[tc::xf_index(line0 + k, 0, tau, P.line_rows)] = Tre[f512_lt(k, t)];
        P.lines[tc::xf_index(line0 + k, 1, tau, P.line_rows)] = Tim[f512_lt(k, t)];
      }
    }
    __syncthreads();                    // the tile's reads are done before the next tile's blocks are written into it
  }
}

// YC: bin-major input (P.yc), 8 consecutive blocks per CTA
template <bool FAST, bool YC>
__global__ void __launch_bounds__(256, 3) k_inv_fft512(InvParams P, const float2* __restrict__ tab512) {
  extern __shared__ float2 pc_smem512[];
  float2* tab = pc_smem512;
  float2* S = pc_smem512 + kF512_TabLen + threadIdx.y * kF512_Xch;
  const int lane = threadIdx.x, tid = threadIdx.y * 32 + lane;
  for (int j = tid; j < kF512_TabLen; j += 256) tab[j] = tab512[j];
  __syncthreads();
  const int c = blockIdx.y;
  OutSpec o;
  o.dst = P.dst + (long long)c * P.dst_cstride;
  o.lo = P.lo; o.hi = P.hi; o.mask = P.mask;
  o.n_add = P.n_add;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    o.add[a] = a < P.n_add ? P.add[a] + (long long)c * P.add_cstride[a] : nullptr;
    o.add_mask[a] = P.add_mask[a];
  }
  if (YC) {
    // bin-major input: the CTA takes 8 consecutive blocks t0 ... t0 + 7, reads per bin the 9 spectra t0 - 1 ... t0 + 7
    // of its line, and leaves the merged W[t] = Y[t] + (-1)^k Y[t - 1] in the exchange buffer of the warp of block t
    float2* S0 = pc_smem512 + kF512_TabLen;
    const int ngroups = (P.nblocks + 7) / 8;
    for (int g = blockIdx.x; g < ngroups; g += gridDim.x) {
      const int t0 = 8 * g;
      const bool full = t0 + 8 <= P.nblocks;
      __syncthreads();                                              // the previous group's reads of the buffers are done
      for (int k = tid; k < kF512_M; k += 256) {
        const float2* line = P.yc + ((long long)c * kF512_M + k) * P.yc_stride;
        const long long s = P.yc_slot0 + t0 - 1;                    // slot of Y[t0 - 1]
        float2 v[9];
        if (full && (s & 1) == 0) {                                 // v[0 .. 7] in four aligned float4
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(line + s) + u);
            v[2 * u] = make_float2(f.x, f.y); v[2 * u + 1] = make_float2(f.z, f.w);
          }
          v[8] = __ldg(line + s + 8);
        } else if (full) {                                          // v[1 .. 8] in four aligned float4
          v[0] = __ldg(line + s);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(line + s + 1) + u);
            v[2 * u + 1] = make_float2(f.x, f.y); v[2 * u + 2] = make_float2(f.z, f.w);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 9; ++j) v[j] = t0 - 1 + j < P.nblocks ? __ldg(line + s + j) : make_float2(0.0f, 0.0f);
        }
        if (t0 == 0 && P.yc_prev_row) v[0] = P.Y[(long long)c * P.y_cstride + (P.yrow0 - 1) * P.y_rstride + k];
        const float sg = (k & 1) ? -1.0f : 1.0f;
#pragma unroll
        for (int w = 0; w < 8; ++w) S0[w * kF512_Xch + k] = f512_ola(v[w + 1], v[w], sg);
      }
      __syncthreads();
      const int blk = t0 + threadIdx.y;
      if (blk >= P.nblocks) continue;
      o.index0 = P.index0 + (long long)blk * kF512_M;
      o.abs0 = P.abs0 + (long long)blk * kF512_M;
      {
        const int la = f512_la(lane), lb = f512_lb(lane);
        float2 A[8], B[8];
#pragma unroll
        for (int q1 = 0; q1 < 8; ++q1) { A[q1] = S[la + 64 * q1]; B[q1] = S[lb + 64 * q1]; }
        __syncwarp();
        f512_inv_p1_core(lane, A, B, S, tab);
      }
      __syncwarp();
      float2 A[8], B[8];
      f512_mid_load<true>(lane, S, tab, A, B);
      __syncwarp();
      f512_mid_store<true>(lane, S, A, B);
      __syncwarp();
      f512_inv_p3<FAST>(lane, S, P.scale, o);
    }
  } else {
    for (int blk = blockIdx.x * 8 + threadIdx.y; blk < P.nblocks; blk += gridDim.x * 8) {
      o.index0 = P.index0 + (long long)blk * kF512_M;
      o.abs0 = P.abs0 + (long long)blk * kF512_M;
      const float2* Yt = P.Y + (long long)c * P.y_cstride + (P.yrow0 + blk) * P.y_rstride;
      f512_inv_p1(lane, Yt, Yt - P.y_rstride, S, tab);
      __syncwarp();
      float2 A[8], B[8];
      f512_mid_load<true>(lane, S, tab, A, B);
      __syncwarp();
      f512_mid_store<true>(lane, S, A, B);
      __syncwarp();
      f512_inv_p3<FAST>(lane, S, P.scale, o);
      __syncwarp();
    }
  }
}
#else
// CPU emulation (tests/emu): the lanes of a warp become loops, __syncwarp() the loop boundaries
inline void emu_fwd_fft512(int nblocks, int C, const FwdParams& P, const float2* tab) {
  float2 S[kF512_Xch];
  float2 A[32][8], B[32][8];
  for (int c = 0; c < C; ++c) {
    const long long nv_total = P.nvalid_c ? (long long)P.nvalid_c[c] : P.nvalid;
    const float* src_c = P.src + (long long)(P.use_cmap ? P.cmap[c] : c) * P.src_cstride;
    for (int blk = 0; blk < nblocks; ++blk) {
      const long long rem = nv_total - (long long)blk * kF512_M;
      const int nv = rem <= 0 ? 0 : (rem > kF512_M ? kF512_M : (int)rem);
      const float* src = src_c + (long long)blk * kF512_M;
      for (int l = 0; l < 32; ++l) {
        float2 a[8];
        f512_fwd_load(l, src, nv, false, a);
        f512_fwd_p1(l, a, S, tab);
      }
      for (int l = 0; l < 32; ++l) f512_mid_load<false>(l, S, tab, A[l], B[l]);
      for (int l = 0; l < 32; ++l) f512_mid_store<false>(l, S, A[l], B[l]);
      for (int l = 0; l < 32; ++l) f512_fwd_p3(l, S, tab, P.dst + (long long)c * P.dst_cstride + (P.dst_row0 + blk) * (long long)kF512_M);
    }
  }
}

inline void emu_inv_fft512(int nblocks, int C, const InvParams& P, const float2* tab, bool fast) {
  float2 S[kF512_Xch];
  float2 A[32][8], B[32][8];
  for (int c = 0; c < C; ++c) {
    OutSpec o;
    o.dst = P.dst + (long long)c * P.dst_cstride;
    o.lo = P.lo; o.hi = P.hi; o.mask = P.mask;
    o.n_add = P.n_add;
    for (int a = 0; a < 3; ++a) {
      o.add[a] = a < P.n_add ? P.add[a] + (long long)c * P.add_cstride[a] : nullptr;
      o.add_mask[a] = P.add_mask[a];
    }
    for (int blk = 0; blk < nblocks; ++blk) {
      o.index0 = P.index0 + (long long)blk * kF512_M;
      o.abs0 = P.abs0 + (long long)blk * kF512_M;
      const float2* Yt = P.Y + (long long)c * P.y_cstride + (P.yrow0 + blk) * P.y_rstride;
      for (int l = 0; l < 32; ++l) f512_inv_p1(l, Yt, Yt - P.y_rstride, S, tab);
      for (int l = 0; l < 32; ++l) f512_mid_load<true>(l, S, tab, A[l], B[l]);
      for (int l = 0; l < 32; ++l) f512_mid_store<true>(l, S, A[l], B[l]);
      for (int l = 0; l < 32; ++l) {
        if (fast) f512_inv_p3<true>(l, S, P.scale, o); else f512_inv_p3<false>(l, S, P.scale, o);
      }
    }
  }
}
#endif

}  // namespace pc
