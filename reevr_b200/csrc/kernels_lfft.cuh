// kernels_lfft.cuh — K2f: the batched sweep of long launch groups as an FFT convolution along the block index.
//
// Per frequency bin k the sweep is a 1-D convolution of the bin's time line with its P partition values
// (kernels_tc.cuh): y_k[s] = sum_p H[p][k] * x_k[s + Q - p], for the outputs s < Lty of the line.  K2f computes it by
// overlap-save with kN-point complex FFTs along the line (nested partitioned convolution):
//
//   segment q: window x_k[w0 ... w0 + kN - 1], w0 = q L + Q - (P - 1);  c = IFFT(FFT(window) . FFT(H[.][k] zero-padded))
//              outputs s = q L + m - (P - 1) = c[m] for m = P - 1 ... kN - 1 (the L = kN - P + 1 valid ones)
//
// Samples past the line's Lt read as zeros; the last segment is partial.  The time lines are the FP32 planes
// k_tc_split_x and k_fwd_fft512_lines write (xf_index), the result goes to the bin-major slots k_tc_sweep writes
// (kYLead + s), so everything before and after the sweep is that of the tensor-core form.
//
// Transform: kN = 4096 = 16^3, 256 threads per CTA with 16 complex values each, three radix-16 Stockham passes (DFT-16
// in registers, twiddles, exchange through 34 KB of padded shared memory between passes).  The last forward pass leaves
// thread j holding bins j + 256 r, which is exactly what the first inverse pass reads: the pointwise product with the
// line's spectrum happens in registers, and the inverse's output (natural order) goes straight to global memory.
// The inverse is conj(FFT(conj(Y))); 1/kN (exact) is folded into the stored spectra.
//
// Entry 0 of each channel packs DC and Nyquist as two real lines (y = (D1, D2) = (Hr * xr, Hi * xi)).  With
// Z = FFT(xr + i xi) and HR, HI the spectra of the real sequences Hr, Hi:
//   FFT(y) = Z[f] (HR + HI) / 2 + conj(Z[-f]) (HR - HI) / 2
// k_lfft_build_h stores (HR + HI) / 2 as the line's spectrum and (HR - HI) / 2 in an extra slot per channel.
//
// Kernels: k_lfft_build_h (H -> line spectra, once per IR and stage), k_lfft_sweep (one CTA per (line, segment),
// segments of a line consecutive in the grid so that the line's spectrum is read from HBM once and from L2 after).
#pragma once

#include "kernels_tc.cuh"

namespace pc {
namespace lfft {

constexpr int kN = 4096;                            // transform size
constexpr int kThreads = 256;                       // kN / 16: one DFT-16 per thread and pass
constexpr int kSmemFloats = kN + kN / 16;           // one pad float per 16: conflict-free stores of both passes

// Segment plan of a line.  L valid outputs per segment; segment q reads the window from tau = w0(q), its output m
// (m >= P - 1) is sweep output q L + m - (P - 1); outputs reach Lty (the slots k_tc_sweep writes).
struct Plan {
  int P, Q, L, nseg;
  long long Lt, Lty;
};

PC_TC_HD Plan make_plan(int P, int nb) {
  const tc::Geom g = tc::make_geom(P, nb);
  Plan p;
  p.P = P; p.Q = g.Q; p.Lt = g.Lt; p.Lty = g.Lty;
  p.L = kN - (P - 1);
  p.nseg = (int)((g.Lty + p.L - 1) / p.L);
  return p;
}
PC_TC_HD bool plan_ok(int P) { return P >= 1 && P <= kN / 2; }
PC_TC_HD long long window_start(const Plan& p, int q) { return (long long)q * p.L + p.Q - (p.P - 1); }
// sweep output of the segment's circular-convolution index m, or -1 when m is not a valid output (m < P - 1 or past Lty)
PC_TC_HD long long output_of(const Plan& p, int q, int m) {
  if (m < p.P - 1) return -1;
  const long long s = (long long)q * p.L + m - (p.P - 1);
  return s < p.Lty ? s : -1;
}
// line spectra: [C * B lines + C][kN] float2 (the C extra lines: (HR - HI) / 2 of each channel's entry 0)
PC_TC_HD size_t spectra_bytes(size_t lines, int C) { return (lines + (size_t)C) * kN * 8; }

#if defined(__CUDACC__)

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// 4-point DFT (forward sign) of a[i0], a[i0 + s], a[i0 + 2 s], a[i0 + 3 s], in place
template <int I0, int S>
__device__ __forceinline__ void dft4(float2 (&a)[16]) {
  const float2 x0 = a[I0], x1 = a[I0 + S], x2 = a[I0 + 2 * S], x3 = a[I0 + 3 * S];
  const float2 s02 = make_float2(x0.x + x2.x, x0.y + x2.y), d02 = make_float2(x0.x - x2.x, x0.y - x2.y);
  const float2 s13 = make_float2(x1.x + x3.x, x1.y + x3.y), d13 = make_float2(x1.x - x3.x, x1.y - x3.y);
  a[I0] = make_float2(s02.x + s13.x, s02.y + s13.y);
  a[I0 + 2 * S] = make_float2(s02.x - s13.x, s02.y - s13.y);
  a[I0 + S] = make_float2(d02.x + d13.y, d02.y - d13.x);        // d02 - i d13
  a[I0 + 3 * S] = make_float2(d02.x - d13.y, d02.y + d13.x);    // d02 + i d13
}

// multiply by W16^e = exp(-2 pi i e / 16), e in 0 ... 9
template <int E>
__device__ __forceinline__ float2 w16(float2 v) {
  constexpr float c1 = 0.92387953251128674f, s1 = 0.38268343236508978f, h = 0.70710678118654752f;
  if constexpr (E == 0) return v;
  else if constexpr (E == 4) return make_float2(v.y, -v.x);
  else if constexpr (E == 2) return make_float2(h * (v.x + v.y), h * (v.y - v.x));
  else if constexpr (E == 6) return make_float2(h * (v.y - v.x), -h * (v.x + v.y));
  else {
    constexpr float c = E == 1 ? c1 : E == 3 ? s1 : E == 9 ? -c1 : 0.0f;
    constexpr float s = E == 1 ? s1 : E == 3 ? c1 : E == 9 ? -s1 : 0.0f;   // W = c - i s
    static_assert(E == 1 || E == 3 || E == 9, "W16 exponent");
    return make_float2(v.x * c + v.y * s, v.y * c - v.x * s);
  }
}

// in-place 16-point DFT, natural order in and out: r = r0 + 4 r1, k = k1 + 4 k0
__device__ __forceinline__ void dft16(float2 (&a)[16]) {
  dft4<0, 4>(a); dft4<1, 4>(a); dft4<2, 4>(a); dft4<3, 4>(a);        // over r1: a[r0 + 4 k1]
  a[5] = w16<1>(a[5]); a[6] = w16<2>(a[6]); a[7] = w16<3>(a[7]);      // W16^(r0 k1)
  a[9] = w16<2>(a[9]); a[10] = w16<4>(a[10]); a[11] = w16<6>(a[11]);
  a[13] = w16<3>(a[13]); a[14] = w16<6>(a[14]); a[15] = w16<9>(a[15]);
  dft4<0, 1>(a); dft4<4, 1>(a); dft4<8, 1>(a); dft4<12, 1>(a);        // over r0: a[4 k1 + k0] = V[k1 + 4 k0]
  float2 t[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) t[i] = a[i];
#pragma unroll
  for (int k1 = 0; k1 < 4; ++k1)
#pragma unroll
    for (int k0 = 0; k0 < 4; ++k0) a[k1 + 4 * k0] = t[4 * k1 + k0];
}

// a[r] *= w^r, r = 1 ... 15, with the powers built by products of depth <= 4 from w
__device__ __forceinline__ void twiddle(float2 (&a)[16], float2 w) {
  // rebuilt at every pass: kept live across the passes, the 30 powers of both bases would not fit the register budget
  asm volatile("" : "+f"(w.x), "+f"(w.y));
  const float2 w2 = cmul(w, w), w4 = cmul(w2, w2), w8 = cmul(w4, w4);
  const float2 w3 = cmul(w2, w);
  const float2 lo[8] = {make_float2(1.0f, 0.0f), w, w2, w3, w4, cmul(w4, w), cmul(w4, w2), cmul(w4, w3)};
  a[1] = cmul(a[1], w); a[2] = cmul(a[2], w2); a[3] = cmul(a[3], w3); a[4] = cmul(a[4], w4);
  a[5] = cmul(a[5], lo[5]); a[6] = cmul(a[6], lo[6]); a[7] = cmul(a[7], lo[7]); a[8] = cmul(a[8], w8);
#pragma unroll
  for (int r = 9; r < 16; ++r) a[r] = cmul(a[r], cmul(w8, lo[r - 8]));
}

__device__ __forceinline__ int pad(int i) { return i + (i >> 4); }

// Stockham exchange after the pass with stride ns: V[k] of thread j goes to (j / ns) ns 16 + j % ns + k ns, then
// thread j reads elements j + 256 r.  The first barrier protects the previous reads of the buffer
template <int NS>
__device__ __forceinline__ void exchange(float2 (&a)[16], float* sre, float* sim, int j) {
  const int base = (j / NS) * NS * 16 + j % NS;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 16; ++k) { sre[pad(base + k * NS)] = a[k].x; sim[pad(base + k * NS)] = a[k].y; }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 16; ++r) a[r] = make_float2(sre[pad(j + 256 * r)], sim[pad(j + 256 * r)]);
}

// forward kN-point DFT: thread j holds x[j + 256 r] in a[r] on entry and X[j + 256 r] on exit.  tw1, tw2: the
// twiddle bases of passes 2 and 3, exp(-2 pi i (j % 16) / 256) and exp(-2 pi i j / 4096)
__device__ __forceinline__ void fft4096(float2 (&a)[16], float* sre, float* sim, int j, float2 tw1, float2 tw2) {
  dft16(a);
  exchange<1>(a, sre, sim, j);
  twiddle(a, tw1);
  dft16(a);
  exchange<16>(a, sre, sim, j);
  twiddle(a, tw2);
  dft16(a);
}

__device__ __forceinline__ void twiddle_bases(int j, float2& tw1, float2& tw2) {
  float s, c;
  sincospif(-(float)(j & 15) / 128.0f, &s, &c);
  tw1 = make_float2(c, s);
  sincospif(-(float)j / 2048.0f, &s, &c);
  tw2 = make_float2(c, s);
}

// ---- H -> line spectra (once per IR and stage) -----------------------------------------------------------------
struct BuildHParams {
  const float2* H;          // [C][Prows][B]
  long long h_cstride;
  int B, P, C;
  float2* S;                // [C * B + C][kN]
};

// grid (B, C), block kThreads.  Spectra carry the inverse transform's 1 / kN
__global__ void __launch_bounds__(kThreads, 1) k_lfft_build_h(BuildHParams p) {
  __shared__ float sre[kSmemFloats], sim[kSmemFloats];
  const int j = threadIdx.x, k = blockIdx.x, ch = blockIdx.y;
  const long long line = (long long)ch * p.B + k;
  const float2* Hk = p.H + (long long)ch * p.h_cstride + k;
  float2 tw1, tw2;
  twiddle_bases(j, tw1, tw2);
  constexpr float inv_n = 1.0f / (float)kN;
  float2 a[16], b[16];
  for (int part = 0; part < (k == 0 ? 2 : 1); ++part) {
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int pp = j + 256 * r;
      float2 h = pp < p.P ? Hk[(long long)pp * p.B] : make_float2(0.0f, 0.0f);
      if (k == 0) h = make_float2(part == 0 ? h.x : h.y, 0.0f);       // entry 0: the real lines Hr, Hi
      a[r] = h;
    }
    fft4096(a, sre, sim, j, tw1, tw2);
    if (k == 0 && part == 0) {
#pragma unroll
      for (int r = 0; r < 16; ++r) b[r] = a[r];
    }
  }
  float2* S = p.S + line * kN;
  if (k == 0) {                                   // b = HR, a = HI
    float2* S2 = p.S + ((long long)p.C * p.B + ch) * kN;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const float hn = 0.5f * inv_n;
      S[j + 256 * r] = make_float2((b[r].x + a[r].x) * hn, (b[r].y + a[r].y) * hn);
      S2[j + 256 * r] = make_float2((b[r].x - a[r].x) * hn, (b[r].y - a[r].y) * hn);
    }
  } else {
#pragma unroll
    for (int r = 0; r < 16; ++r) S[j + 256 * r] = make_float2(a[r].x * inv_n, a[r].y * inv_n);
  }
}

// ---- the sweep ------------------------------------------------------------------------------------------------
struct SweepParams {
  const float* Xt;          // FP32 time lines (tc::xf_index)
  const float2* S;          // line spectra (k_lfft_build_h)
  float2* Yc;               // [lines][ystride] complex result, bin-major (tc::kYLead)
  long long ystride;
  int rows, B, C;
  Plan plan;
};

// grid (lines * nseg), block kThreads: item = line * nseg + segment
__global__ void __launch_bounds__(kThreads, 2) k_lfft_sweep(SweepParams p) {
  __shared__ float sre[kSmemFloats], sim[kSmemFloats];
  const int j = threadIdx.x;
  const int line = (int)(blockIdx.x / (unsigned)p.plan.nseg), q = (int)(blockIdx.x - (unsigned)line * p.plan.nseg);
  const long long w0 = window_start(p.plan, q);
  const float* xr = p.Xt + tc::xf_index(line, 0, 0, p.rows);
  const float* xi = p.Xt + tc::xf_index(line, 1, 0, p.rows);
  float2 a[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const long long tau = w0 + j + 256 * r;
    a[r] = tau < p.plan.Lt ? make_float2(__ldg(xr + tau), __ldg(xi + tau)) : make_float2(0.0f, 0.0f);
  }
  float2 tw1, tw2;
  twiddle_bases(j, tw1, tw2);
  fft4096(a, sre, sim, j, tw1, tw2);
  const float2* S = p.S + (size_t)line * kN;
  if (line % p.B == 0) {                          // DC / Nyquist: Z[f] S[f] + conj(Z[-f]) S2[f]
    const float2* S2 = p.S + ((size_t)p.C * p.B + line / p.B) * kN;
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; ++r) { sre[pad(j + 256 * r)] = a[r].x; sim[pad(j + 256 * r)] = a[r].y; }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int f = (kN - (j + 256 * r)) & (kN - 1);
      const float2 zm = make_float2(sre[pad(f)], -sim[pad(f)]);
      const float2 y = cmul(a[r], __ldg(S + j + 256 * r)), y2 = cmul(zm, __ldg(S2 + j + 256 * r));
      a[r] = make_float2(y.x + y2.x, -(y.y + y2.y));                  // conj: the inverse as a forward transform
    }
  } else {
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const float2 y = cmul(a[r], __ldg(S + j + 256 * r));
      a[r] = make_float2(y.x, -y.y);
    }
  }
  fft4096(a, sre, sim, j, tw1, tw2);
  float2* dst = p.Yc + (size_t)line * p.ystride + tc::kYLead;
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const long long s = output_of(p.plan, q, j + 256 * r);
    if (s >= 0) dst[s] = make_float2(a[r].x, -a[r].y);
  }
}

#endif  // __CUDACC__

}  // namespace lfft
}  // namespace pc
