// fft16.cuh -- register-resident radix-16 building blocks and the 256-point
// complex FFT executed by one HALF-WARP (16 lanes x 16 values), used as the
// N/2-point transform behind the 512-point real STFT / iSTFT of the fused
// kernels.
//
//   z[m], m = 16*m1 + m2            lane = m2 holds v[m1]          (pass 1 in)
//   A[k1; m2] = sum_m1 z W16^{m1 k1}, times W256^{m2 k1}           (pass 1)
//   exchange through a 16 x 17 float2 tile (conflict free both ways)
//   Z[k1 + 16 k2] = sum_m2 A[k1; m2] W16^{m2 k2}   lane = k1       (pass 2)
//
// dft16 leaves its outputs in "slot" order: slot s holds frequency
// kof(s) = (s >> 2) + 4 * (s & 3).
#pragma once
#include "common.cuh"

namespace setk {

#define SETK_C16_1R 0.92387953251128674f
#define SETK_C16_1I 0.38268343236508977f
#define SETK_SQRT1_2 0.70710678118654752f

__device__ __forceinline__ constexpr int kof(int s) { return (s >> 2) + 4 * (s & 3); }
__device__ __forceinline__ constexpr int slot_of(int k) { return ((k & 3) << 2) + (k >> 2); }

// forward 4-point DFT in place (W4 = -i)
__device__ __forceinline__ void dft4(float2& a, float2& b, float2& c, float2& d) {
  const float2 e = cadd(a, c), f = csub(a, c), g = cadd(b, d), h = csub(b, d);
  const float2 r = make_float2(h.y, -h.x);           // -i h: a swizzle on the consumer's operand
  a = cadd(e, g);
  c = csub(e, g);
  b = cadd(f, r);
  d = csub(f, r);
}

// v <- v * W16^m  (forward twiddle, compile-time m)
template <int M>
__device__ __forceinline__ float2 mul_w16(float2 v) {
  if (M == 0) return v;
  // W16^m = (cos, -sin)(2 pi m / 16) as a compile-time constant
  if (M == 1) return cmul(v, make_float2(SETK_C16_1R, -SETK_C16_1I));
  if (M == 2) return cmul(v, make_float2(SETK_SQRT1_2, -SETK_SQRT1_2));
  if (M == 3) return cmul(v, make_float2(SETK_C16_1I, -SETK_C16_1R));
  if (M == 4) return make_float2(v.y, -v.x);
  if (M == 6) return cmul(v, make_float2(-SETK_SQRT1_2, -SETK_SQRT1_2));
  if (M == 9) return cmul(v, make_float2(-SETK_C16_1R, SETK_C16_1I));
  return v;
}

// forward 16-point DFT, input natural order v[n], output in slot order.
__device__ __forceinline__ void dft16(float2 (&v)[16]) {
#pragma unroll
  for (int b = 0; b < 4; ++b) dft4(v[b], v[4 + b], v[8 + b], v[12 + b]);
  // now v[4c + b] = T[c; b]; twiddle by W16^{b c}
  v[5] = mul_w16<1>(v[5]);   v[6] = mul_w16<2>(v[6]);   v[7] = mul_w16<3>(v[7]);
  v[9] = mul_w16<2>(v[9]);   v[10] = mul_w16<4>(v[10]); v[11] = mul_w16<6>(v[11]);
  v[13] = mul_w16<3>(v[13]); v[14] = mul_w16<6>(v[14]); v[15] = mul_w16<9>(v[15]);
#pragma unroll
  for (int c = 0; c < 4; ++c) dft4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
}

// pitch of the exchange tile in float2 units (odd -> conflict-free transposed reads)
#define SETK_XPITCH 17
#define SETK_ZSLOT (16 * SETK_XPITCH)   // float2 per half-warp FFT slot (272 >= 256)

// Multiply slot s of v by w^{kof(s)} where w = W256^{lane16} (w1), using a
// depth-<=4 power tree.
__device__ __forceinline__ void twiddle_pass1(float2 (&v)[16], float2 w1) {
  float2 p[16];
  p[1] = w1;
  p[2] = cmul(w1, w1);
  p[3] = cmul(p[2], w1);
  p[4] = cmul(p[2], p[2]);
  p[5] = cmul(p[4], w1);
  p[6] = cmul(p[4], p[2]);
  p[7] = cmul(p[4], p[3]);
  p[8] = cmul(p[4], p[4]);
  p[9] = cmul(p[8], w1);
  p[10] = cmul(p[8], p[2]);
  p[11] = cmul(p[8], p[3]);
  p[12] = cmul(p[8], p[4]);
  p[13] = cmul(p[8], p[5]);
  p[14] = cmul(p[8], p[6]);
  p[15] = cmul(p[8], p[7]);
#pragma unroll
  for (int s = 1; s < 16; ++s) {
    const int k = kof(s);
    if (k != 0) v[s] = cmul(v[s], p[k]);
  }
}

// The same multiplication with the powers read from a shared-memory table
// tab[k * 16 + lane16] = W256^{lane16 * k}, k = 1..15 (tab[0..15] unused): 15
// broadcast-friendly 8-byte loads instead of 15 complex multiplies for the power
// tree, and no registers held for it (the fused covariance kernel needs them for
// its accumulators to keep two CTAs per SM).
__device__ __forceinline__ void twiddle_pass1_tab(float2 (&v)[16], const float2* tab, int lane16) {
  const float2* t = tab + lane16;              // one base register, immediate offsets
#pragma unroll
  for (int s = 1; s < 16; ++s) {
    const int k = kof(s);
    if (k != 0) v[s] = cmul(v[s], t[k * 16]);
  }
}
// fill the table (any number of threads; sincospif is exact to an ulp)
__device__ __forceinline__ void twiddle_table_fill(float2* tab, int tid, int nthreads) {
  for (int e = tid; e < 256; e += nthreads) {
    const int k = e >> 4, l = e & 15;
    float sn, cs;
    sincospif((float)((k * l) & 255) / 128.0f, &sn, &cs);
    tab[e] = make_float2(cs, -sn);
  }
}

// 256-point forward complex FFT by one half-warp.
//   v     in : v[m1] = z[16*m1 + lane16]
//         out: slot s = Z[lane16 + 16*kof(s)]
//   xch   : this half-warp's SETK_ZSLOT float2 exchange tile in shared memory
//   w1    : W256^{lane16} = (cos(2 pi lane16/256), -sin(2 pi lane16/256))
// All 32 lanes of the warp must call this together (it uses __syncwarp).
// tab != nullptr: inter-pass twiddles from the shared-memory table instead of w1's power tree
template <bool TAB = false>
__device__ __forceinline__ void halfwarp_fft256(float2 (&v)[16], float2* xch, int lane16, float2 w1,
                                                const float2* tab = nullptr) {
  dft16(v);
  if (TAB) twiddle_pass1_tab(v, tab, lane16);
  else twiddle_pass1(v, w1);
#pragma unroll
  for (int s = 0; s < 16; ++s) xch[kof(s) * SETK_XPITCH + lane16] = v[s];
  __syncwarp();
#pragma unroll
  for (int m2 = 0; m2 < 16; ++m2) v[m2] = xch[lane16 * SETK_XPITCH + m2];
  __syncwarp();
  dft16(v);
}

// The same transform in two halves, for kernels that must wait for the exchange
// tile to become free between them (stft_cov_ws.cu: the tile is a ring slot):
//   a: first radix-16 pass + inter-pass twiddles, registers only
//   b: exchange through xch + second radix-16 pass
__device__ __forceinline__ void halfwarp_fft256_a(float2 (&v)[16], const float2* tab, int lane16) {
  dft16(v);
  twiddle_pass1_tab(v, tab, lane16);
}
__device__ __forceinline__ void halfwarp_fft256_b(float2 (&v)[16], float2* xch, int lane16) {
#pragma unroll
  for (int s = 0; s < 16; ++s) xch[kof(s) * SETK_XPITCH + lane16] = v[s];
  __syncwarp();
#pragma unroll
  for (int m2 = 0; m2 < 16; ++m2) v[m2] = xch[lane16 * SETK_XPITCH + m2];
  __syncwarp();
  dft16(v);
}

}  // namespace setk
