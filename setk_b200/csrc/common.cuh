// common.cuh -- plan object, frame bookkeeping and small complex helpers shared
// by every kernel of libsetk_b200.
#pragma once
#include "compat.cuh"
#include "../../include/setk_b200.h"

namespace setk {

// float32 machine epsilon: EPSILON of the reference (libs/utils.py:16)
#define SETK_EPS32 1.1920928955078125e-07f
#define SETK_EPS32_D 1.1920928955078125e-07
// numpy.finfo(float32).tiny: librosa.util.tiny for a float32 iSTFT buffer
#define SETK_TINY32 1.17549435e-38f

// internal flag (not part of the C-ABI): use 1 - mask (after clipping)
#define SETK_F_ONE_MINUS_INTERNAL 0x80000000u

struct Geometry {   // passed by value to kernels
  int C;            // channels
  int n_fft;        // FFT size (power of two)
  int log2n;
  int hop;
  int pad;          // n_fft/2 if center else 0
  int F;            // n_fft/2 + 1
};

// T of librosa.stft for an utterance of n samples (SURVEY.md App. A);
// <= 0 when the utterance is too short for one frame / for reflect padding.
SETK_HD inline int frames_of(int n, int n_fft, int hop, int pad) {
  if (pad > 0 && n < pad + 1) return 0;   // np.pad(reflect) needs n > pad
  int padded = n + 2 * pad;
  if (padded < n_fft) return 0;
  return 1 + (padded - n_fft) / hop;
}

// frames of the STFT that librosa.istft reads for an n_out-sample output; a T-frame input uses
// min(T, this) of its frames (the ones after them reach only trimmed samples)
inline int istft_frame_cap(const Geometry& g, int n_out) { return (n_out + 2 * g.pad + g.hop - 1) / g.hop; }

// row pitch (complex values) of the bin-major STFT workspaces [B][T][C][pitch]: F rounded up to a
// multiple of 8 -- 264 for 257 bins (n_fft 512), 520 for 513 (n_fft 1024)
SETK_HD constexpr int bin_pitch(int F) { return (F + 7) & ~7; }

// n rounded up to a multiple of 256: the alignment of the regions carved from one scratch allocation
inline size_t up256(size_t n) { return (n + 255) / 256 * 256; }

// index into the un-padded signal of padded position p (np.pad mode="reflect")
SETK_HD inline int reflect_index(int p, int pad, int n) {
  int i = p - pad;
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

struct cf { float x, y; };  // not used for storage; float2 is

// ---------------------------------------------------------------------------
// fp32 pairs, element-wise.  sm_90a has no packed fp32 instructions: each
// helper is two scalar FADD / FMUL / FFMA, and the (re, im) shuffles written
// below are register renames.  Every element is rounded once (fmaf is fused),
// so a complex multiply is one FMUL + one FFMA per part.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float2 f2add(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2sub(float2 a, float2 b) {
  return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2mul(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return f2add(a, b); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return f2sub(a, b); }
// a * b = (ax bx, ay bx) + (-ay by, ax by)
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return f2fma(make_float2(a.y, a.x), make_float2(-b.y, b.y), f2mul(a, make_float2(b.x, b.x)));
}
// a * b + c
__device__ __forceinline__ float2 cmad(float2 a, float2 b, float2 c) {
  return f2fma(make_float2(a.y, a.x), make_float2(-b.y, b.y), f2fma(a, make_float2(b.x, b.x), c));
}
// a * conj(b) = (ax bx, ay bx) + (ay by, -ax by)
__device__ __forceinline__ float2 cmul_conj(float2 a, float2 b) {
  return f2fma(make_float2(a.y, a.x), make_float2(b.y, -b.y), f2mul(a, make_float2(b.x, b.x)));
}
// conj(w) * x + c = (wx xx, wx xy) + (wy xy, -wy xx) + c
__device__ __forceinline__ float2 cmad_conjw(float2 w, float2 x, float2 c) {
  return f2fma(make_float2(x.y, x.x), make_float2(w.y, -w.y), f2fma(x, make_float2(w.x, w.x), c));
}

}  // namespace setk

// The opaque plan of the C-ABI.
struct setk_plan {
  setk_config_t cfg;
  setk::Geometry geo;
  float* d_window;       // [n_fft] analysis window, centred zero-padded, float32
  float* d_wsq;          // [n_fft] window squared (rounded from float64)
  // lazily grown workspaces (device)
  float* d_partials;     size_t partials_bytes;   // fused stft_cov partial sums
  float2* d_stft_ws;     size_t stft_ws_bytes;    // generic path STFT spill [B][C][F][T]
  float2* d_enh_ws;      size_t enh_ws_bytes;     // generic path enhanced STFT [B][F][T]
  float* d_frames_ws;    size_t frames_ws_bytes;  // generic iSTFT frames [B][T][n_fft]
  unsigned* d_peak;      size_t peak_bytes;       // [B] max|y| as uint bits
  double* d_cgmm_ws;     size_t cgmm_ws_bytes;    // CGMM posteriors, partials, R^-1 (cgmm.cu)
  int* d_tile_prefix;   size_t tile_prefix_bytes;   // ragged batches: tiles before each utterance
  float* d_wave_ws;     size_t wave_ws_bytes;       // un-normalised wave of the PCM-16 output path
  int* d_mel;           int num_mel, mel_weights;   // setk_plan_set_mel: [num_mel][4] bands, then the weights
  int sm_count;
};
