// generic.cu -- shape-generic kernels behind the reference's per-call Python
// API (any C <= 16, any power-of-two n_fft in [32, 4096], any hop, center
// on/off): explicit STFT, compute_covar on an explicit STFT, beamform on an
// explicit STFT, iSTFT.  They exist so that every reference entry point
// (forward_stft, compute_covar, Beamformer.beamform, inverse_stft) has a CUDA
// implementation with the reference's array layouts; the batch hot path uses
// the fused kernels in stft_cov_fused.cu / apply_istft_fused.cu instead.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

// ---------------------------------------------------------------------------
// In-place radix-2 DIT FFT of n = 2^log2n complex points in shared memory by
// the whole CTA.  Input must be in bit-reversed order.  sign = -1 forward,
// +1 inverse (unscaled).
// ---------------------------------------------------------------------------
__device__ inline void block_fft(float2* s, int log2n, float sign) {
  const int n = 1 << log2n;
  for (int st = 1; st <= log2n; ++st) {
    const int half = 1 << (st - 1);
    __syncthreads();
    for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
      const int j = i & (half - 1);
      const int i0 = ((i >> (st - 1)) << st) + j;
      const int i1 = i0 + half;
      float sn, cs;
      sincospif((float)j / (float)half, &sn, &cs);
      const float2 w = make_float2(cs, sign * sn);
      const float2 t = cmul(w, s[i1]);
      const float2 u = s[i0];
      s[i0] = cadd(u, t);
      s[i1] = csub(u, t);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ int bitrev(int v, int log2n) {
  return (int)(__brev((unsigned)v) >> (32 - log2n));
}

// ---------------------------------------------------------------------------
// n_fft that is not a power of two (--round-power-of-two false, utils.py:115: n_fft =
// frame_len, e.g. 400): direct real DFT / inverse real DFT by the CTA, O(n^2) with a
// shared-memory twiddle table W[k] = exp(-2 pi i k / n) indexed by (f n) mod n.  A rarely
// used option of a 0.1 ms kernel: simplicity over speed; fp32 sums of <= 4096 terms with
// exactly reduced arguments (rel. error ~1e-6).  s holds n floats (signal) + n float2 (table).
// ---------------------------------------------------------------------------
__device__ inline void dft_table(float2* tab, int n) {
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    float sn, cs;
    sincospif(2.0f * (float)k / (float)n, &sn, &cs);
    tab[k] = make_float2(cs, -sn);
  }
}
// X[f] = sum_n x[n] W^{f n}, f = 0 .. n/2
__device__ inline float2 dft_bin(const float* x, const float2* tab, int n, int f) {
  float re = 0.f, im = 0.f;
  int idx = 0;
  for (int i = 0; i < n; ++i) {
    const float2 w = tab[idx];
    re = fmaf(x[i], w.x, re);
    im = fmaf(x[i], w.y, im);
    idx += f;
    if (idx >= n) idx -= n;
  }
  return make_float2(re, im);
}
// x[i] = (1/n) (Re X0 + (-1)^i Re X_{n/2} + 2 sum_{k=1}^{n/2-1} Re(X_k conj(W)^{k i}))   (n even)
__device__ inline float idft_sample(const float2* X, const float2* tab, int n, int i) {
  float acc = 0.f;
  int idx = i % n;
  const int step = idx;
  for (int k = 1; k < n / 2; ++k) {
    const float2 w = tab[idx];                 // W^{k i} = (cos, -sin): Re(X conj(W)) = Xr c - Xi s ... s = -w.y
    acc = fmaf(X[k].x, w.x, acc);
    acc = fmaf(X[k].y, w.y, acc);
    idx += step;
    if (idx >= n) idx -= n;
  }
  const float nyq = (i & 1) ? -X[n / 2].x : X[n / 2].x;
  return (X[0].x + nyq + 2.0f * acc) / (float)n;
}

// forward_stft (utils.py:96-138) for every (frame, channel, utterance).
// grid (T, C, B); dynamic smem n_fft * 8 B.
__global__ void stft_generic_kernel(Geometry g, const float* __restrict__ audio,
                                    const int* __restrict__ n_samples, int N, int T,
                                    const float* __restrict__ window, float2* __restrict__ out) {
  SETK_DYN_SMEM(float2, s);
  const int t = blockIdx.x, c = blockIdx.y, b = blockIdx.z;
  const int nb = n_samples ? n_samples[b] : N;
  const int Tb = frames_of(nb, g.n_fft, g.hop, g.pad);
  float2* o = out + (((long long)b * g.C + c) * g.F) * T + t;
  if (t >= Tb) {
    for (int f = threadIdx.x; f < g.F; f += blockDim.x) o[(long long)f * T] = make_float2(0.f, 0.f);
    return;
  }
  const float* x = audio + ((long long)b * g.C + c) * N;
  if (g.log2n < 0) {                       // n_fft is not a power of two: direct DFT
    float2* tab = s;
    float* xs = reinterpret_cast<float*>(s + g.n_fft);
    dft_table(tab, g.n_fft);
    for (int n = threadIdx.x; n < g.n_fft; n += blockDim.x) {
      const int p = t * g.hop + n;
      const int i = g.pad ? reflect_index(p, g.pad, nb) : p;
      xs[n] = window[n] * x[i];
    }
    __syncthreads();
    for (int f = threadIdx.x; f < g.F; f += blockDim.x) o[(long long)f * T] = dft_bin(xs, tab, g.n_fft, f);
    return;
  }
  for (int n = threadIdx.x; n < g.n_fft; n += blockDim.x) {
    const int p = t * g.hop + n;
    const int i = g.pad ? reflect_index(p, g.pad, nb) : p;
    s[bitrev(n, g.log2n)] = make_float2(window[n] * x[i], 0.f);
  }
  block_fft(s, g.log2n, -1.f);
  for (int f = threadIdx.x; f < g.F; f += blockDim.x) o[(long long)f * T] = s[f];
}

// compute_covar (beamformer.py:87-103) on an explicit STFT.
// grid (F, B); block C*C threads (>= 32); thread (i, j) accumulates
// sum_t m x_i conj(x_j) in double over T tiles staged in shared memory.
#define SETK_COV_TILE 64
__global__ void cov_generic_kernel(const float2* __restrict__ stft, const float* __restrict__ mask,
                                   unsigned flags, int C, int F, int T, float2* __restrict__ R) {
  __shared__ float2 sx[SETK_MAX_CHANNELS][SETK_COV_TILE];
  __shared__ float sm[SETK_COV_TILE];
  const int f = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x;
  const int i = tid / C, j = tid % C;
  const bool active = tid < C * C;
  double ar = 0.0, ai = 0.0, msum = 0.0;
  for (int t0 = 0; t0 < T; t0 += SETK_COV_TILE) {
    const int nt = imin(SETK_COV_TILE, T - t0);
    __syncthreads();
    for (int e = tid; e < C * SETK_COV_TILE; e += blockDim.x) {
      const int c = e / SETK_COV_TILE, tt = e % SETK_COV_TILE;
      if (tt < nt) sx[c][tt] = stft[(((long long)b * C + c) * F + f) * T + t0 + tt];
    }
    for (int tt = tid; tt < nt; tt += blockDim.x) {
      float m = (flags & SETK_F_MASK_FT) ? mask[((long long)b * F + f) * T + t0 + tt]
                                         : mask[((long long)b * T + t0 + tt) * F + f];
      if (flags & SETK_F_CLIP_MASK) m = fminf(m, 1.0f);
      if (flags & SETK_F_ONE_MINUS_INTERNAL) m = 1.0f - m;
      sm[tt] = m;
    }
    __syncthreads();
    if (active) {
      for (int tt = 0; tt < nt; ++tt) {
        const float2 xi = sx[i][tt], xj = sx[j][tt];
        const double m = (double)sm[tt];
        // (m x_i) conj(x_j)
        ar += m * ((double)xi.x * xj.x + (double)xi.y * xj.y);
        ai += m * ((double)xi.y * xj.x - (double)xi.x * xj.y);
        msum += m;
      }
    }
  }
  if (active) {
    const double den = fmax(msum, 1e-6);
    R[(((long long)b * F + f) * C + i) * C + j] = make_float2((float)(ar / den), (float)(ai / den));
  }
}

// Beamformer.beamform (beamformer.py:220-234) (+ optional post-mask,
// apply_adaptive_beamformer.py:174-175).  One thread per (b, f, t), t fastest.
__global__ void apply_generic_kernel(const float2* __restrict__ stft, const void* __restrict__ w,
                                     int w_dtype, const float* __restrict__ post_mask, int B, int C,
                                     int F, int T, float2* __restrict__ enh) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * F * T) return;
  const int t = (int)(idx % T);
  const int f = (int)((idx / T) % F);
  const int b = (int)(idx / ((long long)T * F));
  float yr = 0.f, yi = 0.f;
  for (int c = 0; c < C; ++c) {
    float wr, wi;
    const long long wi_ = ((long long)b * F + f) * C + c;
    if (w_dtype == SETK_C128) {
      const double* wp = reinterpret_cast<const double*>(w) + 2 * wi_;
      wr = (float)wp[0]; wi = (float)wp[1];
    } else {
      const float* wp = reinterpret_cast<const float*>(w) + 2 * wi_;
      wr = wp[0]; wi = wp[1];
    }
    const float2 x = stft[(((long long)b * C + c) * F + f) * T + t];
    // conj(w) * x
    yr += wr * x.x + wi * x.y;
    yi += wr * x.y - wi * x.x;
  }
  if (post_mask) {
    const float m = post_mask[((long long)b * T + t) * F + f];
    yr *= m; yi *= m;
  }
  enh[idx] = make_float2(yr, yi);
}

// irfft of one enhanced frame x synthesis window -> frames[b][t][n]
// (librosa.istft: ytmp = ifft_window * irfft(stft_matrix)).  grid (T_used, B).
// enh element (b, f, t) lives at  b*sb + f*sf + t*st  (the API layout [B][F][T]
// or the bin-major workspace of stft_spill.cu).
__global__ void istft_frames_kernel(Geometry g, const float2* __restrict__ enh, long long sb,
                                    long long sf, long long st,
                                    const float* __restrict__ window, float* __restrict__ frames,
                                    int T_used) {
  SETK_DYN_SMEM(float2, s);
  const int t = blockIdx.x, b = blockIdx.y;
  const float2* e = enh + (long long)b * sb + (long long)t * st;
  const int n = g.n_fft;
  if (g.log2n < 0) {                       // n_fft is not a power of two: direct inverse DFT
    float2* tab = s;
    float2* X = s + n;
    dft_table(tab, n);
    for (int k = threadIdx.x; k < g.F; k += blockDim.x) X[k] = e[(long long)k * sf];
    __syncthreads();
    float* o = frames + ((long long)b * T_used + t) * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) o[i] = window[i] * idft_sample(X, tab, n, i);
    return;
  }
  for (int k = threadIdx.x; k < g.F; k += blockDim.x) {
    float2 v = e[(long long)k * sf];
    if (k == 0 || k == n / 2) v.y = 0.f;      // c2r ignores these imaginary parts
    s[bitrev(k, g.log2n)] = v;
    if (k > 0 && k < n / 2) s[bitrev(n - k, g.log2n)] = make_float2(v.x, -v.y);
  }
  block_fft(s, g.log2n, 1.f);
  float* o = frames + ((long long)b * T_used + t) * n;
  const float inv = 1.0f / (float)n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) o[i] = window[i] * (s[i].x * inv);
}

// overlap-add + window-sum-square normalisation + trim / fix_length
// (librosa.istft steps 2-4, SURVEY.md App. A), and the running peak for the
// later `norm` rescale (utils.py:166-168).  One thread per output sample.
__global__ void istft_ola_kernel(Geometry g, const float* __restrict__ frames,
                                 const float* __restrict__ wsq, int T_used, int n_out,
                                 const int* __restrict__ n_samples, float* __restrict__ wave,
                                 unsigned* __restrict__ peak) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  // a ragged batch: each utterance overlap-adds its own frames only
  const int Tu = n_samples ? imin(T_used, frames_of(n_samples[b], g.n_fft, g.hop, g.pad)) : T_used;
  float val = 0.f;
  if (q < n_out) {
    const int p = q + g.pad;
    const int expected = Tu > 0 ? g.n_fft + g.hop * (Tu - 1) : 0;
    // a ragged utterance ends where its own istft(length=None) would (center: the trailing
    // n_fft/2 is trimmed); what lies beyond is zero and must not reach the peak
    const int limit = n_samples ? expected - g.pad : expected;
    if (p < limit) {
      const int t_lo = (p >= g.n_fft) ? (p - g.n_fft) / g.hop + 1 : 0;
      const int t_hi = imin(Tu - 1, p / g.hop);
      float wss = 0.f;
      for (int t = t_lo; t <= t_hi; ++t) {
        const int n = p - t * g.hop;
        val += frames[((long long)b * T_used + t) * g.n_fft + n];
        wss += wsq[n];
      }
      if (wss > SETK_TINY32) val /= wss;
    }
    wave[(long long)b * n_out + q] = val;
  }
  if (peak) {
    float m = fabsf(val);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(peak + b, __float_as_uint(m));
  }
}

// samps * norm / (max|samps| + EPSILON)  (utils.py:166-168); norm == 0 -> skip
// ("if norm:").
__global__ void peak_scale_kernel(float* __restrict__ wave, int n_out, const float* __restrict__ norm,
                                  const unsigned* __restrict__ peak) {
  const int b = blockIdx.y;
  const float nm = norm[b];
  if (nm == 0.f) return;
  const float den = __uint_as_float(peak[b]) + SETK_EPS32;
  float* y = wave + (long long)b * n_out;
  if ((n_out & 3) == 0 && (reinterpret_cast<uintptr_t>(wave) & 15) == 0) {
    float4* y4 = reinterpret_cast<float4*>(y);
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < (n_out >> 2); q += gridDim.x * blockDim.x) {
      float4 v = y4[q];
      v.x = (v.x * nm) / den; v.y = (v.y * nm) / den; v.z = (v.z * nm) / den; v.w = (v.w * nm) / den;
      y4[q] = v;
    }
    return;
  }
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n_out; q += gridDim.x * blockDim.x)
    y[q] = (y[q] * nm) / den;
}

// The same rescale fused with write_wav's float -> PCM-16 conversion (utils.py:45-62:
// soundfile's default subtype, floor(y * 32768) clipped, SURVEY.md finding 3): the float wave
// is read once and 2 bytes per sample are written.  norm == null or norm[b] == 0: no rescale.
__global__ void peak_scale_pcm16_kernel(const float* __restrict__ wave, int n_out,
                                        const float* __restrict__ norm, const unsigned* __restrict__ peak,
                                        int16_t* __restrict__ pcm) {
  const int b = blockIdx.y;
  const float nm = norm ? norm[b] : 0.f;
  const float den = nm != 0.f ? __uint_as_float(peak[b]) + SETK_EPS32 : 1.f;
  const float* y = wave + (long long)b * n_out;
  int16_t* o = pcm + (long long)b * n_out;
  auto conv = [&](float v) {
    if (nm != 0.f) v = (v * nm) / den;
    v = floorf(v * 32768.0f);
    return (int)fminf(fmaxf(v, -32768.0f), 32767.0f);
  };
  if ((n_out & 3) == 0 && (reinterpret_cast<uintptr_t>(wave) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(pcm) & 7) == 0) {
    const float4* y4 = reinterpret_cast<const float4*>(y);
    int2* o2 = reinterpret_cast<int2*>(o);
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < (n_out >> 2); q += gridDim.x * blockDim.x) {
      const float4 v = y4[q];
      const int a0 = conv(v.x), a1 = conv(v.y), a2 = conv(v.z), a3 = conv(v.w);
      o2[q] = make_int2((a0 & 0xffff) | (a1 << 16), (a2 & 0xffff) | (a3 << 16));
    }
    return;
  }
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n_out; q += gridDim.x * blockDim.x)
    o[q] = (int16_t)conv(y[q]);
}

// max |sample| over all channels of each utterance (data_handler.py:398-400)
__global__ void maxabs_kernel(const float* __restrict__ audio, const int* __restrict__ n_samples, int C,
                              int N, unsigned* __restrict__ bits) {
  const int b = blockIdx.y;
  const int nb = n_samples ? n_samples[b] : N;
  float m = 0.f;
  for (int c = 0; c < C; ++c) {
    const float* x = audio + ((long long)b * C + c) * N;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += gridDim.x * blockDim.x)
      m = fmaxf(m, fabsf(x[i]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(bits + b, __float_as_uint(m));
}

__global__ void bits_to_float_kernel(const unsigned* __restrict__ bits, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __uint_as_float(bits[i]);
}

__global__ void float_to_pcm16_kernel(const float* __restrict__ wave, long long n, int16_t* __restrict__ pcm) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = floorf(wave[i] * 32768.0f);
  v = fminf(fmaxf(v, -32768.0f), 32767.0f);
  pcm[i] = (int16_t)v;
}

__global__ void pcm16_to_float_kernel(const int16_t* __restrict__ pcm, long long n, float* __restrict__ wave) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  wave[i] = (float)pcm[i] * (1.0f / 32768.0f);
}

// 8 samples per thread: one 16-byte load, two 16-byte stores
__global__ void pcm16_to_float_vec_kernel(const int4* __restrict__ pcm8, long long n8,
                                          float4* __restrict__ wave4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const int4 p = pcm8[i];
  const float s = 1.0f / 32768.0f;
  float4 a, b;
  a.x = (float)(short)(p.x & 0xffff) * s; a.y = (float)(short)(p.x >> 16) * s;
  a.z = (float)(short)(p.y & 0xffff) * s; a.w = (float)(short)(p.y >> 16) * s;
  b.x = (float)(short)(p.z & 0xffff) * s; b.y = (float)(short)(p.z >> 16) * s;
  b.z = (float)(short)(p.w & 0xffff) * s; b.w = (float)(short)(p.w >> 16) * s;
  wave4[2 * i] = a;
  wave4[2 * i + 1] = b;
}

// ---------------------------------------------------------------------------
// host-side launchers (called from api.cu)
// ---------------------------------------------------------------------------
cudaError_t run_stft_generic(const setk_plan* pl, const float* audio, const int* n_samples, int B,
                             int N, int T, float2* out, void* stream) {
  const Geometry& g = pl->geo;
  dim3 grid(T, g.C, B), block(imin(256, g.n_fft / 2));
  return launch(stft_generic_kernel, grid, block, (size_t)g.n_fft * sizeof(float2) * (g.log2n < 0 ? 2 : 1),
                stream, false, g,
                audio, n_samples, N, T, (const float*)pl->d_window, out);
}

cudaError_t run_cov_generic(const float2* stft, const float* mask, unsigned flags, int B, int C, int F,
                            int T, float2* R, void* stream) {
  int threads = ((C * C + 31) / 32) * 32;
  if (threads < 64) threads = 64;
  return launch(cov_generic_kernel, dim3(F, B), dim3(threads), 0, stream, false, stft, mask, flags, C,
                F, T, R);
}

cudaError_t run_apply_generic(const float2* stft, const void* w, int w_dtype, const float* post_mask,
                              int B, int C, int F, int T, float2* enh, void* stream) {
  long long n = (long long)B * F * T;
  return launch(apply_generic_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                stft, w, w_dtype, post_mask, B, C, F, T, enh);
}

cudaError_t run_istft_strided(const setk_plan* pl, const float2* enh, long long sb, long long sf,
                              long long st, int B, int T_used, int n_out, const int* n_samples,
                              float* frames_ws, float* wave, unsigned* peak, void* stream) {
  const Geometry& g = pl->geo;
  cudaError_t e = launch(istft_frames_kernel, dim3(T_used, B), dim3(imin(256, g.n_fft / 2)),
                         (size_t)g.n_fft * sizeof(float2) * (g.log2n < 0 ? 2 : 1), stream, false, g, enh,
                         sb, sf, st,
                         (const float*)pl->d_window, frames_ws, T_used);
  if (e != cudaSuccess) return e;
  return launch(istft_ola_kernel, dim3((n_out + 255) / 256, B), dim3(256), 0, stream, false, g,
                (const float*)frames_ws, (const float*)pl->d_wsq, T_used, n_out, n_samples, wave, peak);
}

cudaError_t run_istft_generic(const setk_plan* pl, const float2* enh, int B, int T, int T_used,
                              int n_out, const int* n_samples, float* frames_ws, float* wave,
                              unsigned* peak, void* stream) {
  return run_istft_strided(pl, enh, (long long)pl->geo.F * T, T, 1, B, T_used, n_out, n_samples,
                           frames_ws, wave, peak, stream);
}

cudaError_t run_peak_scale(float* wave, int B, int n_out, const float* norm, const unsigned* peak,
                           void* stream) {
  int gx = imin(64, (n_out + 255) / 256);
  return launch(peak_scale_kernel, dim3(gx, B), dim3(256), 0, stream, true, wave, n_out, norm, peak);
}

cudaError_t run_bits_to_float(const unsigned* bits, int n, float* out, void* stream) {
  return launch(bits_to_float_kernel, dim3((n + 127) / 128), dim3(128), 0, stream, true, bits, n, out);
}

cudaError_t maxabs_generic(const float* audio, const int* n_samples, int B, int C, int N, unsigned* bits,
                           float* out, void* stream) {
  cudaError_t e = launch(maxabs_kernel, dim3(imin(64, (N + 255) / 256), B), dim3(256), 0, stream, false,
                         audio, n_samples, C, N, bits);
  if (e != cudaSuccess) return e;
  return run_bits_to_float(bits, B, out, stream);
}

cudaError_t run_peak_scale_pcm16(const float* wave, int B, int n_out, const float* norm,
                                 const unsigned* peak, int16_t* pcm, void* stream) {
  int gx = (n_out / 4 + 255) / 256;
  if (gx < 1) gx = 1;
  if (gx > 64) gx = 64;
  return launch(peak_scale_pcm16_kernel, dim3(gx, B), dim3(256), 0, stream, true, wave, n_out, norm, peak,
                pcm);
}
cudaError_t run_float_to_pcm16(const float* wave, long long n, int16_t* pcm, void* stream) {
  return launch(float_to_pcm16_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                wave, n, pcm);
}
cudaError_t run_pcm16_to_float(const int16_t* pcm, long long n, float* wave, void* stream) {
  if ((n & 7) == 0 && (reinterpret_cast<uintptr_t>(pcm) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(wave) & 15) == 0) {
    const long long n8 = n >> 3;
    return launch(pcm16_to_float_vec_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, stream,
                  true, reinterpret_cast<const int4*>(pcm), n8, reinterpret_cast<float4*>(wave));
  }
  return launch(pcm16_to_float_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                pcm, n, wave);
}

}  // namespace setk
