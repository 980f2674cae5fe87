// simu.cu -- speech + RIR + noise mixture simulation: the reference's scripts/sptk/wav_simulate.py on the
// device, for batches of mixtures.
//
// K14a, setk_convolve: batched long linear convolution y_b[m][n] = sum_k x_b[n - k] h_b[m][k], n < n_out_b,
// by uniformly partitioned overlap-save (a frequency-domain delay line) with block P = kConvP:
//   * conv_filter_spectra_kernel: the spectrum of every P-tap partition p of every filter channel, once
//     per (problem, channel): FFT of h[pP, (p+1)P) zero-padded to 2P;
//   * conv_source_spectra_kernel: the spectrum of every 2P-sample input segment x[(j-1)P, (j+1)P), once per
//     problem and shared by its M channels;
//   * conv_output_kernel: per output block j, Y = sum_{p = 0..min(j, parts-1)} X[j - p] H[p] in that fixed
//     order, the inverse FFT, and the last P samples (the first P are the circular wrap).
// Spectra keep bins 0..P of the real signals (Hermitian symmetry gives the rest).  The FFT is one CTA's
// radix-2 over 2P complex points in shared memory with a table of exact twiddles (sincospif); the
// real input rides in the real part.  fp32 throughout and no atomics: the same call gives the same
// bits, and a problem gives the same bits alone or inside a batch.
//
// K14b, setk_simulate_mix: mixing and normalisation over a per-mixture term table (speakers, point
// noises, an isotropic noise), on one stream and without host synchronisation:
//   1. simu_power_kernel         channel-0 power of every term's image over its range, fp64, fixed-order tree;
//   2. simu_speaker_coeff_kernel coeff_snr of every speaker against the first;
//   3. simu_spk_power_kernel     P_spk partial sums of the scaled speakers' channel-0 sum, per chunk;
//   4. simu_noise_coeff_kernel   P_spk in a fixed order, coeff_snr of every noise against it;
//   5. simu_peak_kernel          max |mix| over every channel (integer-bit atomicMax of the fp64 value);
//   6. simu_write_kernel         mix, speaker references and noise reference times norm / (peak + eps).
// Every pass evaluates a sample through the same function, adding the terms in table order in fp64.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

#ifndef SETK_CONV_BLOCK
#define SETK_CONV_BLOCK 1024   // P: the block and partition length (the CPU tier also tests 64)
#endif
constexpr int ilog2_const(int n) { return n <= 1 ? 0 : 1 + ilog2_const(n / 2); }
constexpr int kConvP = SETK_CONV_BLOCK;
constexpr int kConvN = 2 * kConvP;           // FFT length
constexpr int kConvLog2N = ilog2_const(kConvN);
constexpr int kConvBins = kConvP + 1;        // stored bins of a real signal's spectrum
constexpr int kConvThreads = 256;
static_assert((kConvP & (kConvP - 1)) == 0 && kConvP >= 32 && kConvP <= 2048,
              "SETK_CONV_BLOCK must be a power of two in [32, 2048]");

constexpr int kMixThreads = 256;
constexpr int kMixChunk = 2048;              // mixture samples per CTA of the per-sample passes

int conv_block() { return kConvP; }

struct ConvArgs {
  const float* x;      // [B][Sx]
  const float* h;      // [B][M][Lh]
  float* y;            // [B][M][Ny]
  const int* len;      // [B][3]: S_b, L_b, n_out_b
  float2* X;           // [B][nblk][kConvBins]
  float2* H;           // [B][M][npart][kConvBins]
  int B, M, Sx, Lh, Ny, nblk, npart;
};

size_t conv_spectra_bytes(int B, int M, int Lh, int Ny) {
  const size_t nblk = (size_t)(Ny + kConvP - 1) / kConvP, npart = (size_t)(Lh + kConvP - 1) / kConvP;
  return up256(sizeof(float2) * kConvBins * B * nblk) + up256(sizeof(float2) * kConvBins * B * M * npart);
}

__device__ __forceinline__ int conv_bitrev(int v) { return (int)(__brev((unsigned)v) >> (32 - kConvLog2N)); }

// tw[k] = exp(-2 pi i k / N), k < N / 2 (the argument k / (N/2) is exact in float)
__device__ inline void conv_twiddles(float2* tw) {
  for (int k = threadIdx.x; k < kConvN / 2; k += blockDim.x) {
    float s, c;
    sincospif((float)k / (float)(kConvN / 2), &s, &c);
    tw[k] = make_float2(c, -s);
  }
}

// in-place radix-2 DIT FFT of kConvN points given in bit-reversed order; inverse = conjugate twiddles,
// unscaled.  Starts and ends with a barrier.
__device__ inline void conv_fft(float2* s, const float2* tw, bool inverse) {
  for (int st = 1; st <= kConvLog2N; ++st) {
    const int half = 1 << (st - 1);
    __syncthreads();
    for (int i = threadIdx.x; i < kConvN / 2; i += blockDim.x) {
      const int j = i & (half - 1);
      const int i0 = ((i >> (st - 1)) << st) + j, i1 = i0 + half;
      float2 w = tw[j << (kConvLog2N - st)];
      if (inverse) w.y = -w.y;
      const float2 t = cmul(w, s[i1]);
      const float2 u = s[i0];
      s[i0] = cadd(u, t);
      s[i1] = csub(u, t);
    }
  }
  __syncthreads();
}

// grid (nblk, B): X[b][j] = FFT of x_b[(j-1)P, (j+1)P), zero outside [0, S_b)
__global__ void __launch_bounds__(kConvThreads) conv_source_spectra_kernel(ConvArgs a) {
  SETK_DYN_SMEM(float2, s);
  float2* tw = s + kConvN;
  const int j = blockIdx.x, b = blockIdx.y;
  const int S = a.len[3 * b], nb = (a.len[3 * b + 2] + kConvP - 1) / kConvP;
  if (j >= nb) return;   // the whole CTA
  conv_twiddles(tw);
  const float* x = a.x + (size_t)b * a.Sx;
  for (int i = threadIdx.x; i < kConvN; i += blockDim.x) {
    const long long t = (long long)(j - 1) * kConvP + i;
    s[conv_bitrev(i)] = make_float2(t >= 0 && t < S ? x[t] : 0.f, 0.f);
  }
  conv_fft(s, tw, false);
  float2* X = a.X + ((size_t)b * a.nblk + j) * kConvBins;
  for (int k = threadIdx.x; k < kConvBins; k += blockDim.x) X[k] = s[k];
}

// grid (npart, M, B): H[b][m][p] = FFT of h_b[m][pP, (p+1)P) (zero past L_b) padded with P zeros
__global__ void __launch_bounds__(kConvThreads) conv_filter_spectra_kernel(ConvArgs a) {
  SETK_DYN_SMEM(float2, s);
  float2* tw = s + kConvN;
  const int p = blockIdx.x, m = blockIdx.y, b = blockIdx.z;
  const int L = a.len[3 * b + 1];
  if (p >= (L + kConvP - 1) / kConvP) return;
  conv_twiddles(tw);
  const float* h = a.h + ((size_t)b * a.M + m) * a.Lh;
  for (int i = threadIdx.x; i < kConvN; i += blockDim.x) {
    const long long t = (long long)p * kConvP + i;
    s[conv_bitrev(i)] = make_float2(i < kConvP && t < L ? h[t] : 0.f, 0.f);
  }
  conv_fft(s, tw, false);
  float2* H = a.H + (((size_t)b * a.M + m) * a.npart + p) * kConvBins;
  for (int k = threadIdx.x; k < kConvBins; k += blockDim.x) H[k] = s[k];
}

// grid (ceil(Ny / P), M, B): output block j of channel m; blocks past n_out write zeros
__global__ void __launch_bounds__(kConvThreads) conv_output_kernel(ConvArgs a) {
  SETK_DYN_SMEM(float2, s);
  float2* tw = s + kConvN;
  const int j = blockIdx.x, m = blockIdx.y, b = blockIdx.z;
  const int L = a.len[3 * b + 1], n_out = a.len[3 * b + 2];
  float* y = a.y + ((size_t)b * a.M + m) * a.Ny;
  const int n0 = j * kConvP;
  if (n0 >= n_out) {
    for (int i = threadIdx.x; i < kConvP && n0 + i < a.Ny; i += blockDim.x) y[n0 + i] = 0.f;
    return;
  }
  conv_twiddles(tw);
  const int p_hi = imin(j, (L + kConvP - 1) / kConvP - 1);
  const float2* X = a.X + (size_t)b * a.nblk * kConvBins;
  const float2* H = a.H + ((size_t)b * a.M + m) * a.npart * kConvBins;
  for (int k = threadIdx.x; k < kConvBins; k += blockDim.x) {
    float2 acc = make_float2(0.f, 0.f);
    for (int p = 0; p <= p_hi; ++p)
      acc = cmad(X[(size_t)(j - p) * kConvBins + k], H[(size_t)p * kConvBins + k], acc);
    s[conv_bitrev(k)] = acc;
    if (k > 0 && k < kConvP) s[conv_bitrev(kConvN - k)] = make_float2(acc.x, -acc.y);
  }
  conv_fft(s, tw, true);
  const float scale = 1.0f / (float)kConvN;
  for (int i = threadIdx.x; i < kConvP && n0 + i < a.Ny; i += blockDim.x)
    y[n0 + i] = n0 + i < n_out ? s[kConvP + i].x * scale : 0.f;
}

static cudaError_t conv_launch(void (*k)(ConvArgs), dim3 grid, const ConvArgs& a, void* stream) {
  const size_t smem = sizeof(float2) * (kConvN + kConvN / 2);
#ifndef SETK_EMU
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
#endif
  return launch(k, grid, dim3(kConvThreads), smem, stream, false, a);
}

cudaError_t run_convolve(const float* x, int Sx, const float* h, int Lh, int B, int M, const int* len, float* y,
                         int Ny, char* ws, void* stream) {
  ConvArgs a;
  a.x = x; a.h = h; a.y = y; a.len = len;
  a.B = B; a.M = M; a.Sx = Sx; a.Lh = Lh; a.Ny = Ny;
  a.nblk = (Ny + kConvP - 1) / kConvP;
  a.npart = (Lh + kConvP - 1) / kConvP;
  a.X = reinterpret_cast<float2*>(ws);
  a.H = reinterpret_cast<float2*>(ws + up256(sizeof(float2) * kConvBins * B * (size_t)a.nblk));
  cudaError_t e = conv_launch(conv_filter_spectra_kernel, dim3(a.npart, M, B), a, stream);
  if (e == cudaSuccess) e = conv_launch(conv_source_spectra_kernel, dim3(a.nblk, B), a, stream);
  if (e == cudaSuccess) e = conv_launch(conv_output_kernel, dim3(a.nblk, M, B), a, stream);
  return e;
}

// ---------------------------------------------------------------------------------------------------
// K14b: mixing and normalisation
// ---------------------------------------------------------------------------------------------------
struct MixArgs {
  const float* pool;
  const setk_simu_mix_t* mixes;    // [B]
  const setk_simu_term_t* terms;   // [n_terms]
  double* power;                   // [n_terms] channel-0 power of each image
  double* coeff;                   // [n_terms]
  double* partial;                 // [B][nchunk] P_spk partial sums
  unsigned long long* peak;        // [B] max |mix| as fp64 bits
  int B, n_terms, M, K, n_pitch, nchunk, pcm16;
  void* mix;                       // f32 | i16 [B][M][n_pitch]
  void* spk;                       // f32 | i16 [B][K][n_pitch] or null
  void* noise;                     // f32 | i16 [B][n_pitch] or null
  double* factor;                  // [B] or null
};

size_t simu_scratch_bytes(int B, int n_terms, int n_pitch) {
  const size_t nchunk = (size_t)(n_pitch + kMixChunk - 1) / kMixChunk;
  return up256(sizeof(setk_simu_mix_t) * B) + up256(sizeof(setk_simu_term_t) * n_terms) +
         2 * up256(sizeof(double) * n_terms) + up256(sizeof(double) * B * nchunk) +
         up256(sizeof(unsigned long long) * B);
}

// coeff_snr of wav_simulate.py:17-26: sqrt(ref / (sig 10^(snr/10) + EPSILON))
__device__ __forceinline__ double coeff_snr(double sig, double ref, double snr) {
  return sqrt(ref / (sig * pow(10.0, snr / 10.0) + SETK_EPS32_D));
}

// fixed-order tree over the CTA (kMixThreads values in red)
__device__ inline double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  for (int w = kMixThreads / 2; w > 0; w >>= 1) {
    __syncthreads();
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
  }
  __syncthreads();
  const double r = red[0];
  __syncthreads();
  return r;
}

// grid (n_terms): power[t] = mean of image channel 0 over [power_begin, power_end)
__global__ void __launch_bounds__(kMixThreads) simu_power_kernel(MixArgs a) {
  __shared__ double red[kMixThreads];
  const setk_simu_term_t t = a.terms[blockIdx.x];
  const float* img = a.pool + t.src;
  double acc = 0.0;
  for (int i = t.power_begin + (int)threadIdx.x; i < t.power_end; i += kMixThreads) {
    const double v = (double)img[i];
    acc = fma(v, v, acc);
  }
  const double sum = block_sum(acc, red);
  if (threadIdx.x == 0) a.power[blockIdx.x] = sum / (double)(t.power_end - t.power_begin);
}

// one thread per mixture: the first speaker 1, every other coeff_snr(P_k, P_0, sdr_k)  (wav_simulate.py:87-92)
__global__ void simu_speaker_coeff_kernel(MixArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const setk_simu_mix_t mx = a.mixes[b];
  const double p0 = a.power[mx.first_term];
  for (int i = 0; i < mx.n_terms; ++i) {
    const int t = mx.first_term + i;
    if (a.terms[t].kind != SETK_SIMU_SPEAKER) break;
    a.coeff[t] = i == 0 ? 1.0 : coeff_snr(a.power[t], p0, a.terms[t].level_db);
  }
}

struct MixCtx {   // a mixture's terms in shared memory
  setk_simu_term_t t[SETK_SIMU_MAX_TERMS];
  double c[SETK_SIMU_MAX_TERMS];
  int n;
};

__device__ inline void load_mix(const MixArgs& a, int b, MixCtx& ctx, bool coeffs) {
  const setk_simu_mix_t mx = a.mixes[b];
  for (int i = threadIdx.x; i < mx.n_terms; i += blockDim.x) {
    ctx.t[i] = a.terms[mx.first_term + i];
    ctx.c[i] = coeffs ? a.coeff[mx.first_term + i] : 0.0;
  }
  if (threadIdx.x == 0) ctx.n = mx.n_terms;
  __syncthreads();
}

__device__ __forceinline__ double image_at(const float* pool, const setk_simu_term_t& t, int c, int n) {
  const int i = n - t.begin;
  if (i < 0 || i >= t.length) return 0.0;
  const int ch = t.n_channels == 1 ? 0 : c;
  return (double)pool[t.src + (long long)ch * t.pitch + (t.repeat ? 0 : i)];
}

// sample n of channel c: spk = sum of the scaled speakers (sum(spk), :252), noise = sum of the scaled point
// noises (add_point_noise, :139-142) plus the isotropic term, mix = (spk + point noises) + isotropic
// (:270, :297).  Any output may be null.
__device__ inline void eval_sample(const float* pool, const MixCtx& ctx, int c, int n, double* mix, double* noise,
                                   double* spk_sum) {
  double spk = 0.0, pnoise = 0.0, iso = 0.0;
  for (int i = 0; i < ctx.n; ++i) {
    const setk_simu_term_t& t = ctx.t[i];
    const double v = ctx.c[i] * image_at(pool, t, c, n);
    if (t.kind == SETK_SIMU_SPEAKER) spk += v;
    else if (t.kind == SETK_SIMU_POINT_NOISE) pnoise += v;
    else iso = v;
  }
  if (spk_sum) *spk_sum = spk;
  if (mix) *mix = (spk + pnoise) + iso;
  if (noise) *noise = pnoise + iso;
}

// grid (nchunk, B): partial[b][chunk] = sum over the chunk of (sum_k spk_k[0][n])^2
__global__ void __launch_bounds__(kMixThreads) simu_spk_power_kernel(MixArgs a) {
  __shared__ MixCtx ctx;
  __shared__ double red[kMixThreads];
  const int b = blockIdx.y, n0 = blockIdx.x * kMixChunk;
  const int n_mix = a.mixes[b].n_samples;
  load_mix(a, b, ctx, true);
  double acc = 0.0;
  for (int n = n0 + threadIdx.x; n < imin(n0 + kMixChunk, n_mix); n += kMixThreads) {
    double s;
    eval_sample(a.pool, ctx, 0, n, nullptr, nullptr, &s);
    acc = fma(s, s, acc);
  }
  const double sum = block_sum(acc, red);
  if (threadIdx.x == 0) a.partial[(size_t)b * a.nchunk + blockIdx.x] = sum;
}

// one thread per mixture: P_spk = mean(spk_utt[0]^2) (:255), noises coeff_snr(P_noise, P_spk, snr) (:141, :296)
__global__ void simu_noise_coeff_kernel(MixArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const setk_simu_mix_t mx = a.mixes[b];
  double sum = 0.0;
  for (int c = 0; c < a.nchunk; ++c) sum += a.partial[(size_t)b * a.nchunk + c];
  const double p_spk = sum / (double)mx.n_samples;
  for (int i = 0; i < mx.n_terms; ++i) {
    const int t = mx.first_term + i;
    if (a.terms[t].kind != SETK_SIMU_SPEAKER) a.coeff[t] = coeff_snr(a.power[t], p_spk, a.terms[t].level_db);
  }
}

// grid (nchunk, B): peak[b] = max |mix| over every channel and sample (:304)
__global__ void __launch_bounds__(kMixThreads) simu_peak_kernel(MixArgs a) {
  __shared__ MixCtx ctx;
  __shared__ double red[kMixThreads];
  const int b = blockIdx.y, n0 = blockIdx.x * kMixChunk;
  const setk_simu_mix_t mx = a.mixes[b];
  load_mix(a, b, ctx, true);
  double m = 0.0;
  const int n1 = imin(n0 + kMixChunk, mx.n_samples);
  for (int n = n0 + threadIdx.x; n < n1; n += kMixThreads)
    for (int c = 0; c < mx.n_channels; ++c) {
      double v;
      eval_sample(a.pool, ctx, c, n, &v, nullptr, nullptr);
      m = fmax(m, fabs(v));
    }
  red[threadIdx.x] = m;
  for (int w = kMixThreads / 2; w > 0; w >>= 1) {
    __syncthreads();
    if ((int)threadIdx.x < w) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + w]);
  }
  // |v| >= 0: the fp64 bits order as unsigned integers
  if (threadIdx.x == 0 && red[0] > 0.0) atomicMax(a.peak + b, (unsigned long long)__double_as_longlong(red[0]));
}

__device__ __forceinline__ void put(void* base, bool pcm16, size_t i, double v) {
  const float f = (float)v;
  if (pcm16) {
    const float q = floorf(f * 32768.0f);   // write_wav's PCM-16 (setk_float_to_pcm16)
    static_cast<int16_t*>(base)[i] = (int16_t)fminf(fmaxf(q, -32768.0f), 32767.0f);
  } else {
    static_cast<float*>(base)[i] = f;
  }
}

// grid (nchunk, B): every output sample times factor = norm / (peak + EPSILON) (:304-312); zeros past the
// mixture's samples, channels and speakers
__global__ void __launch_bounds__(kMixThreads) simu_write_kernel(MixArgs a) {
  __shared__ MixCtx ctx;
  const int b = blockIdx.y, n0 = blockIdx.x * kMixChunk;
  const setk_simu_mix_t mx = a.mixes[b];
  load_mix(a, b, ctx, true);
  const double factor = mx.norm_factor / (__longlong_as_double((long long)a.peak[b]) + SETK_EPS32_D);
  if (a.factor && blockIdx.x == 0 && threadIdx.x == 0) a.factor[b] = factor;
  const bool pcm = a.pcm16 != 0;
  for (int n = n0 + threadIdx.x; n < imin(n0 + kMixChunk, a.n_pitch); n += kMixThreads) {
    const bool in = n < mx.n_samples;
    for (int c = 0; c < a.M; ++c) {
      double v = 0.0, nz = 0.0;
      if (in && c < mx.n_channels) eval_sample(a.pool, ctx, c, n, &v, &nz, nullptr);
      put(a.mix, pcm, ((size_t)b * a.M + c) * a.n_pitch + n, v * factor);
      if (c == 0 && a.noise) put(a.noise, pcm, (size_t)b * a.n_pitch + n, nz * factor);
    }
    if (!a.spk) continue;
    int k = 0;   // speaker k's channel 0, the same product as in eval_sample
    for (int i = 0; i < ctx.n && k < a.K; ++i)
      if (ctx.t[i].kind == SETK_SIMU_SPEAKER)
        put(a.spk, pcm, ((size_t)b * a.K + k++) * a.n_pitch + n,
            in ? ctx.c[i] * image_at(a.pool, ctx.t[i], 0, n) * factor : 0.0);
    for (; k < a.K; ++k) put(a.spk, pcm, ((size_t)b * a.K + k) * a.n_pitch + n, 0.0);
  }
}

cudaError_t run_simulate_mix(const float* pool, int B, int n_terms, int M, int K, int n_pitch, int pcm16,
                             char* ws, const setk_simu_mix_t* mixes_host, const setk_simu_term_t* terms_host,
                             void* mix, void* spk, void* noise, double* factor, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MixArgs a;
  a.pool = pool; a.B = B; a.n_terms = n_terms; a.M = M; a.K = K; a.n_pitch = n_pitch; a.pcm16 = pcm16;
  a.nchunk = (n_pitch + kMixChunk - 1) / kMixChunk;
  a.mix = mix; a.spk = spk; a.noise = noise; a.factor = factor;
  char* p = ws;
  a.mixes = reinterpret_cast<const setk_simu_mix_t*>(p);
  cudaError_t e = cudaMemcpyAsync(p, mixes_host, sizeof(setk_simu_mix_t) * B, cudaMemcpyHostToDevice, st);
  p += up256(sizeof(setk_simu_mix_t) * B);
  a.terms = reinterpret_cast<const setk_simu_term_t*>(p);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(p, terms_host, sizeof(setk_simu_term_t) * n_terms, cudaMemcpyHostToDevice, st);
  p += up256(sizeof(setk_simu_term_t) * n_terms);
  a.power = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * n_terms);
  a.coeff = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * n_terms);
  a.partial = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * B * (size_t)a.nchunk);
  a.peak = reinterpret_cast<unsigned long long*>(p);
  if (e == cudaSuccess) e = cudaMemsetAsync(a.peak, 0, sizeof(unsigned long long) * B, st);
  const dim3 per_b((B + 127) / 128), grid(a.nchunk, B);
  if (e == cudaSuccess) e = launch(simu_power_kernel, dim3(n_terms), dim3(kMixThreads), 0, stream, false, a);
  if (e == cudaSuccess) e = launch(simu_speaker_coeff_kernel, per_b, dim3(128), 0, stream, true, a);
  if (e == cudaSuccess) e = launch(simu_spk_power_kernel, grid, dim3(kMixThreads), 0, stream, false, a);
  if (e == cudaSuccess) e = launch(simu_noise_coeff_kernel, per_b, dim3(128), 0, stream, true, a);
  if (e == cudaSuccess) e = launch(simu_peak_kernel, grid, dim3(kMixThreads), 0, stream, false, a);
  if (e == cudaSuccess) e = launch(simu_write_kernel, grid, dim3(kMixThreads), 0, stream, false, a);
  return e;
}

}  // namespace setk
