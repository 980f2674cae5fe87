// feats.cu -- spectral features: the magnitude / power / log spectrogram and the mel filterbank of
// every channel of a batch (forward_stft with apply_abs / apply_pow / apply_log, utils.py:96-138, as
// compute_spectrogram.py:19-40 calls it; np.dot(mel, |X|) and log(max(., EPSILON)) of
// compute_fbank.py:22-61).
//
// Per (frame, channel) the tail is
//   v = |X| * scale  (sqrt(re^2 + im^2), each step rounded as numpy does in float32)
//   v = v * v                    (SETK_FEAT_POW)
//   v = sum_k mel[m][k] v[k]     (SETK_FEAT_MEL: over the row's non-zero band only)
//   v = log(max(v, FLT_EPSILON)) (SETK_FEAT_LOG)
// written as out[b][c][t][0..D).  Frames past an utterance's own count are zero rows.
//
//   feats512_kernel<CG,TT>, feats1024_kernel<CG>  grid (chunks, channel groups of <= 4, B): the tile STFT
//       of stft_tile.cuh (TMA-staged audio, half-warp FFTs, split_bin) with the tail on the tile in
//       shared memory; the STFT never reaches HBM.  The geometries of stft_spill_supported.
//   feats_stft_kernel  grid (frame blocks, C, B): the same tail over run_stft_generic's [B][C][F][T]
//       output, for every other geometry.
// The mel band table (a [first bin, bins, offset] triple per filter) is staged in shared memory once
// per CTA, and so are its weights when they fit (kMelSmemWeights); else they are read from global.
#include "common.cuh"
#include "stft_tile.cuh"
#include "launchers.cuh"

namespace setk {

constexpr int kMelSmemWeights = 12288;   // weights staged in shared memory (48 KB) when W <= this
constexpr int kGenFrames = 8;            // frames per CTA of feats_stft_kernel

struct FeatArgs {
  Geometry g;
  const float* audio; const int* n_samples; int N;
  int T;                     // frames of an N-sample utterance (rows of every output block)
  int frames_per_chunk;
  const float* window;
  const int* mel;            // [M][4] {first bin, bins, weight offset, 0}, then the W packed weights; or null
  int M, W;
  unsigned flags; float scale;
  float* out;                // [B][C][T][D], D = M with a mel table, else F
};

// Forward FFT of every (frame, channel) of a 1024-point tile, as stft_spill1024_kernel runs it: job = (frame, channel, parity) on one
// half-warp, all JOBS in one round of 288 threads.  A dead frame (fr >= nt) transforms zeros.
template <int CG>
__device__ __forceinline__ void fft_tile1024(const Tile1024<CG>& sm, int buf, int nt, int hop, float2 w1,
                                             float& amax) {
  constexpr int JOBS = Tile1024<CG>::JOBS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lane16 = lane & 15, half = lane >> 4;
  const int job = warp * 2 + half;                  // (frame, channel, parity)
  if (job - half < JOBS) {                          // warp-uniform
    const int fr = job / (2 * CG), rem = job - fr * 2 * CG;
    const int ch = rem >> 1;                        // parity == half: both halves share the loads
    float2 v[16];
    const float* src = sm.abuf(buf) + ch * sm.Lp + fr * hop + 4 * lane16;
    const float* wsrc = sm.win + 4 * lane16;
    const bool live = fr < nt;
#pragma unroll
    for (int m1 = 0; m1 < 16; ++m1) {
      float2 x = make_float2(0.f, 0.f);
      if (live) {
        const float4 s = *reinterpret_cast<const float4*>(src + 64 * m1);
        const float4 w = *reinterpret_cast<const float4*>(wsrc + 64 * m1);
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(s.x), fabsf(s.y)), fmaxf(fabsf(s.z), fabsf(s.w))));
        x = half ? make_float2(s.y * w.y, s.w * w.w) : make_float2(s.x * w.x, s.z * w.z);
      }
      v[m1] = x;
    }
    float2* zs = sm.z + job * SETK_ZSLOT;
    halfwarp_fft256(v, zs, lane16, w1);
#pragma unroll
    for (int s = 0; s < 16; ++s) zs[lane16 + 16 * kof(s)] = v[s];
  }
}

// X[k] of a 1024-point tile from the even / odd half spectra ze, ze + SETK_ZSLOT of one (frame,
// channel): zk, zn, tw are those of the 512-point bin kk = min(k, 512 - k), cj = k > 256, wk = W1024^k
__device__ __forceinline__ float2 bin1024(const float2* ze, int k, int zk, int zn, float2 tw, bool cj,
                                          float2 wk) {
  const float2* zo = ze + SETK_ZSLOT;
  float2 e = split_bin(ze[zk], ze[zn], tw);
  float2 o = split_bin(zo[zk], zo[zn], tw);
  if (cj) { e.y = -e.y; o.y = -o.y; }
  float2 x = make_float2(e.x + wk.x * o.x - wk.y * o.y,
                         e.y + wk.x * o.y + wk.y * o.x);
  if (k == 0 || k == kNfft2 / 2) x.y = 0.f;
  return x;
}

__device__ __forceinline__ float feat_mag(float2 x, float scale, bool pw) {
  const float v = __fmul_rn(sqrtf(__fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y))), scale);
  return pw ? __fmul_rn(v, v) : v;
}

// shared-memory floats of the mel table: bands (4 ints per filter) and, when they fit, the weights
SETK_HD inline size_t mel_smem_floats(int M, int W) { return 4 * (size_t)M + (W <= kMelSmemWeights ? W : 0); }

// all threads: copy the band table (and the weights when they fit) to shared memory; returns the
// weights' base, shared or global
__device__ __forceinline__ const float* stage_mel(const FeatArgs& a, int* band) {
  if (!a.mel) return nullptr;
  for (int i = threadIdx.x; i < 4 * a.M; i += blockDim.x) band[i] = a.mel[i];
  const float* wg = reinterpret_cast<const float*>(a.mel + 4 * a.M);
  if (a.W > kMelSmemWeights) return wg;
  float* ws = reinterpret_cast<float*>(band + 4 * a.M);
  for (int i = threadIdx.x; i < a.W; i += blockDim.x) ws[i] = wg[i];
  return ws;
}

// all threads: rows [0, nrows) of spec (leading dim ld, F linear values each) -> out rows.  Row r is
// (frame r / CG, channel r % CG) of the tile; out_row(r) gives its D-float destination.
template <class OutRow>
__device__ __forceinline__ void emit_rows(const FeatArgs& a, const float* spec, int ld, int nrows,
                                          const int* band, const float* w, OutRow out_row) {
  const int D = a.mel ? a.M : a.g.F;
  const bool lg = (a.flags & SETK_FEAT_LOG) != 0;
  for (int i = threadIdx.x; i < nrows * D; i += blockDim.x) {
    const int r = i / D, d = i - r * D;
    const float* s = spec + r * ld;
    float v;
    if (band) {
      const int k0 = band[4 * d], nk = band[4 * d + 1], o = band[4 * d + 2];
      v = 0.f;
      for (int k = 0; k < nk; ++k) v = fmaf(w[o + k], s[k0 + k], v);
    } else {
      v = s[d];
    }
    if (lg) v = logf(fmaxf(v, SETK_EPS32));
    out_row(r)[d] = v;
  }
}

// zero rows [t_from, t_to) of channels [c0, c0 + cg) of utterance b
__device__ __forceinline__ void zero_rows(const FeatArgs& a, int b, int c0, int cg, int t_from, int t_to) {
  const int D = a.mel ? a.M : a.g.F;
  const int n = imax(t_to - t_from, 0) * D;
  for (int c = 0; c < cg; ++c) {
    float* o = a.out + (((long long)b * a.g.C + c0 + c) * a.T + t_from) * D;
    for (int i = threadIdx.x; i < n; i += blockDim.x) o[i] = 0.f;
  }
}

template <int CG, int TT>
__global__ void __launch_bounds__(288) feats512_kernel(FeatArgs a) {
  SETK_DYN_SMEM(float, smem);
  const int hop = a.g.hop, pad = a.g.pad, C = a.g.C;
  TileSmem<CG, TT> sm;
  sm.carve(smem, hop);
  float* spec = sm.end();                                         // [TT * CG][kBins]
  int* band = reinterpret_cast<int*>(spec + TT * CG * kBins);
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, chunk = blockIdx.x, c0 = blockIdx.y * 4;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, kNfft, hop, pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, a.T);
  const int D = a.mel ? a.M : kBins;
  const bool pw = (a.flags & SETK_FEAT_POW) != 0;

  for (int n = tid; n < kNfft; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
  const float* w = stage_mel(a, band);
  float w1s, w1c;
  sincospif((float)(lane & 15) / 128.0f, &w1s, &w1c);
  const float2 w1 = make_float2(w1c, -w1s);
  const int bin = tid;
  const bool bin_thread = bin < kBins;
  const float2 tw = split_twiddle(bin);
  const int zk = bin & (kM - 1), zn = (kM - bin) & (kM - 1);
  float amax = 0.f;
  const float* xb = a.audio + ((long long)b * C + c0) * a.N;
  const bool vec_ok = ((a.N & 3) == 0) && ((hop & 3) == 0) && ((pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  const int t_live_end = imin(t_end, Tb);
  unsigned par = 0;
  bool async_cur = false;
  if (t_begin < t_live_end)
    async_cur = stage_tile_begin<CG, TT>(sm, 0, xb, a.N, nb, t_begin, imin(TT, t_live_end - t_begin),
                                         hop, pad, vec_ok);
  int buf = 0;
  for (int t0 = t_begin; t0 < t_live_end; t0 += TT, buf ^= 1) {
    const int nt = imin(TT, t_live_end - t0);
    __syncthreads();
    bool async_next = false;
    if (t0 + TT < t_live_end)
      async_next = stage_tile_begin<CG, TT>(sm, buf ^ 1, xb, a.N, nb, t0 + TT,
                                            imin(TT, t_live_end - t0 - TT), hop, pad, vec_ok);
    if (async_cur) {
      mbar_wait(&sm.bar[buf], (par >> buf) & 1u);
      par ^= 1u << buf;
    }
    if (warp < 8) fft_tile<CG, TT>(sm, buf, nt, hop, w1, amax);
    async_cur = async_next;
    __syncthreads();
    if (bin_thread) {
#pragma unroll
      for (int j = 0; j < TT; ++j) {
        if (j < nt) {
#pragma unroll
          for (int c = 0; c < CG; ++c) {
            const float2* z = sm.z + (j * CG + c) * SETK_ZSLOT;
            float2 x = split_bin(z[zk], z[zn], tw);
            if (bin == 0 || bin == kM) x.y = 0.f;
            spec[(j * CG + c) * kBins + bin] = feat_mag(x, a.scale, pw);
          }
        }
      }
    }
    __syncthreads();
    emit_rows(a, spec, kBins, nt * CG, a.mel ? band : nullptr, w, [&](int r) {
      const int j = r / CG, c = r - j * CG;
      return a.out + (((long long)b * C + c0 + c) * a.T + t0 + j) * D;
    });
  }
  zero_rows(a, b, c0, CG, imax(t_begin, t_live_end), t_end);
}

template <int CG>
__global__ void __launch_bounds__(288) feats1024_kernel(FeatArgs a) {
  SETK_DYN_SMEM(float, smem);
  constexpr int TT = Tile1024<CG>::TT;
  static_assert(Tile1024<CG>::JOBS <= 16, "one round of half-warp jobs");
  const int hop = a.g.hop, pad = a.g.pad, C = a.g.C;   // hop % 4 == 0 (stft_spill_supported)
  Tile1024<CG> sm;
  sm.carve(smem, hop);
  float* spec = reinterpret_cast<float*>(sm.z + Tile1024<CG>::JOBS * SETK_ZSLOT);   // [TT * CG][kBins2]
  int* band = reinterpret_cast<int*>(spec + TT * CG * kBins2);
  const int tid = threadIdx.x;
  const int lane16 = tid & 15;
  const int b = blockIdx.z, chunk = blockIdx.x, c0 = blockIdx.y * 4;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, kNfft2, hop, pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, a.T);
  const int D = a.mel ? a.M : kBins2;
  const bool pw = (a.flags & SETK_FEAT_POW) != 0;

  for (int n = tid; n < kNfft2; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
  const float* w = stage_mel(a, band);
  float w1s, w1c;
  sincospif((float)lane16 / 128.0f, &w1s, &w1c);
  const float2 w1 = make_float2(w1c, -w1s);
  int zk[2], zn[2];                                   // this thread's bins  k = tid, tid + 288
  float2 tw[2], wk[2];
  bool cj[2];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int k = tid + s * 288;
    const int kk = k <= 256 ? k : 512 - k;
    cj[s] = k > 256;
    zk[s] = kk & (kM - 1); zn[s] = (kM - kk) & (kM - 1);
    tw[s] = split_twiddle(kk);
    float sn, cs;
    sincospif((float)k / 512.0f, &sn, &cs);
    wk[s] = make_float2(cs, -sn);
  }
  float amax = 0.f;
  const float* xb = a.audio + ((long long)b * C + c0) * a.N;
  const bool vec_ok = ((a.N & 3) == 0) && ((pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  const int t_live_end = imin(t_end, Tb);
  unsigned par = 0;
  bool async_cur = false;
  if (t_begin < t_live_end)
    async_cur = stage_tile1024<CG>(sm, 0, xb, a.N, nb, t_begin, imin(TT, t_live_end - t_begin), hop, pad,
                                   vec_ok);
  int buf = 0;
  for (int t0 = t_begin; t0 < t_live_end; t0 += TT, buf ^= 1) {
    const int nt = imin(TT, t_live_end - t0);
    __syncthreads();
    bool async_next = false;
    if (t0 + TT < t_live_end)
      async_next = stage_tile1024<CG>(sm, buf ^ 1, xb, a.N, nb, t0 + TT, imin(TT, t_live_end - t0 - TT),
                                      hop, pad, vec_ok);
    if (async_cur) {
      mbar_wait(&sm.bar[buf], (par >> buf) & 1u);
      par ^= 1u << buf;
    }
    fft_tile1024<CG>(sm, buf, nt, hop, w1, amax);
    async_cur = async_next;
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int k = tid + s * 288;
      if (k < kBins2) {
#pragma unroll
        for (int j = 0; j < TT; ++j) {
          if (j < nt) {
#pragma unroll
            for (int c = 0; c < CG; ++c) {
              const float2 x = bin1024(sm.z + ((j * CG + c) * 2) * SETK_ZSLOT, k, zk[s], zn[s], tw[s], cj[s],
                                       wk[s]);
              spec[(j * CG + c) * kBins2 + k] = feat_mag(x, a.scale, pw);
            }
          }
        }
      }
    }
    __syncthreads();
    emit_rows(a, spec, kBins2, nt * CG, a.mel ? band : nullptr, w, [&](int r) {
      const int j = r / CG, c = r - j * CG;
      return a.out + (((long long)b * C + c0 + c) * a.T + t0 + j) * D;
    });
  }
  zero_rows(a, b, c0, CG, imax(t_begin, t_live_end), t_end);
}

// the tail over an explicit STFT X [B][C][F][T]: kGenFrames frames of one (utterance, channel) per CTA
__global__ void __launch_bounds__(256) feats_stft_kernel(FeatArgs a, const float2* __restrict__ X) {
  SETK_DYN_SMEM(float, smem);
  const int F = a.g.F, C = a.g.C, T = a.T;
  const int t0 = blockIdx.x * kGenFrames, c = blockIdx.y, b = blockIdx.z;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad);
  const int t_blk = imin(kGenFrames, T - t0);
  const int nt = imax(imin(t_blk, Tb - t0), 0);                  // live frames of this block
  float* spec = smem;                                            // [kGenFrames][F]
  int* band = reinterpret_cast<int*>(spec + kGenFrames * F);
  const float* w = stage_mel(a, band);
  const bool pw = (a.flags & SETK_FEAT_POW) != 0;
  const float2* xs = X + ((long long)b * C + c) * F * T + t0;
  for (int i = threadIdx.x; i < F * kGenFrames; i += blockDim.x) {
    const int f = i / kGenFrames, j = i - f * kGenFrames;
    if (j < nt) spec[j * F + f] = feat_mag(xs[(long long)f * T + j], a.scale, pw);
  }
  __syncthreads();
  const int D = a.mel ? a.M : F;
  emit_rows(a, spec, F, nt, a.mel ? band : nullptr, w, [&](int r) {
    return a.out + (((long long)b * C + c) * T + t0 + r) * D;
  });
  zero_rows(a, b, c, 1, t0 + nt, t0 + t_blk);
}

bool feats_fused_supported(const Geometry& g) { return stft_spill_supported(g); }

// dynamic shared memory of a fused CTA of CG channels with `mel` floats of mel table
template <int CG>
static size_t feats_smem(const Geometry& g, size_t mel) {
  if (g.n_fft == kNfft2) return sizeof(float) * (Tile1024<CG>::floats(g.hop) + Tile1024<CG>::TT * CG * kBins2 + mel);
  return sizeof(float) * (TileSmem<CG, 4>::floats(g.hop) + 4 * CG * kBins + mel);
}

template <int CG>
static cudaError_t run_feats_t(FeatArgs a, int B, int n_chunks, void* stream, int first_group, int count) {
  FeatArgs s = a;
  s.audio = a.audio + (long long)first_group * 4 * a.N;     // the kernels take c0 from blockIdx.y
  s.out = a.out + (long long)first_group * 4 * a.T * (a.mel ? a.M : a.g.F);
  const size_t smem = feats_smem<CG>(a.g, a.mel ? mel_smem_floats(a.M, a.W) : 0);
  if (a.g.n_fft == kNfft2) {
    cudaError_t e = cudaFuncSetAttribute(feats1024_kernel<CG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
    return launch(feats1024_kernel<CG>, dim3(n_chunks, count, B), dim3(288), smem, stream, false, s);
  }
  cudaError_t e = cudaFuncSetAttribute(feats512_kernel<CG, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  return launch(feats512_kernel<CG, 4>, dim3(n_chunks, count, B), dim3(288), smem, stream, false, s);
}

cudaError_t run_feats_fused(const setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                            unsigned flags, float scale, float* out, void* stream) {
  const Geometry& g = pl->geo;
  FeatArgs a;
  a.g = g;
  a.audio = audio; a.n_samples = n_samples; a.N = N; a.T = T;
  a.window = pl->d_window;
  a.mel = (flags & SETK_FEAT_MEL) ? pl->d_mel : nullptr;
  a.M = pl->num_mel; a.W = pl->mel_weights;
  a.flags = flags; a.scale = scale;
  a.out = out;
  // stft_cov_pick_chunks sizes the grid for 2 CTAs per SM.  A CTA whose shared memory leaves room for only
  // one (a large mel table staged: sm_90 has 228 KB per SM, 1 KB of it reserved per CTA) counts twice.
  const size_t mel = a.mel ? mel_smem_floats(a.M, a.W) : 0;
  size_t smem;
  switch (imin(g.C, 4)) {
    case 1: smem = feats_smem<1>(g, mel); break;
    case 2: smem = feats_smem<2>(g, mel); break;
    case 3: smem = feats_smem<3>(g, mel); break;
    default: smem = feats_smem<4>(g, mel); break;
  }
  const int per_cta = 2 * (smem + 1024) > 228 * 1024 ? 2 : 1;
  const int TT = g.n_fft == kNfft2 ? 2 : 4;
  const int groups = (g.C + 3) / 4;
  const int n_chunks = stft_cov_pick_chunks(pl, B * groups * per_cta, T);
  const int fpc = (T + n_chunks - 1) / n_chunks;
  a.frames_per_chunk = ((fpc + TT - 1) / TT) * TT;
  const int full = g.C / 4, rem = g.C % 4;
  cudaError_t e = cudaSuccess;
  if (full > 0) e = run_feats_t<4>(a, B, n_chunks, stream, 0, full);
  if (e != cudaSuccess) return e;
  switch (rem) {
    case 1: return run_feats_t<1>(a, B, n_chunks, stream, full, 1);
    case 2: return run_feats_t<2>(a, B, n_chunks, stream, full, 1);
    case 3: return run_feats_t<3>(a, B, n_chunks, stream, full, 1);
    default: return e;
  }
}

cudaError_t run_feats_stft(const setk_plan* pl, const float2* stft, const int* n_samples, int B, int N, int T,
                           unsigned flags, float scale, float* out, void* stream) {
  const Geometry& g = pl->geo;
  FeatArgs a;
  a.g = g;
  a.audio = nullptr; a.n_samples = n_samples; a.N = N; a.T = T;
  a.frames_per_chunk = kGenFrames;
  a.window = nullptr;
  a.mel = (flags & SETK_FEAT_MEL) ? pl->d_mel : nullptr;
  a.M = pl->num_mel; a.W = pl->mel_weights;
  a.flags = flags; a.scale = scale;
  a.out = out;
  const size_t smem = sizeof(float) * ((size_t)kGenFrames * g.F + (a.mel ? mel_smem_floats(a.M, a.W) : 0));
  cudaError_t e = cudaFuncSetAttribute(feats_stft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch(feats_stft_kernel, dim3((T + kGenFrames - 1) / kGenFrames, g.C, B), dim3(256), smem, stream, false,
                a, stft);
}

}  // namespace setk
