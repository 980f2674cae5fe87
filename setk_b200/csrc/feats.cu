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
//   feats512_kernel<CG,TT>, feats1024_kernel<CG>  grid (chunks, channel groups of <= 4, B): the chunk
//       driver tile_stft of stft_tile.cuh, as the spill kernels run it, with the tail on each tile in
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

struct FeatArgs : TileChunkArgs {
  const int* mel;            // [M][4] {first bin, bins, weight offset, 0}, then the W packed weights; or null
  int M, W;
  unsigned flags; float scale;
  float* out;                // [B][C][T][D], D = M with a mel table, else F
};
// moves a's audio and output on by c channels (launch_tile_chunks)
static void shift_channels(FeatArgs& a, int c) {
  a.audio += (long long)c * a.N;
  a.out += (long long)c * a.T * (a.mel ? a.M : a.g.F);
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

// Both fused feature kernels: the tile STFT of one chunk, its features per tile through spec (shared
// memory), zero rows for the frames past the utterance's end.
template <int CG, int TT, int NFFT>
__device__ __forceinline__ void feats_chunk(const FeatArgs& a) {
  constexpr int F = NFFT / 2 + 1;
  SETK_DYN_SMEM(float, smem);
  TileSmem<CG, TT, NFFT> sm;
  sm.carve(smem, a.g.hop);
  float* spec = sm.end();                                         // [TT * CG][F]
  int* band = reinterpret_cast<int*>(spec + TT * CG * F);
  const TileChunk ck = tile_chunk<NFFT>(a);
  const bool pw = (a.flags & SETK_FEAT_POW) != 0;
  const float* w = stage_mel(a, band);
  float amax = 0.f;                                               // not used
  tile_stft(sm, a, ck, amax, [&](int, int j, int c, int k, float2 x) {
    spec[(j * CG + c) * F + k] = feat_mag(x, a.scale, pw);
  }, [&](int t0, int nt) {
    __syncthreads();
    emit_rows(a, spec, F, nt * CG, a.mel ? band : nullptr, w, [&](int r) {
      const int j = r / CG, c = r - j * CG, D = a.mel ? a.M : F;
      return a.out + (((long long)ck.b * a.g.C + ck.c0 + c) * a.T + t0 + j) * D;
    });
  });
  zero_rows(a, ck.b, ck.c0, CG, imax(ck.t_begin, ck.t_live_end), ck.t_end);
}

template <int CG, int TT>
__global__ void __launch_bounds__(kChunkThreads) feats512_kernel(FeatArgs a) { feats_chunk<CG, TT, kNfft>(a); }

template <int CG>
__global__ void __launch_bounds__(kChunkThreads) feats1024_kernel(FeatArgs a) {
  feats_chunk<CG, 2, kNfft2>(a);   // hop % 4 == 0 (stft_spill_supported)
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
  if (g.n_fft == kNfft2) return sizeof(float) * (TileSmem<CG, 2, kNfft2>::floats(g.hop) + 2 * CG * kBins2 + mel);
  return sizeof(float) * (TileSmem<CG, 4>::floats(g.hop) + 4 * CG * kBins + mel);
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
  const int groups = (g.C + 3) / 4;
  const int n_chunks = stft_cov_pick_chunks(pl, B * groups * per_cta, T);
  return launch_tile_chunks(a, B, n_chunks, stream, [&](auto cg) {
    constexpr int CG = decltype(cg)::value;
    return TileLaunch<FeatArgs>{g.n_fft == kNfft2 ? feats1024_kernel<CG> : feats512_kernel<CG, 4>,
                                feats_smem<CG>(g, mel)};
  });
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
