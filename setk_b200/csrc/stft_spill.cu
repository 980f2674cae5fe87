// stft_spill.cu -- the "many channels" route of the covariance pass (C > 4):
// a fast multichannel STFT into a bin-major HBM workspace, then a covariance
// kernel that streams it.
//
// With C > 4 the per-bin accumulators of the fused kernel (2 C^2 floats per
// thread) no longer fit in registers, so the STFT is materialised once --
// written and read back at full coalescing -- and the covariance is computed
// by one thread per (bin, matrix row).  Replaces the same reference code as
// stft_cov_fused.cu (data_handler.py:492-503, beamformer.py:87-103,279-281).
//
//   stft_spill_kernel<CG,TT>, stft_spill1024_kernel<CG>  grid (chunks, channel
//       groups of <= 4, B): the chunk driver tile_stft of stft_tile.cuh, whose
//       X[k] are stored as  Xws[b][t][c][FP]  (c64, FP = 264 or 520: rows of
//       bins are contiguous, 8-byte coalesced stores);  max|x|.
//   cov_spill_kernel<C>       grid (chunks, C rows, B), thread per bin: row i
//       accumulates  sum_t m x_i conj(x_j), j >= i  for (m_s, m_n) in fp32.
//   cov_spill_finalize<C>     fixed-order sum over chunks, / max(sum m, 1e-6),
//       Hermitian fill.
// Algorithmic bytes per utterance (as for the fused kernel) 4CN + 4TF + 16FC^2;
// this route moves 2 * 8*C*F*T more (the spill), which DESIGN.md reports.
#include <cstdlib>
#include "common.cuh"
#include "stft_tile.cuh"
#include "cov_spill_args.cuh"
#include "launchers.cuh"

namespace setk {

struct StftSpillArgs : TileChunkArgs {
  float2* xws;           // [B][T][C][bin_pitch(F)]
  unsigned* maxabs_bits; // [B] or null
};
// moves a's audio and workspace on by c channels (launch_tile_chunks)
static void shift_channels(StftSpillArgs& a, int c) {
  a.audio += (long long)c * a.N;
  a.xws += (long long)c * bin_pitch(a.g.F);
}

// Both spill kernels: the tile STFT of one chunk into the workspace, zeros for the frames past the
// utterance's end, and max|x| into maxabs_bits.
template <int CG, int TT, int NFFT>
__device__ __forceinline__ void stft_spill_chunk(const StftSpillArgs& a) {
  constexpr int F = NFFT / 2 + 1, P = bin_pitch(F);
  SETK_DYN_SMEM(float, smem);
  const int hop = a.g.hop, pad = a.g.pad, C = a.g.C;
  TileSmem<CG, TT, NFFT> sm;
  sm.carve(smem, hop);
  const TileChunk ck = tile_chunk<NFFT>(a);
  float amax = 0.f;
  tile_stft(sm, a, ck, amax, [&](int t0, int j, int c, int k, float2 x) {
    a.xws[(((long long)ck.b * a.T + (t0 + j)) * C + ck.c0 + c) * P + k] = x;
  }, [](int, int) {});
  // frames past this utterance's own count (ragged batch): zeros
  for (int t = imax(ck.t_begin, ck.t_live_end); t < ck.t_end; ++t)
#pragma unroll
    for (int c = 0; c < CG; ++c)
      for (int k = threadIdx.x; k < F; k += kChunkThreads)
        a.xws[(((long long)ck.b * a.T + t) * C + ck.c0 + c) * P + k] = make_float2(0.f, 0.f);
  if (a.maxabs_bits) {
    if (blockIdx.x == gridDim.x - 1) {   // center=False tail that no frame covers
      const int covered = (ck.Tb > 0 ? (ck.Tb - 1) * hop + NFFT - 2 * pad : 0);
      const float* xb = ck.audio(a);
      for (int c = 0; c < CG; ++c)
        for (int i = imax(covered, 0) + threadIdx.x; i < ck.nb; i += blockDim.x)
          amax = fmaxf(amax, fabsf(xb[(long long)c * a.N + i]));
    }
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0 && amax > 0.f) atomicMax(a.maxabs_bits + ck.b, __float_as_uint(amax));
  }
}

template <int CG, int TT>
__global__ void __maxnreg__(96) stft_spill_kernel(StftSpillArgs a) { stft_spill_chunk<CG, TT, kNfft>(a); }

template <int CG>
__global__ void __launch_bounds__(kChunkThreads) stft_spill1024_kernel(StftSpillArgs a) {
  stft_spill_chunk<CG, 2, kNfft2>(a);   // hop % 4 == 0 (stft_spill_supported)
}

// Beamformer.beamform on the workspace (beamformer.py:220-234, optional
// post-mask apply_adaptive_beamformer.py:174-175): thread per bin, the bin's
// weights in registers, a run of frames per CTA.   Y[b][t][pitch].
struct ApplySpillArgs {
  const float2* xws; int pitch;
  const void* w; int w_dtype;
  const float* post_mask;
  int C, F, T, frames_per_chunk;
  float2* yws;
};

template <int C>
__global__ void __launch_bounds__(288) apply_spill_kernel(ApplySpillArgs a) {
  const int nbb = (a.F + blockDim.x - 1) / blockDim.x;
  const int chunk = blockIdx.x / nbb, b = blockIdx.y;
  const int bin = (blockIdx.x - chunk * nbb) * blockDim.x + threadIdx.x;
  if (bin >= a.F) return;
  float2 w[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const long long i = ((long long)b * a.F + bin) * C + c;
    if (a.w_dtype == SETK_C128) {
      const double* p = reinterpret_cast<const double*>(a.w) + 2 * i;
      w[c] = make_float2((float)p[0], (float)p[1]);
    } else {
      w[c] = reinterpret_cast<const float2*>(a.w)[i];
    }
  }
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, a.T);
  const long long pitch = a.pitch;
  for (int t = t_begin; t < t_end; ++t) {
    const float2* xt = a.xws + (((long long)b * a.T + t) * C) * pitch + bin;
    float yr = 0.f, yi = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float2 x = xt[(long long)c * pitch];
      yr += w[c].x * x.x + w[c].y * x.y;       // conj(w) x
      yi += w[c].x * x.y - w[c].y * x.x;
    }
    if (a.post_mask) {
      const float m = a.post_mask[((long long)b * a.T + t) * a.F + bin];
      yr *= m; yi *= m;
    }
    a.yws[((long long)b * a.T + t) * pitch + bin] = make_float2(yr, yi);
  }
}

// workspace [B][T][C][P] -> the API's STFT layout [B][C][F][T] (forward_stft with
// transpose=False, utils.py:96-138): 32 x 32 (t, f) tiles through shared memory
__global__ void __launch_bounds__(256) spill_to_bcft_kernel(const float2* __restrict__ xws, int P, int C,
                                                            int F, int T, float2* __restrict__ out) {
  __shared__ float2 tile[32][33];
  const int bc = blockIdx.z, b = bc / C, c = bc - b * C;
  const int t0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int t = t0 + r, f = f0 + tx;
    if (t < T && f < F) tile[r][tx] = xws[(((long long)b * T + t) * C + c) * P + f];
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int f = f0 + r, t = t0 + tx;
    if (t < T && f < F) out[(((long long)b * C + c) * F + f) * T + t] = tile[tx][r];
  }
}

template <int C>
__global__ void __launch_bounds__(288) cov_spill_kernel(CovSpillArgs a) {
  const int nbb = (a.F + blockDim.x - 1) / blockDim.x;      // bin blocks (2 when F = 513)
  const int chunk = blockIdx.x / nbb, row = blockIdx.y, b = blockIdx.z;
  const int bin = (blockIdx.x - chunk * nbb) * blockDim.x + threadIdx.x;
  const long long pitch = a.pitch;
  if (bin >= a.F) return;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(imin(t_begin + a.frames_per_chunk, a.T), Tb);
  const bool has_mn = a.mask_n != nullptr;
  const bool clip = (a.flags & SETK_F_CLIP_MASK) != 0;
  const long long m_bs = (a.flags & SETK_F_MASK_FT) ? a.T : 1;
  const long long m_ts = (a.flags & SETK_F_MASK_FT) ? 1 : a.F;
  const float* ms_p = a.mask_s + (long long)b * a.T * a.F + bin * m_bs;
  const float* mn_p = has_mn ? a.mask_n + (long long)b * a.T * a.F + bin * m_bs : nullptr;
  float2 as[C], an[C];
#pragma unroll
  for (int j = 0; j < C; ++j) { as[j] = make_float2(0.f, 0.f); an[j] = make_float2(0.f, 0.f); }
  float sum_s = 0.f, sum_n = 0.f;
  const float2* xp = a.xws + ((long long)b * a.T * C) * pitch + bin;
  for (int t = t_begin; t < t_end; ++t) {
    const float2* xt = xp + ((long long)t * C) * pitch;
    float m_s = ms_p[t * m_ts];
    if (clip) m_s = fminf(m_s, 1.0f);
    const float m_n = has_mn ? mn_p[t * m_ts] : 1.0f - m_s;
    sum_s += m_s; sum_n += m_n;
    const float2 xi = xt[(long long)row * pitch];
#pragma unroll
    for (int j = 0; j < C; ++j) {
      if (j >= row) {
        const float2 xj = xt[(long long)j * pitch];
        const float pr = xi.x * xj.x + xi.y * xj.y;      // x_i conj(x_j)
        const float pi = xi.y * xj.x - xi.x * xj.y;
        as[j].x += m_s * pr; as[j].y += m_s * pi;
        an[j].x += m_n * pr; an[j].y += m_n * pi;
      }
    }
  }
  const int W = 2 * C + 1;
  float* pp = a.partials + ((((long long)b * a.n_chunks + chunk) * C + row) * 2) * W * a.F + bin;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    pp[(long long)(2 * j) * a.F] = as[j].x;
    pp[(long long)(2 * j + 1) * a.F] = as[j].y;
    pp[(long long)(W + 2 * j) * a.F] = an[j].x;
    pp[(long long)(W + 2 * j + 1) * a.F] = an[j].y;
  }
  pp[(long long)(2 * C) * a.F] = sum_s;
  pp[(long long)(W + 2 * C) * a.F] = sum_n;
}

// thread per (b, f, row): fixed-order sum over chunks, normalise, Hermitian fill
template <int C>
__global__ void cov_spill_finalize_kernel(const float* __restrict__ partials, int B, int F, int n_chunks,
                                          float2* __restrict__ Rs, float2* __restrict__ Rn) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * F * C) return;
  const int f = (int)(idx % F);
  const int row = (int)((idx / F) % C);
  const int b = (int)(idx / ((long long)F * C));
  const int W = 2 * C + 1;
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    double acc[2 * C + 1];   // short fp32 runs are combined in double
#pragma unroll
    for (int i = 0; i < W; ++i) acc[i] = 0.0;
    for (int ch = 0; ch < n_chunks; ++ch) {
      const float* pp = partials + (((((long long)b * n_chunks + ch) * C + row) * 2 + which) * W) * F + f;
#pragma unroll
      for (int i = 0; i < W; ++i) acc[i] += pp[(long long)i * F];
    }
    const double inv = 1.0 / fmax(acc[2 * C], 1e-6);
    float2* R = (which == 0 ? Rs : Rn) + ((long long)b * F + f) * (C * C);
#pragma unroll
    for (int j = 0; j < C; ++j) {
      if (j == row) {
        R[row * C + row] = make_float2((float)(acc[2 * j] * inv), 0.f);
      } else if (j > row) {
        const float re = (float)(acc[2 * j] * inv), im = (float)(acc[2 * j + 1] * inv);
        R[row * C + j] = make_float2(re, im);
        R[j * C + row] = make_float2(re, -im);
      }
    }
  }
}

bool stft_spill_supported(const Geometry& g) {
  if (g.C < 1 || g.C > SETK_MAX_CHANNELS) return false;
  if (g.n_fft == 512) return g.hop >= 2 && g.hop <= 512 && !(g.hop & 1);
  if (g.n_fft == 1024) return g.hop >= 4 && g.hop <= 1024 && !(g.hop & 3);
  return false;
}

size_t stft_spill_bytes(const Geometry& g, int B, int T) {
  return sizeof(float2) * (size_t)B * T * g.C * bin_pitch(g.F);
}
size_t apply_spill_bytes(const Geometry& g, int B, int T) {
  return sizeof(float2) * (size_t)B * T * bin_pitch(g.F);
}

cudaError_t run_stft_spill(setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                           int n_chunks, float2* xws, unsigned* maxabs_bits, void* stream) {
  StftSpillArgs a;
  a.g = pl->geo;
  a.audio = audio; a.n_samples = n_samples; a.N = N; a.T = T;
  a.window = pl->d_window;
  a.xws = xws;
  a.maxabs_bits = maxabs_bits;
  const int hop = a.g.hop;
  const bool n1024 = a.g.n_fft == kNfft2;
  return launch_tile_chunks(a, B, n_chunks, stream, [&](auto cg) {
    constexpr int CG = decltype(cg)::value;
    if (n1024)
      return TileLaunch<StftSpillArgs>{stft_spill1024_kernel<CG>, sizeof(float) * TileSmem<CG, 2, kNfft2>::floats(hop)};
    return TileLaunch<StftSpillArgs>{stft_spill_kernel<CG, 4>, sizeof(float) * TileSmem<CG, 4>::floats(hop)};
  });
}

// C >= 5: the covariance is a real dense contraction (2C x 2C Gram blocks over T frames) and runs
// on the tensor cores (cov_mma.cu); C <= 4 keeps the CUDA-core cov_spill_kernel
static bool use_cov_mma(int C) { return C >= 5; }

// chunks of frames per utterance for the covariance pass over the workspace
int cov_spill_chunks(const setk_plan* pl, int B, int T) {
  const Geometry& g = pl->geo;
  if (use_cov_mma(g.C)) {
    // fp32 tensor-core accumulators run over the whole utterance unless the launch would leave
    // the machine empty (small batches): then cut T so that ~4 CTAs per SM exist
    const int nbb = (g.F + cov_mma_bins_per_cta(g.C) - 1) / cov_mma_bins_per_cta(g.C);
    int chunks = (4 * pl->sm_count + B * nbb - 1) / (B * nbb);
    if (chunks > 16) chunks = 16;
    if (chunks > (T + 7) / 8) chunks = (T + 7) / 8;
    return chunks < 1 ? 1 : chunks;
  }
  int chunks = stft_cov_pick_chunks(pl, B * g.C * ((g.F + 287) / 288), T);
  if (chunks < 16) chunks = 16;
  if (chunks > T) chunks = T;
  return chunks;
}

template <int C>
static cudaError_t run_cov_spill_t(const CovSpillArgs& a, int B, float2* Rs, float2* Rn, void* stream) {
  cudaError_t e;
  if constexpr (C >= 5) {
    e = run_cov_mma(a, B, stream);
  } else {
    const int nbb = (a.F + 287) / 288;
    e = launch(cov_spill_kernel<C>, dim3(a.n_chunks * nbb, C, B), dim3(288), 0, stream, true, a);
  }
  if (e != cudaSuccess) return e;
  const long long n = (long long)B * a.F * C;
  return launch(cov_spill_finalize_kernel<C>, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, stream,
                true, (const float*)a.partials, B, a.F, a.n_chunks, Rs, Rn);
}

size_t cov_spill_partial_bytes(const Geometry& g, int B, int n_chunks) {
  return sizeof(float) * cov_spill_partial_floats(g.C, g.F) * (size_t)B * n_chunks;
}

cudaError_t run_cov_spill(setk_plan* pl, const float2* xws, const float* mask_s, const float* mask_n,
                          unsigned flags, const int* n_samples, int B, int N, int T, int n_chunks,
                          float* partials, float2* Rs, float2* Rn, void* stream) {
  CovSpillArgs a;
  a.xws = xws; a.pitch = bin_pitch(pl->geo.F);
  a.mask_s = mask_s; a.mask_n = mask_n; a.flags = flags;
  a.n_samples = n_samples; a.N = N; a.g = pl->geo;
  a.T = T; a.F = pl->geo.F;
  a.n_chunks = n_chunks;
  a.frames_per_chunk = (T + n_chunks - 1) / n_chunks;
  a.partials = partials;
  switch (pl->geo.C) {
#define SETK_CASE(k) case k: return run_cov_spill_t<k>(a, B, Rs, Rn, stream);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t run_spill_to_bcft(const setk_plan* pl, const float2* xws, int B, int T, float2* out, void* stream) {
  const Geometry& g = pl->geo;
  return launch(spill_to_bcft_kernel, dim3((T + 31) / 32, (g.F + 31) / 32, B * g.C), dim3(256), 0, stream,
                false, xws, bin_pitch(g.F), g.C, g.F, T, out);
}

// y = w^H x over the workspace -> yws [B][T][pitch]
cudaError_t run_apply_spill(setk_plan* pl, const float2* xws, const void* w, int w_dtype,
                            const float* post_mask, int B, int T, float2* yws, void* stream) {
  ApplySpillArgs a;
  a.xws = xws; a.pitch = bin_pitch(pl->geo.F);
  a.w = w; a.w_dtype = w_dtype; a.post_mask = post_mask;
  a.C = pl->geo.C; a.F = pl->geo.F; a.T = T;
  const int nbb = (a.F + 287) / 288;
  int chunks = (4 * pl->sm_count + B * nbb - 1) / (B * nbb);   // ~4 CTAs per SM
  if (chunks < 1) chunks = 1;
  if (chunks > T) chunks = T;
  a.frames_per_chunk = (T + chunks - 1) / chunks;
  chunks = (T + a.frames_per_chunk - 1) / a.frames_per_chunk;
  a.yws = yws;
  const dim3 grid(chunks * nbb, B);
  switch (a.C) {
#define SETK_CASE(k) case k: return launch(apply_spill_kernel<k>, grid, dim3(288), 0, stream, true, a);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
