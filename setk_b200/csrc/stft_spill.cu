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
//   stft_spill_kernel<CG,TT>  grid (chunks, channel groups of <= 4, B): the
//       tile STFT of stft_tile.cuh (TMA-streamed audio, half-warp FFTs),
//       split into X[k] and stored as  Xws[b][t][c][FP]  (c64, FP = 264:
//       rows of bins are contiguous, 8-byte coalesced stores);  max|x|.
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

constexpr int kSpillPitch = bin_pitch(kBins);
constexpr int kSpillPitch2 = bin_pitch(kBins2);

struct StftSpillArgs {
  Geometry g;
  const float* audio; const int* n_samples; int N;
  int T;                 // frames of an N-sample utterance (workspace leading dim)
  int frames_per_chunk, n_chunks;
  const float* window;
  float2* xws;           // [B][T][C][kSpillPitch]
  unsigned* maxabs_bits; // [B] or null
};

template <int CG, int TT>
__global__ void __maxnreg__(96) stft_spill_kernel(StftSpillArgs a) {
  SETK_DYN_SMEM(float, smem);
  const int hop = a.g.hop, pad = a.g.pad, C = a.g.C;
  TileSmem<CG, TT> sm;
  sm.carve(smem, hop);
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, chunk = blockIdx.x, c0 = blockIdx.y * 4;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, kNfft, hop, pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, a.T);   // frames >= Tb are written as zeros

  for (int n = tid; n < kNfft; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
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
            a.xws[(((long long)b * a.T + (t0 + j)) * C + c0 + c) * kSpillPitch + bin] = x;
          }
        }
      }
    }
  }
  // frames past this utterance's own count (ragged batch): zeros
  if (bin_thread) {
    for (int t = imax(t_begin, t_live_end); t < t_end; ++t)
#pragma unroll
      for (int c = 0; c < CG; ++c)
        a.xws[(((long long)b * a.T + t) * C + c0 + c) * kSpillPitch + bin] = make_float2(0.f, 0.f);
  }
  if (a.maxabs_bits) {
    if (chunk == a.n_chunks - 1) {   // center=False tail that no frame covers
      const int covered = (Tb > 0 ? (Tb - 1) * hop + kNfft - 2 * pad : 0);
      for (int c = 0; c < CG; ++c)
        for (int i = imax(covered, 0) + tid; i < nb; i += blockDim.x)
          amax = fmaxf(amax, fabsf(xb[(long long)c * a.N + i]));
    }
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if (lane == 0 && amax > 0.f) atomicMax(a.maxabs_bits + b, __float_as_uint(amax));
  }
}

template <int CG>
__global__ void __launch_bounds__(288) stft_spill1024_kernel(StftSpillArgs a) {
  SETK_DYN_SMEM(float, smem);
  constexpr int TT = Tile1024<CG>::TT, JOBS = Tile1024<CG>::JOBS;
  static_assert(JOBS <= 16, "one round of half-warp jobs");
  const int hop = a.g.hop, pad = a.g.pad, C = a.g.C;   // hop % 4 == 0 (stft_spill_supported)
  Tile1024<CG> sm;
  sm.carve(smem, hop);
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int lane16 = lane & 15, half = lane >> 4;
  const int b = blockIdx.z, chunk = blockIdx.x, c0 = blockIdx.y * 4;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, kNfft2, hop, pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, a.T);

  for (int n = tid; n < kNfft2; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
  float w1s, w1c;
  sincospif((float)lane16 / 128.0f, &w1s, &w1c);
  const float2 w1 = make_float2(w1c, -w1s);
  // this thread's bins  k = tid, tid + 288  and their constants
  int zk[2], zn[2];
  float2 tw[2], wk[2];
  bool cj[2];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int k = tid + s * 288;
    const int kk = k <= 256 ? k : 512 - k;           // bin of the 512-point halves
    cj[s] = k > 256;
    zk[s] = kk & (kM - 1); zn[s] = (kM - kk) & (kM - 1);
    tw[s] = split_twiddle(kk);
    float sn, cs;
    sincospif((float)k / 512.0f, &sn, &cs);           // W1024^k
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
              const float2* ze = sm.z + ((j * CG + c) * 2) * SETK_ZSLOT;
              const float2* zo = ze + SETK_ZSLOT;
              float2 e = split_bin(ze[zk[s]], ze[zn[s]], tw[s]);
              float2 o = split_bin(zo[zk[s]], zo[zn[s]], tw[s]);
              if (cj[s]) { e.y = -e.y; o.y = -o.y; }
              float2 x = make_float2(e.x + wk[s].x * o.x - wk[s].y * o.y,
                                     e.y + wk[s].x * o.y + wk[s].y * o.x);
              if (k == 0 || k == kNfft2 / 2) x.y = 0.f;
              a.xws[(((long long)b * a.T + (t0 + j)) * C + c0 + c) * kSpillPitch2 + k] = x;
            }
          }
        }
      }
    }
  }
  for (int s = 0; s < 2; ++s) {
    const int k = tid + s * 288;
    if (k < kBins2)
      for (int t = imax(t_begin, t_live_end); t < t_end; ++t)
#pragma unroll
        for (int c = 0; c < CG; ++c)
          a.xws[(((long long)b * a.T + t) * C + c0 + c) * kSpillPitch2 + k] = make_float2(0.f, 0.f);
  }
  if (a.maxabs_bits) {
    if (chunk == a.n_chunks - 1) {
      const int covered = (Tb > 0 ? (Tb - 1) * hop + kNfft2 - 2 * pad : 0);
      for (int c = 0; c < CG; ++c)
        for (int i = imax(covered, 0) + tid; i < nb; i += blockDim.x)
          amax = fmaxf(amax, fabsf(xb[(long long)c * a.N + i]));
    }
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if (lane == 0 && amax > 0.f) atomicMax(a.maxabs_bits + b, __float_as_uint(amax));
  }
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

// channel groups [first_group, first_group + count) of CG channels each
template <int CG>
static cudaError_t run_spill_t(StftSpillArgs a, int B, void* stream, int first_group, int count) {
  StftSpillArgs s = a;
  s.audio = a.audio + (long long)first_group * 4 * a.N;      // the kernels take c0 from blockIdx.y
  s.xws = a.xws + (long long)first_group * 4 * bin_pitch(a.g.F);
  if (a.g.n_fft == kNfft2) {
    const size_t smem = sizeof(float) * Tile1024<CG>::floats(a.g.hop);
    cudaError_t e = cudaFuncSetAttribute(stft_spill1024_kernel<CG>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return launch(stft_spill1024_kernel<CG>, dim3(a.n_chunks, count, B), dim3(288), smem, stream, false, s);
  }
  constexpr int TT = 4;
  const size_t smem = sizeof(float) * TileSmem<CG, TT>::floats(a.g.hop);
  cudaError_t e = cudaFuncSetAttribute(stft_spill_kernel<CG, TT>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch(stft_spill_kernel<CG, TT>, dim3(a.n_chunks, count, B), dim3(288), smem, stream, false, s);
}

cudaError_t run_stft_spill(setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                           int n_chunks, float2* xws, unsigned* maxabs_bits, void* stream) {
  const int TT = pl->geo.n_fft == kNfft2 ? 2 : 4;
  StftSpillArgs a;
  a.g = pl->geo;
  a.audio = audio; a.n_samples = n_samples; a.N = N; a.T = T;
  a.n_chunks = n_chunks;
  int fpc = (T + n_chunks - 1) / n_chunks;
  a.frames_per_chunk = ((fpc + TT - 1) / TT) * TT;
  a.window = pl->d_window;
  a.xws = xws;
  a.maxabs_bits = maxabs_bits;
  const int C = pl->geo.C;
  const int full = C / 4, rem = C % 4;
  cudaError_t e = cudaSuccess;
  if (full > 0) e = run_spill_t<4>(a, B, stream, 0, full);
  if (e != cudaSuccess) return e;
  switch (rem) {
    case 1: return run_spill_t<1>(a, B, stream, full, 1);
    case 2: return run_spill_t<2>(a, B, stream, full, 1);
    case 3: return run_spill_t<3>(a, B, stream, full, 1);
    default: return e;
  }
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
