// stft_tile.cuh -- the on-chip STFT of one tile of TT frames x C channels,
// shared by the two fused kernels (stft_cov_fused.cu, apply_istft_fused.cu).
//
//   stage_tile_begin : audio (global, f32 [C][N]) -> shared.  Interior tiles are
//                streamed by TMA 1-D bulk copies (one elected thread, completion
//                on an mbarrier) into one of two buffers, one tile ahead of the
//                math; tiles that touch librosa's center=True reflect padding
//                (np.pad(y, n_fft//2, "reflect"), SURVEY.md App. A step 2) or a
//                ragged end are written element-wise.
//   fft_tile   : 512-point real FFT of every (frame, channel) as a 256-point
//                complex FFT on one half-warp (fft16.cuh); the *unsplit*
//                half-size spectrum Z stays in shared memory
//   split_bin  : X[k] (and X[256-k]) from Z[k], Z[256-k] with the bin's
//                constant twiddle
//   Tile1024, stage_tile1024 : the 1024-point tile of stft_spill.cu and feats.cu
#pragma once
#include "async_copy.cuh"
#include "common.cuh"
#include "fft16.cuh"

namespace setk {

constexpr int kNfft = 512;      // frame size of the fused kernels
constexpr int kM = 256;         // half-size complex transform
constexpr int kBins = 257;

// ---------------------------------------------------------------------------
// Balanced persistent schedule.  The work of a launch is the sequence of
// (utterance, tile) pairs, utterance-major; every utterance has >= 1 tile (a
// too-short one gets an empty tile so that its outputs are still initialised).
// CTA g of G owns the tiles [g*q, (g+1)*q) of that sequence, q = the quota
// below: all CTAs carry the same load (no last partial wave, which cost 14 % at
// 256 utterances on 296 CTA slots) and an utterance is cut only where a CTA
// range ends.  q >= min_quota bounds how many CTAs can share one utterance.
// ---------------------------------------------------------------------------
struct TileSched {
  const int* prefix;   // [B+1] tiles before utterance b (ragged batch), or null
  int tiles_u;         // tiles of every utterance when prefix == null
  int B;
  int min_quota;       // lower bound of q
};
SETK_HD inline int sched_tiles_of(int frames, int TT) { return frames > 0 ? (frames + TT - 1) / TT : 1; }
__device__ __forceinline__ int sched_prefix(const TileSched& s, int b) {
  return s.prefix ? s.prefix[b] : b * s.tiles_u;
}
__device__ __forceinline__ int sched_quota(const TileSched& s, int n_ctas) {
  const int total = sched_prefix(s, s.B);
  return imax((total + n_ctas - 1) / n_ctas, imax(s.min_quota, 1));
}
// utterance that holds tile x (0 <= x < total)
__device__ __forceinline__ int sched_find(const TileSched& s, int x) {
  if (!s.prefix) return x / s.tiles_u;
  int lo = 0, hi = s.B;                 // prefix[lo] <= x < prefix[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (s.prefix[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}
// slots of per-utterance partial results a launch with n_ctas CTA slots needs
SETK_HD inline int sched_slots(int n_ctas, int B) {
  int s = (n_ctas + B - 1) / B + 3;
  return s < 4 ? 4 : (s > 18 ? 18 : s);
}
SETK_HD inline int sched_min_quota(int tiles_max, int slots) { return (tiles_max + slots - 3) / (slots - 2); }
// CTAs to launch for at most total_max tiles
SETK_HD inline int sched_grid(int total_max, int n_ctas, int min_quota) {
  int q = (total_max + n_ctas - 1) / n_ctas;
  if (q < min_quota) q = min_quota;
  if (q < 1) q = 1;
  return (total_max + q - 1) / q;
}

// Shared-memory carve-up common to both fused kernels.
template <int C, int TT>
struct TileSmem {
  int Lp;            // staged samples per channel (padded to a multiple of 4)
  MBar* bar;         // [2] one per audio buffer
  float* win;        // [512]  analysis window x 0.5
  float* audio0;     // [2][C][Lp] double buffered (kept as base + offset so the
                     // compiler keeps shared-memory addressing, LDS not LD)
  float2* z;         // [TT*C][SETK_ZSLOT]
  SETK_HD static int staged_len(int hop) { return ((TT - 1) * hop + kNfft + 3) & ~3; }
  SETK_HD static size_t floats(int hop) {
    return 4 + (size_t)kNfft + 2 * (size_t)C * staged_len(hop) + 2 * (size_t)TT * C * SETK_ZSLOT;
  }
  __device__ void carve(float* base, int hop) {
    Lp = staged_len(hop);
    bar = reinterpret_cast<MBar*>(base);
    win = base + 4;
    audio0 = win + kNfft;
    z = reinterpret_cast<float2*>(audio0 + 2 * C * Lp);
  }
  __device__ float* abuf(int buf) const { return audio0 + buf * (C * Lp); }
  __device__ float* end() { return reinterpret_cast<float*>(z + TT * C * SETK_ZSLOT); }
};

// Begin staging the samples of frames [t0, t0+nt) of every channel into
// audio[buf].  Called by ALL threads (uniform).  Returns true when the tile is
// delivered asynchronously (consumers must mbar_wait on bar[buf]); false when
// it was written with ordinary stores (visible after the next __syncthreads).
template <int C, int TT>
__device__ __forceinline__ bool stage_tile_begin(const TileSmem<C, TT>& sm, int buf,
                                                 const float* __restrict__ xb, int N, int nb, int t0,
                                                 int nt, int hop, int pad, bool vec_ok) {
  const int p0 = t0 * hop;                      // first padded position of the tile
  const int need = (nt - 1) * hop + kNfft;      // samples actually used
  const int i0 = p0 - pad;
  float* dst = sm.abuf(buf);
  if (vec_ok && i0 >= 0 && i0 + need <= nb) {
    if (threadIdx.x == 0) {
      fence_proxy_async();
      mbar_expect_tx(&sm.bar[buf], (unsigned)(C * need * sizeof(float)));
#pragma unroll
      for (int c = 0; c < C; ++c)
        bulk_g2s(dst + c * sm.Lp, xb + (long long)c * N + i0, (unsigned)(need * sizeof(float)),
                 &sm.bar[buf]);
    }
    return true;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float* src = xb + (long long)c * N;
    for (int q = threadIdx.x; q < need; q += blockDim.x) {
      const int i = pad ? reflect_index(p0 + q, pad, nb) : (p0 + q);
      dst[c * sm.Lp + q] = src[i];
    }
  }
  return false;
}

// The same decision and the two delivery paths as separate pieces, for kernels
// that give the bulk-copy issue to one producer warp.
__device__ __forceinline__ bool tile_bulk_ok(int t0, int nt, int hop, int pad, int nb, bool vec_ok) {
  const int i0 = t0 * hop - pad;
  return vec_ok && i0 >= 0 && i0 + (nt - 1) * hop + kNfft <= nb;
}
template <int C, int TT>
__device__ __forceinline__ void stage_tile_bulk(const TileSmem<C, TT>& sm, int buf,
                                                const float* __restrict__ xb, int N, int t0, int nt,
                                                int hop, int pad) {   // ONE thread
  const int need = (nt - 1) * hop + kNfft;
  const int i0 = t0 * hop - pad;
  float* dst = sm.abuf(buf);
  fence_proxy_async();
  mbar_expect_tx(&sm.bar[buf], (unsigned)(C * need * sizeof(float)));
#pragma unroll
  for (int c = 0; c < C; ++c)
    bulk_g2s(dst + c * sm.Lp, xb + (long long)c * N + i0, (unsigned)(need * sizeof(float)),
             &sm.bar[buf]);
}
template <int C, int TT>
__device__ __forceinline__ void stage_tile_scalar(const TileSmem<C, TT>& sm, int buf,
                                                  const float* __restrict__ xb, int N, int nb, int t0,
                                                  int nt, int hop, int pad) {   // ALL threads
  const int p0 = t0 * hop;
  const int need = (nt - 1) * hop + kNfft;
  float* dst = sm.abuf(buf);
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float* src = xb + (long long)c * N;
    for (int q = threadIdx.x; q < need; q += blockDim.x) {
      const int i = pad ? reflect_index(p0 + q, pad, nb) : (p0 + q);
      dst[c * sm.Lp + q] = src[i];
    }
  }
}

// Forward FFT of every (frame, channel) of the tile by warps 0..NW-1, reading
// audio[buf].  All threads of those warps must call it; hop must be even.
// amax accumulates max |sample| of everything the tile reads.
template <int C, int TT, bool TAB = false, int NW = 8>
__device__ __forceinline__ void fft_tile(const TileSmem<C, TT>& sm, int buf, int nt, int hop,
                                         float2 w1, float& amax, const float2* twtab = nullptr) {
  constexpr int JOBS = TT * C;
  static_assert(JOBS % 2 == 0, "half-warp jobs must pair up per warp");
  constexpr int ROUNDS = (JOBS + 2 * NW - 1) / (2 * NW);       // warps 0..NW-1 call this
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lane16 = lane & 15, half = lane >> 4;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    const int job = r * (2 * NW) + warp * 2 + half;
    if (job - half < JOBS) {                    // warp-uniform
      const int fr = job / C, ch = job - fr * C;
      // a dead frame (fr >= nt, only in an utterance's last tile) re-transforms the last live one:
      // its spectrum is never read, max|x| sees nothing new, and every tile runs ONE straight-line
      // path -- no zero-fill branch, no second instantiation whose rounding could differ
      const int fr_src = imin(fr, nt - 1);
      float2 v[16];
      const float* src = sm.abuf(buf) + ch * sm.Lp + fr_src * hop + 2 * lane16;
      const float* wsrc = sm.win + 2 * lane16;
      float2* zs = sm.z + job * SETK_ZSLOT;
#pragma unroll
      for (int m1 = 0; m1 < 16; ++m1) {
        const float2 s = *reinterpret_cast<const float2*>(src + 32 * m1);
        const float2 w = *reinterpret_cast<const float2*>(wsrc + 32 * m1);
        amax = fmaxf(amax, fmaxf(fabsf(s.x), fabsf(s.y)));
        v[m1] = f2mul(s, w);
      }
      halfwarp_fft256<TAB>(v, zs, lane16, w1, twtab);
#pragma unroll
      for (int s = 0; s < 16; ++s) zs[lane16 + 16 * kof(s)] = v[s];
    }
  }
}

// Twiddle of bin k for the real-FFT split: -i W512^k = (-sin t, -cos t), t = 2 pi k / 512.
__device__ __forceinline__ float2 split_twiddle(int k) {
  float s, c;
  sincospif((float)k / 256.0f, &s, &c);
  return make_float2(-s, -c);
}

// X[k] from the half-size spectrum (Z was computed from samples x 0.5):
//   X[k] = (Zk + conj(Zn)) + (-i W^k)(Zk - conj(Zn)),  Zn = Z[(256-k) & 255]
__device__ __forceinline__ float2 split_bin(float2 zk, float2 zn, float2 tw) {
  const float2 cn = make_float2(zn.x, -zn.y);               // conj(Zn): an operand modifier
  return cmad(f2sub(zk, cn), tw, f2add(zk, cn));            // E + tw D
}
// the mirrored bin from the same pair: X[256-k] = conj(E - P), P = (-iW^k) D
__device__ __forceinline__ void split_pair(float2 zk, float2 zn, float2 tw, float2& xk, float2& xm) {
  const float2 cn = make_float2(zn.x, -zn.y);
  const float2 e = f2add(zk, cn);
  const float2 p = cmul(f2sub(zk, cn), tw);
  xk = f2add(e, p);
  const float2 m = f2sub(e, p);
  xm = make_float2(m.x, -m.y);
}

constexpr int kNfft2 = 1024;       // the second tile size (BASELINE config 3)
constexpr int kBins2 = 513;

// ---------------------------------------------------------------------------
// n_fft = 1024 (513 bins): the same tile scheme with TT = 2 frames.  A
// 1024-point real FFT is two 512-point real FFTs of the even and the odd
// samples, i.e. two half-warp jobs  z_e[m] = x[4m] + i x[4m+2],
// z_o[m] = x[4m+1] + i x[4m+3]  that share their (16-byte) shared-memory loads;
//   X[k] = E[k] + W1024^k O[k],  E[k] = conj(E[512-k]) for k > 256.
// ---------------------------------------------------------------------------
template <int CG>
struct Tile1024 {
  static constexpr int TT = 2;
  static constexpr int JOBS = TT * CG * 2;
  int Lp; MBar* bar; float* win; float* audio0; float2* z;
  SETK_HD static int staged_len(int hop) { return ((TT - 1) * hop + kNfft2 + 3) & ~3; }
  SETK_HD static size_t floats(int hop) {
    return 4 + (size_t)kNfft2 + 2 * (size_t)CG * staged_len(hop) + 2 * (size_t)JOBS * SETK_ZSLOT;
  }
  __device__ void carve(float* base, int hop) {
    Lp = staged_len(hop);
    bar = reinterpret_cast<MBar*>(base);
    win = base + 4;
    audio0 = win + kNfft2;
    z = reinterpret_cast<float2*>(audio0 + 2 * CG * Lp);
  }
  __device__ float* abuf(int buf) const { return audio0 + buf * (CG * Lp); }
};

// all threads; true -> delivered by TMA on bar[buf]
template <int CG>
__device__ __forceinline__ bool stage_tile1024(const Tile1024<CG>& sm, int buf, const float* __restrict__ xb,
                                               int N, int nb, int t0, int nt, int hop, int pad, bool vec_ok) {
  const int p0 = t0 * hop;
  const int need = (nt - 1) * hop + kNfft2;
  const int i0 = p0 - pad;
  float* dst = sm.abuf(buf);
  if (vec_ok && i0 >= 0 && i0 + need <= nb) {
    if (threadIdx.x == 0) {
      fence_proxy_async();
      mbar_expect_tx(&sm.bar[buf], (unsigned)(CG * need * sizeof(float)));
#pragma unroll
      for (int c = 0; c < CG; ++c)
        bulk_g2s(dst + c * sm.Lp, xb + (long long)c * N + i0, (unsigned)(need * sizeof(float)),
                 &sm.bar[buf]);
    }
    return true;
  }
#pragma unroll
  for (int c = 0; c < CG; ++c) {
    const float* src = xb + (long long)c * N;
    for (int q = threadIdx.x; q < need; q += blockDim.x) {
      const int i = pad ? reflect_index(p0 + q, pad, nb) : (p0 + q);
      dst[c * sm.Lp + q] = src[i];
    }
  }
  return false;
}

}  // namespace setk
