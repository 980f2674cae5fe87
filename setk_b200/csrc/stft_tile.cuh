// stft_tile.cuh -- the on-chip STFT of one tile of TT frames x C channels, shared by the fused
// kernels (stft_cov_fused.cu, stft_cov_ws.cu, apply_istft_fused.cu) and the chunk-grid kernels
// (stft_spill.cu, feats.cu).
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
//   fft_tile1024, bin1024 : the same for n_fft 1024 (TT = 2)
//   tile_stft  : one CTA's chunk of frames of a chunk-grid launch, staged, transformed and handed
//                to the caller's per-bin sink tile by tile; launch_tile_chunks launches such a
//                kernel over every channel group of a batch
#pragma once
#include "async_copy.cuh"
#include "common.cuh"
#include "fft16.cuh"
#include <type_traits>

namespace setk {

constexpr int kNfft = 512;      // frame size of the fused kernels
constexpr int kM = 256;         // half-size complex transform
constexpr int kBins = 257;
constexpr int kNfft2 = 1024;    // the second tile size (BASELINE config 3)
constexpr int kBins2 = 513;

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

// Shared-memory carve-up of a tile of NFFT-point frames.  An NFFT-point frame keeps NFFT / 512
// half-size spectra Z (n_fft 1024: the even and the odd samples' 512-point transforms).
template <int C, int TT, int NFFT = kNfft>
struct TileSmem {
  static constexpr int kZ = NFFT / kNfft;   // Z slots per (frame, channel)
  int Lp;            // staged samples per channel (padded to a multiple of 4)
  MBar* bar;         // [2] one per audio buffer
  float* win;        // [NFFT]  analysis window x 0.5
  float* audio0;     // [2][C][Lp] double buffered (kept as base + offset so the
                     // compiler keeps shared-memory addressing, LDS not LD)
  float2* z;         // [TT*C*kZ][SETK_ZSLOT]
  SETK_HD static int staged_len(int hop) { return ((TT - 1) * hop + NFFT + 3) & ~3; }
  SETK_HD static size_t floats(int hop) {
    return 4 + (size_t)NFFT + 2 * (size_t)C * staged_len(hop) + 2 * (size_t)TT * C * kZ * SETK_ZSLOT;
  }
  __device__ void carve(float* base, int hop) {
    Lp = staged_len(hop);
    bar = reinterpret_cast<MBar*>(base);
    win = base + 4;
    audio0 = win + NFFT;
    z = reinterpret_cast<float2*>(audio0 + 2 * C * Lp);
  }
  __device__ float* abuf(int buf) const { return audio0 + buf * (C * Lp); }
  __device__ float* end() { return reinterpret_cast<float*>(z + TT * C * kZ * SETK_ZSLOT); }
};

// True when frames [t0, t0+nt) of NFFT samples lie inside the signal and vec_ok allows 16-byte
// copies: the tile is then delivered by TMA bulk copies, else element-wise.
template <int NFFT = kNfft>
__device__ __forceinline__ bool tile_bulk_ok(int t0, int nt, int hop, int pad, int nb, bool vec_ok) {
  const int i0 = t0 * hop - pad;
  return vec_ok && i0 >= 0 && i0 + (nt - 1) * hop + NFFT <= nb;
}

// Begin staging the samples of frames [t0, t0+nt) of every channel into
// audio[buf].  Called by ALL threads (uniform).  Returns true when the tile is
// delivered asynchronously (consumers must mbar_wait on bar[buf]); false when
// it was written with ordinary stores (visible after the next __syncthreads).
template <int C, int TT, int NFFT>
__device__ __forceinline__ bool stage_tile_begin(const TileSmem<C, TT, NFFT>& sm, int buf,
                                                 const float* __restrict__ xb, int N, int nb, int t0,
                                                 int nt, int hop, int pad, bool vec_ok) {
  const int p0 = t0 * hop;                      // first padded position of the tile
  const int need = (nt - 1) * hop + NFFT;       // samples actually used
  const int i0 = p0 - pad;
  float* dst = sm.abuf(buf);
  if (tile_bulk_ok<NFFT>(t0, nt, hop, pad, nb, vec_ok)) {
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

// ---------------------------------------------------------------------------
// n_fft = 1024 (513 bins): the same tile scheme with TT = 2 frames.  A
// 1024-point real FFT is two 512-point real FFTs of the even and the odd
// samples, i.e. two half-warp jobs  z_e[m] = x[4m] + i x[4m+2],
// z_o[m] = x[4m+1] + i x[4m+3]  that share their (16-byte) shared-memory loads;
//   X[k] = E[k] + W1024^k O[k],  E[k] = conj(E[512-k]) for k > 256.
// ---------------------------------------------------------------------------
// Forward FFT of every (frame, channel) of a 1024-point tile: job = (frame, channel, parity) on one
// half-warp, all jobs in one round of 288 threads.  A dead frame (fr >= nt) transforms zeros.
template <int CG>
__device__ __forceinline__ void fft_tile1024(const TileSmem<CG, 2, kNfft2>& sm, int buf, int nt, int hop,
                                             float2 w1, float& amax) {
  constexpr int JOBS = 2 * CG * 2;
  static_assert(JOBS <= 16, "one round of half-warp jobs");
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

// ---------------------------------------------------------------------------
// Chunk grid (stft_spill.cu, feats.cu): grid (chunks, channel groups, B) of kChunkThreads-thread
// CTAs.  CTA (x, y, z) runs frames [x * frames_per_chunk, +frames_per_chunk) of the CG channels from
// 4y (counted from the launch's first channel) of utterance z, with TT = 4 frames per tile at n_fft
// 512 and 2 at 1024.
// ---------------------------------------------------------------------------
constexpr int kChunkThreads = 288;

struct TileChunkArgs {
  Geometry g;
  const float* audio; const int* n_samples; int N;
  int T;                 // frames of an N-sample utterance (rows of every output block)
  int frames_per_chunk;  // a multiple of TT
  const float* window;
};

struct TileChunk {       // one CTA's share of a chunk-grid launch
  int b, c0;             // utterance, first channel of the group
  int nb, Tb;            // the utterance's samples and frames
  int t_begin, t_end;    // the chunk's frames
  int t_live_end;        // min(t_end, Tb): frames [t_live_end, t_end) are past the utterance's end
  __device__ const float* audio(const TileChunkArgs& a) const {   // channel c0 of utterance b
    return a.audio + ((long long)b * a.g.C + c0) * a.N;
  }
};

// this CTA's chunk
template <int NFFT>
__device__ __forceinline__ TileChunk tile_chunk(const TileChunkArgs& a) {
  TileChunk ck;
  ck.b = blockIdx.z;
  ck.c0 = blockIdx.y * 4;
  ck.nb = a.n_samples ? a.n_samples[ck.b] : a.N;
  ck.Tb = frames_of(ck.nb, NFFT, a.g.hop, a.g.pad);
  ck.t_begin = blockIdx.x * a.frames_per_chunk;
  ck.t_end = imin(ck.t_begin + a.frames_per_chunk, a.T);
  ck.t_live_end = imin(ck.t_end, ck.Tb);
  return ck;
}

// All threads: the tile STFT of chunk ck, two audio buffers deep (the next tile is staged while this
// one is transformed).  For every tile of frames [t0, t0 + nt), bin(t0, j, c, k, X) runs for each
// live frame t0 + j, channel c0 + c and bin k = threadIdx.x + 288 s of this thread, then tile(t0, nt)
// runs on all threads.  amax gathers max |sample| of the frames read.
template <int CG, int TT, int NFFT, class Bin, class Tile>
__device__ __forceinline__ void tile_stft(const TileSmem<CG, TT, NFFT>& sm, const TileChunkArgs& a,
                                          const TileChunk& ck, float& amax, Bin bin, Tile tile) {
  constexpr int S = NFFT / kNfft;                       // bins per thread
  const int hop = a.g.hop, pad = a.g.pad;
  const int tid = threadIdx.x;
  for (int n = tid; n < NFFT; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
  float w1s, w1c;
  sincospif((float)(tid & 15) / 128.0f, &w1s, &w1c);
  const float2 w1 = make_float2(w1c, -w1s);
  // the split constants of this thread's bins: those of the 512-point bin kk, and at n_fft 1024
  // the fold cj = k > 256 and the twiddle wk = W1024^k
  int zk[S], zn[S];
  float2 tw[S], wk[S];
  bool cj[S];
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const int k = tid + s * kChunkThreads;
    const int kk = (S == 1 || k <= kM) ? k : kNfft - k;
    zk[s] = kk & (kM - 1); zn[s] = (kM - kk) & (kM - 1);
    tw[s] = split_twiddle(kk);
    if constexpr (S == 2) {
      cj[s] = k > kM;
      float sn, cs;
      sincospif((float)k / 512.0f, &sn, &cs);
      wk[s] = make_float2(cs, -sn);
    }
  }
  const float* xb = ck.audio(a);
  const bool vec_ok = ((a.N & 3) == 0) && ((hop & 3) == 0) && ((pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  unsigned par = 0;
  bool async_cur = false;
  if (ck.t_begin < ck.t_live_end)
    async_cur = stage_tile_begin(sm, 0, xb, a.N, ck.nb, ck.t_begin, imin(TT, ck.t_live_end - ck.t_begin),
                                 hop, pad, vec_ok);
  int buf = 0;
  for (int t0 = ck.t_begin; t0 < ck.t_live_end; t0 += TT, buf ^= 1) {
    const int nt = imin(TT, ck.t_live_end - t0);
    __syncthreads();
    bool async_next = false;
    if (t0 + TT < ck.t_live_end)
      async_next = stage_tile_begin(sm, buf ^ 1, xb, a.N, ck.nb, t0 + TT, imin(TT, ck.t_live_end - t0 - TT),
                                    hop, pad, vec_ok);
    if (async_cur) {
      mbar_wait(&sm.bar[buf], (par >> buf) & 1u);
      par ^= 1u << buf;
    }
    if constexpr (S == 1) {
      if (tid < 256) fft_tile<CG, TT>(sm, buf, nt, hop, w1, amax);   // warps 0..7
    } else {
      fft_tile1024<CG>(sm, buf, nt, hop, w1, amax);
    }
    async_cur = async_next;
    __syncthreads();
#pragma unroll
    for (int s = 0; s < S; ++s) {
      const int k = tid + s * kChunkThreads;
      if (k < NFFT / 2 + 1) {
#pragma unroll
        for (int j = 0; j < TT; ++j) {
          if (j < nt) {
#pragma unroll
            for (int c = 0; c < CG; ++c) {
              const float2* z = sm.z + (j * CG + c) * S * SETK_ZSLOT;
              float2 x;
              if constexpr (S == 1) {
                x = split_bin(z[zk[s]], z[zn[s]], tw[s]);
                if (k == 0 || k == kM) x.y = 0.f;
              } else {
                x = bin1024(z, k, zk[s], zn[s], tw[s], cj[s], wk[s]);
              }
              bin(t0, j, c, k, x);
            }
          }
        }
      }
    }
    tile(t0, nt);
  }
}

// Host: a chunk-grid kernel and its dynamic shared memory
template <class Args>
struct TileLaunch {
  void (*kernel)(Args);
  size_t smem;
};

// Host: runs a chunk-grid kernel over B utterances in n_chunks chunks of frames: one launch for the
// C / 4 groups of 4 channels, one for the group of the C % 4 left, whose arguments are moved on to
// its first channel by shift_channels(Args&, c).  pick(cg) gives the TileLaunch for groups of cg
// channels (cg a std::integral_constant).
template <class Args, class Pick>
cudaError_t launch_tile_chunks(Args a, int B, int n_chunks, void* stream, Pick pick) {
  const int TT = a.g.n_fft == kNfft2 ? 2 : 4;
  const int fpc = (a.T + n_chunks - 1) / n_chunks;
  a.frames_per_chunk = ((fpc + TT - 1) / TT) * TT;
  auto run = [&](auto cg, int group0, int groups) -> cudaError_t {
    const TileLaunch<Args> l = pick(cg);
    cudaError_t e = cudaFuncSetAttribute(l.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l.smem);
    if (e != cudaSuccess) return e;
    Args s = a;
    shift_channels(s, 4 * group0);
    return launch(l.kernel, dim3(n_chunks, groups, B), dim3(kChunkThreads), l.smem, stream, false, s);
  };
  const int full = a.g.C / 4;
  cudaError_t e = cudaSuccess;
  if (full > 0) e = run(std::integral_constant<int, 4>(), 0, full);
  if (e != cudaSuccess) return e;
  switch (a.g.C % 4) {
    case 1: return run(std::integral_constant<int, 1>(), full, 1);
    case 2: return run(std::integral_constant<int, 2>(), full, 1);
    case 3: return run(std::integral_constant<int, 3>(), full, 1);
    default: return e;
  }
}

}  // namespace setk
