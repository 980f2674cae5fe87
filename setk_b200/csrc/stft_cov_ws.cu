// stft_cov_ws.cu -- THE METRIC KERNEL, warp-specialised build (round 2): multichannel
// STFT fused with the mask-weighted spatial covariance; the STFT never touches HBM.
//
// Replaces (scripts/sptk): SpectrogramReader._load (libs/data_handler.py:492-503,
// forward_stft per channel, libs/utils.py:96-138 -> librosa.stft) followed by
// SupervisedBeamformer.run's two compute_covar calls (libs/beamformer.py:279-281,
// 87-103); C++ twin: ShortTimeFTComputer::Compute (include/stft.cc:28-66) +
// EstimatePsd (include/beamformer.cc:91-120).
//
// Same maths, schedule (TileSched) and outputs as stft_cov_fused.cu; what changed is who
// does what.  There every thread carried the FFT's 32 values AND 34 covariance
// accumulators (96 registers, 20 warps / SM) and the two phases alternated behind two
// CTA-wide barriers per tile.  Here the roles live in different warps with their own
// register budgets (setmaxnreg) and meet only through a ring of Z tiles:
//
//   384 threads = 8 FFT warps (64 registers) + 4 covariance warps (112 registers, the
//   highest warp ids: the issue arbiter favours them and they are the critical role);
//   launched at 80 registers ⇒ two CTAs per SM (24 warps)
//   tile = 16 half-warp FFT jobs = TT frames x C channels (C = 4: 4 frames)
//
//   FFT warps   wait audio tile (TMA bulk copy, mbarrier) -> 16 samples x window per lane
//               -> named barrier among the FFT warps (the single audio buffer is free:
//               one thread issues the bulk copy of the NEXT tile) -> first radix-16 pass +
//               twiddles in registers -> wait z_empty[slot] -> exchange + second pass in
//               the slot itself -> Z -> arrive z_full[slot]
//   masks       the TT mask rows of a tile are one contiguous run of a [B][T][F] array: the
//               FFT warps' elected thread fetches them with ONE bulk copy per tile (rounded
//               out to 16-byte boundaries) that completes on z_full[slot] together with the
//               Z tile -- no per-thread cp.async, no address arithmetic in the covariance
//               warps.  (F,T)-layout masks, unaligned arrays and an utterance's last,
//               partial tile are read by the covariance threads with plain loads instead.
//   cov warps   thread k owns the bin PAIR (k, 256-k), k = 0..127 (k = 0: DC and Nyquist):
//               one split serves both bins and every Z value is read once.  Per tile:
//               wait z_full[slot], TT rank-1 updates of 2 x (Rs, Rn) upper triangles in 68
//               fp32 registers, arrive z_empty[slot].  The 129th job -- bin 128, its own mirror -- goes to lanes
//               0..TT-1 (one frame each) of cov warp (tile mod 4); its accumulators live in
//               shared memory, one row per (warp, lane), summed in fixed order at the end.
//   end of an utterance's run: partial sums -> workspace [B][slot][acc][F], reduced by
//   cov_finalize_kernel exactly as before (deterministic, no float atomics).
//
// Algorithmic bytes per utterance: 4*C*N + 4*T*F (+4*T*F with mask_n) + 2*8*F*C^2.
#include "common.cuh"
#include "stft_tile.cuh"
#include "stft_cov_args.cuh"
#include "launchers.cuh"

namespace setk {

// Register budgets.  The CTA's pool is what it was launched with (80 x 384 = 30 720, two
// CTAs per SM); after the re-budgeting 8 x 32 x 64 + 4 x 32 x 112 = 30 720 exactly.
constexpr int kWsFftRegs = 64, kWsCovRegs = 112;
#define SETK_WS_LAUNCH_REGS 80
constexpr int kWsCovThreads = 128, kWsFftThreads = 256, kWsThreads = 384;
constexpr int kWsBarFft = 1, kWsBarCov = 2;   // named barriers (0 is __syncthreads)
#ifndef SETK_TABLE_CHUNK
#define SETK_TABLE_CHUNK 128       // tile descriptors per table fill (the CPU test tier builds with 8)
#endif
constexpr int kWsChunk = SETK_TABLE_CHUNK;
constexpr int kWsMaskRegion = 1036;           // floats of one mask tile in shared memory: 4 x 257 rounded
                                              // out to 16-byte boundaries at both ends (<= 1032), padded

template <int C>
struct WsShape {
  static_assert(16 % C == 0, "16 half-warp jobs per tile");
  static constexpr int TT = 16 / C;                 // frames per tile
  static constexpr int NOFF = C * (C - 1) / 2;
  static constexpr int NACC = C * C;
  static constexpr int NPAIR = C + 2 * NOFF + 1;    // float2 accumulators of one bin
  static constexpr int ROWS128 = 4 * TT;            // (cov warp, lane) rows of bin 128
};

// What the two roles need to know about one tile of the CTA's run, computed once per tile by
// one thread (table fill) instead of by every thread of both roles on every tile.
enum : unsigned {
  WS_NT = 0xfu,               // live frames (0 for the empty tile of a too-short utterance)
  WS_AUDIO_BULK = 1u << 4,    // samples arrive by bulk copy (else element-wise: reflect padding, ragged end)
  WS_MASK_BULK = 1u << 5,     // mask rows arrive by bulk copy (else plain loads in the covariance warps)
  WS_SEG_BEGIN = 1u << 6,     // first tile of an utterance's part of this CTA's run: accumulators restart
  WS_SEG_END = 1u << 7,       // last tile of that part: partial sums and max|x| are flushed
  WS_UTT_END = 1u << 8,       // ... and it is also the utterance's last tile
  WS_SHIFT_POS = 9,           // 2 bits: floats between the 16-byte aligned mask copy and frame t0, bin 0
  WS_SLOT_POS = 16            // 8 bits: partial-sum slot of this CTA for the utterance
};
struct alignas(16) WsTile { int b, t0, nb; unsigned flags; };

// Shared-memory carve-up (C = 4, hop 256: 110 960 B, 115 104 B with mask_n rows).
template <int C>
struct WsSmem {
  static constexpr int TT = WsShape<C>::TT;
  WsTile* tiles;     // [kWsChunk + 1]
  MBar* bar_audio;   // [1]  bulk copy of the audio tile
  MBar* z_full;      // [2]  8 arrivals: one per FFT warp
  MBar* z_empty;     // [2]  4 arrivals: one per covariance warp
  float* win;        // [512] analysis window x 0.5
  float2* twtab;     // [256] W256^{lane16 k}
  float* audio;      // [C][Lp]
  float2* z;         // [2][16][SETK_ZSLOT]
  float* mask;       // [mslots][mrows][kWsMaskRegion], mslots = 3 (2 with mask_n rows)
  float2* acc128;    // [ROWS128][NPAIR]
  int Lp, mrows;
  SETK_HD static int staged_len(int hop) { return ((TT - 1) * hop + kNfft + 3) & ~3; }
  SETK_HD static int mask_slots(int mrows) { return mrows > 1 ? 2 : 3; }
  SETK_HD static size_t bytes(int hop, int mrows) {
    return 64 + sizeof(WsTile) * (kWsChunk + 2) + sizeof(float) * kNfft + sizeof(float2) * 256 +
           sizeof(float) * C * staged_len(hop) + sizeof(float2) * 2 * 16 * SETK_ZSLOT +
           sizeof(float) * mask_slots(mrows) * mrows * kWsMaskRegion +
           sizeof(float2) * WsShape<C>::ROWS128 * WsShape<C>::NPAIR;
  }
  __device__ void carve(float* base, int hop, int mrows_) {
    Lp = staged_len(hop);
    mrows = mrows_;
    MBar* bars = reinterpret_cast<MBar*>(base);
    bar_audio = bars; z_full = bars + 1; z_empty = bars + 3;
    tiles = reinterpret_cast<WsTile*>(base + 16);
    win = base + 16 + 4 * (kWsChunk + 2);
    twtab = reinterpret_cast<float2*>(win + kNfft);
    audio = reinterpret_cast<float*>(twtab + 256);
    z = reinterpret_cast<float2*>(audio + C * Lp);
    mask = reinterpret_cast<float*>(z + 2 * 16 * SETK_ZSLOT);
    acc128 = reinterpret_cast<float2*>(mask + mask_slots(mrows) * mrows * kWsMaskRegion);
  }
};

// Can the TT mask rows of tile (b, frames t0..) arrive as one bulk copy?  They are TT * F
// consecutive floats of a [B][T][F] array starting at float index `first`; the copy starts at
// the 16-byte boundary below (`shift` floats earlier) and ends at the one above, which must
// still lie inside the array.
__device__ __forceinline__ bool ws_mask_bulk(const StftCovArgs& a, int b, int t0, int nt, int TT,
                                             long long& first, int& shift) {
  first = ((long long)b * a.T + t0) * kBins;
  shift = (int)(first & 3);
  if (nt != TT || (a.flags & SETK_F_MASK_FT)) return false;
  if ((reinterpret_cast<uintptr_t>(a.mask_s) & 15) ||
      (a.mask_n && (reinterpret_cast<uintptr_t>(a.mask_n) & 15)))
    return false;
  const long long end = first + (long long)TT * kBins;
  return ((end + 3) & ~3LL) <= (long long)a.sched.B * a.T * kBins;
}

// Descriptor of linear tile x of the launch (x in this CTA's run [lo, hi); q = its quota).
template <int C>
__device__ __forceinline__ WsTile ws_describe(const StftCovArgs& a, int x, int lo, int hi, int q,
                                              bool vec_ok) {
  constexpr int TT = WsShape<C>::TT;
  WsTile d;
  const int b = sched_find(a.sched, x);
  const int pb = sched_prefix(a.sched, b), pe = sched_prefix(a.sched, b + 1);
  d.b = b;
  d.nb = a.n_samples ? a.n_samples[b] : a.N;
  d.t0 = (x - pb) * TT;
  const int nt = imax(0, imin(TT, frames_of(d.nb, kNfft, a.g.hop, a.g.pad) - d.t0));
  unsigned f = (unsigned)nt;
  if (nt > 0 && tile_bulk_ok(d.t0, nt, a.g.hop, a.g.pad, d.nb, vec_ok)) f |= WS_AUDIO_BULK;
  long long first;
  int shift;
  if (ws_mask_bulk(a, b, d.t0, nt, TT, first, shift)) f |= WS_MASK_BULK;
  f |= (unsigned)shift << WS_SHIFT_POS;
  if (x == imax(lo, pb)) f |= WS_SEG_BEGIN;
  if (x + 1 == imin(hi, pe)) f |= WS_SEG_END;
  if (x + 1 == pe) f |= WS_UTT_END;
  f |= (unsigned)((int)blockIdx.x - pb / q) << WS_SLOT_POS;
  d.flags = f;
  return d;
}
// Both roles call this between two __syncthreads(): descriptors of tiles [c0, c0 + count).
template <int C>
__device__ __forceinline__ void ws_fill_table(const StftCovArgs& a, const WsSmem<C>& sm, int c0, int count,
                                              int lo, int hi, int q, bool vec_ok) {
  for (int i = threadIdx.x; i < count; i += kWsThreads) sm.tiles[i] = ws_describe<C>(a, c0 + i, lo, hi, q, vec_ok);
}

// ---- audio staging by the FFT warps (threads 0..255) ----
template <int C>
__device__ __forceinline__ void ws_stage_bulk(const WsSmem<C>& sm, const float* __restrict__ xb, int N,
                                              int t0, int nt, int hop, int pad) {   // ONE thread
  const int need = (nt - 1) * hop + kNfft;
  const int i0 = t0 * hop - pad;
  fence_proxy_async();
  mbar_expect_tx(sm.bar_audio, (unsigned)(C * need * sizeof(float)));
#pragma unroll
  for (int c = 0; c < C; ++c)
    bulk_g2s(sm.audio + c * sm.Lp, xb + (long long)c * N + i0, (unsigned)(need * sizeof(float)),
             sm.bar_audio);
}
template <int C>
__device__ __forceinline__ void ws_stage_scalar(const WsSmem<C>& sm, const float* __restrict__ xb, int N,
                                                int nb, int t0, int nt, int hop, int pad, int ftid) {
  const int p0 = t0 * hop;
  const int need = (nt - 1) * hop + kNfft;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float* src = xb + (long long)c * N;
    for (int q = ftid; q < need; q += kWsFftThreads) {
      const int i = pad ? reflect_index(p0 + q, pad, nb) : (p0 + q);
      sm.audio[c * sm.Lp + q] = src[i];
    }
  }
}

// ---------------------------------------------------------------------------
// FFT role: threads 0..255, half-warp job = thread / 16 = frame * C + channel
// ---------------------------------------------------------------------------
template <int C, bool HAS_MN>
__device__ __forceinline__ void ws_fft_role(const StftCovArgs& a, const WsSmem<C>& sm, int lo, int hi, int q,
                                            bool vec_ok) {
  constexpr int TT = WsShape<C>::TT;
  constexpr int NR = HAS_MN ? 2 : 1, MS = HAS_MN ? 2 : 3;
  const int ftid = (int)threadIdx.x;
  const int lane = ftid & 31, lane16 = lane & 15;
  const int fwarp = ftid >> 5;
  const int half = lane >> 4;
  const int job = 2 * fwarp + half;
  static_assert(C % 2 == 0, "a warp's two jobs are channels (c, c + 1) of one frame");
  const int fr = (2 * fwarp) / C, ch = (2 * fwarp) % C + half;
  const int hop = a.g.hop, pad = a.g.pad;
  float amax = 0.f;
  unsigned apar = 0;

  // one thread: the mask rows of tile d (local number nn) -> mask slot nn % MS, completing on
  // z_full[nn & 1] together with that tile's Z
  auto issue_mask = [&](const WsTile& d, int nn, int mslot) {
    const int shift = (int)(d.flags >> WS_SHIFT_POS) & 3;
    const long long a0 = ((long long)d.b * a.T + d.t0) * kBins - shift;
    const unsigned bytes = (unsigned)(((shift + TT * kBins + 3) & ~3) * sizeof(float));
    float* dst = sm.mask + mslot * NR * kWsMaskRegion;
    MBar* bar = &sm.z_full[nn & 1];
    fence_proxy_async();
    mbar_add_tx(bar, bytes * (unsigned)NR);
    bulk_g2s(dst, a.mask_s + a0, bytes, bar);
    if (HAS_MN) bulk_g2s(dst + kWsMaskRegion, a.mask_n + a0, bytes, bar);
  };
  auto stage = [&](const WsTile& d) -> bool {       // true: written with ordinary stores
    const int nt = (int)(d.flags & WS_NT);
    if (nt <= 0) return false;
    const float* xb = a.audio + (long long)d.b * C * a.N;
    if (d.flags & WS_AUDIO_BULK) {
      if (ftid == 0) ws_stage_bulk<C>(sm, xb, a.N, d.t0, nt, hop, pad);
      return false;
    }
    ws_stage_scalar<C>(sm, xb, a.N, d.nb, d.t0, nt, hop, pad, ftid);
    return true;
  };

  int n = 0, m3 = 0;                               // local tile number, n % MS
  for (int c0 = lo; c0 < hi; c0 += kWsChunk) {
    const int cnt = imin(kWsChunk, hi - c0);
    __syncthreads();                               // the previous table is consumed by both roles
    ws_fill_table<C>(a, sm, c0, cnt + (c0 + cnt < hi ? 1 : 0), lo, hi, q, vec_ok);
    __syncthreads();
    if (c0 == lo) {                                // the run's first tile: nobody staged it yet
      const WsTile d = sm.tiles[0];
      if (stage(d)) named_bar_sync(kWsBarFft, kWsFftThreads);
      if (MS == 3 && ftid == 0 && (d.flags & WS_MASK_BULK)) issue_mask(d, 0, 0);
    }
    for (int i = 0; i < cnt; ++i, ++n) {
      const WsTile d = sm.tiles[i];
      const int nt = (int)(d.flags & WS_NT);
      float2 v[16];
      if (nt > 0) {
        if (d.flags & WS_AUDIO_BULK) { mbar_wait(sm.bar_audio, apar); apar ^= 1u; }
        // a dead frame (fr >= nt, only in an utterance's last tile) re-transforms the last live
        // one: its spectrum is never read and max|x| sees nothing new
        const int fr_src = imin(fr, nt - 1);
        // max|x|: with hop = n_fft / 2 the first halves of the frames tile the signal, so only an
        // utterance's last frame looks at its second half as well
        const bool amax_full = hop != kM || ((d.flags & WS_UTT_END) && fr >= nt - 1);
        const float* src = sm.audio + ch * sm.Lp + fr_src * hop + 2 * lane16;
        const float* wsrc = sm.win + 2 * lane16;
#pragma unroll
        for (int m1 = 0; m1 < 16; ++m1) v[m1] = *reinterpret_cast<const float2*>(src + 32 * m1);
#pragma unroll
        for (int m1 = 0; m1 < 16; ++m1) {
          if (m1 < 8 || amax_full) amax = fmaxf(amax, fmaxf(fabsf(v[m1].x), fabsf(v[m1].y)));
          v[m1] = f2mul(v[m1], *reinterpret_cast<const float2*>(wsrc + 32 * m1));
        }
      }
      // every FFT warp holds its samples: the staging buffer is free
      named_bar_sync(kWsBarFft, kWsFftThreads);
      const bool has_next = c0 + i + 1 < hi;
      bool scalar_next = false;
      if (has_next) scalar_next = stage(sm.tiles[i + 1]);
      if (nt > 0) halfwarp_fft256_a(v, sm.twtab, lane16);
      const int s = n & 1;
      mbar_wait(&sm.z_empty[s], ((unsigned)(n >> 1) & 1u) ^ 1u);
      // the covariance warps are done with tile n - 2: its Z slot, and the mask slot tile n + 1
      // (three mask slots) or tile n (two) will use, are free
      if (ftid == 0) {
        if (MS == 3) {
          if (has_next && (sm.tiles[i + 1].flags & WS_MASK_BULK))
            issue_mask(sm.tiles[i + 1], n + 1, m3 == 2 ? 0 : m3 + 1);
        } else if (d.flags & WS_MASK_BULK) {
          issue_mask(d, n, s);
        }
      }
      if (nt > 0) {
        float2* zs = sm.z + (s * 16 + job) * SETK_ZSLOT;
        halfwarp_fft256_b(v, zs, lane16);
#pragma unroll
        for (int p = 0; p < 16; ++p) zs[lane16 + 16 * kof(p)] = v[p];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.z_full[s]);

      // end of this utterance's part of the CTA's run: max|x| (SpectrogramReader.maxabs)
      if ((d.flags & WS_SEG_END) && a.maxabs_bits) {
        if (d.flags & WS_UTT_END) {                 // center=False leaves a tail no frame covers
          const int Tb = frames_of(d.nb, kNfft, hop, pad);
          const int covered = (Tb > 0 ? (Tb - 1) * hop + kNfft - 2 * pad : 0);
          const float* xb = a.audio + (long long)d.b * C * a.N;
          for (int c = 0; c < C; ++c)
            for (int k = imax(covered, 0) + ftid; k < d.nb; k += kWsFftThreads)
              amax = fmaxf(amax, fabsf(xb[(long long)c * a.N + k]));
        }
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0 && amax > 0.f) atomicMax(a.maxabs_bits + d.b, __float_as_uint(amax));
        amax = 0.f;
      }
      if (scalar_next) named_bar_sync(kWsBarFft, kWsFftThreads);
      m3 = (m3 == MS - 1) ? 0 : m3 + 1;
    }
  }
}

// ---------------------------------------------------------------------------
// covariance role: threads 256..383, thread 256 + k owns bins (k, 256 - k)
// ---------------------------------------------------------------------------
// one frame of one bin: A += m x x^H for (m_s, m_n); A = [diag | off_s | off_n | mask sums]
template <int C>
__device__ __forceinline__ void ws_update(float2* A, const float2* x, float ms, float mn) {
  constexpr int NOFF = WsShape<C>::NOFF;
  const float2 msn = make_float2(ms, mn);
  const float2 mss = make_float2(ms, ms), mnn = make_float2(mn, mn);
  A[C + 2 * NOFF] = f2add(A[C + 2 * NOFF], msn);
  int o = 0;
#pragma unroll
  for (int i = 0; i < C; ++i) {
    const float pii = x[i].x * x[i].x + x[i].y * x[i].y;
    A[i] = f2fma(msn, make_float2(pii, pii), A[i]);
#pragma unroll
    for (int k = i + 1; k < C; ++k) {
      const float2 pr = cmul_conj(x[i], x[k]);          // x_i conj(x_k)
      A[C + o] = f2fma(pr, mss, A[C + o]);
      A[C + NOFF + o] = f2fma(pr, mnn, A[C + NOFF + o]);
      ++o;
    }
  }
}
// accumulator p of a bin -> its two rows in the partial-sum workspace [2*NACC + 2][F]
template <int C>
__device__ __forceinline__ void ws_store_pair(float* pp, int p, float2 v) {
  constexpr int NOFF = WsShape<C>::NOFF, NACC = WsShape<C>::NACC, F = kBins;
  int i0, i1;
  if (p < C) { i0 = p; i1 = NACC + p; }
  else if (p < C + NOFF) { i0 = C + 2 * (p - C); i1 = i0 + 1; }
  else if (p < C + 2 * NOFF) { i0 = NACC + C + 2 * (p - C - NOFF); i1 = i0 + 1; }
  else { i0 = 2 * NACC; i1 = i0 + 1; }
  pp[(long long)i0 * F] = v.x;
  pp[(long long)i1 * F] = v.y;
}

// The TT frames of one tile for this thread's bin pair (+ bin 128 on the handler lanes).
//   BULK : masks from the tile's shared-memory copy (ms: frame t0, bin 0 of the m_s rows; the m_n
//          rows kWsMaskRegion floats later), else from the registers g* (loaded by the caller)
//   FULL : nt == TT (straight-line code)
template <int C, bool HAS_MN, bool BULK, bool FULL>
__device__ __forceinline__ void ws_cov_tile(float2* ak, float2* am, float2* my128, const float2* zt,
                                            const float* ms, const float* gk, const float* gm,
                                            const float* g128, int nt, bool clip, int bk, int bm, int zk,
                                            int zn, float2 tw, bool handler, int lane) {
  constexpr int TT = WsShape<C>::TT, F = kBins;
  constexpr int NR = HAS_MN ? 2 : 1;
#pragma unroll
  for (int j = 0; j < TT; ++j) {
    if (FULL || j < nt) {
      float2 xk[C], xm[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float2* z = zt + (j * C + c) * SETK_ZSLOT;
        split_pair(z[zk], z[zn], tw, xk[c], xm[c]);
      }
      const float rk = BULK ? ms[j * F + bk] : gk[j * NR];
      const float rm = BULK ? ms[j * F + bm] : gm[j * NR];
      const float msk = clip ? fminf(rk, 1.0f) : rk, msm = clip ? fminf(rm, 1.0f) : rm;
      float mnk, mnm;
      if (HAS_MN) {
        mnk = BULK ? ms[kWsMaskRegion + j * F + bk] : gk[j * NR + 1];
        mnm = BULK ? ms[kWsMaskRegion + j * F + bm] : gm[j * NR + 1];
      } else {
        mnk = 1.0f - msk;
        mnm = 1.0f - msm;
      }
      ws_update<C>(ak, xk, msk, mnk);
      ws_update<C>(am, xm, msm, mnm);
    }
  }
  if (handler && lane < nt) {                       // bin 128, frame `lane`
    float2 x128[C];
    const float2 tw128 = make_float2(-1.0f, -0.0f);       // split_twiddle(128)
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float2 z = zt[(lane * C + c) * SETK_ZSLOT + 128];
      x128[c] = split_bin(z, z, tw128);
    }
    const float r = BULK ? ms[lane * F + 128] : g128[0];
    const float m1 = clip ? fminf(r, 1.0f) : r;
    const float m2 = HAS_MN ? (BULK ? ms[kWsMaskRegion + lane * F + 128] : g128[1]) : 1.0f - m1;
    ws_update<C>(my128, x128, m1, m2);
  }
}

template <int C, bool HAS_MN>
__device__ __forceinline__ void ws_cov_role(const StftCovArgs& a, const WsSmem<C>& sm, int lo, int hi,
                                            int q, bool vec_ok) {
  constexpr int TT = WsShape<C>::TT, NPAIR = WsShape<C>::NPAIR, NACC = WsShape<C>::NACC;
  constexpr int ROWS128 = WsShape<C>::ROWS128, F = kBins;
  constexpr int NR = HAS_MN ? 2 : 1, MS = HAS_MN ? 2 : 3;
  const int tid = (int)threadIdx.x - kWsFftThreads, lane = tid & 31, warp = tid >> 5;
  const int bk = tid, bm = kM - tid;                       // the pair's bins
  const int zk = tid, zn = (kM - tid) & (kM - 1);          // their half-size spectrum entries
  const float2 tw = split_twiddle(tid);
  const bool clip = (a.flags & SETK_F_CLIP_MASK) != 0;
  const bool mask_ft = (a.flags & SETK_F_MASK_FT) != 0;
  float2 ak[NPAIR], am[NPAIR];
  float2* my128 = sm.acc128 + (warp * TT + imin(lane, TT - 1)) * NPAIR;

  int n = 0, m3 = 0;                                       // local tile number, n % MS
  for (int c0 = lo; c0 < hi; c0 += kWsChunk) {
    const int cnt = imin(kWsChunk, hi - c0);
    __syncthreads();
    ws_fill_table<C>(a, sm, c0, cnt + (c0 + cnt < hi ? 1 : 0), lo, hi, q, vec_ok);
    __syncthreads();
    for (int i = 0; i < cnt; ++i, ++n) {
      const WsTile d = sm.tiles[i];
      const int nt = (int)(d.flags & WS_NT);
      if (d.flags & WS_SEG_BEGIN) {
#pragma unroll
        for (int p = 0; p < NPAIR; ++p) { ak[p] = make_float2(0.f, 0.f); am[p] = make_float2(0.f, 0.f); }
        if (lane < TT) {
#pragma unroll
          for (int p = 0; p < NPAIR; ++p) my128[p] = make_float2(0.f, 0.f);
        }
      }
      const bool handler = warp == (n & 3);
      const bool bulk = (d.flags & WS_MASK_BULK) != 0;
      // masks the bulk copy does not bring: plain loads, issued before the wait for the Z tile
      float gk[TT * NR], gm[TT * NR], g128[NR];
      if (!bulk && nt > 0) {
        const long long mstride = mask_ft ? 1 : F, fmul = mask_ft ? a.T : 1;
        const long long base = mask_ft ? (long long)d.b * F * a.T + d.t0 : ((long long)d.b * a.T + d.t0) * F;
#pragma unroll
        for (int j = 0; j < TT; ++j) {
          const long long o = base + imin(j, nt - 1) * mstride;
          gk[j * NR] = a.mask_s[o + bk * fmul];
          gm[j * NR] = a.mask_s[o + bm * fmul];
          if (HAS_MN) { gk[j * NR + 1] = a.mask_n[o + bk * fmul]; gm[j * NR + 1] = a.mask_n[o + bm * fmul]; }
        }
        const long long o128 = base + imin(lane, nt - 1) * mstride + 128 * fmul;
        g128[0] = a.mask_s[o128];
        if (HAS_MN) g128[1] = a.mask_n[o128];
      }
      const int s = n & 1;
      mbar_wait(&sm.z_full[s], (unsigned)(n >> 1) & 1u);
      const float2* zt = sm.z + s * 16 * SETK_ZSLOT;
      const float* ms = sm.mask + m3 * NR * kWsMaskRegion + ((d.flags >> WS_SHIFT_POS) & 3);
      if (bulk)
        ws_cov_tile<C, HAS_MN, true, true>(ak, am, my128, zt, ms, gk, gm, g128, nt, clip, bk, bm, zk, zn,
                                           tw, handler, lane);
      else if (nt == TT)
        ws_cov_tile<C, HAS_MN, false, true>(ak, am, my128, zt, ms, gk, gm, g128, nt, clip, bk, bm, zk, zn,
                                            tw, handler, lane);
      else if (nt > 0)
        ws_cov_tile<C, HAS_MN, false, false>(ak, am, my128, zt, ms, gk, gm, g128, nt, clip, bk, bm, zk, zn,
                                             tw, handler, lane);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.z_empty[s]);

      if (d.flags & WS_SEG_END) {
        // ---- partial sums of this segment -> slot ----
        const int slot = (int)(d.flags >> WS_SLOT_POS) & 0xff;
        float* pp = a.partials + (((long long)d.b * a.slots + slot) * (2 * NACC + 2)) * F;
#pragma unroll
        for (int p = 0; p < NPAIR; ++p) {
          ws_store_pair<C>(pp + bk, p, ak[p]);
          ws_store_pair<C>(pp + bm, p, am[p]);
        }
        named_bar_sync(kWsBarCov, kWsCovThreads);     // every warp's bin-128 rows are final
        if (tid < NPAIR) {
          float2 sum = make_float2(0.f, 0.f);
#pragma unroll
          for (int r = 0; r < ROWS128; ++r) sum = f2add(sum, sm.acc128[r * NPAIR + tid]);
          ws_store_pair<C>(pp + 128, tid, sum);
        }
        named_bar_sync(kWsBarCov, kWsCovThreads);     // rows may be zeroed again
      }
      m3 = (m3 == MS - 1) ? 0 : m3 + 1;
    }
  }
}

template <int C, bool HAS_MN>
__global__ void __maxnreg__(SETK_WS_LAUNCH_REGS) stft_cov_ws_kernel(StftCovArgs a) {
  SETK_DYN_SMEM(float, smem);
  WsSmem<C> sm;
  sm.carve(smem, a.g.hop, HAS_MN ? 2 : 1);
  const int tid = threadIdx.x;

  // this CTA's run of the (utterance, tile) sequence
  const int q = sched_quota(a.sched, gridDim.x);
  const int total = sched_prefix(a.sched, a.sched.B);
  const int lo = blockIdx.x * q;
  const int hi = imin(lo + q, total);
  if (lo >= hi) return;

  for (int n = tid; n < kNfft; n += kWsThreads)
    sm.win[n] = 0.5f * a.window[n];
  twiddle_table_fill(sm.twtab, tid, kWsThreads);
  if (tid == 0) {
    mbar_init(sm.bar_audio, 1);
    mbar_init(&sm.z_full[0], kWsFftThreads / 32);
    mbar_init(&sm.z_full[1], kWsFftThreads / 32);
    mbar_init(&sm.z_empty[0], kWsCovThreads / 32);
    mbar_init(&sm.z_empty[1], kWsCovThreads / 32);
  }
  __syncthreads();
  const bool vec_ok = ((a.N & 3) == 0) && ((a.g.hop & 3) == 0) && ((a.g.pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  if (tid >= kWsFftThreads) {
    setmaxnreg_inc<kWsCovRegs>();
    ws_cov_role<C, HAS_MN>(a, sm, lo, hi, q, vec_ok);
  } else {
    setmaxnreg_dec<kWsFftRegs>();
    ws_fft_role<C, HAS_MN>(a, sm, lo, hi, q, vec_ok);
  }
}

// ---- host side ----
static_assert(WsShape<4>::TT == stft_cov_tt(4),
              "run_stft_cov_fused schedules the C = 4 launch in tiles of this kernel's TT frames");

template <int C, bool HAS_MN>
static cudaError_t run_ws_t(const StftCovArgs& a, int n_ctas, void* stream) {
  const size_t smem = WsSmem<C>::bytes(a.g.hop, HAS_MN ? 2 : 1);
  cudaError_t e = cudaFuncSetAttribute(stft_cov_ws_kernel<C, HAS_MN>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch(stft_cov_ws_kernel<C, HAS_MN>, dim3(n_ctas), dim3(kWsThreads), smem, stream, false, a);
}

// the C = 4 launch of the fused pass; run_stft_cov_fused prepares a and runs the finalize after it
cudaError_t run_stft_cov_ws(const StftCovArgs& a, int n_ctas, void* stream) {
  if (a.mask_n) return run_ws_t<4, true>(a, n_ctas, stream);
  return run_ws_t<4, false>(a, n_ctas, stream);
}

}  // namespace setk
