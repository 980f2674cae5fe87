// stft_cov_fused.cu -- THE METRIC KERNEL: multichannel STFT fused with the
// mask-weighted spatial covariance; the STFT never touches HBM.
//
// Replaces (scripts/sptk): SpectrogramReader._load (libs/data_handler.py:492-503,
// forward_stft per channel, libs/utils.py:96-138 -> librosa.stft) followed by
// SupervisedBeamformer.run's two compute_covar calls (libs/beamformer.py:279-281,
// 87-103); C++ twin: ShortTimeFTComputer::Compute (include/stft.cc:28-66) +
// EstimatePsd (include/beamformer.cc:91-120).
//
// Mapping (template <C, 512-point frames, TT frames per tile>), 320 threads at TT = 5 (even C)
// or 288 at TT = 4, 96 registers, two CTAs per SM:
//   grid = 2 x SMs persistent CTAs; the (utterance, tile) sequence of the batch is
//   cut into equal runs (TileSched, stft_tile.cuh), so a CTA owns a run of frames
//   of one to three consecutive utterances and there is no partial last wave.
//   per tile of TT frames
//     stage   (TT-1)*hop + n_fft samples x C channels -> smem by TMA bulk copies one
//             tile ahead; reflect padding / ragged ends element-wise; running max|x|
//     FFT     one half-warp per (frame, channel): 512-point real FFT as a
//             256-point complex FFT, 16 values per lane in registers, one
//             conflict-free smem exchange (fft16.cuh); Z stays in smem
//     cov     one thread per bin k < 256 (the Nyquist bin: one lane of warp 8 per
//             frame): split Z -> X_c[k] with the thread-constant twiddle,
//             accumulate the Hermitian upper triangle of  sum m x x^H  for
//             (m_s, m_n) in fp32 registers
//   end of an utterance's run: partial sums -> workspace [B][slot][acc][F];
//   cov_finalize_kernel reduces the slots in fixed order, normalises by
//   max(sum m, 1e-6), writes Rs, Rn c64 [B][F][C][C].
// Algorithmic bytes per utterance: 4*C*N + 4*T*F (+4*T*F with mask_n) + 2*8*F*C^2.
#include "common.cuh"
#include "stft_tile.cuh"
#include "stft_cov_args.cuh"
#include "launchers.cuh"

namespace setk {

// registers per thread of the fused kernel: 288 threads occupy 10 warp slots of the
// register file (allocation granularity: 2 warps), so two CTAs per SM need
// <= 65536 / (2 * 10 * 32) = 102 -> 96 registers (ncu: 112 left ONE CTA per SM)
constexpr int kScRegs = 96;

// tiles before every utterance of a ragged batch (one CTA; B is small)
__global__ void tile_prefix_kernel(const int* __restrict__ n_samples, int B, Geometry g, int TT,
                                   int T_cap, int* __restrict__ prefix) {
  __shared__ int s_scan[2][256];
  __shared__ int s_run;
  const int tid = threadIdx.x;
  if (tid == 0) { s_run = 0; prefix[0] = 0; }
  __syncthreads();
  for (int base = 0; base < B; base += 256) {
    const int b = base + tid;
    int v = 0;
    if (b < B) v = sched_tiles_of(imin(frames_of(n_samples[b], g.n_fft, g.hop, g.pad), T_cap), TT);
    int cur = 0;
    s_scan[0][tid] = v;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const int x = s_scan[cur][tid] + (tid >= o ? s_scan[cur][tid - o] : 0);
      s_scan[cur ^ 1][tid] = x;
      cur ^= 1;
      __syncthreads();
    }
    const int run = s_run;
    if (b < B) prefix[b + 1] = run + s_scan[cur][tid];
    __syncthreads();
    if (tid == 255) s_run = run + s_scan[cur][255];
    __syncthreads();
  }
}

template <int C, int TT>
__global__ void __maxnreg__(kScRegs) stft_cov_kernel(StftCovArgs a) {
  constexpr int NACC = CovAcc<C>::NACC;
  constexpr int F = kBins;
  static_assert(TT <= 8, "Nyquist lanes: one frame per lane, butterfly sum over 8 lanes");
  constexpr int NW = 2 * TT;                 // FFT warps: TT * C <= 4 TT half-warp jobs, one round
  SETK_DYN_SMEM(float, smem);
  const int hop = a.g.hop, pad = a.g.pad;
  TileSmem<C, TT> sm;
  sm.carve(smem, hop);

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;

  // this CTA's run of the (utterance, tile) sequence
  const int q = sched_quota(a.sched, gridDim.x);
  const int total = sched_prefix(a.sched, a.sched.B);
  int cur = blockIdx.x * q;
  const int hi = imin(cur + q, total);
  if (cur >= hi) return;

  for (int n = tid; n < kNfft; n += blockDim.x) sm.win[n] = 0.5f * a.window[n];
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }

  // cov role: threads 0..255 own bins 0..255 (all frames of a tile); the Nyquist
  // bin is spread over the lanes of warp 8, one FRAME per lane, so that warp
  // issues the accumulation once per tile instead of once per frame
  const bool nyq = warp == 8;
  const bool cov_idle = warp > 8;            // a tenth warp only transforms
  const int bin = nyq ? kM : tid;
  const float2 tw = split_twiddle(bin);
  const int zk = bin & (kM - 1), zn = (kM - bin) & (kM - 1);

  // accumulators as (m_s, m_n) pairs: dg[i] = (sum m_s |x_i|^2, sum m_n |x_i|^2),
  // os[p] / on[p] = sum m x_i conj(x_k) for the p-th (i < k), sm2 = (sum m_s, sum m_n)
  constexpr int NOFF = C * (C - 1) / 2;
  float2 dg[C], os[NOFF > 0 ? NOFF : 1], on[NOFF > 0 ? NOFF : 1];
  float2 sm2;
  float amax = 0.f;

  const bool vec_ok = ((a.N & 3) == 0) && ((hop & 3) == 0) && ((pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  const bool has_mn = a.mask_n != nullptr;
  const bool clip = (a.flags & SETK_F_CLIP_MASK) != 0;
  const long long mstride = (a.flags & SETK_F_MASK_FT) ? 1 : F;
  float* s_mask = sm.end();                        // [TT][2][MPITCH]
  constexpr int MPITCH = 260;
  float2* s_twtab = reinterpret_cast<float2*>(s_mask + TT * 2 * MPITCH);   // [16][16] W256^{lane16 k}
  twiddle_table_fill(s_twtab, tid, blockDim.x);

  // one frame of this thread's bin: split Z -> X_c[bin], rank-1 update for (m_s, m_n)
  auto accumulate = [&](int j) {
    float2 x[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float2* z = sm.z + (j * C + c) * SETK_ZSLOT;
      x[c] = split_bin(z[zk], z[zn], tw);
    }
    // DC / Nyquist need no special case: with Zk == Zn the split's difference has an
    // exactly zero real part, its sum an exactly zero imaginary part, and the bin's
    // twiddle is (-0, -+1), so Im X comes out as an exact (signed) zero
    const float m_raw = s_mask[(2 * j) * MPITCH + bin];
    const float m_s = clip ? fminf(m_raw, 1.0f) : m_raw;
    // the second row is loaded whether or not it was filled (a select, not a branch, keeps the
    // frames of a tile in one basic block for the scheduler)
    const float m_n_row = s_mask[(2 * j + 1) * MPITCH + bin];
    const float m_n = has_mn ? m_n_row : 1.0f - m_s;
    const float2 msn = make_float2(m_s, m_n);
    const float2 mss = make_float2(m_s, m_s), mnn = make_float2(m_n, m_n);
    sm2 = f2add(sm2, msn);
    int o = 0;
#pragma unroll
    for (int i = 0; i < C; ++i) {
      const float pii = x[i].x * x[i].x + x[i].y * x[i].y;
      dg[i] = f2fma(msn, make_float2(pii, pii), dg[i]);
#pragma unroll
      for (int k = i + 1; k < C; ++k) {
        const float2 pr = cmul_conj(x[i], x[k]);        // x_i conj(x_k)
        os[o] = f2fma(pr, mss, os[o]);
        on[o] = f2fma(pr, mnn, on[o]);
        ++o;
      }
    }
  };

  unsigned par = 0;                 // mbarrier phase parity per buffer (bit b)
  int buf = 0;
  int b = sched_find(a.sched, cur);
  while (cur < hi) {
    // ---- next segment: the part of utterance b inside [cur, hi) ----
    int pb = sched_prefix(a.sched, b), pe = sched_prefix(a.sched, b + 1);
    while (pe <= cur) { ++b; pb = pe; pe = sched_prefix(a.sched, b + 1); }
    const int seg_end = imin(hi, pe);
    const int nb = a.n_samples ? a.n_samples[b] : a.N;
    const int Tb = frames_of(nb, kNfft, hop, pad);
    const int t_begin = (cur - pb) * TT;
    const int t_end = imin((seg_end - pb) * TT, Tb);
    const int slot = (int)blockIdx.x - pb / q;
    const float* xb = a.audio + (long long)b * C * a.N;

#pragma unroll
    for (int i = 0; i < C; ++i) dg[i] = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < NOFF; ++i) { os[i] = make_float2(0.f, 0.f); on[i] = make_float2(0.f, 0.f); }
    sm2 = make_float2(0.f, 0.f);

    // software pipeline: tile i+1 streams into the other audio buffer while tile i
    // is transformed and accumulated.  (All FFT reads of both audio buffers are
    // behind a barrier here, also when a previous segment just ended.)
    bool async_cur = false;
    if (t_begin < t_end)
      async_cur = stage_tile_begin<C, TT>(sm, buf, xb, a.N, nb, t_begin, imin(TT, t_end - t_begin), hop,
                                          pad, vec_ok);
    // mask rows of this thread's bin.  They are fetched with 4-byte cp.async
    // straight into shared memory at the top of the tile and first touched after
    // the FFT phase, so their latency costs neither registers nor issue slots
    const long long mbase = (a.flags & SETK_F_MASK_FT) ? ((long long)b * F + bin) * a.T
                                                       : (long long)b * a.T * F + bin;
    for (int t0 = t_begin; t0 < t_end; t0 += TT, buf ^= 1) {
      const int nt = imin(TT, t_end - t0);
      __syncthreads();   // tile i-1 fully consumed: sm.z and audio[buf^1] are free
      bool async_next = false;
      if (t0 + TT < t_end)
        async_next = stage_tile_begin<C, TT>(sm, buf ^ 1, xb, a.N, nb, t0 + TT,
                                             imin(TT, t_end - t0 - TT), hop, pad, vec_ok);
      if (cov_idle) {
      } else if (!nyq) {
        const float* mps = a.mask_s + mbase + (long long)t0 * mstride;
        const float* mpn = has_mn ? a.mask_n + mbase + (long long)t0 * mstride : nullptr;
        if (nt == TT) {
#pragma unroll
          for (int j = 0; j < TT; ++j) {
            cp_async_f32(s_mask + (2 * j) * MPITCH + bin, mps + j * mstride);
            if (has_mn) cp_async_f32(s_mask + (2 * j + 1) * MPITCH + bin, mpn + j * mstride);
          }
        } else {
#pragma unroll
          for (int j = 0; j < TT; ++j) {
            if (j < nt) {
              cp_async_f32(s_mask + (2 * j) * MPITCH + bin, mps + j * mstride);
              if (has_mn) cp_async_f32(s_mask + (2 * j + 1) * MPITCH + bin, mpn + j * mstride);
            }
          }
        }
      } else if (lane < nt) {
        const long long mo = mbase + (long long)(t0 + lane) * mstride;
        cp_async_f32(s_mask + (2 * lane) * MPITCH + bin, a.mask_s + mo);
        if (has_mn) cp_async_f32(s_mask + (2 * lane + 1) * MPITCH + bin, a.mask_n + mo);
      }
      if (async_cur) {
        mbar_wait(&sm.bar[buf], (par >> buf) & 1u);
        par ^= 1u << buf;
      }
      // inter-pass twiddles from s_twtab (the w1 argument is unused)
      if (warp < NW) fft_tile<C, TT, true, NW>(sm, buf, nt, hop, make_float2(1.f, 0.f), amax, s_twtab);
      async_cur = async_next;
      cp_async_wait_all();
      __syncthreads();
      // ---- covariance ----
      if (cov_idle) {
      } else if (!nyq) {
        if (nt == TT) {          // every tile but an utterance's last: straight-line code
#pragma unroll
          for (int j = 0; j < TT; ++j) accumulate(j);
        } else {
#pragma unroll
          for (int j = 0; j < TT; ++j)
            if (j < nt) accumulate(j);
        }
      } else if (lane < nt) {
        accumulate(lane);
      }
    }

    // center=False leaves a tail no frame covers; max|x| must still see it
    if (a.maxabs_bits && t_end >= Tb) {
      const int covered = (Tb > 0 ? (Tb - 1) * hop + kNfft - 2 * pad : 0);
      for (int c = 0; c < C; ++c)
        for (int i = imax(covered, 0) + tid; i < nb; i += blockDim.x)
          amax = fmaxf(amax, fabsf(xb[(long long)c * a.N + i]));
    }

    // ---- partial sums of this segment -> slot ----
    if (nyq) {
      // the Nyquist lanes hold one frame class each: fixed-order butterfly sum
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) {      // lanes >= TT hold zeros
#pragma unroll
        for (int i = 0; i < C; ++i) {
          dg[i].x += __shfl_xor_sync(0xffffffffu, dg[i].x, o);
          dg[i].y += __shfl_xor_sync(0xffffffffu, dg[i].y, o);
        }
#pragma unroll
        for (int i = 0; i < NOFF; ++i) {
          os[i].x += __shfl_xor_sync(0xffffffffu, os[i].x, o);
          os[i].y += __shfl_xor_sync(0xffffffffu, os[i].y, o);
          on[i].x += __shfl_xor_sync(0xffffffffu, on[i].x, o);
          on[i].y += __shfl_xor_sync(0xffffffffu, on[i].y, o);
        }
        sm2.x += __shfl_xor_sync(0xffffffffu, sm2.x, o);
        sm2.y += __shfl_xor_sync(0xffffffffu, sm2.y, o);
      }
    }
    if (warp < 8 || (nyq && lane == 0)) {
      float* pp = a.partials + (((long long)b * a.slots + slot) * (2 * NACC + 2)) * F + bin;
#pragma unroll
      for (int i = 0; i < C; ++i) { pp[(long long)i * F] = dg[i].x; pp[(long long)(NACC + i) * F] = dg[i].y; }
#pragma unroll
      for (int i = 0; i < NOFF; ++i) {
        pp[(long long)(C + 2 * i) * F] = os[i].x;        pp[(long long)(C + 2 * i + 1) * F] = os[i].y;
        pp[(long long)(NACC + C + 2 * i) * F] = on[i].x; pp[(long long)(NACC + C + 2 * i + 1) * F] = on[i].y;
      }
      pp[(long long)(2 * NACC) * F] = sm2.x;
      pp[(long long)(2 * NACC + 1) * F] = sm2.y;
    }
    if (a.maxabs_bits) {
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      if (lane == 0 && amax > 0.f) atomicMax(a.maxabs_bits + b, __float_as_uint(amax));
      amax = 0.f;
    }
    cur = seg_end;
  }
}

// Deterministic reduction over the segments of an utterance + normalisation + Hermitian fill.
// One thread per (matrix, b, f) -- Rs and Rn of a bin are reduced by different threads (half the
// dependent loads per thread, twice the threads in flight); a thread writes its C x C matrix as
// 16-byte stores (rows of the row-major matrix are contiguous).
template <int C>
__global__ void cov_finalize_kernel(const float* __restrict__ partials, int B, int F, TileSched sched,
                                    int n_ctas, int slots, float2* __restrict__ Rs,
                                    float2* __restrict__ Rn) {
  constexpr int NACC = CovAcc<C>::NACC;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)B * F;
  if (gid >= 2 * n) return;
  const int which = gid >= n ? 1 : 0;
  const long long idx = gid - which * n;
  const int b = (int)(idx / F), f = (int)(idx % F);
  // the CTAs of the main kernel that held tiles of utterance b wrote slots 0..n_used-1
  const int q = sched_quota(sched, n_ctas);
  const int pb = sched_prefix(sched, b), pe = sched_prefix(sched, b + 1);
  const int n_used = (pe - 1) / q - pb / q + 1;
  float acc[NACC + 1];                                   // this matrix's sums, then its mask sum
#pragma unroll
  for (int i = 0; i <= NACC; ++i) acc[i] = 0.f;
  for (int ch = 0; ch < n_used; ++ch) {
    const float* pp = partials + (((long long)b * slots + ch) * (2 * NACC + 2)) * F + f;
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] += pp[(long long)(which * NACC + i) * F];
    acc[NACC] += pp[(long long)(2 * NACC + which) * F];
  }
  const float inv = 1.0f / fmaxf(acc[NACC], 1e-6f);
  float2 M[C * C];
  int o = C;
#pragma unroll
  for (int i = 0; i < C; ++i) {
    M[i * C + i] = make_float2(acc[i] * inv, 0.f);
#pragma unroll
    for (int k = i + 1; k < C; ++k) {
      const float re = acc[o] * inv, im = acc[o + 1] * inv;
      M[i * C + k] = make_float2(re, im);
      M[k * C + i] = make_float2(re, -im);
      o += 2;
    }
  }
  float2* R = (which == 0 ? Rs : Rn) + idx * (C * C);
  if ((C * C) % 2 == 0 && (reinterpret_cast<uintptr_t>(R) & 15) == 0) {
#pragma unroll
    for (int e = 0; e < C * C; e += 2)
      *reinterpret_cast<float4*>(R + e) = make_float4(M[e].x, M[e].y, M[e + 1].x, M[e + 1].y);
  } else {
#pragma unroll
    for (int e = 0; e < C * C; ++e) R[e] = M[e];
  }
}

template <int C>
static cudaError_t run_cov_finalize_t(const float* partials, int B, int F, TileSched sched, int n_ctas,
                                      int slots, float2* Rs, float2* Rn, void* stream) {
  const long long n = (long long)B * F;
  return launch(cov_finalize_kernel<C>, dim3((unsigned)((2 * n + 127) / 128)), dim3(128), 0, stream, true,
                partials, B, F, sched, n_ctas, slots, Rs, Rn);
}
static cudaError_t run_cov_finalize(int C, const float* partials, int B, int F, TileSched sched, int n_ctas,
                                    int slots, float2* Rs, float2* Rn, void* stream) {
  switch (C) {
    case 1: return run_cov_finalize_t<1>(partials, B, F, sched, n_ctas, slots, Rs, Rn, stream);
    case 2: return run_cov_finalize_t<2>(partials, B, F, sched, n_ctas, slots, Rs, Rn, stream);
    case 3: return run_cov_finalize_t<3>(partials, B, F, sched, n_ctas, slots, Rs, Rn, stream);
    case 4: return run_cov_finalize_t<4>(partials, B, F, sched, n_ctas, slots, Rs, Rn, stream);
    default: return cudaErrorInvalidValue;
  }
}

template <int C, int TT>
static size_t stft_cov_smem_bytes(int hop) {
  return sizeof(float) * (TileSmem<C, TT>::floats(hop) + (size_t)TT * 2 * 260 + 2 * 256);
}

template <int C, int TT>
static cudaError_t run_stft_cov_t(const StftCovArgs& a, int n_ctas, void* stream) {
  const size_t smem = stft_cov_smem_bytes<C, TT>(a.g.hop);
  cudaError_t e = cudaFuncSetAttribute(stft_cov_kernel<C, TT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  return launch(stft_cov_kernel<C, TT>, dim3(n_ctas), dim3(TT > 4 ? 320 : 288), smem, stream, false, a);
}

// Does a fused instantiation exist for this geometry?
bool stft_cov_fused_supported(const Geometry& g) {
  if (g.n_fft != 512) return false;
  if (g.C < 1 || g.C > 4) return false;
  if (g.hop < 2 || g.hop > 512 || (g.hop & 1)) return false;   // float2 frame loads
  return true;
}

// partial-sum workspace: floats per (utterance, chunk)
static size_t stft_cov_partial_floats(const Geometry& g) { return (size_t)(2 * g.C * g.C + 2) * g.F; }

int stft_cov_pick_chunks(const setk_plan* pl, int B, int T) {
  // (chunk, utterance) grids of the workspace routes: all CTAs are equally long, so
  // the launch costs ceil(CTAs / slots) waves of frames-per-chunk each.  Pick the
  // chunk count (<= 16 per utterance) that minimises that product -- "two waves
  // or more" alone left up to a third of the last wave empty.
  const int slots = 2 * pl->sm_count;
  int max_chunks = (T + 3) / 4;
  if (max_chunks > 16) max_chunks = 16;
  if (max_chunks < 1) max_chunks = 1;
  int best = 1;
  long long best_cost = -1;
  for (int c = 1; c <= max_chunks; ++c) {
    const long long waves = ((long long)B * c + slots - 1) / slots;
    const int fpc = (((T + c - 1) / c + 3) / 4) * 4 + 4;     // + per-chunk prologue
    const long long cost = waves * fpc;
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = c; }
  }
  return best;
}

// The persistent schedule of a fused pass over B utterances of <= T frames, TT frames per tile and
// at most T_cap frames of each used: the TileSched, the CTAs to launch and the partial-sum slots per
// utterance.  A ragged batch (n_samples != null) keeps its lengths on the device, so this also
// launches tile_prefix_kernel, which writes the tiles before every utterance to tile_prefix [B + 1].
cudaError_t fused_schedule(const setk_plan* pl, int B, int T, int TT, int T_cap, const int* n_samples,
                           int* tile_prefix, void* stream, TileSched* sched, int* n_ctas, int* slots) {
  const int G = 2 * pl->sm_count;   // CTA slots: 2 CTAs per SM resident (registers and shared memory)
  const int tiles_max = sched_tiles_of(imin(T, T_cap), TT);
  *slots = sched_slots(G, B);
  sched->prefix = n_samples ? tile_prefix : nullptr;
  sched->tiles_u = tiles_max;
  sched->B = B;
  sched->min_quota = sched_min_quota(tiles_max, *slots);
  *n_ctas = sched_grid(B * tiles_max, G, sched->min_quota);
  if (!n_samples) return cudaSuccess;
  return launch(tile_prefix_kernel, dim3(1), dim3(256), 0, stream, false, n_samples, B, pl->geo, TT, T_cap,
                tile_prefix);
}

static const int kNoFrameCap = 0x7fffffff;

size_t stft_cov_partial_bytes(const setk_plan* pl, int B, int T) {
  TileSched sched;
  int n_ctas, slots;
  fused_schedule(pl, B, T, stft_cov_tt(pl->geo.C), kNoFrameCap, nullptr, nullptr, nullptr, &sched, &n_ctas,
                 &slots);
  return sizeof(float) * stft_cov_partial_floats(pl->geo) * (size_t)slots * B;
}

cudaError_t run_stft_cov_fused(setk_plan* pl, const float* audio, const int* n_samples, int B, int N,
                               int T, const float* mask_s, const float* mask_n, unsigned flags,
                               int* tile_prefix, float* partials, unsigned* maxabs_bits, float2* Rs,
                               float2* Rn, float* maxabs, void* stream) {
  const Geometry& g = pl->geo;
  StftCovArgs a;
  a.g = g;
  a.audio = audio; a.n_samples = n_samples; a.N = N;
  a.mask_s = mask_s; a.mask_n = mask_n; a.flags = flags;
  a.T = T;
  a.window = pl->d_window;
  a.partials = partials;
  a.maxabs_bits = maxabs_bits;
  int n_ctas;
  cudaError_t e = fused_schedule(pl, B, T, stft_cov_tt(g.C), kNoFrameCap, n_samples, tile_prefix, stream,
                                 &a.sched, &n_ctas, &a.slots);
  if (e != cudaSuccess) return e;
  switch (g.C) {
    case 1: e = run_stft_cov_t<1, stft_cov_tt(1)>(a, n_ctas, stream); break;
    case 2: e = run_stft_cov_t<2, stft_cov_tt(2)>(a, n_ctas, stream); break;
    case 3: e = run_stft_cov_t<3, stft_cov_tt(3)>(a, n_ctas, stream); break;
    case 4: e = run_stft_cov_ws(a, n_ctas, stream); break;   // the warp-specialised build (stft_cov_ws.cu)
    default: return cudaErrorInvalidValue;
  }
  if (e == cudaSuccess) e = run_cov_finalize(g.C, partials, B, g.F, a.sched, n_ctas, a.slots, Rs, Rn, stream);
  if (e == cudaSuccess && maxabs) e = run_bits_to_float(maxabs_bits, B, maxabs, stream);
  return e;
}

}  // namespace setk
