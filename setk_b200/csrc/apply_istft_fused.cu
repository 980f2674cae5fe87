// apply_istft_fused.cu -- beamform apply fused with the inverse STFT, driven
// from the multichannel AUDIO: the STFT is recomputed on chip (same tile code as
// the covariance pass), so neither the C-channel STFT nor the enhanced STFT
// ever exists in HBM.
//
// Replaces (scripts/sptk): Beamformer.beamform (libs/beamformer.py:220-234),
// the optional post-mask (apply_adaptive_beamformer.py:174-175) and
// inverse_stft (libs/utils.py:142-173 -> librosa.istft: irfft, x window,
// overlap-add, / window-sum-square, trim) up to the peak of |y| needed by the
// `norm` rescale (utils.py:166-168), which peak_scale_kernel then applies (a
// rescale by the CTA that completes an utterance was measured slower: the
// utterance's first samples have left L2 by then, 17 % of the kernel's samples
// sat in that loop).
// C++ twin: Beamform (include/beamformer.cc:215-230) + InverseShortTimeFT
// (include/stft.cc:154-198).
//
// 320 threads, two barriers per tile of <= TT frames, audio streamed one tile
// ahead by TMA bulk copies (stft_tile.cuh).  Software pipeline over tiles:
//   phase A(i)  warps 0-7 : forward FFT of tile i            (Z_i in smem)
//               warps 8-9 : inverse FFT of tile i-1 (one half-warp per frame:
//                           conj . FFT256 . conj) x synthesis window -> frames
//   phase B(i)  all       : apply items (frame, k<=128) of tile i: split Z ->
//                           X_c[k], X_c[256-k]; y = w^H x for both bins;
//                           inverse split -> half-size spectrum Zi[k], Zi[256-k]
//                           flush tile i-1: gather overlap-add of its frames +
//                           carry; positions no later frame can touch are
//                           divided by the window-sum-square, trimmed and
//                           written (coalesced rows); the rest is the next carry
// Persistent CTAs (2 per SM) over equal runs of the batch's (utterance, tile)
// sequence (TileSched, stft_tile.cuh): no partial last wave; the weights of an
// utterance are reloaded where a run crosses into the next utterance.
// Deterministic: no atomics on data.  A CTA owns the output positions of its
// own frames; the <= ceil(n_fft/hop)-1 frames before the first frame of a run
// are recomputed as a halo tile.
// Algorithmic bytes per utterance: 4*C*N (audio) + 8*F*C (w) + 4*n_out (wave)
// (+ 4*T*F with a post-mask).
#include <type_traits>
#include "common.cuh"
#include "stft_tile.cuh"
#include "apply_istft_args.cuh"
#include "launchers.cuh"

namespace setk {

constexpr int kApplyThreads = 320;
constexpr int kWPitch = 260;          // float2 pitch of the per-channel weight rows

template <int C, int TT>
__global__ void __maxnreg__(96) apply_istft_kernel(ApplyIstftArgs a) {
  static_assert(TT == 4, "two inverse-FFT warps serve exactly four frames");
  constexpr int F = kBins;
  constexpr int NPAIR = kM / 2 + 1;     // 129 bin pairs (k, 256-k)
  SETK_DYN_SMEM(float, smem);
  const int hop = a.g.hop, pad = a.g.pad;
  TileSmem<C, TT> sm;
  sm.carve(smem, hop);
  const int carry_len = kNfft - hop;
  float2* s_w = reinterpret_cast<float2*>(sm.end());          // [C][kWPitch]
  float2* s_zi = s_w + C * kWPitch;                           // [TT][SETK_ZSLOT]
  float2* s_tw = s_zi + TT * SETK_ZSLOT;                      // [130] split twiddles (129 used)
  float* s_frames = reinterpret_cast<float*>(s_tw + NPAIR + 1);   // [TT][512]
  float* s_wsyn = s_frames + TT * kNfft;                      // [512] window / 512
  float* s_wsq = s_wsyn + kNfft;                              // [512]
  float* s_rw = s_wsq + kNfft;                                // [256] 1 / (wsq[r] + wsq[r+256])
  float* s_carry = s_rw + kM;                                 // [2][carry_len]

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int lane16 = lane & 15, half = lane >> 4;

  // this CTA's run of the (utterance, tile) sequence (TileSched, stft_tile.cuh)
  const int q = sched_quota(a.sched, gridDim.x);
  const int total = sched_prefix(a.sched, a.sched.B);
  int cur_tile = blockIdx.x * q;
  const int hi_tile = imin(cur_tile + q, total);
  if (cur_tile >= hi_tile) return;

  // frames librosa.istft would use for this output length
  const int T_cap = (a.n_out + 2 * pad + hop - 1) / hop;
  // per-segment state (set at the top of the segment loop)
  int b = 0, nb = 0, T_used = 0, own_begin = 0;
  int n_lim = a.n_out;      // output samples of the current utterance (a ragged one ends earlier)
  float* yb = nullptr;
  float peak = 0.f;

  for (int n = tid; n < kNfft; n += blockDim.x) {
    const float w = a.window[n];
    sm.win[n] = 0.5f * w;
    s_wsyn[n] = w * (1.0f / 512.0f);
    s_wsq[n] = a.wsq[n];
  }
  for (int n = tid; n < kM; n += blockDim.x) {
    const float s = a.wsq[n] + a.wsq[n + kM];
    s_rw[n] = s > SETK_TINY32 ? 1.0f / s : 1.0f;
  }
  if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); }
  for (int k = tid; k < NPAIR; k += blockDim.x) s_tw[k] = split_twiddle(k);
  float w1s, w1c;
  sincospif((float)lane16 / 128.0f, &w1s, &w1c);
  const float2 w1 = make_float2(w1c, -w1s);
  const bool vec_ok = ((a.N & 3) == 0) && ((hop & 3) == 0) && ((pad & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.audio) & 15) == 0);
  const bool fast_hop = (hop == kM);               // 50 % overlap: every position has two frames
  const bool out_vec = ((a.n_out & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.wave) & 15) == 0);

  // ---- inverse FFT of the frames of the pending tile (warps 8, 9) ----
  auto ifft_tile = [&](int p_nt) {
    const int job = (warp - 8) * 2 + half;         // frame inside the tile
    float2 v[16];
    float2* zi = s_zi + job * SETK_ZSLOT;
    if (job < p_nt) {                              // ONE branch per job, not one per load
#pragma unroll
      for (int m1 = 0; m1 < 16; ++m1) {
        const float2 x = zi[16 * m1 + lane16];
        v[m1] = make_float2(x.x, -x.y);
      }
    } else {
#pragma unroll
      for (int m1 = 0; m1 < 16; ++m1) v[m1] = make_float2(0.f, 0.f);
    }
    __syncwarp();                                  // slot is free: reuse it as the exchange tile
    halfwarp_fft256(v, zi, lane16, w1);
    float* fr = s_frames + job * kNfft;
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      const int m = lane16 + 16 * kof(s);
      const float2 ws = *reinterpret_cast<const float2*>(s_wsyn + 2 * m);
      *reinterpret_cast<float2*>(fr + 2 * m) = make_float2(v[s].x * ws.x, -v[s].y * ws.y);
    }
  };

  // ---- flush of a finished tile: overlap-add, normalise, trim, write ----
  int cur = 0;                                     // which carry buffer is the input
  auto flush_tile = [&](int p_t0, int p_nt) {
    const int p_tile = p_t0 * hop;
    const bool last_tile = (p_t0 + p_nt == T_used);
    const float* cin = s_carry + cur * carry_len;
    float* cout = s_carry + (cur ^ 1) * carry_len;
    // interior tile of a 50 %-overlap transform: every row is owned, inside the output, has two
    // frames and a following tile takes the last half frame -- one check per tile, none per sample
    const bool interior = fast_hop && out_vec && !a.accumulate && p_nt == TT && !last_tile &&
                          p_t0 >= 1 && p_t0 + p_nt < T_used && p_tile >= own_begin && p_tile >= pad &&
                          p_tile - pad + p_nt * kM <= n_lim;
    if (interior) {
      static_assert((TT + 1) * (kM / 4) == kApplyThreads, "one flush item per thread");
      const int jj = tid >> 6, r = (tid & 63) * 4;
      float4 val = jj >= 1 ? *reinterpret_cast<const float4*>(s_frames + (jj - 1) * kNfft + kM + r)
                           : *reinterpret_cast<const float4*>(cin + r);
      if (jj < TT) {
        const float4 f = *reinterpret_cast<const float4*>(s_frames + jj * kNfft + r);
        const float4 rw = *reinterpret_cast<const float4*>(s_rw + r);
        val.x = (val.x + f.x) * rw.x; val.y = (val.y + f.y) * rw.y;
        val.z = (val.z + f.z) * rw.z; val.w = (val.w + f.w) * rw.w;
        *reinterpret_cast<float4*>(yb + (p_tile - pad + jj * kM + r)) = val;
        peak = fmaxf(peak, fmaxf(fmaxf(fabsf(val.x), fabsf(val.y)), fmaxf(fabsf(val.z), fabsf(val.w))));
      } else {
        *reinterpret_cast<float4*>(cout + r) = val;
      }
    } else if (fast_hop) {
      // rows of 256 positions; row jj gets frame jj (n = r) and frame jj-1 (n = r + 256).
      // Four consecutive positions per thread: 16-byte shared loads and (when the
      // output rows allow it) 16-byte global stores; pad and own_begin are multiples
      // of 256 here, so the four share every row condition
      for (int item = tid; item < (p_nt + 1) * (kM / 4); item += blockDim.x) {
        const int jj = item >> 6, r = (item & 63) * 4;
        float4 val = jj >= 1 ? *reinterpret_cast<const float4*>(s_frames + (jj - 1) * kNfft + kM + r)
                             : *reinterpret_cast<const float4*>(cin + r);
        if (jj < p_nt) {
          const float4 f = *reinterpret_cast<const float4*>(s_frames + jj * kNfft + r);
          val.x += f.x; val.y += f.y; val.z += f.z; val.w += f.w;
        }
        if (jj < p_nt || last_tile) {
          const int p = p_tile + jj * kM + r;
          const int q = p - pad;
          if (p >= own_begin && q >= 0 && q < n_lim) {
            const int t = p_t0 + jj;               // frame starting at this row
            float vv[4] = {val.x, val.y, val.z, val.w};
            if (t >= 1 && t < T_used) {
              const float4 rw = *reinterpret_cast<const float4*>(s_rw + r);
              vv[0] *= rw.x; vv[1] *= rw.y; vv[2] *= rw.z; vv[3] *= rw.w;
            } else {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float wss = (t < T_used ? s_wsq[r + i] : 0.f) + (t >= 1 ? s_wsq[kM + r + i] : 0.f);
                if (wss > SETK_TINY32) vv[i] /= wss;
              }
            }
            if (out_vec && q + 4 <= n_lim) {
              float4* dst = reinterpret_cast<float4*>(yb + q);
              if (a.accumulate) {
                const float4 o = *dst;
                vv[0] += o.x; vv[1] += o.y; vv[2] += o.z; vv[3] += o.w;
              }
              *dst = make_float4(vv[0], vv[1], vv[2], vv[3]);
              peak = fmaxf(peak, fmaxf(fmaxf(fabsf(vv[0]), fabsf(vv[1])), fmaxf(fabsf(vv[2]), fabsf(vv[3]))));
            } else {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                if (q + i < n_lim) {
                  float v1 = vv[i];
                  if (a.accumulate) v1 += yb[q + i];
                  yb[q + i] = v1;
                  peak = fmaxf(peak, fabsf(v1));
                }
              }
            }
          }
        } else {
          *reinterpret_cast<float4*>(cout + r) = val;
        }
      }
    } else {
      const int span = (p_nt - 1) * hop + kNfft;         // positions touched by this tile
      const int final_len = last_tile ? span : p_nt * hop;
      for (int jj = 0; jj * hop < span; ++jj) {          // hop-sized rows of positions
        const int rmax = imin(hop, span - jj * hop);
        for (int r = tid; r < rmax; r += blockDim.x) {
          const int rel = jj * hop + r;
          float val = rel < carry_len ? cin[rel] : 0.f;
          float wss = 0.f;
          // frames t = (p_t0 + jj) - d overlap position p at sample n = r + d*hop
          for (int d = 0, n = r; n < kNfft; ++d, n += hop) {
            const int j = jj - d;                        // index inside this tile
            const int t = p_t0 + j;                      // absolute frame
            if (j >= 0 && j < p_nt) val += s_frames[j * kNfft + n];
            if (t >= 0 && t < T_used) wss += s_wsq[n];
          }
          if (rel < final_len) {
            const int p = p_tile + rel;
            const int q = p - pad;
            if (p >= own_begin && q >= 0 && q < n_lim) {
              if (wss > SETK_TINY32) val /= wss;
              if (a.accumulate) val += yb[q];
              yb[q] = val;
              peak = fmaxf(peak, fabsf(val));
            }
          } else {
            cout[rel - p_nt * hop] = val;
          }
        }
      }
    }
    cur ^= 1;
  };

  const int R = (kNfft + hop - 1) / hop - 1;       // frames before t that overlap frame t
  unsigned par = 0;
  float amax_unused = 0.f;
  int buf = 0;
  b = sched_find(a.sched, cur_tile);
  while (cur_tile < hi_tile) {
    // ---- next segment: the part of utterance b inside [cur_tile, hi_tile) ----
    int pb = sched_prefix(a.sched, b), pe = sched_prefix(a.sched, b + 1);
    while (pe <= cur_tile) { ++b; pb = pe; pe = sched_prefix(a.sched, b + 1); }
    const int seg_end = imin(hi_tile, pe);
    nb = a.n_samples ? a.n_samples[b] : a.N;
    const int Tb = frames_of(nb, kNfft, hop, pad);
    T_used = imin(Tb, T_cap);
    const int t_begin = (cur_tile - pb) * TT;
    const int t_end = imin((seg_end - pb) * TT, T_used);
    const int expected = T_used > 0 ? kNfft + hop * (T_used - 1) : 0;   // padded signal length
    // a ragged utterance ends where its own istft(length=None) would (center: the trailing
    // n_fft/2 is trimmed); what lies beyond is zero-filled and must not reach the peak
    n_lim = a.n_samples ? imin(a.n_out, imax(expected - 2 * pad, 0)) : a.n_out;
    own_begin = t_begin * hop;
    yb = a.wave + (long long)b * a.n_out;
    const float* xb = a.audio + ((long long)b * a.c_total + a.c0) * a.N;

    __syncthreads();   // the previous segment's last flush has read carry / frames / weights
    for (int n = tid; n < 2 * carry_len; n += blockDim.x) s_carry[n] = 0.f;
    cur = 0;
    for (int e = tid; e < F * C; e += blockDim.x) {
      const int k = e / C, c = e - k * C;
      const long long wi = ((long long)b * F + k) * a.c_total + a.c0 + c;
      float2 v;
      if (a.w_dtype == SETK_C128) {
        const double* p = reinterpret_cast<const double*>(a.w) + 2 * wi;
        v = make_float2((float)p[0], (float)p[1]);
      } else {
        const float* p = reinterpret_cast<const float*>(a.w) + 2 * wi;
        v = make_float2(p[0], p[1]);
      }
      s_w[c * kWPitch + k] = v;
    }

    // tile sequence: an optional halo tile [t_begin-R, t_begin), then full tiles
    int t0 = imax(0, t_begin - R);
    if (t_begin >= t_end) t0 = t_end;                // nothing to do for this segment
    int nt = (t0 < t_begin) ? (t_begin - t0) : imin(TT, t_end - t0);
    bool async_cur = false;
    if (t0 < t_end) async_cur = stage_tile_begin<C, TT>(sm, buf, xb, a.N, nb, t0, nt, hop, pad, vec_ok);
    int prev_t0 = 0, prev_nt = 0;                    // tile whose Zi is waiting for its inverse FFT
    while (t0 < t_end) {
      const int t_next = t0 + nt;
      const int nt_next = imin(TT, t_end - t_next);
      __syncthreads();   // phase B of the previous tile is complete
      bool async_next = false;
      if (t_next < t_end)
        async_next = stage_tile_begin<C, TT>(sm, buf ^ 1, xb, a.N, nb, t_next, nt_next, hop, pad, vec_ok);
      if (async_cur) {
        mbar_wait(&sm.bar[buf], (par >> buf) & 1u);
        par ^= 1u << buf;
      }
      // ---- phase A: forward FFT of this tile || inverse FFT of the previous one ----
      if (warp < 8) {
        fft_tile<C, TT, false, 8>(sm, buf, nt, hop, w1, amax_unused, nullptr);
      } else if (prev_nt > 0) {
        ifft_tile(prev_nt);
      }
      __syncthreads();
      // ---- phase B: apply + inverse split of this tile ----
      // thread = (bin pair k, frame parity g): the pair's weights and twiddle are
      // loaded once and serve frames g, g + 2
      if (tid < 2 * NPAIR) {
        const int g = tid >= NPAIR ? 1 : 0;
        const int k = tid - g * NPAIR;
        const int km = kM - k;                              // mirrored bin 256-k
        const float2 tw = s_tw[k];
        float2 wk[C], wm[C];
#pragma unroll
        for (int c = 0; c < C; ++c) { wk[c] = s_w[c * kWPitch + k]; wm[c] = s_w[c * kWPitch + km]; }
        // one (pair, frame) item; a full tile is two straight-line items per thread (frames g, g + 2)
        auto item = [&](int j, auto pm_tag) {      // pm_tag: post-mask or not, decided per tile, not per item
          float2 yk = make_float2(0.f, 0.f), ym = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < C; ++c) {
            const float2* z = sm.z + (j * C + c) * SETK_ZSLOT;
            float2 xk, xm;
            // (k = 0: zk = zn = Z[0] and tw = (-0, -1) give X[0], X[256] with imaginary parts that are
            // exact zeros for finite data -- no special case, as in the covariance kernels)
            split_pair(z[k & (kM - 1)], z[km & (kM - 1)], tw, xk, xm);
            yk = cmad_conjw(wk[c], xk, yk);                    // += conj(w) x
            ym = cmad_conjw(wm[c], xm, ym);
          }
          if constexpr (decltype(pm_tag)::value) {
            const float* pm = a.post_mask + ((long long)b * a.T + (t0 + j)) * F;
            const float mk = pm[k], mm = pm[km];
            yk = f2mul(yk, make_float2(mk, mk)); ym = f2mul(ym, make_float2(mm, mm));
          }
          float2* zi = s_zi + j * SETK_ZSLOT;
          if (k == 0) {
            // irfft ignores Im Y[0], Im Y[256]
            zi[0] = make_float2(yk.x + ym.x, yk.x - ym.x);
          } else {
            // Zi[k]   = (Yk + conj(Ym)) + conj(tw) (Yk - conj(Ym))
            const float2 cm = make_float2(ym.x, -ym.y);
            const float2 e = f2add(yk, cm), d = f2sub(yk, cm);
            const float2 p = cmul_conj(d, tw);                 // conj(tw) D
            zi[k] = f2add(e, p);
            if (k != kM / 2) {
              // Zi[256-k] = (Ym + conj(Yk)) + tw (Ym - conj(Yk)) = conj(E) - tw conj(D) = conj(E - conj(tw) D)
              const float2 qq = f2sub(e, p);
              zi[km] = make_float2(qq.x, -qq.y);
            }
          }
        };
        if (nt == TT && !a.post_mask) {
          item(g, std::false_type{});
          item(g + 2, std::false_type{});
        } else if (a.post_mask) {
          for (int j = g; j < nt; j += 2) item(j, std::true_type{});
        } else {
          for (int j = g; j < nt; j += 2) item(j, std::false_type{});
        }
      }
      // ---- phase B: flush of the previous tile (its frames were made in phase A) ----
      if (prev_nt > 0) flush_tile(prev_t0, prev_nt);
      prev_t0 = t0; prev_nt = nt;
      t0 = t_next;
      nt = nt_next;
      async_cur = async_next;
      buf ^= 1;
    }
    // ---- drain the pipeline: the last tile's inverse FFT and flush ----
    if (prev_nt > 0) {
      __syncthreads();
      if (warp >= 8) ifft_tile(prev_nt);
      __syncthreads();
      flush_tile(prev_t0, prev_nt);
    }

    // zero-fill what no frame reaches (fix_length padding / too-short input)
    if (t_end >= T_used && !a.accumulate) {
      const int q0 = a.n_samples ? n_lim : imax(expected - pad, 0);
      for (int qq = q0 + tid; qq < a.n_out; qq += blockDim.x) yb[qq] = 0.f;
    }
    if (a.peak) {
      for (int o = 16; o > 0; o >>= 1) peak = fmaxf(peak, __shfl_xor_sync(0xffffffffu, peak, o));
      if (lane == 0 && peak > 0.f) atomicMax(a.peak + b, __float_as_uint(peak));
      peak = 0.f;
    }
    cur_tile = seg_end;
  }
}

template <int C, int TT>
static size_t apply_istft_smem_bytes(int hop) {
  size_t fl = TileSmem<C, TT>::floats(hop);
  fl += 2 * (size_t)C * kWPitch;          // s_w
  fl += 2 * (size_t)TT * SETK_ZSLOT;      // s_zi
  fl += 2 * (size_t)(kM / 2 + 2);         // s_tw
  fl += (size_t)TT * kNfft;               // s_frames
  fl += 2 * (size_t)kNfft;                // s_wsyn, s_wsq
  fl += (size_t)kM;                       // s_rw
  fl += 2 * (size_t)(kNfft - hop);        // carry x2
  return fl * sizeof(float);
}

template <int C, int TT>
static cudaError_t run_apply_istft_t(const ApplyIstftArgs& a, int n_ctas, void* stream) {
  const size_t smem = apply_istft_smem_bytes<C, TT>(a.g.hop);
  cudaError_t e = cudaFuncSetAttribute(apply_istft_kernel<C, TT>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch(apply_istft_kernel<C, TT>, dim3(n_ctas), dim3(kApplyThreads), smem, stream, false, a);
}

bool apply_istft_fused_supported(const Geometry& g) {
  if (g.n_fft != 512) return false;
  if (g.C < 1 || g.C > SETK_MAX_CHANNELS) return false;   // C > 4: channel blocks of <= 4, accumulated
  if (g.hop < 128 || g.hop > 512 || (g.hop & 1)) return false;   // halo <= TT frames
  return true;
}

// Warp-specialised builds of this pass (FFT / apply+flush / inverse-FFT roles on mbarrier rings) were
// slower than this kernel (DESIGN.md K4+K5): four short stages per frame make the hand-overs cost more
// than the two barriers they replace.  They are not part of the library.
cudaError_t run_apply_istft_fused(setk_plan* pl, const float* audio, const int* n_samples, int B, int N,
                                  int T, const void* w, int w_dtype, const float* post_mask, int n_out,
                                  int* tile_prefix, float* wave, unsigned* peak, void* stream) {
  constexpr int TT = 4;
  ApplyIstftArgs a;
  a.g = pl->geo;
  a.audio = audio; a.n_samples = n_samples; a.N = N;
  a.w = w; a.w_dtype = w_dtype;
  a.post_mask = post_mask; a.T = T;
  // persistent schedule over the frames librosa.istft uses for this output length
  int n_ctas, slots_unused;
  cudaError_t e = fused_schedule(pl, B, T, TT, istft_frame_cap(a.g, n_out), n_samples, tile_prefix, stream,
                                 &a.sched, &n_ctas, &slots_unused);
  if (e != cudaSuccess) return e;
  a.window = pl->d_window;
  a.wsq = pl->d_wsq;
  a.n_out = n_out;
  a.wave = wave;
  // channel blocks of <= 4: the first block writes, the others accumulate; the
  // peak is taken by the last block (it sees the complete sums)
  const int Ctot = pl->geo.C;
  a.c_total = Ctot;
  for (int c0 = 0; c0 < Ctot && e == cudaSuccess; c0 += 4) {
    const int cb = Ctot - c0 < 4 ? Ctot - c0 : 4;
    a.c0 = c0;
    a.accumulate = c0 > 0;
    a.peak = (c0 + cb >= Ctot) ? peak : nullptr;
    switch (cb) {
      case 1: e = run_apply_istft_t<1, TT>(a, n_ctas, stream); break;
      case 2: e = run_apply_istft_t<2, TT>(a, n_ctas, stream); break;
      case 3: e = run_apply_istft_t<3, TT>(a, n_ctas, stream); break;
      default: e = run_apply_istft_t<4, TT>(a, n_ctas, stream); break;
    }
  }
  return e;
}

}  // namespace setk
