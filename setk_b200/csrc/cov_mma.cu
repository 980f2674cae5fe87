// cov_mma.cu -- mask-weighted spatial covariance for C >= 5 channels on the TENSOR CORES.
//
// Replaces compute_covar (scripts/sptk/libs/beamformer.py:87-103; C++ twin EstimatePsd,
// include/beamformer.cc:91-120) where the per-bin update stops being a handful of rank-1 terms
// and becomes a real dense contraction (north_star: "tensor cores only where C >= 8 makes it a
// real dense contraction"; used from C = 5, padded to 8 or 16 channels):
//
//   per bin f, with u_t = [Re x_t ; Im x_t] (2C real components of frame t)
//       G = sum_t  m_t u_t u_t^T            (2C x 2C real Gram matrix over the T frames)
//       Re R = G_rr + G_ii ,  Im R = G_ir - G_ri
//   = a [2C x T] . [T x 2C] matrix product per bin and mask: mma.sync.m16n8k8 TF32 with the
//   3xTF32 operand split (mma_tf32.cuh), i.e. fp32-accurate products, fp32 accumulators.
//
// Input is the bin-major STFT workspace of the tile STFT (stft_spill.cu): Xws[b][t][c][pitch].
// Why the STFT round trip stays for C > 4: the accumulator state of one utterance is
// 257 bins x 2 masks x (2C)^2 fp32 = 131 KB (C = 8) / 526 KB (C = 16) -- more than the register
// file or shared memory of an SM can hold next to the FFT -- so frames must be revisited bin by bin.
//
// Mapping: CTA = 8 warps = NB bins x one chunk of frames of one utterance; per step of 8 frames
//   stage   8 frames x C channels x NB bins, 8-byte cp.async (zero-filled past the utterance),
//           bin-major in shared memory (pitch 8*CP+1: conflict-free both ways), a ring of four
//           steps (three in flight); the step's raw mask values by 4-byte cp.async (clip and
//           1 - m at use) -- round 2's first build double-buffered and fetched the masks with
//           ordinary loads: every step then waited out one DRAM latency (0.49 ms per 64 x 8 ch)
//   mma     warp w owns bins [w*BPW, (w+1)*BPW): lane (g, q) reads channel g (and g+8) of frames
//           q and q+4 -- exactly its A and B fragment elements -- splits them and issues
//           12 (C <= 8) or 48 (C <= 16) HMMA per bin for both masks
//   end     R entries are sums / differences of accumulators of the SAME thread; they go to the
//           partial-sum workspace of cov_spill_finalize_kernel (stft_spill.cu), which combines
//           the chunks in fp64 and normalises by max(sum m, 1e-6).
#include "common.cuh"
#include "async_copy.cuh"
#include "cov_spill_args.cuh"
#include "launchers.cuh"
#include "mma_tf32.cuh"

namespace setk {

template <int CP>
struct CovMmaShape {
  static constexpr int BPW = CP == 8 ? 4 : 1;      // bins per warp (64 accumulator registers either way)
  static constexpr int NB = 8 * BPW;               // bins per CTA
  static constexpr int BP = 8 * CP + 1;            // float2 pitch of one bin's [8 frames][CP channels]
  static constexpr int MT = CP / 8;                // 16-row blocks of Re (and of Im) components
  static constexpr int NS = 4;                     // cp.async ring depth: three steps in flight
  static constexpr size_t smem_bytes() {
    return sizeof(float2) * NS * NB * BP + sizeof(float) * NS * 2 * 8 * NB;
  }
};

#ifdef SETK_EMU
__device__ inline void cp_async_8_zfill(void* dst, const void* src, bool valid) {
  if (valid) memcpy(dst, src, 8); else memset(dst, 0, 8);
}
__device__ inline void cp_async_4_zfill(void* dst, const void* src, bool valid) {
  if (valid) memcpy(dst, src, 4); else memset(dst, 0, 4);
}
__device__ inline void cp_async_wait_group2() {}
#else
__device__ __forceinline__ void cp_async_8_zfill(void* dst, const void* src, bool valid) {
  const unsigned n = valid ? 8u : 0u;              // src-size 0: the 8 bytes are zero-filled
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n)
               : "memory");
}
__device__ __forceinline__ void cp_async_4_zfill(void* dst, const void* src, bool valid) {
  const unsigned n = valid ? 4u : 0u;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(n)
               : "memory");
}
// all but the two most recently committed groups have landed
__device__ __forceinline__ void cp_async_wait_group2() { asm volatile("cp.async.wait_group 2;" ::: "memory"); }
#endif

template <int CP>
__global__ void __launch_bounds__(256) cov_mma_kernel(CovSpillArgs a) {
  using S = CovMmaShape<CP>;
  constexpr int BPW = S::BPW, NB = S::NB, BP = S::BP, MT = S::MT, NS = S::NS;
  static_assert(NS == 4, "the wait below leaves NS - 2 = 2 groups in flight");
  SETK_DYN_SMEM(float2, smem);
  float2* xs = smem;                                            // [NS][NB][BP]
  float* msk = reinterpret_cast<float*>(xs + NS * NB * BP);     // [NS][2 (s, n)][8][NB], raw mask values

  const int C = a.g.C, F = a.F;
  const int nbb = (F + NB - 1) / NB;
  const int chunk = blockIdx.x / nbb, f0 = (blockIdx.x - chunk * nbb) * NB, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, q = lane & 3;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(imin(t_begin + a.frames_per_chunk, a.T), Tb);
  const int nk = t_end > t_begin ? (t_end - t_begin + 7) / 8 : 0;
  const bool has_mn = a.mask_n != nullptr;
  const bool clip = (a.flags & SETK_F_CLIP_MASK) != 0;
  const long long m_fs = (a.flags & SETK_F_MASK_FT) ? a.T : 1;
  const long long m_ts = (a.flags & SETK_F_MASK_FT) ? 1 : F;
  const long long pitch = a.pitch;
  const float2* xb = a.xws + ((long long)b * a.T * C) * pitch + f0;
  const float* msb = a.mask_s + (long long)b * a.T * F;
  const float* mnb = has_mn ? a.mask_n + (long long)b * a.T * F : nullptr;

  // One step = 8 frames x CP channels x NB bins of the workspace + the step's raw mask values, all by
  // cp.async (nothing a thread has to wait for at issue time).  A thread keeps its (bin, channel)
  // and walks the frames: pointers advance by constants.
  constexpr int EPT = 8 * CP * NB / 256;           // workspace elements per thread and step
  constexpr int TSTEP = 256 / (CP * NB) > 0 ? 256 / (CP * NB) : 1;   // frames covered by one pass of the CTA
  static_assert(EPT * TSTEP == 8 || (CP * NB >= 256 && EPT == 8), "frame walk of the staging loop");
  const int s_bin = tid % NB, s_c = (tid / NB) % CP, s_t = tid / (NB * CP);
  const bool s_ok = s_c < C && f0 + s_bin < F;
  const int m_bin = tid % NB, m_t = tid / NB;                        // masks: 8 * NB <= 256 values
  // running source pointers: the steps are staged in order, so every call advances them by 8 frames
  const long long walk = (long long)TSTEP * C * pitch;               // float2 between this thread's frames
  const float2* src_next = xb + ((long long)(t_begin + s_t) * C + s_c) * pitch + s_bin;
  const long long m_off = (long long)(t_begin + m_t) * m_ts + (long long)(f0 + m_bin) * m_fs;
  const float* ms_next = msb + m_off;
  const float* mn_next = has_mn ? mnb + m_off : nullptr;
  const bool m_ok = tid < 8 * NB && f0 + m_bin < F;
  float2* const dst0 = xs + s_bin * BP + s_t * CP + s_c;
  float* const md0 = msk + m_t * NB + m_bin;
  int t_next = t_begin;                                              // first frame of the next step
  auto stage = [&](int buf) {
    float2* dst = dst0 + buf * NB * BP;
    const float2* src = src_next;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const bool ok = s_ok && t_next + s_t + i * TSTEP < t_end;
      cp_async_8_zfill(dst + i * TSTEP * CP, ok ? src : a.xws, ok);
      src += walk;
    }
    src_next = src;
    if (tid < 8 * NB) {
      const bool ok = m_ok && t_next + m_t < t_end;
      float* md = md0 + buf * 2 * 8 * NB;
      cp_async_4_zfill(md, ok ? ms_next : a.mask_s, ok);
      if (has_mn) cp_async_4_zfill(md + 8 * NB, ok ? mn_next : a.mask_n, ok);
    }
    ms_next += 8 * m_ts;
    if (has_mn) mn_next += 8 * m_ts;
    t_next += 8;
  };

  // accumulators [bin of this warp][mask][m-tile: Re rows, Im rows][n-tile][4]
  //   CP = 8 : one m-tile (rows g = Re ch g, g + 8 = Im ch g), n-tiles {Re ch, Im ch}
  //   CP = 16: m-tiles {Re ch g / g+8, Im ch g / g+8}, n-tiles {Re 0-7, Re 8-15, Im 0-7, Im 8-15}
  constexpr int NMT = CP == 8 ? 1 : 2, NNT = CP == 8 ? 2 : 4;
  float acc[BPW][2][NMT][NNT][4];
  float sum_s[BPW], sum_n[BPW];
#pragma unroll
  for (int i = 0; i < BPW; ++i) {
    sum_s[i] = 0.f; sum_n[i] = 0.f;
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int mt = 0; mt < NMT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NNT; ++nt)
#pragma unroll
          for (int r = 0; r < 4; ++r) acc[i][m][mt][nt][r] = 0.f;
  }

  // ring of NS steps: NS - 1 are in flight while one is consumed (one commit group per step, empty
  // groups past the end keep the count uniform)
#pragma unroll
  for (int p = 0; p < NS - 1; ++p) {
    if (p < nk) stage(p);
    cp_async_commit();
  }
  for (int ks = 0; ks < nk; ++ks) {
    cp_async_wait_group2();
    __syncthreads();                       // step ks has landed; everyone is done with step ks - 1
    if (ks + NS - 1 < nk) stage((ks + NS - 1) % NS);
    cp_async_commit();
    const float2* xt = xs + (ks % NS) * NB * BP;
    const float* md = msk + (ks % NS) * 2 * 8 * NB;
    const int live = t_end - (t_begin + 8 * ks);            // frames of this step inside the utterance
    const bool v0 = q < live, v1 = q + 4 < live;
#pragma unroll
    for (int i = 0; i < BPW; ++i) {
      const int bin = warp * BPW + i;
      const float2* xbin = xt + bin * BP;
      float s0 = md[q * NB + bin], s1 = md[(q + 4) * NB + bin];   // raw (zero past the utterance)
      if (clip) { s0 = fminf(s0, 1.0f); s1 = fminf(s1, 1.0f); }
      const float n0 = has_mn ? md[(8 + q) * NB + bin] : (v0 ? 1.0f - s0 : 0.f);
      const float n1 = has_mn ? md[(12 + q) * NB + bin] : (v1 ? 1.0f - s1 : 0.f);
      if (g == 0) { sum_s[i] += s0 + s1; sum_n[i] += n0 + n1; }
      if (CP == 8) {
        const float2 x0 = xbin[q * CP + g], x1 = xbin[(q + 4) * CP + g];
        unsigned bh[2][2], bl[2][2];       // [n-tile: Re, Im][b0 (frame q), b1 (frame q + 4)]
        tf32_split(x0.x, bh[0][0], bl[0][0]); tf32_split(x1.x, bh[0][1], bl[0][1]);
        tf32_split(x0.y, bh[1][0], bl[1][0]); tf32_split(x1.y, bh[1][1], bl[1][1]);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const float w0 = m == 0 ? s0 : n0, w1 = m == 0 ? s1 : n1;
          unsigned ah[4], al[4];           // a0 (Re, q) a1 (Im, q) a2 (Re, q+4) a3 (Im, q+4)
          tf32_split(w0 * x0.x, ah[0], al[0]); tf32_split(w0 * x0.y, ah[1], al[1]);
          tf32_split(w1 * x1.x, ah[2], al[2]); tf32_split(w1 * x1.y, ah[3], al[3]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_3xtf32(acc[i][m][0][nt], ah, al, bh[nt], bl[nt]);
        }
      } else {
        const float2 x00 = xbin[q * CP + g], x01 = xbin[q * CP + g + 8];
        const float2 x10 = xbin[(q + 4) * CP + g], x11 = xbin[(q + 4) * CP + g + 8];
        unsigned bh[4][2], bl[4][2];       // n-tiles: Re ch g, Re ch g+8, Im ch g, Im ch g+8
        tf32_split(x00.x, bh[0][0], bl[0][0]); tf32_split(x10.x, bh[0][1], bl[0][1]);
        tf32_split(x01.x, bh[1][0], bl[1][0]); tf32_split(x11.x, bh[1][1], bl[1][1]);
        tf32_split(x00.y, bh[2][0], bl[2][0]); tf32_split(x10.y, bh[2][1], bl[2][1]);
        tf32_split(x01.y, bh[3][0], bl[3][0]); tf32_split(x11.y, bh[3][1], bl[3][1]);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const float w0 = m == 0 ? s0 : n0, w1 = m == 0 ? s1 : n1;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {   // 0: Re rows (ch g, ch g+8), 1: Im rows
            const float v00 = mt == 0 ? x00.x : x00.y, v01 = mt == 0 ? x01.x : x01.y;
            const float v10 = mt == 0 ? x10.x : x10.y, v11 = mt == 0 ? x11.x : x11.y;
            unsigned ah[4], al[4];
            tf32_split(w0 * v00, ah[0], al[0]); tf32_split(w0 * v01, ah[1], al[1]);
            tf32_split(w1 * v10, ah[2], al[2]); tf32_split(w1 * v11, ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) mma_3xtf32(acc[i][m][mt][nt], ah, al, bh[nt], bl[nt]);
          }
        }
      }
    }
  }

  // ---- R entries of this thread -> partial sums [B][n_chunks][C rows][2][2C + 1][F] ----
  const int W = 2 * C + 1;
#pragma unroll
  for (int i = 0; i < BPW; ++i) {
    const int f = f0 + warp * BPW + i;
    // mask sums: lanes with g == 0 hold frames q, q + 4 of every step
    float ss = sum_s[i], sn = sum_n[i];
    ss += __shfl_xor_sync(0xffffffffu, ss, 1); ss += __shfl_xor_sync(0xffffffffu, ss, 2);
    sn += __shfl_xor_sync(0xffffffffu, sn, 1); sn += __shfl_xor_sync(0xffffffffu, sn, 2);
    ss = __shfl_sync(0xffffffffu, ss, 0); sn = __shfl_sync(0xffffffffu, sn, 0);
    if (f >= F) continue;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      float* base = a.partials + ((((long long)b * a.n_chunks + chunk) * C) * 2 + m) * W * F + f;
      auto put = [&](int row, int col, float re, float im) {
        if (row < C && col < C) {
          float* pp = base + (long long)row * 2 * W * F;
          pp[(long long)(2 * col) * F] = re;
          pp[(long long)(2 * col + 1) * F] = im;
        }
      };
      if (CP == 8) {
        const float* dr = acc[i][m][0][0];      // columns Re ch j
        const float* di = acc[i][m][0][1];      // columns Im ch j
        put(g, 2 * q, dr[0] + di[2], dr[2] - di[0]);
        put(g, 2 * q + 1, dr[1] + di[3], dr[3] - di[1]);
      } else {
#pragma unroll
        for (int r = 0; r < 2; ++r)             // row channel g + 8 r  (c0/c1 vs c2/c3)
#pragma unroll
          for (int jj = 0; jj < 2; ++jj)        // column channels 2q + e + 8 jj
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int k = 2 * r + e;
              put(g + 8 * r, 2 * q + e + 8 * jj,
                  acc[i][m][0][jj][k] + acc[i][m][1][2 + jj][k],
                  acc[i][m][1][jj][k] - acc[i][m][0][2 + jj][k]);
            }
      }
      if (q == 0 && g < C) base[(long long)g * 2 * W * F + (long long)(2 * C) * F] = m == 0 ? ss : sn;
      if (CP == 16 && q == 0 && g + 8 < C)
        base[(long long)(g + 8) * 2 * W * F + (long long)(2 * C) * F] = m == 0 ? ss : sn;
    }
  }
}

int cov_mma_bins_per_cta(int C) { return C <= 8 ? CovMmaShape<8>::NB : CovMmaShape<16>::NB; }

template <int CP>
static cudaError_t run_cov_mma_t(const CovSpillArgs& a, int B, void* stream) {
  using S = CovMmaShape<CP>;
  const int nbb = (a.F + S::NB - 1) / S::NB;
  const size_t smem = S::smem_bytes();
  cudaError_t e = cudaFuncSetAttribute(cov_mma_kernel<CP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  return launch(cov_mma_kernel<CP>, dim3(a.n_chunks * nbb, B), dim3(256), smem, stream, false, a);
}

cudaError_t run_cov_mma(const CovSpillArgs& a, int B, void* stream) {
  return a.g.C <= 8 ? run_cov_mma_t<8>(a, B, stream) : run_cov_mma_t<16>(a, B, stream);
}

}  // namespace setk
