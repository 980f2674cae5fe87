// stft_cov_args.cuh -- launch arguments and accumulator bookkeeping shared by the two
// fused STFT + covariance kernels (stft_cov_fused.cu, stft_cov_ws.cu).
#pragma once
#include "common.cuh"
#include "stft_tile.cuh"

namespace setk {

// frames per tile of the fused pass at C channels.  5 at C = 2: 320 threads, 10 FFT warps (the tenth
// warp's registers are allocated either way at 288).  4 at odd C, where 5 would leave an odd number
// of half-warp jobs, and at C = 4, whose warp-specialised build runs 16 half-warp jobs per tile.
// The partial-sum workspace is sized and the kernels are launched with this schedule.
constexpr int stft_cov_tt(int C) { return C == 2 ? 5 : 4; }

template <int C>
struct CovAcc {
  static constexpr int NOFF = C * (C - 1) / 2;
  static constexpr int NACC = C * C;  // C real diagonals + NOFF complex
};

struct StftCovArgs {
  Geometry g;
  const float* audio; const int* n_samples; int N;
  const float* mask_s; const float* mask_n; unsigned flags;
  int T;                 // frames of an N-sample utterance (mask leading dim)
  TileSched sched;       // which (utterance, tile) pairs this CTA owns
  int slots;             // partial-sum slots per utterance
  const float* window;   // [n_fft]
  float* partials;       // [B][slots][2*C*C + 2][F]
  unsigned* maxabs_bits; // [B] or null
};

}  // namespace setk
