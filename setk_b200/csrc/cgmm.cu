// cgmm.cu -- CGMM time-frequency mask estimation (the mask producer of BASELINE
// config 3; SURVEY.md §8(f) rank 1).  Replaces, per utterance and frequency bin,
//   scripts/sptk/libs/cluster.py:94-130   Covariance (eigh, scaled + floored
//                                          eigenvalues, R^-1, log det)
//   scripts/sptk/libs/cluster.py:187-231  CgDistribution.update_parameters / log_pdf
//   scripts/sptk/libs/cluster.py:234-287  Cgmm.update / predict
//   scripts/sptk/libs/cluster.py:396-465  CgmmTrainer (K = 2 start or given posteriors)
//   scripts/sptk/estimate_cgmm_masks.py:36-60  K x F x T -> K x T x F float32
//
// Every bin is an independent EM problem, so the data stay bin-major:
//   X     c64  [B][T][C][P]   the tile STFT's workspace (stft_spill.cu), read-only
//   G, W  f64  [B][K][T][P]   posteriors gamma and M-step weights gamma M / phi
// and one EM iteration is three launches that each touch X at most once:
//   cgmm_cov_kernel     R_k <- sum_t W_k y y^H, sum_t G_k.  A CTA owns 64 bins and
//                       a run of frames; tiles of X go through shared memory once
//                       and the C(C+1)/2 Hermitian entries are dealt to thread
//                       groups, <= 10 per thread, both classes sharing a product.
//   cgmm_factor_kernel  thread per (b, k, f): fixed-order sum of the chunk partials,
//                       / max(sum gamma, eps), Jacobi eigh, eigenvalue scaling and
//                       floor, packed Hermitian R^-1 and log det  (fp64).
//   cgmm_estep_kernel   thread per (bin, frame lane), R^-1 of the CTA's bins in
//                       shared memory: phi_k = max(|y^H R_k^-1 y|, eps)/M, the
//                       posterior (log-sum-exp shifted), G and W for the next pass.
// All arithmetic after the complex64 STFT is fp64, as in the reference.
//
// The CACGMM (cluster.py:290-393, 468-535) runs the same three passes on the unit-norm
// observations z = y / n, n = max(|y|_2, eps), without a normalised copy of X: since
// z z^H = y y^H / n^2 and z^H B^-1 z = y^H B^-1 y / n^2, the covariance pass takes the weight
// W = gamma M / (kappa n^2), kappa = max(|y^H B^-1 y| / n^2, eps), which the E-step writes
// (ACG = true), and the start writes W = gamma M / n^2 (cacgmm_import_kernel).
#include "async_copy.cuh"
#include "common.cuh"
#include "jacobi_coop.cuh"
#include "launchers.cuh"

namespace setk {

// covariance pass: BINS bins per CTA; the upper triangle of R is cut into 2 x 2
// blocks over (row pair I, column pair J >= I) and every thread owns <= NBT of
// them, so four entries share four shared-memory loads:
//   C <= 4 : 64 bins x <= 3 groups of 1 block   (<= 192 threads)
//   C <= 8 : 32 bins x <= 5 groups of 2 blocks  (<= 160 threads)
//   C  > 8 : 32 bins x <= 18 groups of 2 blocks (<= 576 threads)
SETK_HD inline int cgmm_blocks(int C) { const int nb = (C + 1) / 2; return nb * (nb + 1) / 2; }
SETK_HD inline int cgmm_groups(int C, int NBT) { return (cgmm_blocks(C) + NBT - 1) / NBT; }
// packed Hermitian slots of a C x C matrix: [0, C) the real diagonal, then
// (re, im) of the entries above it in row-major order; C*C doubles in all
SETK_HD inline int cgmm_slot(int C, int i, int j) {   // i < j
  return C + 2 * (i * C - i * (i + 1) / 2 + (j - i - 1));
}

struct CgmmCovArgs {
  const float2* X; int P;
  const double* W;          // [B][K][T][P] or null: weight 1 (the K = 2 start)
  const double* G;          // [B][K][T][P] or null: sum gamma = number of frames
  const int* n_samples; int N; Geometry g;
  int T, K, k0;             // this launch accumulates classes k0 and k0 + 1
  int frames_per_chunk, n_chunks, tile_frames;
  double* part;             // [B][n_chunks][K][C*C + 1][F]
};

template <int BINS, int NBT, int MAXT>
__global__ void __launch_bounds__(MAXT) cgmm_cov_kernel(CgmmCovArgs a) {
  SETK_DYN_SMEM(double2, ys);                // [tile_frames][Cp][BINS], converted once per tile
  const int C = a.g.C, F = a.g.F;
  const int NB = (C + 1) / 2, Cp = 2 * NB;   // an odd C gets a zero row
  const int NBK = NB * (NB + 1) / 2;
  const int G = blockDim.x / BINS;
  double* ws = reinterpret_cast<double*>(ys + a.tile_frames * Cp * BINS);    // [2][tile][2][BINS]
  double* gsm = ws + 2 * a.tile_frames * 2 * BINS;                           // [2][tile][2][BINS] gamma
  float2* raw = reinterpret_cast<float2*>(gsm + 2 * a.tile_frames * 2 * BINS);  // [tile][Cp][BINS] in flight
  unsigned char* bi = reinterpret_cast<unsigned char*>(raw + a.tile_frames * Cp * BINS);
  unsigned char* bj = bi + 64;
  const int tid = threadIdx.x;
  const int bl = tid & (BINS - 1), grp = tid / BINS;
  const int nbb = (F + BINS - 1) / BINS;
  const int chunk = blockIdx.x / nbb, bin0 = (blockIdx.x - chunk * nbb) * BINS;
  const int b = blockIdx.y;
  const int bin = bin0 + bl;
  const bool live = bin < F;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = imin(frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad), a.T);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, Tb);
  const int k1 = a.k0 + 1 < a.K ? a.k0 + 1 : a.k0;     // a lone last class is computed twice
  if (tid < NBK) {                                     // block -> (I, J), row-major upper triangle
    int e = tid, i = 0;
    while (e >= NB - i) { e -= NB - i; ++i; }
    bi[tid] = (unsigned char)i; bj[tid] = (unsigned char)(i + e);
  }
  __syncthreads();
  // this thread's blocks: shared-memory row offsets of (2I, 2I+1) and (2J, 2J+1)
  int oa[NBT], ob[NBT];
  bool has[NBT];
#pragma unroll
  for (int n = 0; n < NBT; ++n) {
    const int blk = grp + n * G;
    has[n] = blk < NBK;
    oa[n] = has[n] ? 2 * bi[blk] * BINS : 0;
    ob[n] = has[n] ? 2 * bj[blk] * BINS : 0;
  }
  // acc[n][e][k]: block n, entry e = (row 2I + e/2, column 2J + e%2), class k
  double ar[NBT][4][2], ai[NBT][4][2];
#pragma unroll
  for (int n = 0; n < NBT; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) { ar[n][e][0] = ar[n][e][1] = ai[n][e][0] = ai[n][e][1] = 0.0; }
  double gs0 = 0.0, gs1 = 0.0;
  const long long P = a.P;
  const int f_ld = bin0 + bl;
  const bool f_ok = f_ld < F;
  // Tiles are pipelined: cp.async (LDGSTS) brings tile i+1 of X (raw complex64)
  // and of W into shared memory while tile i is being accumulated; every
  // thread converts the samples it copied itself to fp64 once per tile.
  // thread (bl, grp) owns bin bl of rows grp, grp + G, ... of each tile.
  auto issue = [&](int t0, int wb) {
    const int nt = imin(a.tile_frames, t_end - t0);
    if (f_ok) {
      for (int t = 0; t < nt; ++t) {
        const float2* xr = a.X + (((long long)b * a.T + t0 + t) * C) * P + f_ld;
        for (int c = grp; c < C; c += G) cp_async_8(raw + (t * Cp + c) * BINS + bl, xr + (long long)c * P);
      }
      if (a.W)
        for (int tk = grp; tk < 2 * nt; tk += G) {
          const int t = tk >> 1, k = (tk & 1) ? k1 : a.k0;
          cp_async_8(ws + (wb * a.tile_frames * 2 + tk) * BINS + bl,
                     a.W + (((long long)b * a.K + k) * a.T + t0 + t) * P + f_ld);
          cp_async_8(gsm + (wb * a.tile_frames * 2 + tk) * BINS + bl,
                     a.G + (((long long)b * a.K + k) * a.T + t0 + t) * P + f_ld);
        }
    }
    cp_async_commit();
  };
  if (!f_ok || !a.W) {                        // lanes past F and the weight-1 start: constants
    for (int q = grp; q < 2 * a.tile_frames * 2; q += G) { ws[q * BINS + bl] = 1.0; gsm[q * BINS + bl] = 1.0; }
  }
  if (!f_ok || Cp != C) {                     // zero samples for lanes past F and for the pad row
    for (int q = grp; q < a.tile_frames * Cp; q += G)
      if (!f_ok || (q % Cp) >= C) ys[q * BINS + bl] = make_double2(0.0, 0.0);
  }
  int wb = 0;
  if (t_begin < t_end) issue(t_begin, 0);
  for (int t0 = t_begin; t0 < t_end; t0 += a.tile_frames, wb ^= 1) {
    const int nt = imin(a.tile_frames, t_end - t0);
    cp_async_wait_all();                      // my own copies of this tile have landed
    __syncthreads();                          // everyone is done reading ys of the previous tile
    if (f_ok)
      for (int t = 0; t < nt; ++t)
        for (int c = grp; c < C; c += G) {
          const float2 v = raw[(t * Cp + c) * BINS + bl];
          ys[(t * Cp + c) * BINS + bl] = make_double2((double)v.x, (double)v.y);
        }
    if (t0 + a.tile_frames < t_end) issue(t0 + a.tile_frames, wb ^ 1);
    __syncthreads();
    const double* wt = ws + (wb * a.tile_frames * 2) * BINS + bl;
    const double* gt = gsm + (wb * a.tile_frames * 2) * BINS + bl;
    for (int t = 0; t < nt; ++t) {
      const double2* yt = ys + t * Cp * BINS + bl;
      const double w0 = wt[(2 * t) * BINS], w1 = wt[(2 * t + 1) * BINS];
#pragma unroll
      for (int n = 0; n < NBT; ++n) {
        if (has[n]) {
          double2 ya[2], yb[2];
          ya[0] = yt[oa[n]]; ya[1] = yt[oa[n] + BINS];
          yb[0] = yt[ob[n]]; yb[1] = yt[ob[n] + BINS];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const double2 u = ya[e >> 1], v = yb[e & 1];
            const double pr = u.x * v.x + u.y * v.y;       // y_i conj(y_j)
            const double pm = u.y * v.x - u.x * v.y;
            ar[n][e][0] += w0 * pr; ai[n][e][0] += w0 * pm;
            ar[n][e][1] += w1 * pr; ai[n][e][1] += w1 * pm;
          }
        }
      }
    }
    if (grp == G - 1)                          // the last group has the fewest blocks
      for (int t = 0; t < nt; ++t) { gs0 += gt[(2 * t) * BINS]; gs1 += gt[(2 * t + 1) * BINS]; }
  }
  if (!live) return;
  const int S = C * C + 1;
  double* p0 = a.part + ((((long long)b * a.n_chunks + chunk) * a.K + a.k0) * S) * F + bin;
  double* p1 = a.part + ((((long long)b * a.n_chunks + chunk) * a.K + k1) * S) * F + bin;
#pragma unroll
  for (int n = 0; n < NBT; ++n) {
    const int blk = grp + n * G;
    if (blk < NBK) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 2 * bi[blk] + (e >> 1), j = 2 * bj[blk] + (e & 1);
        if (i > j || j >= C) continue;                     // mirrored entry / the zero row
        if (i == j) {
          p0[(long long)i * F] = ar[n][e][0];
          p1[(long long)i * F] = ar[n][e][1];
        } else {
          const int s = cgmm_slot(C, i, j);
          p0[(long long)s * F] = ar[n][e][0]; p0[(long long)(s + 1) * F] = ai[n][e][0];
          p1[(long long)s * F] = ar[n][e][1]; p1[(long long)(s + 1) * F] = ai[n][e][1];
        }
      }
    }
  }
  if (grp == G - 1) {
    p0[(long long)(C * C) * F] = gs0;
    p1[(long long)(C * C) * F] = gs1;
  }
}

struct CgmmFactorArgs {
  const double* part; int n_chunks;
  const int* n_samples; int N; Geometry g;
  int B, T, K;
  int identity_class;        // >= 0: that class gets R = I (cluster.py:421-425)
  int update_alpha;
  double* Rinv;              // [B][K][C*C][F]
  double* logdet;            // [B][K][F]
  double* alpha;             // [B][K][F]
  unsigned* status;          // [B] or null
};

// One group of Coop<C>::GS threads per (b, k, f); 128 threads per CTA (one
// group per CTA under the CPU execution model, whose barriers are OS-level).
template <int C>
struct FactorCfg {
#ifdef SETK_EMU
  static constexpr int THREADS = Coop<C>::GS;
#else
  static constexpr int THREADS = 128;
#endif
  static constexpr int MPB = THREADS / Coop<C>::GS;      // matrices per CTA
};
template <int C>
__global__ void __launch_bounds__(FactorCfg<C>::THREADS) cgmm_factor_kernel(CgmmFactorArgs a) {
  using K = Coop<C>;
  constexpr int GS = K::GS, LD = K::LD, MPB = FactorCfg<C>::MPB;
  constexpr int S = C * C + 1;
  SETK_DYN_SMEM(double, sm);
  const int F = a.g.F;
  const int tid = threadIdx.x;
  const int grp = tid / GS, r = tid - grp * GS;
  cd* A = reinterpret_cast<cd*>(sm) + (size_t)grp * 2 * K::MAT;
  cd* V = A + K::MAT;
  double* rot = sm + (size_t)MPB * 4 * K::MAT + grp * K::ROT;
  const long long idx = (long long)blockIdx.x * MPB + grp;   // (b, k, f), f fastest
  const bool active = idx < (long long)a.B * a.K * F;
  const int f = active ? (int)(idx % F) : 0;
  const int k = active ? (int)((idx / F) % a.K) : 0;
  const int b = active ? (int)(idx / ((long long)F * a.K)) : 0;
  const bool row = active && r < C;
  double gsum = 0.0;
  if (row) {
    if (k == a.identity_class) {
      for (int j = 0; j < C; ++j) A[r * LD + j] = cd_make(r == j ? 1.0 : 0.0, 0.0);
    } else {
      cd acc[C];                                  // row r, columns >= r
#pragma unroll
      for (int j = 0; j < C; ++j) acc[j] = cd_make(0.0, 0.0);
      for (int ch = 0; ch < a.n_chunks; ++ch) {
        const double* p = a.part + ((((long long)b * a.n_chunks + ch) * a.K + k) * S) * F + f;
        gsum += p[(long long)(C * C) * F];
#pragma unroll
        for (int j = 0; j < C; ++j) {
          if (j == r) {
            acc[j].x += p[(long long)r * F];
          } else if (j > r) {
            const int sl = cgmm_slot(C, r, j);
            acc[j].x += p[(long long)sl * F];
            acc[j].y += p[(long long)(sl + 1) * F];
          }
        }
      }
      const double inv = 1.0 / fmax(gsum, SETK_EPS32_D);     // cluster.py:200-201
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (j == r) {
          A[r * LD + r] = cd_make(acc[j].x * inv, 0.0);
        } else if (j > r) {
          const cd v = cd_scale(acc[j], inv);
          A[r * LD + j] = v;
          A[j * LD + r] = cd_conj(v);                         // (R + R^H) / 2 of cluster.py:100-102
        }
      }
    }
  }
  __syncwarp();
  const bool ok = jacobi_coop<C>(A, V, rot, r, active);
  if (!row) return;
  if (!ok && r == 0 && a.status) atomicOr(a.status + b, (unsigned)SETK_ST_NO_CONVERGE);
  // eigenvalues scaled by the largest and floored (cluster.py:108-113)
  double wmax = A[0].x;
#pragma unroll
  for (int m = 1; m < C; ++m) wmax = fmax(wmax, A[m * LD + m].x);
  wmax = fmax(wmax, SETK_EPS32_D);
  double winv[C];
  double ld = 0.0;
#pragma unroll
  for (int m = 0; m < C; ++m) {
    const double v = fmax(A[m * LD + m].x / wmax, SETK_EPS32_D);
    ld += log(v);
    winv[m] = 1.0 / v;
  }
  // row r of R^-1 = V diag(1/w) V^H, columns >= r, in packed slots
  double* o = a.Rinv + (((long long)b * a.K + k) * (C * C)) * F + f;
  cd vr[C];
#pragma unroll
  for (int m = 0; m < C; ++m) vr[m] = cd_scale(V[r * LD + m], winv[m]);
#pragma unroll
  for (int j = 0; j < C; ++j) {
    if (j < r) continue;
    cd sacc = cd_make(0.0, 0.0);
#pragma unroll
    for (int m = 0; m < C; ++m) sacc = cd_add(sacc, cd_mulc(vr[m], V[j * LD + m]));
    if (j == r) {
      o[(long long)r * F] = sacc.x;
    } else {
      const int sl = cgmm_slot(C, r, j);
      o[(long long)sl * F] = sacc.x;
      o[(long long)(sl + 1) * F] = sacc.y;
    }
  }
  if (r == 0) {
    a.logdet[((long long)b * a.K + k) * F + f] = ld;
    if (a.update_alpha && k != a.identity_class) {
      const int nb = a.n_samples ? a.n_samples[b] : a.N;
      const int Tb = imin(frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad), a.T);
      a.alpha[((long long)b * a.K + k) * F + f] = gsum / (double)imax(Tb, 1);   // cluster.py:252
    }
  }
}

struct CgmmEstepArgs {
  const float2* X; int P;
  const double* Rinv; const double* logdet; const double* alpha;
  const int* n_samples; int N; Geometry g;
  int T, frames_per_chunk;
  double* G; double* W;      // [B][K][T][P]
};

// BL bins x (256 / BL) frame lanes per CTA; R^-1 of the BL bins in shared memory.
// ACG: the CACGMM's log-pdf and weight (cluster.py:311-337, 367-393) instead of the CGMM's.
template <int C, int K, int BL, bool ACG>
__global__ void __launch_bounds__(256) cgmm_estep_kernel(CgmmEstepArgs a) {
  SETK_DYN_SMEM(double, rs);                 // [K][C*C][BL]
  constexpr int L = 256 / BL, CC = C * C;
  const int F = a.g.F;
  const int tid = threadIdx.x;
  const int bl = tid % BL, lane = tid / BL;
  const int nbb = (F + BL - 1) / BL;
  const int chunk = blockIdx.x / nbb, bin0 = (blockIdx.x - chunk * nbb) * BL;
  const int b = blockIdx.y;
  const int bin = bin0 + bl;
  for (int q = tid; q < K * CC * BL; q += 256) {
    const int l = q % BL, ks = q / BL;       // ks = k * CC + slot
    const int f = bin0 + l;
    rs[q] = f < F ? a.Rinv[((long long)b * K * CC + ks) * F + f] : 0.0;
  }
  __syncthreads();
  if (bin >= F) return;
  const int nb = a.n_samples ? a.n_samples[b] : a.N;
  const int Tb = imin(frames_of(nb, a.g.n_fft, a.g.hop, a.g.pad), a.T);
  const int t_begin = chunk * a.frames_per_chunk;
  const int t_end = imin(t_begin + a.frames_per_chunk, Tb);
  double ld[K], al[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    ld[k] = a.logdet[((long long)b * K + k) * F + bin];
    al[k] = a.alpha[((long long)b * K + k) * F + bin];
  }
  const long long P = a.P;
  const double* r = rs + bl;
  // frames in flight per thread: R^-1 is read once for both.  ACG keeps one: its n^2 per frame would
  // otherwise push most C >= 5 instantiations further into local memory.
  constexpr int FR = ACG ? 1 : 2;
  constexpr bool PF = C <= 8;                // prefetch the next pair of frames (registers allow it)
  float2 nx[FR][PF ? C : 1];
  auto fetch = [&](int t) {
#pragma unroll
    for (int u = 0; u < FR; ++u) {
      const float2* xt = a.X + (((long long)b * a.T + imin(t + u * L, t_end - 1)) * C) * P + bin;
#pragma unroll
      for (int c = 0; c < C; ++c) nx[u][PF ? c : 0] = xt[(long long)c * P];
    }
  };
  if (PF && t_begin + lane < t_end) fetch(t_begin + lane);
#pragma unroll 1
  for (int t = t_begin + lane; t < t_end; t += FR * L) {
    double yr[FR][C], yi[FR][C];
    if (PF) {
#pragma unroll
      for (int u = 0; u < FR; ++u)
#pragma unroll
        for (int c = 0; c < C; ++c) { yr[u][c] = nx[u][PF ? c : 0].x; yi[u][c] = nx[u][PF ? c : 0].y; }
      if (t + FR * L < t_end) fetch(t + FR * L);
    } else {
#pragma unroll
      for (int u = 0; u < FR; ++u) {
        const float2* xt = a.X + (((long long)b * a.T + imin(t + u * L, t_end - 1)) * C) * P + bin;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const float2 v = xt[(long long)c * P];
          yr[u][c] = v.x; yi[u][c] = v.y;
        }
      }
    }
    double q[FR][K];
#pragma unroll
    for (int u = 0; u < FR; ++u)
#pragma unroll
      for (int k = 0; k < K; ++k) q[u][k] = 0.0;
#pragma unroll
    for (int i = 0; i < C; ++i) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double rii = r[(k * CC + i) * BL];
#pragma unroll
        for (int u = 0; u < FR; ++u) q[u][k] += rii * (yr[u][i] * yr[u][i] + yi[u][i] * yi[u][i]);
      }
#pragma unroll
      for (int j = i + 1; j < C; ++j) {
        // conj(y_i) y_j ;  y^H R^-1 y = sum_i R_ii |y_i|^2 + 2 Re sum_{i<j} conj(y_i) R_ij y_j
        double cr[FR], ci[FR];
#pragma unroll
        for (int u = 0; u < FR; ++u) {
          cr[u] = yr[u][i] * yr[u][j] + yi[u][i] * yi[u][j];
          ci[u] = yr[u][i] * yi[u][j] - yi[u][i] * yr[u][j];
        }
        const int s = C + 2 * (i * C - i * (i + 1) / 2 + (j - i - 1));
#pragma unroll
        for (int k = 0; k < K; ++k) {
          const double rr = 2.0 * r[(k * CC + s) * BL], ri = 2.0 * r[(k * CC + s + 1) * BL];
#pragma unroll
          for (int u = 0; u < FR; ++u) q[u][k] += rr * cr[u] - ri * ci[u];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < FR; ++u) {
      const int tt = t + u * L;
      if (tt >= t_end) break;
      double phi[K], lp[K], mx = -1.0e300;
      double n2 = 1.0;                                               // |y|^2 floored (ACG)
      if constexpr (ACG) {
        n2 = 0.0;
#pragma unroll
        for (int c = 0; c < C; ++c) n2 += yr[u][c] * yr[u][c] + yi[u][c] * yi[u][c];
        const double n = fmax(sqrt(n2), SETK_EPS32_D);              // cluster.py:39-45
        n2 = n * n;
      }
#pragma unroll
      for (int k = 0; k < K; ++k) {
        if constexpr (ACG) {
          phi[k] = fmax(fabs(q[u][k]) / n2, SETK_EPS32_D);           // kappa, cluster.py:326-329
          lp[k] = -(double)C * log(phi[k]) - ld[k];                  // cluster.py:331-332
        } else {
          phi[k] = fmax(fabs(q[u][k]), SETK_EPS32_D) / (double)C;    // cluster.py:203-206
          lp[k] = -(double)C * log(phi[k]) - ld[k];                  // cluster.py:228-229
        }
        mx = fmax(mx, lp[k]);
      }
      double den = 0.0;
#pragma unroll
      for (int k = 0; k < K; ++k) { lp[k] = exp(lp[k] - mx) * al[k]; den += lp[k]; }   // cluster.py:276-281
      den = fmax(den, SETK_EPS32_D);
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const double gm = lp[k] / den;
        const long long o = (((long long)b * K + k) * a.T + tt) * P + bin;
        a.G[o] = gm;
        if constexpr (ACG) a.W[o] = gm * (double)C / (phi[k] * n2);  // cluster.py:305-308 on z = y / n
        else a.W[o] = gm * (double)C / phi[k];
      }
    }
  }
}

// init_gamma f32 [B][K][T][F] -> G = W = gamma  (cluster.py:436-440: R = sum gamma y y^H / sum gamma)
__global__ void cgmm_import_kernel(const float* __restrict__ gin, int B, int K, int T, int F, int P,
                                   double* __restrict__ G, double* __restrict__ W) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * K * T * F) return;
  const int f = (int)(idx % F);
  const long long row = idx / F;             // (b * K + k) * T + t
  const double v = gin[idx];
  G[row * P + f] = v;
  W[row * P + f] = v;
}

// CACGMM start, thread per (b, t, f) (cluster.py:508-518): init_gamma f64 [B][K][T][F] -> G = gamma,
// W = gamma M / n^2 (the kernel term is ones); without it (cgmm_init) G = 1, W = 1 / n^2, so that
// the covariance pass forms sum_t z z^H / T_b (cluster.py:495-505).  n as in the E-step.
__global__ void cacgmm_import_kernel(const double* __restrict__ gin, const float2* __restrict__ X, int P, int C,
                                     int B, int K, int T, int F, double* __restrict__ G, double* __restrict__ W) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * T * F) return;
  const int f = (int)(idx % F);
  const long long bt = idx / F;               // b * T + t
  const int b = (int)(bt / T), t = (int)(bt - (long long)b * T);
  const float2* x = X + bt * C * P + f;
  double n2 = 0.0;
  for (int c = 0; c < C; ++c) {
    const double re = x[(long long)c * P].x, im = x[(long long)c * P].y;
    n2 += re * re + im * im;
  }
  const double n = fmax(sqrt(n2), SETK_EPS32_D);
  n2 = n * n;
  for (int k = 0; k < K; ++k) {
    const long long row = ((long long)b * K + k) * T + t;
    const double g = gin ? gin[row * F + f] : 1.0;
    G[row * P + f] = g;
    W[row * P + f] = gin ? g * (double)C / n2 : 1.0 / n2;
  }
}

// G -> masks f32 [B][K][T][F]; frames past the utterance's own count are zero
__global__ void cgmm_export_kernel(const double* __restrict__ G, const int* __restrict__ n_samples, int N,
                                   Geometry g, int B, int K, int T, int P, float* __restrict__ masks) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * K * T * g.F) return;
  const int f = (int)(idx % g.F);
  const long long row = idx / g.F;
  const int t = (int)(row % T);
  const int b = (int)(row / ((long long)T * K));
  const int nb = n_samples ? n_samples[b] : N;
  const int Tb = frames_of(nb, g.n_fft, g.hop, g.pad);
  masks[idx] = t < Tb ? (float)G[row * P + f] : 0.f;
}

__global__ void cgmm_fill_kernel(double* __restrict__ p, long long n, double v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// API layout [B][C][F][T] (forward_stft, transpose=False) -> bin-major workspace
// [B][T][C][P] for callers that bring their own STFT (CgmmTrainer(obs, ...))
__global__ void __launch_bounds__(256) bcft_to_spill_kernel(const float2* __restrict__ in, int P, int C, int F,
                                                            int T, float2* __restrict__ xws) {
  __shared__ float2 tile[32][33];
  const int bc = blockIdx.z, b = bc / C, c = bc - b * C;
  const int t0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const int f = f0 + r, t = t0 + tx;
    if (t < T && f < F) tile[r][tx] = in[(((long long)b * C + c) * F + f) * T + t];
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int t = t0 + r, f = f0 + tx;
    if (t < T && f < F) xws[(((long long)b * T + t) * C + c) * P + f] = tile[tx][r];
  }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
cudaError_t run_bcft_to_spill(const float2* in, int B, int C, int F, int T, int P, float2* xws, void* stream) {
  return launch(bcft_to_spill_kernel, dim3((T + 31) / 32, (F + 31) / 32, B * C), dim3(256), 0, stream, false,
                in, P, C, F, T, xws);
}

struct CgmmWorkspace {
  double *G, *W, *part, *Rinv, *logdet, *alpha;
  int n_chunks;
};

static int cgmm_cov_chunks(const CgCtx* pl, int B, int T) {
  const int bins = pl->geo.C <= 4 ? 64 : 32;
  const int nbb = (pl->geo.F + bins - 1) / bins;
  int chunks = (2 * pl->sm_count + B * nbb - 1) / (B * nbb);
  if (chunks < 1) chunks = 1;
  if (chunks > 8) chunks = 8;
  if (chunks > T) chunks = T;
  return chunks;
}

size_t cgmm_workspace_bytes(const CgCtx* pl, const CgmmModel& m, int B, int T, int K, int P) {
  const Geometry& g = pl->geo;
  const int chunks = cgmm_cov_chunks(pl, B, T);
  size_t n = 2 * (size_t)B * K * T * P;                          // G, W
  n += (size_t)B * chunks * K * (g.C * g.C + 1) * g.F;           // part
  n += (size_t)B * K * g.C * g.C * g.F;                          // Rinv
  n += 2 * (size_t)B * K * g.F;                                  // logdet, alpha
  if (m.acg) n += (size_t)B * K * T;                             // the aligner's centroids
  return n * sizeof(double);
}

static CgmmWorkspace cgmm_carve(const CgCtx* pl, double* base, int B, int T, int K, int P) {
  const Geometry& g = pl->geo;
  CgmmWorkspace w;
  w.n_chunks = cgmm_cov_chunks(pl, B, T);
  w.G = base;
  w.W = w.G + (size_t)B * K * T * P;
  w.part = w.W + (size_t)B * K * T * P;
  w.Rinv = w.part + (size_t)B * w.n_chunks * K * (g.C * g.C + 1) * g.F;
  w.logdet = w.Rinv + (size_t)B * K * g.C * g.C * g.F;
  w.alpha = w.logdet + (size_t)B * K * g.F;
  return w;
}

template <int BINS, int NBT, int MAXT>
static cudaError_t cgmm_cov_t(const CgCtx* pl, CgmmCovArgs a, bool uniform, int B, void* stream) {
  const Geometry& g = pl->geo;
  const int Cp = 2 * ((g.C + 1) / 2);
  int tile = 32768 / (Cp * BINS * (int)sizeof(double2));      // <= 32 KB of converted samples
  if (tile < 2) tile = 2;
  if (tile > 8) tile = 8;
  a.tile_frames = tile;
  const int G = cgmm_groups(g.C, NBT);
  const size_t smem = (size_t)tile * Cp * BINS * (sizeof(double2) + sizeof(float2)) +
                      4 * (size_t)tile * 2 * BINS * sizeof(double) + 128;
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(cgmm_cov_kernel<BINS, NBT, MAXT>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
  if (ea != cudaSuccess) return ea;
#endif
  const int nbb = (g.F + BINS - 1) / BINS;
  const int k_last = uniform ? 1 : a.K;                  // the start needs class 0 only
  for (int k0 = 0; k0 < k_last; k0 += 2) {
    a.k0 = k0;
    cudaError_t e = launch(cgmm_cov_kernel<BINS, NBT, MAXT>, dim3(a.n_chunks * nbb, B), dim3(G * BINS), smem,
                           stream, false, a);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

static cudaError_t cgmm_cov(const CgCtx* pl, const float2* X, int P, const CgmmWorkspace& w,
                            bool uniform, const int* n_samples, int B, int N, int T, int K, void* stream) {
  CgmmCovArgs a;
  a.X = X; a.P = P;
  a.W = uniform ? nullptr : w.W;
  a.G = uniform ? nullptr : w.G;
  a.n_samples = n_samples; a.N = N; a.g = pl->geo;
  a.T = T; a.K = K; a.k0 = 0;
  a.n_chunks = w.n_chunks;
  a.frames_per_chunk = (T + w.n_chunks - 1) / w.n_chunks;
  a.tile_frames = 2;
  a.part = w.part;
  if (pl->geo.C <= 4) return cgmm_cov_t<64, 1, 192>(pl, a, uniform, B, stream);   // <= 3 blocks, one each
  if (pl->geo.C <= 8) return cgmm_cov_t<32, 2, 160>(pl, a, uniform, B, stream);   // <= 10 blocks, 5 groups
  return cgmm_cov_t<32, 2, 576>(pl, a, uniform, B, stream);
}

template <int C>
static cudaError_t cgmm_factor_t(const CgmmFactorArgs& a, void* stream) {
  using K = Coop<C>;
  constexpr int MPB = FactorCfg<C>::MPB;
  const size_t smem = sizeof(double) * ((size_t)MPB * 4 * K::MAT + (size_t)MPB * K::ROT);
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(cgmm_factor_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem);
  if (ea != cudaSuccess) return ea;
#endif
  const long long n = (long long)a.B * a.K * a.g.F;
  return launch(cgmm_factor_kernel<C>, dim3((unsigned)((n + MPB - 1) / MPB)), dim3(FactorCfg<C>::THREADS), smem, stream, false, a);
}

static cudaError_t cgmm_factor(const CgCtx* pl, const CgmmWorkspace& w, int identity_class,
                               int update_alpha, const int* n_samples, int B, int N, int T, int K,
                               unsigned* status, void* stream) {
  CgmmFactorArgs a;
  a.part = w.part; a.n_chunks = w.n_chunks;
  a.n_samples = n_samples; a.N = N; a.g = pl->geo;
  a.B = B; a.T = T; a.K = K;
  a.identity_class = identity_class; a.update_alpha = update_alpha;
  a.Rinv = w.Rinv; a.logdet = w.logdet; a.alpha = w.alpha; a.status = status;
  switch (pl->geo.C) {
#define SETK_CASE(k) case k: return cgmm_factor_t<k>(a, stream);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

template <int C, int K, bool ACG>
static cudaError_t cgmm_estep_t(const CgCtx* pl, CgmmEstepArgs a, int B, void* stream) {
  constexpr int BL = C <= 8 ? 64 : 16;
  const size_t smem = sizeof(double) * K * C * C * BL;
#ifndef SETK_EMU
  cudaError_t e = cudaFuncSetAttribute(cgmm_estep_kernel<C, K, BL, ACG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
#endif
  const int nbb = (a.g.F + BL - 1) / BL;
  int chunks = (4 * pl->sm_count + B * nbb - 1) / (B * nbb);
  if (chunks < 1) chunks = 1;
  if (chunks > a.T) chunks = a.T;
  a.frames_per_chunk = (a.T + chunks - 1) / chunks;
  chunks = (a.T + a.frames_per_chunk - 1) / a.frames_per_chunk;
  return launch(cgmm_estep_kernel<C, K, BL, ACG>, dim3(chunks * nbb, B), dim3(256), smem, stream, false, a);
}

template <int C, bool ACG>
static cudaError_t cgmm_estep_c(const CgCtx* pl, const CgmmEstepArgs& a, int B, int K, void* stream) {
  switch (K) {
    case 2: return cgmm_estep_t<C, 2, ACG>(pl, a, B, stream);
    case 3: return cgmm_estep_t<C, 3, ACG>(pl, a, B, stream);
    case 4: return cgmm_estep_t<C, 4, ACG>(pl, a, B, stream);
    default: return cudaErrorInvalidValue;
  }
}

template <bool ACG>
static cudaError_t cgmm_estep(const CgCtx* pl, const float2* X, int P, const CgmmWorkspace& w,
                              const int* n_samples, int B, int N, int T, int K, void* stream) {
  CgmmEstepArgs a;
  a.X = X; a.P = P;
  a.Rinv = w.Rinv; a.logdet = w.logdet; a.alpha = w.alpha;
  a.n_samples = n_samples; a.N = N; a.g = pl->geo;
  a.T = T; a.frames_per_chunk = T;
  a.G = w.G; a.W = w.W;
  switch (pl->geo.C) {
#define SETK_CASE(k) case k: return cgmm_estep_c<k, ACG>(pl, a, B, K, stream);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

// one pass over the workspace: covariance -> factor -> E-step
static cudaError_t cgmm_pass(const CgCtx* pl, const CgmmModel& m, const float2* X, int P, const CgmmWorkspace& w,
                             bool uniform, int identity_class, int update_alpha, const int* n_samples, int B, int N,
                             int T, int K, unsigned* status, void* stream) {
  cudaError_t e = cgmm_cov(pl, X, P, w, uniform, n_samples, B, N, T, K, stream);
  if (e == cudaSuccess) e = cgmm_factor(pl, w, identity_class, update_alpha, n_samples, B, N, T, K, status, stream);
  if (e != cudaSuccess) return e;
  return m.acg ? cgmm_estep<true>(pl, X, P, w, n_samples, B, N, T, K, stream)
               : cgmm_estep<false>(pl, X, P, w, n_samples, B, N, T, K, stream);
}

// CgmmTrainer start (cluster.py:436-447): the given posteriors, or with none (K = 2)
// R_0 = sum y y^H / T, R_1 = I and one E-step
static cudaError_t cgmm_start(const CgCtx* pl, const CgmmModel& m, const float2* X, int P, const CgmmWorkspace& w,
                              const int* n_samples, int B, int N, int T, int K, unsigned* status, void* stream) {
  const bool uniform = m.gamma32 == nullptr;
  if (!uniform) {
    const long long n = (long long)B * K * T * pl->geo.F;
    cudaError_t e = launch(cgmm_import_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                           m.gamma32, B, K, T, pl->geo.F, P, w.G, w.W);
    if (e != cudaSuccess) return e;
  }
  return cgmm_pass(pl, m, X, P, w, uniform, uniform ? 1 : -1, 0, n_samples, B, N, T, K, status, stream);
}

// CacgmmTrainer start (cluster.py:495-518): the given posteriors, or with cgmm_init (K = 2)
// B_0 = sum_t z z^H / T, B_1 = I and one E-step
static cudaError_t cacgmm_start(const CgCtx* pl, const CgmmModel& m, const float2* X, int P, const CgmmWorkspace& w,
                                const int* n_samples, int B, int N, int T, int K, unsigned* status, void* stream) {
  const Geometry& g = pl->geo;
  const bool from_cgmm = m.cgmm_init && K == 2;
  const long long n = (long long)B * T * g.F;
  cudaError_t e = launch(cacgmm_import_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                         from_cgmm ? nullptr : m.gamma64, X, P, g.C, B, K, T, g.F, w.G, w.W);
  if (e != cudaSuccess || !from_cgmm) return e;
  return cgmm_pass(pl, m, X, P, w, false, 1, 0, n_samples, B, N, T, K, status, stream);
}

// CgmmTrainer / CacgmmTrainer(...).train(num_iters) (cluster.py:396-465, 468-535) over the workspace X
// of B utterances, then the masks, or permu_aligner (cluster.py:48-91) on the fp64 posteriors when
// m.R > 0.
cudaError_t run_cgmm(const CgCtx* pl, const CgmmModel& m, const float2* X, int P, double* ws, const int* n_samples,
                     int B, int N, int T, int K, int num_iters, float* masks, unsigned* status, void* stream) {
  const Geometry& g = pl->geo;
  const CgmmWorkspace w = cgmm_carve(pl, ws, B, T, K, P);
  const long long na = (long long)B * K * g.F;         // alpha = 1 / K  (cluster.py:447, 485)
  cudaError_t e = launch(cgmm_fill_kernel, dim3((unsigned)((na + 255) / 256)), dim3(256), 0, stream, true,
                         w.alpha, na, 1.0 / (double)K);
  if (e == cudaSuccess)
    e = m.acg ? cacgmm_start(pl, m, X, P, w, n_samples, B, N, T, K, status, stream)
              : cgmm_start(pl, m, X, P, w, n_samples, B, N, T, K, status, stream);
  for (int it = 0; it < num_iters && e == cudaSuccess; ++it)
    e = cgmm_pass(pl, m, X, P, w, false, -1, m.update_alpha, n_samples, B, N, T, K, status, stream);
  if (e != cudaSuccess) return e;
  if (m.R > 0) {
    PermuArgs a;
    a.m = w.G; a.ld = P; a.n_frames = nullptr; a.n_samples = n_samples; a.N = N; a.g = g;
    a.K = K; a.T = T; a.F = g.F;
    return run_permu_align(a, B, m.permu_rows, m.R, w.alpha + (size_t)B * K * g.F, masks, nullptr, stream);
  }
  const long long n = (long long)B * K * T * g.F;
  return launch(cgmm_export_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                (const double*)w.G, n_samples, N, g, B, K, T, P, masks);
}

}  // namespace setk
