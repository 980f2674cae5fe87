// sep_eval.cu -- separation metrics: BSS-Eval v3 sources criteria (SDR / SIR / SAR, the definition
// mir_eval.separation.bss_eval_sources implements, used by the reference's scripts/sptk/compute_sdr.py)
// and the scale-invariant SNR of the reference's libs/metric.py (compute_si_snr.py), for batches of
// ragged utterances, in fp64 on float32 samples.
//
// K15, setk_bss_eval: for utterance b with N references s_i and N estimates e_j of S_b samples, and
// the filter length L, A_i is the (S_b + L - 1) x L matrix of the delayed copies s_i[n - a], a < L.
// P_all(j) is e_j's least-squares projection onto span(A_0 .. A_{N-1}), P_spat(j, i) onto span(A_i).
//   1. sep_corr_kernel    r_{ii'}(k) = sum_m s_i[m] s_i'[m + k], i <= i', |k| < L, and
//                         D_{ij}(a) = sum_m s_i[m] e_j[m + a], a < L: direct fixed-order fp64 sums
//                         (each CTA owns 512 lags over the whole utterance; no atomics);
//   2. sep_factor_kernel  one CTA per utterance: G = A^T A (N L square, block Toeplitz in r) in
//                         scratch, a blocked right-looking Cholesky (32-column panels, G streamed
//                         through L2), forward and back substitution for the N right-hand sides
//                         D_j; then the same for every diagonal block G_ii.  A pivot <= tau times the
//                         column's original diagonal marks the column dependent: its row and column
//                         of the factor and its coefficient are zero, so the solution is still the
//                         least-squares projection when references are (numerically) dependent;
//   3. sep_score_kernel   per (256-sample block, utterance): the L-tap FIRs of the coefficients over
//                         the references give P_all(j) and P_spat(j, i) sample by sample; the five
//                         energies |P_spat|^2, |e - P_spat|^2, |P_all - P_spat|^2, |P_all|^2,
//                         |e - P_all|^2 (and |e|^2) are taken from the signals, per warp;
//   4. sep_crit_kernel    sums the per-warp energies in a fixed order and writes
//                         SDR = 10 log10(|P_spat|^2 / |e - P_spat|^2), SIR = .. / |P_all - P_spat|^2,
//                         SAR = 10 log10(|P_all|^2 / |e - P_all|^2), +inf for a zero denominator.
// Every sum has a fixed order and depends only on the utterance's own samples, so the same call gives
// the same bits, and an utterance gives the same bits alone as inside a batch.
//
// K15e, setk_si_snr: per (estimate j, reference i, utterance) CTA, three fixed-order passes: the means,
// then <x, s> and |s|^2 of the zero-mean signals, then |x - t|^2 of the residual itself.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

namespace {

constexpr int kCorrThreads = 64;
constexpr int kCorrLags = 8;                            // lags per thread (a sliding window of samples)
constexpr int kCorrTile = kCorrThreads * kCorrLags;     // lags per CTA
constexpr int kCorrChunk = 512;                         // samples staged per step
constexpr int kCorrY = kCorrChunk + kCorrTile;          // y samples a step reads
constexpr int kNB = 32;                                 // Cholesky panel width
constexpr int kFactorThreads = 256;
constexpr int kScoreT = 256;                            // output samples per score CTA (one per thread)
constexpr int kTapChunk = 64;                           // coefficients staged per step
constexpr int kWarps = kScoreT / 32;
// a pivot <= kSepTau times its column's original diagonal drops the column; the dependent-reference
// test (one reference a 3-sample delay of another) drops columns with it and matches the explicit
// least-squares projection
constexpr double kSepTau = 1e-10;

// index into the padded y stage: stride-8 reads of a warp fall in distinct banks
__device__ __forceinline__ int ypad(int p) { return p + (p >> 4); }

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// fixed-order tree over the CTA's 256 threads (red holds 256 values)
__device__ inline double cta_sum(double v, double* red) {
  red[threadIdx.x] = v;
  for (int w = kScoreT / 2; w > 0; w >>= 1) {
    __syncthreads();
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
  }
  __syncthreads();
  const double r = red[0];
  __syncthreads();
  return r;
}

}  // namespace

struct SepArgs {
  const float* est;       // [B][N][S]
  const float* ref;       // [B][N][S]
  const int* len;         // [B] samples of each utterance
  int B, N, S, L, nblk;
  double tau;
  double* corr;           // [B][corr_stride]: r of the pairs i <= i' (2L - 1 lags each), then D [j][i][L]
  double* G;              // [B][(N L)^2], column major, lower triangle
  double* d0;             // [B][N L] original diagonal
  double* coef;           // [B][2 N^2 L]: C_all [j][N L], then C_spat [j][i][L]
  double* part;           // [B][nblk][kWarps][V] per-warp energies
  double* crit;           // [B][3][N][N]
  int* dropped;           // [B] or null
  unsigned* status;       // [B]
  SETK_HD size_t corr_stride() const { return (size_t)N * (N + 1) / 2 * (2 * L - 1) + (size_t)N * N * L; }
};

static __host__ __device__ inline int n_pairs(int N) { return N * (N + 1) / 2; }
// index of the pair (i, i'), i <= i', in row-major upper-triangle order
static __host__ __device__ inline int pair_index(int N, int i, int ip) { return i * N - i * (i - 1) / 2 + (ip - i); }
static __host__ __device__ inline int n_values(int N) { return 3 * N * N + 3 * N; }
// r_{ii'}(k), i <= i', |k| < L
static __device__ inline double rcorr(const SepArgs& a, const double* corr, int i, int ip, int k) {
  return corr[(size_t)pair_index(a.N, i, ip) * (2 * a.L - 1) + (k + a.L - 1)];
}
static __device__ inline const double* dcorr(const SepArgs& a, const double* corr, int j, int i) {
  return corr + (size_t)n_pairs(a.N) * (2 * a.L - 1) + ((size_t)j * a.N + i) * a.L;
}

size_t sep_eval_scratch_bytes(int B, int N, int S, int L) {
  const size_t n = (size_t)N * L;
  const size_t nblk = (size_t)(S + L - 1 + kScoreT - 1) / kScoreT;
  const size_t corr = (size_t)n_pairs(N) * (2 * L - 1) + (size_t)N * N * L;
  return up256(sizeof(double) * B * corr) + up256(sizeof(double) * B * n * n) + up256(sizeof(double) * B * n) +
         up256(sizeof(double) * B * 2 * N * n) + up256(sizeof(double) * B * nblk * kWarps * n_values(N));
}

// grid (ceil(lags / kCorrTile), pairs + N^2, B): term t < pairs is r_{ii'} over k in [-(L-1), L-1],
// the others D_{ij} over a in [0, L).  Thread t owns lags k0 + 8t .. k0 + 8t + 7 and slides a window of
// y over the staged chunk: one y load and one x broadcast per 8 FMAs.
__global__ void __launch_bounds__(kCorrThreads) sep_corr_kernel(SepArgs a) {
  __shared__ double xs[kCorrChunk];
  __shared__ double ys[kCorrY + kCorrY / 16];
  const int b = blockIdx.z, term = blockIdx.y, N = a.N, L = a.L, S = a.len[b];
  const int P = n_pairs(N);
  const float *x, *y;
  int kmin, nk;
  double* out;
  const float* ref = a.ref + (size_t)b * N * a.S;
  if (term < P) {
    int i = 0, r = term;
    while (r >= N - i) { r -= N - i; ++i; }
    x = ref + (size_t)i * a.S;
    y = ref + (size_t)(i + r) * a.S;
    kmin = -(L - 1);
    nk = 2 * L - 1;
    out = a.corr + b * a.corr_stride() + (size_t)term * (2 * L - 1);
  } else {
    const int j = (term - P) / N, i = (term - P) % N;
    x = ref + (size_t)i * a.S;
    y = a.est + ((size_t)b * N + j) * a.S;
    kmin = 0;
    nk = L;
    out = a.corr + b * a.corr_stride() + (size_t)P * (2 * L - 1) + ((size_t)j * N + i) * L;
  }
  const int l0 = blockIdx.x * kCorrTile;   // first lag of the CTA, relative to kmin
  if (l0 >= nk) return;
  const int k0 = kmin + l0, tl = kCorrLags * threadIdx.x;
  double acc[kCorrLags];
#pragma unroll
  for (int q = 0; q < kCorrLags; ++q) acc[q] = 0.0;
  for (int m0 = 0; m0 < S; m0 += kCorrChunk) {
    __syncthreads();
    for (int u = threadIdx.x; u < kCorrChunk; u += kCorrThreads) {
      const int m = m0 + u;
      xs[u] = m < S ? (double)x[m] : 0.0;
    }
    for (int u = threadIdx.x; u < kCorrY; u += kCorrThreads) {
      const long long m = (long long)m0 + k0 + u;
      ys[ypad(u)] = m >= 0 && m < S ? (double)y[m] : 0.0;
    }
    __syncthreads();
    double w[kCorrLags];
#pragma unroll
    for (int q = 0; q < kCorrLags; ++q) w[q] = ys[ypad(tl + q)];
    const int cn = imin(kCorrChunk, S - m0);
    for (int u = 0; u < cn; ++u) {
      const double xv = xs[u];
#pragma unroll
      for (int q = 0; q < kCorrLags; ++q) acc[q] = fma(xv, w[q], acc[q]);
#pragma unroll
      for (int q = 0; q < kCorrLags - 1; ++q) w[q] = w[q + 1];
      w[kCorrLags - 1] = ys[ypad(u + 1 + tl + kCorrLags - 1)];
    }
  }
#pragma unroll
  for (int q = 0; q < kCorrLags; ++q)
    if (l0 + tl + q < nk) out[l0 + tl + q] = acc[q];
}

namespace {

struct FactorSmem {
  double D[kNB][kNB + 1];   // the diagonal block being factored
  double Pi[kNB][kNB + 1];  // panel rows of the tile's row block
  double Pj[kNB][kNB + 1];  // panel rows of the tile's column block
  double inv[kNB];          // 1 / pivot, 0 for a dropped column
  double red[kFactorThreads / 32][SETK_SEP_MAX_SOURCES];
  double y[SETK_SEP_MAX_SOURCES];
};

// In-place Cholesky G = L L^T of the lower triangle of the column-major n x n matrix A (lda), with the
// dependent-column rule above; returns the number of dropped columns (in thread 0).
__device__ int sep_cholesky(double* A, int n, int lda, const double* d0, double tau, FactorSmem& sm) {
  const int tid = threadIdx.x;
  int drops = 0;
  for (int k0 = 0; k0 < n; k0 += kNB) {
    const int nb = imin(kNB, n - k0);
    for (int e = tid; e < kNB * kNB; e += kFactorThreads) {
      const int r = e % kNB, c = e / kNB;
      if (r < nb && c <= r) sm.D[r][c] = A[(size_t)(k0 + c) * lda + k0 + r];
    }
    __syncthreads();
    for (int c = 0; c < nb; ++c) {
      if (tid == 0) {
        const double d = sm.D[c][c];
        const bool keep = d > tau * d0[k0 + c];
        const double piv = keep ? sqrt(d) : 0.0;
        sm.D[c][c] = piv;
        sm.inv[c] = keep ? 1.0 / piv : 0.0;
        drops += !keep;
      }
      __syncthreads();
      for (int r = c + 1 + tid; r < nb; r += kFactorThreads) sm.D[r][c] *= sm.inv[c];
      __syncthreads();
      for (int e = tid; e < kNB * kNB; e += kFactorThreads) {
        const int r = e % kNB, cc = e / kNB;
        if (cc > c && cc <= r && r < nb) sm.D[r][cc] = fma(-sm.D[r][c], sm.D[cc][c], sm.D[r][cc]);
      }
      __syncthreads();
    }
    for (int e = tid; e < kNB * kNB; e += kFactorThreads) {
      const int r = e % kNB, c = e / kNB;
      if (r < nb && c <= r) A[(size_t)(k0 + c) * lda + k0 + r] = sm.D[r][c];
    }
    // panel: rows x below the block solve x L_kk^T = a with the rule above, through the linear map M of
    // that forward substitution (M[c][k] = its column-c output for a = e_k; lower triangular), in Pj
    __syncthreads();
    if (tid < nb) {
      const int k = tid;
      for (int c = 0; c < nb; ++c) {
        double v = c == k ? 1.0 : 0.0;
        for (int c2 = k; c2 < c; ++c2) v = fma(-sm.D[c][c2], sm.Pj[c2][k], v);
        sm.Pj[c][k] = c < k ? 0.0 : v * sm.inv[c];
      }
    }
    const int tx = tid % 16, ty = tid / 16;
    for (int I = k0 + nb; I < n; I += kNB) {
      __syncthreads();
      for (int e = tid; e < kNB * kNB; e += kFactorThreads) {
        const int rr = e % kNB, c = e / kNB;
        sm.Pi[rr][c] = c < nb && I + rr < n ? A[(size_t)(k0 + c) * lda + I + rr] : 0.0;
      }
      __syncthreads();
#pragma unroll
      for (int v = 0; v < 2; ++v)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int ii = tx + 16 * u, cc = ty + 16 * v;
          if (I + ii < n && cc < nb) {
            double x = 0.0;
            for (int k = 0; k <= cc; ++k) x = fma(sm.Pi[ii][k], sm.Pj[cc][k], x);
            A[(size_t)(k0 + cc) * lda + I + ii] = x;
          }
        }
    }
    __syncthreads();
    // trailing update of the lower triangle, one 32 x 32 tile at a time: A_IJ -= P_I P_J^T
    const int t0 = k0 + nb;
    for (int J = t0; J < n; J += kNB)
      for (int I = J; I < n; I += kNB) {
        for (int e = tid; e < kNB * kNB; e += kFactorThreads) {
          const int rr = e % kNB, c = e / kNB;
          const bool okc = c < nb;
          sm.Pi[rr][c] = okc && I + rr < n ? A[(size_t)(k0 + c) * lda + I + rr] : 0.0;
          sm.Pj[rr][c] = okc && J + rr < n ? A[(size_t)(k0 + c) * lda + J + rr] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int v = 0; v < 2; ++v)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int ii = tx + 16 * u, jj = ty + 16 * v, r = I + ii, col = J + jj;
            if (r < n && col < n && r >= col) {
              double acc = A[(size_t)col * lda + r];
              for (int c = 0; c < nb; ++c) acc = fma(-sm.Pi[ii][c], sm.Pj[jj][c], acc);
              A[(size_t)col * lda + r] = acc;
            }
          }
        __syncthreads();
      }
  }
  return drops;
}

// L y = b in place for nrhs right-hand sides X[j * ldx + r]; a dropped column gives y_k = 0
__device__ void sep_forward(const double* A, int n, int lda, double* X, int nrhs, int ldx, FactorSmem& sm) {
  for (int k = 0; k < n; ++k) {
    const double lkk = A[(size_t)k * lda + k];
    const double inv = lkk > 0.0 ? 1.0 / lkk : 0.0;
    if ((int)threadIdx.x < nrhs) sm.y[threadIdx.x] = X[(size_t)threadIdx.x * ldx + k] * inv;
    __syncthreads();
    if ((int)threadIdx.x < nrhs) X[(size_t)threadIdx.x * ldx + k] = sm.y[threadIdx.x];
    for (int r = k + 1 + threadIdx.x; r < n; r += kFactorThreads) {
      const double l = A[(size_t)k * lda + r];
      for (int j = 0; j < nrhs; ++j) X[(size_t)j * ldx + r] = fma(-l, sm.y[j], X[(size_t)j * ldx + r]);
    }
    __syncthreads();
  }
}

// L^T c = y in place: c_k = (y_k - sum_{r > k} L[r][k] c_r) / L[k][k], each dot product a fixed-order
// reduction (per-thread strided sums, warp butterflies, the warps in order)
__device__ void sep_backward(const double* A, int n, int lda, double* X, int nrhs, int ldx, FactorSmem& sm) {
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
  for (int k = n - 1; k >= 0; --k) {
    double part[SETK_SEP_MAX_SOURCES];
#pragma unroll
    for (int j = 0; j < SETK_SEP_MAX_SOURCES; ++j) part[j] = 0.0;
    for (int r = k + 1 + threadIdx.x; r < n; r += kFactorThreads) {
      const double l = A[(size_t)k * lda + r];
#pragma unroll
      for (int j = 0; j < SETK_SEP_MAX_SOURCES; ++j)
        if (j < nrhs) part[j] = fma(l, X[(size_t)j * ldx + r], part[j]);
    }
#pragma unroll
    for (int j = 0; j < SETK_SEP_MAX_SOURCES; ++j)
      if (j < nrhs) {
        const double s = warp_sum(part[j]);
        if (lane == 0) sm.red[warp][j] = s;
      }
    __syncthreads();
    if ((int)threadIdx.x < nrhs) {
      const int j = threadIdx.x;
      double s = 0.0;
      for (int w = 0; w < kFactorThreads / 32; ++w) s += sm.red[w][j];
      const double lkk = A[(size_t)k * lda + k];
      X[(size_t)j * ldx + k] = lkk > 0.0 ? (X[(size_t)j * ldx + k] - s) / lkk : 0.0;
    }
    __syncthreads();
  }
}

}  // namespace

// one CTA per utterance: C_all from G, then C_spat(:, i) from every G_ii (factored in G's storage)
__global__ void __launch_bounds__(kFactorThreads) sep_factor_kernel(SepArgs a) {
  __shared__ FactorSmem sm;
  const int b = blockIdx.x, N = a.N, L = a.L, n = N * L, tid = threadIdx.x;
  double* G = a.G + (size_t)b * n * n;
  double* d0 = a.d0 + (size_t)b * n;
  const double* corr = a.corr + b * a.corr_stride();
  double* Ca = a.coef + (size_t)b * 2 * N * n;
  double* Cs = Ca + (size_t)N * n;
  // G[(i, a), (i', a')] = r_{i'i}(a' - a) for i' <= i (the lower triangle)
  for (size_t e = tid; e < (size_t)n * n; e += kFactorThreads) {
    const int col = (int)(e / n), row = (int)(e % n);
    if (row < col) continue;
    const int i = row / L, ar = row % L, ic = col / L, ac = col % L;
    G[e] = rcorr(a, corr, ic, i, ac - ar);
  }
  for (int c = tid; c < n; c += kFactorThreads) d0[c] = rcorr(a, corr, c / L, c / L, 0);
  for (int e = tid; e < N * n; e += kFactorThreads) {
    const int j = e / n, i = (e % n) / L, k = e % L;
    Ca[e] = dcorr(a, corr, j, i)[k];
  }
  __syncthreads();
  const int drops = sep_cholesky(G, n, n, d0, a.tau, sm);
  __syncthreads();
  sep_forward(G, n, n, Ca, N, n, sm);
  sep_backward(G, n, n, Ca, N, n, sm);
  for (int i = 0; i < N; ++i) {
    for (int e = tid; e < L * L; e += kFactorThreads) {
      const int col = e / L, row = e % L;
      if (row >= col) G[e] = rcorr(a, corr, i, i, col - row);
    }
    for (int c = tid; c < L; c += kFactorThreads) d0[c] = rcorr(a, corr, i, i, 0);
    for (int e = tid; e < N * L; e += kFactorThreads) {
      const int j = e / L, k = e % L;
      Cs[((size_t)j * N + i) * L + k] = dcorr(a, corr, j, i)[k];
    }
    __syncthreads();
    sep_cholesky(G, L, L, d0, a.tau, sm);
    __syncthreads();
    sep_forward(G, L, L, Cs + (size_t)i * L, N, N * L, sm);
    sep_backward(G, L, L, Cs + (size_t)i * L, N, N * L, sm);
  }
  if (tid == 0 && a.dropped) a.dropped[b] = drops;
}

// grid (nblk, B): samples n0 .. n0 + 255 of the projections (S_b + L - 1 long); per warp, the energies
// V = [(j, i): |P_spat|^2, |e_j - P_spat|^2, |P_all - P_spat|^2] then [j: |P_all|^2, |e_j - P_all|^2, |e_j|^2]
template <int N>
__global__ void __launch_bounds__(kScoreT) sep_score_kernel(SepArgs a) {
  __shared__ double xs[kScoreT + SETK_SEP_MAX_FLEN - 1];
  __shared__ double cs[N][kTapChunk];
  constexpr int V = 3 * N * N + 3 * N;
  const int blk = blockIdx.x, b = blockIdx.y, L = a.L, S = a.len[b], tid = threadIdx.x;
  const int lane = tid % 32, warp = tid / 32;
  const int n0 = blk * kScoreT, n = n0 + tid;
  double* part = a.part + ((size_t)b * a.nblk + blk) * kWarps * V;
  if (n0 >= S + L - 1) {
    for (int v = tid; v < kWarps * V; v += kScoreT) part[v] = 0.0;
    return;
  }
  const float* ref = a.ref + (size_t)b * N * a.S;
  const float* est = a.est + (size_t)b * N * a.S;
  const double* Ca = a.coef + (size_t)b * 2 * N * N * L;
  const double* Cs = Ca + (size_t)N * N * L;
  double e[N], pa[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    e[j] = n < S ? (double)est[(size_t)j * a.S + n] : 0.0;
    pa[j] = 0.0;
  }
  const int span = kScoreT + L - 1;
  auto stage = [&](int i) {
    __syncthreads();
    const float* s = ref + (size_t)i * a.S;
    for (int u = tid; u < span; u += kScoreT) {
      const int m = n0 - (L - 1) + u;
      xs[u] = m >= 0 && m < S ? (double)s[m] : 0.0;
    }
  };
  // acc[j] += sum_a c_j[a] s_i[n - a] with c_j = coef + j * cstride
  auto fir = [&](const double* coef, size_t cstride, double (&acc)[N]) {
    for (int a0 = 0; a0 < L; a0 += kTapChunk) {
      const int na = imin(kTapChunk, L - a0);
      __syncthreads();
      for (int e2 = tid; e2 < N * kTapChunk; e2 += kScoreT) {
        const int j = e2 / kTapChunk, u = e2 % kTapChunk;
        cs[j][u] = u < na ? coef[j * cstride + a0 + u] : 0.0;
      }
      __syncthreads();
      for (int u = 0; u < na; ++u) {
        const double s = xs[tid + L - 1 - (a0 + u)];
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] = fma(cs[j][u], s, acc[j]);
      }
    }
  };
  auto put = [&](int v, double x) {
    const double s = warp_sum(x);
    if (lane == 0) part[warp * V + v] = s;
  };
  for (int i = 0; i < N; ++i) {
    stage(i);
    fir(Ca + (size_t)i * L, (size_t)N * L, pa);
  }
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const double r = e[j] - pa[j];
    put(3 * N * N + 3 * j, pa[j] * pa[j]);
    put(3 * N * N + 3 * j + 1, r * r);
    put(3 * N * N + 3 * j + 2, e[j] * e[j]);
  }
  for (int i = 0; i < N; ++i) {
    stage(i);
    double ps[N];
#pragma unroll
    for (int j = 0; j < N; ++j) ps[j] = 0.0;
    fir(Cs + (size_t)i * L, (size_t)N * L, ps);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const double r = e[j] - ps[j], q = pa[j] - ps[j];
      put(3 * (j * N + i), ps[j] * ps[j]);
      put(3 * (j * N + i) + 1, r * r);
      put(3 * (j * N + i) + 2, q * q);
    }
  }
}

__device__ __forceinline__ double safe_db(double num, double den) {
  return den == 0.0 ? (double)INFINITY : 10.0 * log10(num / den);
}

// grid (B): the energies summed over blocks and warps in order, then the criteria and the status
__global__ void __launch_bounds__(kScoreT) sep_crit_kernel(SepArgs a) {
  __shared__ double tot[3 * SETK_SEP_MAX_SOURCES * SETK_SEP_MAX_SOURCES + 3 * SETK_SEP_MAX_SOURCES];
  __shared__ unsigned st;
  const int b = blockIdx.x, N = a.N, V = n_values(N), tid = threadIdx.x;
  if (tid == 0) st = 0u;
  for (int v = tid; v < V; v += kScoreT) {
    const double* p = a.part + (size_t)b * a.nblk * kWarps * V + v;
    double s = 0.0;
    for (int k = 0; k < a.nblk * kWarps; ++k) s += p[(size_t)k * V];
    tot[v] = s;
  }
  __syncthreads();
  double* crit = a.crit + (size_t)b * 3 * N * N;
  const double* corr = a.corr + b * a.corr_stride();
  for (int p = tid; p < N * N; p += kScoreT) {
    const int j = p / N, i = p % N;
    const double* t = tot + 3 * p;
    const double* u = tot + 3 * N * N + 3 * j;
    const double sdr = safe_db(t[0], t[1]), sir = safe_db(t[0], t[2]), sar = safe_db(u[0], u[1]);
    crit[p] = sdr;
    crit[N * N + p] = sir;
    crit[2 * N * N + p] = sar;
    unsigned bits = 0u;
    if (sdr != sdr || sir != sir || sar != sar) bits |= SETK_ST_NONFINITE;
    if (i == 0 && u[2] == 0.0) bits |= SETK_ST_SILENT;               // estimate j is all zeros
    if (j == 0 && rcorr(a, corr, i, i, 0) == 0.0) bits |= SETK_ST_SILENT;   // reference i is
    if (bits) atomicOr(&st, bits);
  }
  __syncthreads();
  if (tid == 0) a.status[b] = st;
}

// grid (N^2, B): SI-SNR of estimate j against reference i (libs/metric.py si_snr)
__global__ void __launch_bounds__(kScoreT) sep_si_snr_kernel(const float* est, const float* ref, const int* len,
                                                            int N, int S, int remove_dc, double eps,
                                                            double* out) {
  __shared__ double red[kScoreT];
  const int b = blockIdx.y, j = blockIdx.x / N, i = blockIdx.x % N, n = len[b];
  const float* x = est + ((size_t)b * N + j) * S;
  const float* s = ref + ((size_t)b * N + i) * S;
  double mx = 0.0, ms = 0.0;
  if (remove_dc) {
    double ax = 0.0, as = 0.0;
    for (int m = threadIdx.x; m < n; m += kScoreT) {
      ax += (double)x[m];
      as += (double)s[m];
    }
    mx = cta_sum(ax, red) / n;
    ms = cta_sum(as, red) / n;
  }
  double ip = 0.0, ss = 0.0;
  for (int m = threadIdx.x; m < n; m += kScoreT) {
    const double xv = (double)x[m] - mx, sv = (double)s[m] - ms;
    ip = fma(xv, sv, ip);
    ss = fma(sv, sv, ss);
  }
  ip = cta_sum(ip, red);
  ss = cta_sum(ss, red);
  const double alpha = ip / (ss + eps);
  double nn = 0.0;
  for (int m = threadIdx.x; m < n; m += kScoreT) {
    const double r = ((double)x[m] - mx) - alpha * ((double)s[m] - ms);
    nn = fma(r, r, nn);
  }
  nn = cta_sum(nn, red);
  if (threadIdx.x == 0) {
    const double tn = fabs(alpha) * sqrt(ss);
    out[((size_t)b * N + j) * N + i] = 20.0 * log10(tn / (sqrt(nn) + eps) + eps);
  }
}

cudaError_t run_bss_eval(const float* est, const float* ref, const int* len, int B, int N, int S, int L, char* ws,
                         double* crit, int* dropped, unsigned* status, void* stream) {
  SepArgs a;
  a.est = est; a.ref = ref; a.len = len; a.B = B; a.N = N; a.S = S; a.L = L; a.tau = kSepTau;
  a.nblk = (S + L - 1 + kScoreT - 1) / kScoreT;
  a.crit = crit; a.dropped = dropped; a.status = status;
  const size_t n = (size_t)N * L;
  char* p = ws;
  a.corr = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * B * a.corr_stride());
  a.G = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * B * n * n);
  a.d0 = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * B * n);
  a.coef = reinterpret_cast<double*>(p);
  p += up256(sizeof(double) * B * 2 * N * n);
  a.part = reinterpret_cast<double*>(p);
  const dim3 cgrid((2 * L - 1 + kCorrTile - 1) / kCorrTile, n_pairs(N) + N * N, B);
  cudaError_t e = launch(sep_corr_kernel, cgrid, dim3(kCorrThreads), 0, stream, false, a);
  if (e == cudaSuccess) e = launch(sep_factor_kernel, dim3(B), dim3(kFactorThreads), 0, stream, false, a);
  const dim3 sgrid(a.nblk, B);
  if (e == cudaSuccess) {
    switch (N) {
      case 1: e = launch(sep_score_kernel<1>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 2: e = launch(sep_score_kernel<2>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 3: e = launch(sep_score_kernel<3>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 4: e = launch(sep_score_kernel<4>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 5: e = launch(sep_score_kernel<5>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 6: e = launch(sep_score_kernel<6>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      case 7: e = launch(sep_score_kernel<7>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
      default: e = launch(sep_score_kernel<8>, sgrid, dim3(kScoreT), 0, stream, false, a); break;
    }
  }
  if (e == cudaSuccess) e = launch(sep_crit_kernel, dim3(B), dim3(kScoreT), 0, stream, false, a);
  return e;
}

cudaError_t run_si_snr(const float* est, const float* ref, const int* len, int B, int N, int S, int remove_dc,
                       double eps, double* out, void* stream) {
  return launch(sep_si_snr_kernel, dim3(N * N, B), dim3(kScoreT), 0, stream, false, est, ref, len, N, S, remove_dc,
                eps, out);
}

}  // namespace setk
