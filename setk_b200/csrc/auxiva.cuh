// auxiva.cuh -- AuxIVA blind source separation of a multichannel STFT.  Replaces, per
// utterance, auxiva(X, epochs) of scripts/sptk/apply_auxiva.py:24-57 (Ono 2011, the
// pyroomacoustics update rules with the reference's normalisation).
//
// N sources = N channels; W [F][N][N] starts as the identity; y_n = w_n^H x.  Each epoch:
//   auxiva_demix_kernel   power pass: r[n,t] = sqrt(sum_f |y_n[f,t]|^2), Gr = 1 / (r + EPSILON),
//                         a CTA per (utterance, 32 frames), 8 warps over contiguous bin ranges
//                         added in warp order (fixed order: no float atomics)
//   auxiva_update_kernel  a CTA per (utterance, bin): all N weighted covariances
//                         V_n = sum_t Gr[n,t] x_t x_t^H / T from one pass over the bin's frames,
//                         then for n = 0 .. N-1 IN ORDER (column n is updated before n + 1 is solved):
//                           w = solve(W^H V_n, e_n);  W[:, n] = w / (w^H V_n w)
// and after the last epoch the same demix kernel writes Y (complex128, as the reference returns).
//
// The normalisation divides by w^H V w itself -- NOT by its square root as the pyroomacoustics
// original does -- and the divisor is the complex number the reference computes (its imaginary
// part is at the rounding level), so the division is complex (oracle/auxiva_oracle.py).
//
// Everything after the complex64 input is fp64, like the reference's complex128.  The solves use
// lu_factor / lu_solve_vec (hermitian_solve.cuh) on one thread for N <= 4 and the warp-group
// lu_solve_coop (lu_coop.cuh) above; matrices live in shared memory either way.  An exactly zero
// pivot (numpy.linalg.LinAlgError: an all-zero bin, a silent channel) sets SETK_ST_SINGULAR for
// the utterance, a non-finite W SETK_ST_NONFINITE.  Problems never share data across utterances,
// so one utterance's failure leaves the others' results unchanged.
// Built in wpe.cu's translation unit (the other fp64 per-bin iterative front end).
#pragma once
#include "common.cuh"
#include "launchers.cuh"
#include "lu_coop.cuh"

namespace setk {

struct AuxArgs {
  const float2* X;     // [B][N][F][T]
  int B, F, T;
  cd* W;               // [B][F][N][N]: W[m][n], column n demixes source n
  double* gr;          // [B][N][T]: 1 / (r + EPSILON)
  cd* out;             // demix: Y [B][N][F][T] when not null
  unsigned* status;    // [B] or null
};

constexpr int kAuxFrames = 32;   // frames per demix CTA (one per lane)
constexpr int kAuxSlices = 8;    // bin ranges per demix CTA (one per warp)

template <int N>
struct AuxCfg {
  static constexpr int P = N * (N + 1) / 2;                           // covariance entries i <= j
  static constexpr int THREADS = N <= 4 ? 64 : (P > 128 ? 256 : 128);
  static constexpr int S = THREADS / P;                               // frame slices of the V sums
  static constexpr int TC = 128;                                      // frames per chunk
  static constexpr int XP = TC + 1;                                   // row pitch of the chunk (float2)
};

// shared memory of the update kernel, in doubles
template <int N>
SETK_HD inline size_t aux_update_smem_doubles() {
  using K = AuxCfg<N>;
  return (size_t)N * K::XP + (size_t)N * K::TC + 2 * ((size_t)N * N * N + (size_t)N * N +
         (size_t)K::S * K::P * N + (size_t)N * (N + 1) + N);
}

// (i, j), i <= j, of upper-triangle entry p in row-major order
template <int N>
__device__ __forceinline__ void aux_pair(int p, int& i, int& j) {
  i = 0;
  while (p >= N - i) { p -= N - i; ++i; }
  j = i + p;
}

__global__ void auxiva_init_kernel(cd* W, long long bins, int N) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= bins * N * N) return;
  const int e = (int)(q % (N * N));
  W[q] = cd_make(e / N == e % N ? 1.0 : 0.0, 0.0);
}

// y_n[f, t] = sum_m conj(W[f][m][n]) x_m[f, t]; out -> Y, gr -> 1 / (sqrt(sum_f |y_n|^2) + EPSILON)
template <int N>
__global__ void __launch_bounds__(kAuxFrames * kAuxSlices) auxiva_demix_kernel(AuxArgs a) {
  __shared__ double part[kAuxSlices][N][kAuxFrames];
  const int b = blockIdx.y, lane = threadIdx.x, s = threadIdx.y;
  const int t = blockIdx.x * kAuxFrames + lane;
  const bool live = t < a.T;
  const int f0 = (int)((long long)a.F * s / kAuxSlices), f1 = (int)((long long)a.F * (s + 1) / kAuxSlices);
  double acc[N];
#pragma unroll
  for (int n = 0; n < N; ++n) acc[n] = 0.0;
  for (int f = f0; f < f1; ++f) {
    const cd* Wf = a.W + ((long long)b * a.F + f) * N * N;
    cd x[N];
#pragma unroll
    for (int m = 0; m < N; ++m) {
      const float2 v = live ? a.X[(((long long)b * N + m) * a.F + f) * a.T + t] : make_float2(0.f, 0.f);
      x[m] = cd_make((double)v.x, (double)v.y);
    }
#pragma unroll
    for (int n = 0; n < N; ++n) {
      cd y = cd_make(0.0, 0.0);
#pragma unroll
      for (int m = 0; m < N; ++m) y = cd_add(y, cd_mul(cd_conj(Wf[m * N + n]), x[m]));
      acc[n] += cd_abs2(y);
      if (a.out && live) a.out[(((long long)b * N + n) * a.F + f) * a.T + t] = y;
    }
  }
  if (!a.gr) return;                                           // uniform over the CTA
#pragma unroll
  for (int n = 0; n < N; ++n) part[s][n][lane] = acc[n];
  __syncthreads();
  if (s != 0 || !live) return;
  for (int n = 0; n < N; ++n) {
    double p = part[0][n][lane];
    for (int k = 1; k < kAuxSlices; ++k) p += part[k][n][lane];
    a.gr[((long long)b * N + n) * a.T + t] = 1.0 / (sqrt(p) + SETK_EPS32_D);
  }
}

template <int N>
__global__ void __launch_bounds__(AuxCfg<N>::THREADS) auxiva_update_kernel(AuxArgs a) {
  using K = AuxCfg<N>;
  constexpr int P = K::P, S = K::S, TC = K::TC, XP = K::XP, LD = N + 1;
  SETK_DYN_SMEM(double, sm);
  float2* xs = reinterpret_cast<float2*>(sm);                      // [N][XP] frames of the chunk
  double* gs = sm + (size_t)N * XP;                                // [N][TC] Gr of the chunk
  cd* V = reinterpret_cast<cd*>(gs + (size_t)N * TC);              // [N][N][N] V_n
  cd* Ws = V + N * N * N;                                          // [N][N]    W of the bin
  cd* red = Ws + N * N;                                            // [S][P][N] slice partial sums
  cd* M = red + S * P * N;                                         // [N][N + 1] system (CMat<N> for N <= 4)
  cd* wv = M + N * LD;                                             // [N]       solution
  const int bin = blockIdx.x, b = bin / a.F, f = bin - b * a.F;
  const int tid = threadIdx.x;
  cd* Wg = a.W + (long long)bin * N * N;
  for (int q = tid; q < N * N; q += K::THREADS) Ws[q] = Wg[q];

  // ---- V_n[i][j] for i <= j: thread (slice sl, entry pr) sums frames u = sl (mod S) of each chunk ----
  const int pr = tid % P, sl = tid / P;
  const bool acc_on = sl < S;
  int pi, pj;
  aux_pair<N>(pr, pi, pj);
  double ar[N], ai[N];
#pragma unroll
  for (int n = 0; n < N; ++n) { ar[n] = 0.0; ai[n] = 0.0; }
  for (int t0 = 0; t0 < a.T; t0 += TC) {
    const int nf = imin(TC, a.T - t0);
    __syncthreads();                                               // the previous chunk is consumed
    for (int q = tid; q < N * nf; q += K::THREADS) {
      const int m = q / nf, u = q - m * nf;
      xs[m * XP + u] = a.X[(((long long)b * N + m) * a.F + f) * a.T + t0 + u];
      gs[m * TC + u] = a.gr[((long long)b * N + m) * a.T + t0 + u];
    }
    __syncthreads();
    if (acc_on)
      for (int u = sl; u < nf; u += S) {
        const float2 xi = xs[pi * XP + u], xj = xs[pj * XP + u];
        // x_i conj(x_j): the products of float32 values are exact in fp64
        const double pre = (double)xi.x * (double)xj.x + (double)xi.y * (double)xj.y;
        const double pim = (double)xi.y * (double)xj.x - (double)xi.x * (double)xj.y;
#pragma unroll
        for (int n = 0; n < N; ++n) {
          const double g = gs[n * TC + u];
          ar[n] += g * pre;
          ai[n] += g * pim;
        }
      }
  }
  if (acc_on)
#pragma unroll
    for (int n = 0; n < N; ++n) red[(sl * P + pr) * N + n] = cd_make(ar[n], ai[n]);
  __syncthreads();
  for (int q = tid; q < P * N; q += K::THREADS) {                  // slices added in order, / T
    const int e = q / N, n = q - e * N;
    cd v = red[e * N + n];
    for (int k = 1; k < S; ++k) v = cd_add(v, red[(k * P + e) * N + n]);
    v = cd_make(v.x / a.T, v.y / a.T);
    int i, j;
    aux_pair<N>(e, i, j);
    V[(n * N + i) * N + j] = v;
    if (i != j) V[(n * N + j) * N + i] = cd_conj(v);
  }
  __syncthreads();

  // ---- the N sequential solves: w = solve(W^H V_n, e_n), W[:, n] = w / (w^H V_n w) ----
  bool singular = false;
  if constexpr (N <= 4) {
    if (tid == 0) {
      CMat<N>& A = *reinterpret_cast<CMat<N>*>(M);
      CVec<N>& w = *reinterpret_cast<CVec<N>*>(wv);
      for (int n = 0; n < N; ++n) {
        const cd* Vn = V + n * N * N;
#pragma unroll
        for (int r = 0; r < N; ++r)
#pragma unroll
          for (int c = 0; c < N; ++c) {
            cd s = cd_make(0.0, 0.0);
#pragma unroll
            for (int k = 0; k < N; ++k) s = cd_add(s, cd_mul(cd_conj(Ws[k * N + r]), Vn[k * N + c]));
            A.a[r][c] = s;
          }
        int perm[N];
        if (!lu_factor<N>(A, perm)) singular = true;
#pragma unroll
        for (int r = 0; r < N; ++r) w.v[r] = cd_make(r == n ? 1.0 : 0.0, 0.0);
        lu_solve_vec<N>(A, perm, w);
        cd d = cd_make(0.0, 0.0);
#pragma unroll
        for (int r = 0; r < N; ++r) {
          cd u = cd_make(0.0, 0.0);
#pragma unroll
          for (int c = 0; c < N; ++c) u = cd_add(u, cd_mul(Vn[r * N + c], w.v[c]));
          d = cd_add(d, cd_mul(cd_conj(w.v[r]), u));
        }
#pragma unroll
        for (int r = 0; r < N; ++r) Ws[r * N + n] = cd_div(w.v[r], d);
      }
    }
  } else {
    if (tid < 32) {                                                // one group of Coop<N>::GS lanes of warp 0
      const int r = tid;
      const bool row = r < N;
      for (int n = 0; n < N; ++n) {
        const cd* Vn = V + n * N * N;
        if (row) {
          for (int c = 0; c < N; ++c) {
            cd s = cd_make(0.0, 0.0);
            for (int k = 0; k < N; ++k) s = cd_add(s, cd_mul(cd_conj(Ws[k * N + r]), Vn[k * N + c]));
            M[r * LD + c] = s;
          }
          M[r * LD + N] = cd_make(r == n ? 1.0 : 0.0, 0.0);
        }
        __syncwarp();
        const cd x = lu_solve_coop<N>(M, r, row, &singular);
        if (row) wv[r] = x;
        __syncwarp();
        cd t = cd_make(0.0, 0.0);
        if (row) {
          cd u = cd_make(0.0, 0.0);
          for (int c = 0; c < N; ++c) u = cd_add(u, cd_mul(Vn[r * N + c], wv[c]));
          t = cd_mul(cd_conj(x), u);
        }
        const cd d = cd_make(group_sum<Coop<N>::GS>(t.x), group_sum<Coop<N>::GS>(t.y));
        if (row) Ws[r * N + n] = cd_div(x, d);
        __syncwarp();
      }
    }
  }
  __syncthreads();
  bool finite = true;
  for (int q = tid; q < N * N; q += K::THREADS) {
    const cd w = Ws[q];
    Wg[q] = w;
    if (!(isfinite(w.x) && isfinite(w.y))) finite = false;
  }
  if (a.status) {
    if (singular) atomicOr(a.status + b, (unsigned)SETK_ST_SINGULAR);
    if (!finite) atomicOr(a.status + b, (unsigned)SETK_ST_NONFINITE);
  }
}

size_t auxiva_scratch_bytes(int B, int N, int F, int T) {
  return sizeof(cd) * (size_t)B * F * N * N + sizeof(double) * (size_t)B * N * T;
}

template <int N>
static cudaError_t auxiva_t(AuxArgs a, int epochs, cd* out, void* stream) {
  const size_t smem = sizeof(double) * aux_update_smem_doubles<N>();
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(auxiva_update_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem);
  if (ea != cudaSuccess) return ea;
#endif
  const long long bins = (long long)a.B * a.F;
  const long long nw = bins * N * N;
  cudaError_t e = launch(auxiva_init_kernel, dim3((unsigned)((nw + 255) / 256)), dim3(256), 0, stream, true,
                         a.W, bins, N);
  const dim3 dgrid((a.T + kAuxFrames - 1) / kAuxFrames, a.B), dblock(kAuxFrames, kAuxSlices);
  a.out = nullptr;
  for (int it = 0; it < epochs && e == cudaSuccess; ++it) {
    e = launch(auxiva_demix_kernel<N>, dgrid, dblock, 0, stream, false, a);
    if (e == cudaSuccess)
      e = launch(auxiva_update_kernel<N>, dim3((unsigned)bins), dim3(AuxCfg<N>::THREADS), smem, stream, false, a);
  }
  if (e != cudaSuccess) return e;
  a.out = out;
  a.gr = nullptr;
  return launch(auxiva_demix_kernel<N>, dgrid, dblock, 0, stream, true, a);
}

// X [B][N][F][T] c64 -> Y [B][N][F][T] c128; ws: auxiva_scratch_bytes
cudaError_t run_auxiva(const float2* X, int B, int N, int F, int T, int epochs, char* ws, double2* out,
                       unsigned* status, void* stream) {
  AuxArgs a;
  a.X = X; a.B = B; a.F = F; a.T = T;
  a.W = reinterpret_cast<cd*>(ws);
  a.gr = reinterpret_cast<double*>(ws + sizeof(cd) * (size_t)B * F * N * N);
  a.out = nullptr;
  a.status = status;
  cd* Y = reinterpret_cast<cd*>(out);
  switch (N) {
    case 2: return auxiva_t<2>(a, epochs, Y, stream);
    case 3: return auxiva_t<3>(a, epochs, Y, stream);
    case 4: return auxiva_t<4>(a, epochs, Y, stream);
    case 5: return auxiva_t<5>(a, epochs, Y, stream);
    case 6: return auxiva_t<6>(a, epochs, Y, stream);
    case 7: return auxiva_t<7>(a, epochs, Y, stream);
    case 8: return auxiva_t<8>(a, epochs, Y, stream);
    case 9: return auxiva_t<9>(a, epochs, Y, stream);
    case 10: return auxiva_t<10>(a, epochs, Y, stream);
    case 11: return auxiva_t<11>(a, epochs, Y, stream);
    case 12: return auxiva_t<12>(a, epochs, Y, stream);
    case 13: return auxiva_t<13>(a, epochs, Y, stream);
    case 14: return auxiva_t<14>(a, epochs, Y, stream);
    case 15: return auxiva_t<15>(a, epochs, Y, stream);
    case 16: return auxiva_t<16>(a, epochs, Y, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
