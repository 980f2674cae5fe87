// ssl.cuh -- mask-informed sound source localisation: the three DoA estimators of the reference's
// libs/ssl.py (ml_ssl :12-43, srp_ssl :46-77, music_ssl :80-110) as driven by do_ssl.py.
//
// Every backend reduces to a score per (utterance, mask, frame window, direction) followed by an
// arg-extreme.  A frame window [s, e) is the whole utterance offline, or one chunk of do_ssl.py's
// online mode (:103-111); ragged batches are windows that stop at each utterance's own length.
//
//   ML     ssl_ml_kernel: one CTA per (utterance, 32-frame tile, 8-direction tile) loops over all
//          bins; per bin it stages x[:, f, tile] and the tile's normalised steering vectors in
//          shared memory and evaluates the per-cell log-likelihood in registers, accumulating
//          P[n][a][t] = sum_f mask_n[t][f] ll[a][t][f] in fixed bin order.  The A x T x F
//          likelihood tensor of the reference never exists.  ssl_window_kernel then sums P over
//          each window in frame order.
//   SRP    cos(o - r) = cos o cos r + sin o sin r moves the masked frame sum inside:
//          ssl_srp_accum_kernel forms C_p[w][f] = sum_{t in w} m cos o_p, S_p likewise (one pass
//          over the STFT), ssl_srp_score_kernel adds sum_f sum_p (cos r C_p + sin r S_p) / P.
//          Cost T F P + W A F P instead of the reference's A T F P.
//   MUSIC  ssl_music_cov_kernel: the per-window covariance sum_t (m x)(m x)^H / len in fp64;
//          the principal eigenvector comes from the weight solver's fp64 Jacobi (setk_weights,
//          SETK_BF_PEVD); ssl_music_score_kernel adds sum_f | ||s||^2 - |u^H s|^2 |, i.e.
//          s^H (I - u u^H) s, the projector the reference builds from the M - 1 minor eigenvectors.
//
// Rounding: the reference's float32 steps are reproduced operation by operation where numpy's
// result is IEEE-defined -- |x| and x / max(|x|, eps) of norm=True (a multiply by the float32
// reciprocal, numpy's complex-by-real division), and ssh = sum_m (re re + im im) in channel order
// with no FMA contraction (the idiom of cm_mask.cu).  The float32 phase of SRP is the correctly
// rounded angle (atan2 in fp64, rounded once): numpy's float32 arctan2 is a vectorised
// approximation that is not reproducible elsewhere.  Everything else is fp64.  No float atomics:
// two identical calls give bit-identical scores.
//
// Built as part of spatial.cu's translation unit (included once, at its end): localisation is the
// spatial analysis that turns these features into a direction.
#pragma once
#include "common.cuh"
#include "launchers.cuh"
#include <math.h>

namespace setk {

#define SETK_SSL_TT 32          // frames per ML CTA
#define SETK_SSL_TA 8           // directions per ML CTA
#define SETK_SSL_MAX_MASKS 8

// ---- steering tables ----
// ML: table[f][a][m] = sv[a][m][f] / ||sv[a][:, f]|| (ml_ssl :27), the reciprocal multiplied like
// numpy's complex-by-real division
__global__ void ssl_ml_table_kernel(const double2* __restrict__ sv, int A, int M, int F,
                                    double2* __restrict__ table) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * A) return;
  const int f = (int)(i / A), a = (int)(i - (long long)f * A);
  double n2 = 0.0;
  for (int m = 0; m < M; ++m) {
    const double2 s = sv[((long long)a * M + m) * F + f];
    n2 += s.x * s.x + s.y * s.y;
  }
  const double scl = 1.0 / sqrt(n2);
  for (int m = 0; m < M; ++m) {
    const double2 s = sv[((long long)a * M + m) * F + f];
    table[i * M + m] = make_double2(s.x * scl, s.y * scl);
  }
}

// SRP: table[f][p][a] = (cos, sin) of the oracle IPD angle(sv[a][l]) - angle(sv[a][r]) (srp_ssl :66-70)
__global__ void ssl_srp_table_kernel(const double2* __restrict__ sv, const int* __restrict__ pairs, int P,
                                     int A, int M, int F, double2* __restrict__ table) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * P * A) return;
  const int a = (int)(i % A);
  const int p = (int)((i / A) % P);
  const int f = (int)(i / ((long long)A * P));
  const double2 sl = sv[((long long)a * M + pairs[2 * p]) * F + f];
  const double2 sr = sv[((long long)a * M + pairs[2 * p + 1]) * F + f];
  double s, c;
  sincos(atan2(sl.y, sl.x) - atan2(sr.y, sr.x), &s, &c);
  table[i] = make_double2(c, s);
}

// ---- ML ----
// grid (ceil(T / TT), ceil(A / TA), B), block TT * TA.  P [B][N][A][T] fp64.
__global__ void __launch_bounds__(SETK_SSL_TT * SETK_SSL_TA)
ssl_ml_kernel(const float2* __restrict__ stft, const double2* __restrict__ table,
              const float* __restrict__ mask, int N, int M, int F, int T, int A, int norm,
              double compression, double eps, double inv_1pe, double* __restrict__ P) {
  __shared__ float2 sx[SETK_MAX_CHANNELS][SETK_SSL_TT];
  __shared__ double2 ssv[SETK_SSL_TA][SETK_MAX_CHANNELS];
  __shared__ float smk[SETK_SSL_MAX_MASKS][SETK_SSL_TT];
  const int tid = threadIdx.x, tt = tid % SETK_SSL_TT, ta = tid / SETK_SSL_TT;
  const int t0 = blockIdx.x * SETK_SSL_TT, a0 = blockIdx.y * SETK_SSL_TA, b = blockIdx.z;
  const float eps_f = (float)eps;      // np.maximum(float32 array, python float) stays float32
  double acc[SETK_SSL_MAX_MASKS];
#pragma unroll
  for (int n = 0; n < SETK_SSL_MAX_MASKS; ++n) acc[n] = 0.0;
  const float2* xb = stft + (long long)b * M * F * T;
  const float* mb = mask ? mask + (long long)b * N * T * F : nullptr;
  for (int f = 0; f < F; ++f) {
    for (int e = tid; e < M * SETK_SSL_TT; e += blockDim.x) {
      const int m = e / SETK_SSL_TT, k = e - m * SETK_SSL_TT;
      float2 x = make_float2(0.f, 0.f);
      if (t0 + k < T) {
        x = xb[((long long)m * F + f) * T + t0 + k];
        if (norm) {   // stft / max(cmat_abs(stft), eps): ml_ssl :28-29, utils.py:42
          // sqrtf is IEEE round-to-nearest (nvcc's default -prec-sqrt=true)
          const float mag = sqrtf(__fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)));
          const float scl = __fdiv_rn(1.0f, mag < eps_f ? eps_f : mag);
          x = make_float2(__fmul_rn(x.x, scl), __fmul_rn(x.y, scl));
        }
      }
      sx[m][k] = x;
    }
    for (int e = tid; e < SETK_SSL_TA * M; e += blockDim.x) {
      const int k = e / M, m = e - k * M;
      ssv[k][m] = a0 + k < A ? table[((long long)f * A + a0 + k) * M + m] : make_double2(0.0, 0.0);
    }
    if (mb)
      for (int e = tid; e < N * SETK_SSL_TT; e += blockDim.x) {
        const int n = e / SETK_SSL_TT, k = e - n * SETK_SSL_TT;
        smk[n][k] = t0 + k < T ? mb[((long long)n * T + t0 + k) * F + f] : 0.f;
      }
    __syncthreads();
    // ssh = |sum_m x conj(x)| in complex64 (ml_ssl :30): the imaginary parts cancel exactly
    float ssh = 0.f;
    double re = 0.0, im = 0.0;
    for (int m = 0; m < M; ++m) {
      const float2 x = sx[m][tt];
      ssh = __fadd_rn(ssh, __fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)));
      // s conj(x) in fp64 (ml_ssl :31)
      const double2 s = ssv[ta][m];
      const double xr = (double)x.x, xi = (double)x.y;
      re += s.x * xr + s.y * xi;
      im += s.y * xr - s.x * xi;
    }
    const double delta = (double)ssh - (re * re + im * im) * inv_1pe;   // ml_ssl :33
    double ll;
    if (compression <= 0.0) ll = -log(delta < eps ? eps : delta);       // NaN stays NaN
    else ll = -pow(delta, compression);                                  // delta < 0 -> NaN
    if (mb) {
#pragma unroll
      for (int n = 0; n < SETK_SSL_MAX_MASKS; ++n)
        if (n < N) acc[n] += (double)smk[n][tt] * ll;
    } else {
      acc[0] += ll;
    }
    __syncthreads();
  }
  const int t = t0 + tt, a = a0 + ta;
  if (t < T && a < A) {
    const int nn = mb ? N : 1;
#pragma unroll
    for (int n = 0; n < SETK_SSL_MAX_MASKS; ++n)   // constant indices keep acc[] in registers
      if (n < nn) P[(((long long)b * nn + n) * A + a) * T + t] = acc[n];
  }
}

// scores[b][n][w][a] = sum_{t in window w} P[b][n][a][t], frame order
__global__ void ssl_window_kernel(const double* __restrict__ P, const int* __restrict__ win, int N, int W,
                                  int A, int T, long long total, double* __restrict__ scores) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int a = (int)(i % A);
  const int w = (int)((i / A) % W);
  const long long bn = i / ((long long)A * W);
  const int b = (int)(bn / N);
  const int s = win[((long long)b * W + w) * 2], e = win[((long long)b * W + w) * 2 + 1];
  const double* row = P + (bn * A + a) * T;
  double acc = 0.0;
  for (int t = s; t < e; ++t) acc += row[t];
  scores[i] = acc;
}

// index[r] = numpy's argmax (want_min == 0) / argmin of scores[r][:]: the first extreme, or the
// first NaN when there is one
__global__ void ssl_argext_kernel(const double* __restrict__ scores, long long rows, int A, int want_min,
                                  int* __restrict__ index) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const double* v = scores + r * A;
  int best = 0;
  double bv = v[0];
  if (bv == bv) {
    for (int a = 1; a < A; ++a) {
      const double x = v[a];
      if (x != x) { best = a; break; }
      if (want_min ? x < bv : x > bv) { bv = x; best = a; }
    }
  }
  index[r] = best;
}

// ---- SRP ----
// CS[b][w][p][f] = (sum_{t in w} m cos o, sum_{t in w} m sin o), o = angle(x_l) - angle(x_r) in
// float32 (srp_ssl :64-68), promoted to fp64 where the reference subtracts the fp64 oracle IPD (:72)
__device__ __forceinline__ float ssl_angle_f(float2 z) { return (float)atan2((double)z.y, (double)z.x); }

__global__ void ssl_srp_accum_kernel(const float2* __restrict__ stft, const float* __restrict__ mask,
                                     const int* __restrict__ win, const int* __restrict__ pairs, int P,
                                     int W, int M, int F, int T, long long total, double2* __restrict__ CS) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int f = (int)(i % F);
  const int p = (int)((i / F) % P);
  const long long bw = i / ((long long)F * P);
  const int b = (int)(bw / W);
  const int s = win[bw * 2], e = win[bw * 2 + 1];
  const float2* xl = stft + (((long long)b * M + pairs[2 * p]) * F + f) * T;
  const float2* xr = stft + (((long long)b * M + pairs[2 * p + 1]) * F + f) * T;
  const float* mb = mask ? mask + (long long)b * T * F + f : nullptr;
  double c = 0.0, sn = 0.0;
  for (int t = s; t < e; ++t) {
    const float o = __fsub_rn(ssl_angle_f(xl[t]), ssl_angle_f(xr[t]));
    double so, co;
    sincos((double)o, &so, &co);
    const double m = mb ? (double)mb[(long long)t * F] : 1.0;
    c += m * co;
    sn += m * so;
  }
  CS[i] = make_double2(c, sn);
}

// scores[b][w][a] = sum_f sum_p (cos r C_p + sin r S_p) / P   (the mean over pairs, srp_ssl :74-76)
__global__ void ssl_srp_score_kernel(const double2* __restrict__ CS, const double2* __restrict__ table,
                                     int P, int A, int F, long long total, double* __restrict__ scores) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int a = (int)(i % A);
  const long long bw = i / A;
  const double2* cs = CS + bw * P * F;
  double acc = 0.0;
  for (int f = 0; f < F; ++f) {
    double cell = 0.0;
    for (int p = 0; p < P; ++p) {
      const double2 r = table[((long long)f * P + p) * A + a];
      const double2 v = cs[(long long)p * F + f];
      cell += r.x * v.x + r.y * v.y;
    }
    acc += cell / (double)P;
  }
  scores[i] = acc;
}

// ---- MUSIC ----
// R[b][w][f][i][j] = sum_{t in w} (m x_i) conj(m x_j) / (e - s)   (music_ssl :94-96), fp64
__global__ void ssl_music_cov_kernel(const float2* __restrict__ stft, const float* __restrict__ mask,
                                     const int* __restrict__ win, int W, int M, int F, int T, long long total,
                                     double2* __restrict__ R) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int j = (int)(idx % M);
  const int i = (int)((idx / M) % M);
  const int f = (int)((idx / ((long long)M * M)) % F);
  const long long bw = idx / ((long long)M * M * F);
  const int b = (int)(bw / W);
  const int s = win[bw * 2], e = win[bw * 2 + 1];
  const float2* xi = stft + (((long long)b * M + i) * F + f) * T;
  const float2* xj = stft + (((long long)b * M + j) * F + f) * T;
  const float* mb = mask ? mask + (long long)b * T * F + f : nullptr;
  double ar = 0.0, ai = 0.0;
  for (int t = s; t < e; ++t) {
    const double m = mb ? (double)mb[(long long)t * F] : 1.0;
    const float2 u = xi[t], v = xj[t];
    const double ur = m * u.x, ui = m * u.y, vr = m * v.x, vi = m * v.y;   // exact products
    ar += ur * vr + ui * vi;
    ai += ui * vr - ur * vi;
  }
  const double len = (double)(e - s);
  R[idx] = make_double2(ar / len, ai / len);
}

// scores[b][w][a] = sum_f | ||s||^2 - |u^H s|^2 |, steering vectors as given (music_ssl :104-109).
// A bin whose covariance is exactly zero gets u = e_{M-1}: LAPACK's eigenvectors of the zero matrix
// are the identity and the reference keeps the last column as the signal subspace.
__global__ void ssl_music_score_kernel(const double2* __restrict__ sv, const double2* __restrict__ R,
                                       const double2* __restrict__ U, int M, int F, int A, long long total,
                                       double* __restrict__ scores) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int a = (int)(i % A);
  const long long bw = i / A;
  double acc = 0.0;
  for (int f = 0; f < F; ++f) {
    const double2* r = R + (bw * F + f) * M * M;
    const double2* u = U + (bw * F + f) * M;
    double tr = 0.0;
    for (int m = 0; m < M; ++m) tr += r[m * M + m].x;
    const bool zero = tr == 0.0;
    double ns = 0.0, pr = 0.0, pi = 0.0;
    for (int m = 0; m < M; ++m) {
      const double2 s = sv[((long long)a * M + m) * F + f];
      ns += s.x * s.x + s.y * s.y;
      const double2 um = zero ? make_double2(m == M - 1 ? 1.0 : 0.0, 0.0) : u[m];
      pr += um.x * s.x + um.y * s.y;          // conj(u) s
      pi += um.x * s.y - um.y * s.x;
    }
    acc += fabs(ns - (pr * pr + pi * pi));
  }
  scores[i] = acc;
}

static unsigned blocks_of(long long n, int bs) { return (unsigned)((n + bs - 1) / bs); }

// Scratch (stream-ordered): device copies of the windows / pairs, then the backend's tables.
size_t ssl_scratch_bytes(int backend, int B, int N, int M, int F, int T, int A, int W, int P) {
  size_t n = up256(sizeof(int) * 2 * (size_t)B * W) + up256(sizeof(int) * 2 * (size_t)(P > 0 ? P : 1));
  if (backend == SETK_SSL_ML)
    n += up256(sizeof(double2) * (size_t)F * A * M) + up256(sizeof(double) * (size_t)B * N * A * T);
  else if (backend == SETK_SSL_SRP)
    n += up256(sizeof(double2) * (size_t)F * P * A) + up256(sizeof(double2) * (size_t)B * W * P * F);
  else
    n += up256(sizeof(double2) * (size_t)B * W * F * M * M) + up256(sizeof(double2) * (size_t)B * W * F * M) +
         up256(sizeof(unsigned) * (size_t)B * W);
  return n;
}

cudaError_t run_ssl(int backend, const float2* stft, int B, int M, int F, int T, const double2* sv, int A,
                    const float* mask, int N, const int* windows_host, int W, const int* pairs_host, int P,
                    double compression, double eps, int normalize, char* ws, double* scores, int* index,
                    void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* win = reinterpret_cast<int*>(ws);
  ws += up256(sizeof(int) * 2 * (size_t)B * W);
  int* pairs = reinterpret_cast<int*>(ws);
  ws += up256(sizeof(int) * 2 * (size_t)(P > 0 ? P : 1));
  cudaError_t e = cudaMemcpyAsync(win, windows_host, sizeof(int) * 2 * (size_t)B * W, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && P > 0)
    e = cudaMemcpyAsync(pairs, pairs_host, sizeof(int) * 2 * (size_t)P, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  const int NN = mask ? N : 1;
  const long long rows = (long long)B * NN * W;
  if (backend == SETK_SSL_ML) {
    double2* table = reinterpret_cast<double2*>(ws);
    double* Pt = reinterpret_cast<double*>(ws + up256(sizeof(double2) * (size_t)F * A * M));
    e = launch(ssl_ml_table_kernel, dim3(blocks_of((long long)F * A, 128)), dim3(128), 0, stream, true, sv, A,
               M, F, table);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((T + SETK_SSL_TT - 1) / SETK_SSL_TT), (unsigned)((A + SETK_SSL_TA - 1) / SETK_SSL_TA),
                    (unsigned)B);
    e = launch(ssl_ml_kernel, grid, dim3(SETK_SSL_TT * SETK_SSL_TA), 0, stream, false, stft,
               (const double2*)table, mask, NN, M, F, T, A, normalize, compression, eps, 1.0 / (1.0 + eps), Pt);
    if (e != cudaSuccess) return e;
    e = launch(ssl_window_kernel, dim3(blocks_of(rows * A, 128)), dim3(128), 0, stream, true, (const double*)Pt,
               (const int*)win, NN, W, A, T, rows * A, scores);
  } else if (backend == SETK_SSL_SRP) {
    double2* table = reinterpret_cast<double2*>(ws);
    double2* CS = reinterpret_cast<double2*>(ws + up256(sizeof(double2) * (size_t)F * P * A));
    e = launch(ssl_srp_table_kernel, dim3(blocks_of((long long)F * P * A, 128)), dim3(128), 0, stream, true, sv,
               (const int*)pairs, P, A, M, F, table);
    if (e != cudaSuccess) return e;
    const long long ncs = (long long)B * W * P * F;
    e = launch(ssl_srp_accum_kernel, dim3(blocks_of(ncs, 128)), dim3(128), 0, stream, true, stft, mask,
               (const int*)win, (const int*)pairs, P, W, M, F, T, ncs, CS);
    if (e != cudaSuccess) return e;
    e = launch(ssl_srp_score_kernel, dim3(blocks_of(rows * A, 128)), dim3(128), 0, stream, true,
               (const double2*)CS, (const double2*)table, P, A, F, rows * A, scores);
  } else {
    double2* R = reinterpret_cast<double2*>(ws);
    ws += up256(sizeof(double2) * (size_t)B * W * F * M * M);
    double2* U = reinterpret_cast<double2*>(ws);
    ws += up256(sizeof(double2) * (size_t)B * W * F * M);
    unsigned* status = reinterpret_cast<unsigned*>(ws);
    e = cudaMemsetAsync(status, 0, sizeof(unsigned) * (size_t)B * W, st);
    if (e != cudaSuccess) return e;
    const long long nr = (long long)B * W * F * M * M;
    e = launch(ssl_music_cov_kernel, dim3(blocks_of(nr, 128)), dim3(128), 0, stream, true, stft, mask,
               (const int*)win, W, M, F, T, nr, R);
    if (e != cudaSuccess) return e;
    e = weights_run(SETK_BF_PEVD, 0.0, -1, SETK_RANK1_NONE, 0, R, nullptr, nullptr, SETK_C128, B * W, F, M, U,
                    SETK_C128, status, nullptr, stream);
    if (e != cudaSuccess) return e;
    e = launch(ssl_music_score_kernel, dim3(blocks_of(rows * A, 128)), dim3(128), 0, stream, true, sv,
               (const double2*)R, (const double2*)U, M, F, A, rows * A, scores);
  }
  if (e != cudaSuccess) return e;
  return launch(ssl_argext_kernel, dim3(blocks_of(rows, 128)), dim3(128), 0, stream, true, (const double*)scores,
                rows, A, backend == SETK_SSL_MUSIC ? 1 : 0, index);
}

}  // namespace setk
