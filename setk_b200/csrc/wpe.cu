// wpe.cu -- WPE dereverberation of a multichannel STFT (the pre-processor of
// BASELINE config 4; SURVEY.md §8(f) rank 2).  Replaces, per utterance and bin,
//   scripts/sptk/libs/wpe.py:14-30   compute_tap_mat (the delayed stack, never built here)
//   scripts/sptk/libs/wpe.py:33-56   compute_lambda  (channel-mean power, +-context box, floor)
//   scripts/sptk/libs/wpe.py:59-79   wpe_step        (R, r, G = solve(R, r), z = x - G^H yt)
//   scripts/sptk/libs/wpe.py:82-110  wpe             (num_iters steps)
//
// Every bin is an independent problem of size NK = channels x taps, so a CTA
// owns ONE (utterance, bin) and keeps that bin's time series in shared memory
// as fp64 (converted once; rows carry taps + delay frames of history, zeros
// before frame 0, so the delayed stack yt[k N + n, t] = x[n, t - k - delay] is
// just an offset).  An utterance that does not fit is walked in chunks of Tc
// frames (each reloaded with its history and +-context halo); the sums run over
// t in the same order either way, so chunking does not change a bit:
//   wpe_corr_kernel    prologue: previous filter G -> z -> lambda (or lambda of x);
//                      then [R | r] = sum_t a_i conj(a_j) / lambda, 4 x 4 register tiles
//                      over the upper block triangle of the augmented matrix
//   wpe_solve_kernel   LU with partial pivoting of [R | r], four threads per row
//                      (numpy.linalg.solve), column-oriented back substitution -> G
//   wpe_filter_kernel  z = x - G^H yt, written in the API layout [B][C][F][T]
// All arithmetic is fp64 (the reference computes in the dtype of its input,
// complex64; see oracle/wpe_oracle.py).
#include <cstdlib>
#include "common.cuh"
#include "hermitian_solve.cuh"
#include "launchers.cuh"

namespace setk {

struct WpeArgs {
  const float2* X; int P;        // bin-major workspace [B][T][C][P]
  int B, C, F, T;
  int taps, delay, ctx;
  int NK;                        // C * taps
  int Tc;                        // frames per chunk (>= T: the whole utterance at once)
  int Wp;                        // row length in shared memory: Tc + 2 ctx + taps + delay
  int use_filter;                // corr: lambda from z = x - G^H yt (iterations > 0)
  const double* G;               // [B*F][NK][C] complex (interleaved)
  double* Raug;                  // [B*F][NK][NK + C] complex
  float2* out;                   // filter: [B][C][F][T]
  unsigned* status;              // [B]
  const float2* lam_src;         // corr, first pass only: lambda = max(|e|^2, eps) of this [B][F][T]
                                 // spectrum (facted_wpd, wpe.py:150-153) instead of compute_lambda
  float* linv_out;               // corr: 1 / lambda -> [B][T][F] f32 (weights of Rd, wpe.py:165), or null
};

// shared memory: xs [C][Wp] cd | linv [Tc] | L [Tc + 2 ctx] | Gs [NK][C] cd
__device__ __forceinline__ void wpe_carve(double* sm, const WpeArgs& a, cd*& xs, double*& linv, double*& L, cd*& Gs) {
  xs = reinterpret_cast<cd*>(sm);
  linv = sm + 2 * (size_t)a.C * a.Wp;
  L = linv + a.Tc;
  const int nl = a.Tc + 2 * a.ctx;
  Gs = reinterpret_cast<cd*>(L + nl + ((a.Tc + nl) & 1));
}
SETK_HD inline size_t wpe_smem_bytes(int C, int Tc, int ctx, int hist, int NK) {
  const size_t nl = (size_t)Tc + 2 * ctx;
  return sizeof(double) * (2 * (size_t)C * (nl + hist) + Tc + nl + ((Tc + nl) & 1) + 2 * (size_t)NK * C);
}

// frames [base, base + Wp) of bin (b, f) of the workspace -> xs (fp64, zeros outside [0, T))
__device__ __forceinline__ void wpe_load_bin(const WpeArgs& a, int b, int f, cd* xs, int base) {
  for (int q = threadIdx.x; q < a.C * a.Wp; q += blockDim.x) {
    const int n = q / a.Wp, g = base + (q - n * a.Wp);
    cd v = cd_make(0.0, 0.0);
    if (g >= 0 && g < a.T) {
      const float2 x = a.X[(((long long)b * a.T + g) * a.C + n) * a.P + f];
      v = cd_make((double)x.x, (double)x.y);
    }
    xs[q] = v;
  }
}

// z_n[t] = x_n[t] - sum_m conj(G[m][n]) yt[m][t]   (wpe.py:78); p = position of frame t in xs
__device__ __forceinline__ cd wpe_filtered(const WpeArgs& a, const cd* xs, const cd* Gs, int n, int p) {
  cd z = xs[n * a.Wp + p];
  for (int k = 0; k < a.taps; ++k) {
    const int pp = p - k - a.delay;                // >= 0: every row carries taps + delay frames of history
    for (int c = 0; c < a.C; ++c)
      z = cd_sub(z, cd_mul(cd_conj(Gs[(k * a.C + c) * a.C + n]), xs[c * a.Wp + pp]));
  }
  return z;
}

// One chunk of frames [t0, t0 + n) of bin (b, f): load it (with history and context halo) and
// compute 1 / lambda for its frames (wpe.py:33-56).  All threads of the CTA; ends with a barrier.
__device__ __forceinline__ void wpe_chunk_prologue(const WpeArgs& a, int b, int f, int t0, int n, cd* xs,
                                                   double* linv, double* L, const cd* Gs) {
  const int tid = threadIdx.x, C = a.C;
  const int hist = a.taps + a.delay;
  const int base = t0 - a.ctx - hist;                   // frame at position 0 of xs
  __syncthreads();                                       // the previous chunk is consumed
  wpe_load_bin(a, b, f, xs, base);
  __syncthreads();
  // ---- channel-mean power of frames [t0 - ctx, t0 + n + ctx) ----
  for (int u = tid; u < n + 2 * a.ctx; u += blockDim.x) {
    const int t = t0 - a.ctx + u;
    double p = 0.0;
    if (t >= 0 && t < a.T)
      for (int c = 0; c < C; ++c) {
        const cd z = a.use_filter ? wpe_filtered(a, xs, Gs, c, u + hist) : xs[c * a.Wp + u + hist];
        p += z.x * z.x + z.y * z.y;
      }
    L[u] = p / (double)C;
  }
  __syncthreads();
  for (int u = tid; u < n; u += blockDim.x) {
    const int t = t0 + u;
    double lam;
    if (a.lam_src && !a.use_filter) {
      const float2 ev = a.lam_src[((long long)b * a.F + f) * a.T + t];
      lam = (double)ev.x * (double)ev.x + (double)ev.y * (double)ev.y;
    } else {
      double s = 0.0;
      int cnt = 0;
      for (int c = -a.ctx; c <= a.ctx; ++c)
        if (t + c >= 0 && t + c < a.T) { s += L[u + a.ctx + c]; ++cnt; }
      lam = s / (double)cnt;
    }
    linv[u] = 1.0 / fmax(lam, SETK_EPS32_D);
    if (a.linv_out) a.linv_out[((long long)b * a.T + t) * a.F + f] = (float)linv[u];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(512) wpe_corr_kernel(WpeArgs a) {
  SETK_DYN_SMEM(double, sm);
  cd* xs; double* linv; double* L; cd* Gs;
  wpe_carve(sm, a, xs, linv, L, Gs);
  const int bin = blockIdx.x, b = bin / a.F, f = bin - b * a.F;
  const int tid = threadIdx.x;
  const int hist = a.taps + a.delay, C = a.C, NK = a.NK, NA = NK + C;
  if (a.use_filter)
    for (int q = tid; q < NK * C; q += blockDim.x) {
      const double* g = a.G + ((long long)bin * NK * C + q) * 2;
      Gs[q] = cd_make(g[0], g[1]);
    }
  // ---- [R | r]: 4 x 4 tiles (I, J >= I) of the NK x (NK + C) augmented matrix ----
  const int RT = (NK + 3) / 4, CT = (NA + 3) / 4;
  int I = 0, e = tid;
  while (I < RT && e >= CT - I) { e -= CT - I; ++I; }
  const bool tile = I < RT;
  const int J = I + e;
  // row m of the augmented operand: m < NK -> x_{m % C} delayed by m / C + delay; else x_{m - NK}
  // (offsets relative to the position of frame t)
  int oi[4], oj[4];
  bool vi[4], vj[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int mi = 4 * I + u, mj = 4 * J + u;
    vi[u] = tile && mi < NK;
    vj[u] = tile && mj < NA;
    oi[u] = vi[u] ? (mi % C) * a.Wp - (mi / C) - a.delay : 0;
    oj[u] = vj[u] ? (mj < NK ? (mj % C) * a.Wp - (mj / C) - a.delay : (mj - NK) * a.Wp) : 0;
  }
  double ar[4][4], ai[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) { ar[u][v] = 0.0; ai[u][v] = 0.0; }

  for (int t0 = 0; t0 < a.T; t0 += a.Tc) {
    const int n = imin(a.Tc, a.T - t0);
    wpe_chunk_prologue(a, b, f, t0, n, xs, linv, L, Gs);
    if (tile) {
      const cd* xt = xs + a.ctx + hist;                    // position of frame t0
      for (int u = 0; u < n; ++u) {
        const double w = linv[u];
        cd p[4], q[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          p[k] = vi[k] ? xt[oi[k] + u] : cd_make(0.0, 0.0);
          q[k] = vj[k] ? xt[oj[k] + u] : cd_make(0.0, 0.0);
          p[k].x *= w; p[k].y *= w;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int v = 0; v < 4; ++v) {                     // p conj(q)
            ar[k][v] += p[k].x * q[v].x + p[k].y * q[v].y;
            ai[k][v] += p[k].y * q[v].x - p[k].x * q[v].y;
          }
      }
    }
  }
  if (!tile) return;
  double* R = a.Raug + (long long)bin * NK * NA * 2;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = 4 * I + u, j = 4 * J + v;
      if (i >= NK || j >= NA) continue;
      if (j >= i) { R[((long long)i * NA + j) * 2] = ar[u][v]; R[((long long)i * NA + j) * 2 + 1] = ai[u][v]; }
      if (j > i && j < NK) {                              // Hermitian mirror (the solve reads the full matrix)
        R[((long long)j * NA + i) * 2] = ar[u][v];
        R[((long long)j * NA + i) * 2 + 1] = -ai[u][v];
      }
    }
}

// CTA per bin; thread (r, cg) = (tid / 4, tid % 4) owns columns j = cg (mod 4) of row r of
// the augmented [R | r].  The multipliers are used and dropped (the right-hand sides
// ride along), so a step costs three barriers: pivot vote, row swap, elimination.
__global__ void __launch_bounds__(512) wpe_solve_kernel(WpeArgs a, double* Gout) {
  SETK_DYN_SMEM(double, sm);
  const int NK = a.NK, C = a.C, NA = NK + C, LD = NA + 1;
  cd* M = reinterpret_cast<cd*>(sm);                         // [NK][LD]
  double* red_v = sm + 2 * (size_t)NK * LD;                  // [16 warps]
  int* red_i = reinterpret_cast<int*>(red_v + 16);
  const int bin = blockIdx.x, b = bin / a.F;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = (blockDim.x + 31) >> 5;
  const int r = tid >> 2, cg = tid & 3;
  const bool row = r < NK;
  const double* R = a.Raug + (long long)bin * NK * NA * 2;
  for (int q = tid; q < NK * NA; q += blockDim.x) {
    const int i = q / NA, j = q - i * NA;
    M[i * LD + j] = cd_make(R[2 * (long long)q], R[2 * (long long)q + 1]);
  }
  __syncthreads();
  bool singular = false;
  for (int k = 0; k < NK; ++k) {
    double m = (cg == 0 && row && r >= k) ? fabs(M[r * LD + k].x) + fabs(M[r * LD + k].y) : -1.0;
    int piv = r;
    for (int o = 16; o > 0; o >>= 1) {                        // izamax: first index on ties
      const double m2 = __shfl_xor_sync(0xffffffffu, m, o);
      const int p2 = __shfl_xor_sync(0xffffffffu, piv, o);
      if (m2 > m || (m2 == m && p2 < piv)) { m = m2; piv = p2; }
    }
    if (lane == 0) { red_v[wid] = m; red_i[wid] = piv; }
    __syncthreads();
    m = red_v[0]; piv = red_i[0];
    for (int w = 1; w < nw; ++w)
      if (red_v[w] > m || (red_v[w] == m && red_i[w] < piv)) { m = red_v[w]; piv = red_i[w]; }
    if (piv != k)
      for (int j = tid; j < NA; j += blockDim.x) { const cd t = M[k * LD + j]; M[k * LD + j] = M[piv * LD + j]; M[piv * LD + j] = t; }
    __syncthreads();
    if (m == 0.0) singular = true;
    if (row && r > k && m != 0.0) {
      const cd l = cd_mul(M[r * LD + k], cd_div(cd_make(1.0, 0.0), M[k * LD + k]));   // column k is read-only here
      for (int j = k + 1 + cg; j < NA; j += 4) M[r * LD + j] = cd_sub(M[r * LD + j], cd_mul(l, M[k * LD + j]));
    }
    __syncthreads();
  }
  for (int i = NK - 1; i >= 0; --i) {                         // back substitution, all C right-hand sides
    if (tid < C) M[i * LD + NK + tid] = cd_div(M[i * LD + NK + tid], M[i * LD + i]);
    __syncthreads();
    if (row && r < i)
      for (int n = cg; n < C; n += 4)
        M[r * LD + NK + n] = cd_sub(M[r * LD + NK + n], cd_mul(M[r * LD + i], M[i * LD + NK + n]));
    __syncthreads();
  }
  double* G = Gout + (long long)bin * NK * C * 2;
  if (row)
    for (int n = cg; n < C; n += 4) {
      const cd g = M[r * LD + NK + n];
      G[((long long)r * C + n) * 2] = g.x;
      G[((long long)r * C + n) * 2 + 1] = g.y;
      if (!(isfinite(g.x) && isfinite(g.y))) singular = true;
    }
  if (singular && a.status) atomicOr(a.status + b, (unsigned)SETK_ST_SINGULAR);
}

__global__ void __launch_bounds__(256) wpe_filter_kernel(WpeArgs a) {
  SETK_DYN_SMEM(double, sm);
  cd* xs; double* linv; double* L; cd* Gs;
  wpe_carve(sm, a, xs, linv, L, Gs);
  const int bin = blockIdx.x, b = bin / a.F, f = bin - b * a.F;
  const int hist = a.taps + a.delay;
  for (int q = threadIdx.x; q < a.NK * a.C; q += blockDim.x) {
    const double* g = a.G + ((long long)bin * a.NK * a.C + q) * 2;
    Gs[q] = cd_make(g[0], g[1]);
  }
  for (int t0 = 0; t0 < a.T; t0 += a.Tc) {
    const int n = imin(a.Tc, a.T - t0);
    __syncthreads();
    wpe_load_bin(a, b, f, xs, t0 - a.ctx - hist);
    __syncthreads();
    for (int q = threadIdx.x; q < a.C * n; q += blockDim.x) {
      const int c = q / n, u = q - c * n;
      const cd z = wpe_filtered(a, xs, Gs, c, u + a.ctx + hist);
      a.out[(((long long)b * a.C + c) * a.F + f) * a.T + t0 + u] = make_float2((float)z.x, (float)z.y);
    }
  }
}

// ---------------------------------------------------------------------------
// what the kernels can hold: tiles <= 512 threads, matrices within shared memory
static const size_t kWpeSmemCap = 200 * 1024;
// frames per chunk: the whole utterance when it fits, else the largest multiple of 32 that does
static int wpe_chunk_frames(int C, int T, int taps, int delay, int ctx) {
  const int NK = C * taps, hist = taps + delay;
  if (wpe_smem_bytes(C, T, ctx, hist, NK) <= kWpeSmemCap) return T;
  int tc = 32;
  while (wpe_smem_bytes(C, tc + 32, ctx, hist, NK) <= kWpeSmemCap) tc += 32;
  return tc;
}
bool wpe_supported(int C, int T, int taps, int delay, int ctx) {
  (void)T;                       // any length: long utterances are walked in chunks
  const int NK = C * taps, NA = NK + C, RT = (NK + 3) / 4, CT = (NA + 3) / 4;
  if (NK > 128 || RT * CT - RT * (RT - 1) / 2 > 512) return false;
  if (ctx < 0 || wpe_smem_bytes(C, 32, ctx, taps + delay, NK) > kWpeSmemCap) return false;
  return sizeof(double) * (2 * (size_t)NK * (NA + 1) + 16) + 64 <= kWpeSmemCap;
}

size_t wpe_workspace_bytes(int B, int C, int F, int taps) {
  const size_t NK = (size_t)C * taps;
  return sizeof(double) * 2 * (size_t)B * F * (NK * (NK + C) + NK * C);
}

// reverb -> dereverberated STFT, both [B][C][F][T] c64; X is the bin-major copy of reverb
cudaError_t run_wpe(const float2* X, int P, int B, int C, int F, int T, int taps, int delay, int ctx,
                    int num_iters, double* ws, float2* out, unsigned* status, const float2* lam_src,
                    float* linv_out, void* stream) {
  WpeArgs a;
  a.lam_src = lam_src; a.linv_out = linv_out;
  a.X = X; a.P = P; a.B = B; a.C = C; a.F = F; a.T = T;
  a.taps = taps; a.delay = delay; a.ctx = ctx;
  a.NK = C * taps;
  a.Tc = wpe_chunk_frames(C, T, taps, delay, ctx);
  if (const char* env = getenv("SETK_WPE_CHUNK")) {     // test knob: force chunking of short inputs
    const int v = (atoi(env) + 3) & ~3;                   // a multiple of 4 frames
    if (v >= 4 && v < a.Tc) a.Tc = v;
  }
  a.Wp = a.Tc + 2 * ctx + taps + delay;
  a.Raug = ws;
  double* G = ws + 2 * (size_t)B * F * a.NK * (a.NK + C);
  a.G = G;
  a.out = out; a.status = status;
  const size_t smem = wpe_smem_bytes(C, a.Tc, ctx, taps + delay, a.NK);
  const int NA = a.NK + C, RT = (a.NK + 3) / 4, CT = (NA + 3) / 4;
  const int ntiles = RT * CT - RT * (RT - 1) / 2;
  const int corr_threads = ((ntiles + 31) / 32) * 32;
  const int solve_threads = 4 * (((a.NK + 7) / 8) * 8);             // 4 column groups per row, whole warps
  const size_t solve_smem = sizeof(double) * (2 * (size_t)a.NK * (NA + 1) + 16) + sizeof(int) * 16;
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(wpe_corr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (ea == cudaSuccess)
    ea = cudaFuncSetAttribute(wpe_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (ea == cudaSuccess)
    ea = cudaFuncSetAttribute(wpe_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem);
  if (ea != cudaSuccess) return ea;
#endif
  cudaError_t e = cudaSuccess;
  for (int it = 0; it < num_iters && e == cudaSuccess; ++it) {
    a.use_filter = it > 0;
    e = launch(wpe_corr_kernel, dim3(B * F), dim3(corr_threads), smem, stream, false, a);
    if (e == cudaSuccess)
      e = launch(wpe_solve_kernel, dim3(B * F), dim3(solve_threads), solve_smem, stream, false, a, G);
  }
  if (e != cudaSuccess) return e;
  a.use_filter = num_iters > 0;
  return launch(wpe_filter_kernel, dim3(B * F), dim3(256), smem, stream, false, a);
}

}  // namespace setk

// AuxIVA blind source separation (setk_auxiva_stft): its kernels build in this translation unit
#include "auxiva.cuh"
