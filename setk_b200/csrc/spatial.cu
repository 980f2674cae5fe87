// spatial.cu -- spatial features of the reference's libs/spatial.py on explicit
// STFTs (SURVEY.md section 8f rank 3; north_star "subsystems replaced":
// scripts/sptk/libs/spatial.py):
//
//   ipd               spatial.py:163-181   angle(si) - angle(sj), wrapped | cos | [cos, sin]
//   directional_feats spatial.py:184-208   mean over pairs of cos(dphase_obs - dphase_steer)
//   gcc_phat_*        spatial.py:37-92     Re(exp(j dphase) @ exp(-j omega tau)), per-call
//                                          max-normalisation and floor; srp_phat_linear
//                                          (95-123) accumulates pairs through `accumulate`
//   msc               spatial.py:126-160   magnitude squared coherence over a frame context
//
// Element-wise / small-contraction kernels: bytes and flops are tiny next to the
// beamformer path, so they are written for clarity and determinism (fixed-order
// reductions, no float atomics on data), not tuned.  Phase differences are taken
// in float32 like the reference (np.angle of complex64), everything the
// reference promotes to float64 (the GCC transform, MSC) is float64 here too.
#include "common.cuh"
#include "launchers.cuh"
#include <math.h>

namespace setk {

#define SETK_PI_F 3.14159265358979323846f
#define SETK_PI_D 3.14159265358979323846

__device__ __forceinline__ float angle_f(float2 z) { return atan2f(z.y, z.x); }

// numpy.mod for floats (npy_divmod): result has the sign of the divisor
__device__ __forceinline__ float np_modf(float a, float b) {
  float m = fmodf(a, b);
  if (m != 0.f) {
    if ((b < 0.f) != (m < 0.f)) m += b;
  } else {
    m = copysignf(0.f, b);
  }
  return m;
}

// ---- ipd ----
// si, sj [rows][F] c64; mode 0: wrapped difference, 1: cos, 2: out [rows][2F] = [cos | sin]
__global__ void ipd_kernel(const float2* __restrict__ si, const float2* __restrict__ sj, long long n,
                           int F, int mode, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float d = angle_f(si[i]) - angle_f(sj[i]);
  if (mode == 0) {
    // np.mod(d + pi, 2 pi) - pi, float32 arithmetic (np.pi is a weak python scalar)
    out[i] = np_modf(d + SETK_PI_F, 2.0f * SETK_PI_F) - SETK_PI_F;
  } else if (mode == 1) {
    out[i] = cosf(d);
  } else {
    const long long row = i / F;
    const int f = (int)(i - row * F);
    out[row * 2 * F + f] = cosf(d);
    out[row * 2 * F + F + f] = sinf(d);
  }
}

cudaError_t run_ipd(const float2* si, const float2* sj, long long rows, int F, int mode, float* out,
                    void* stream) {
  const long long n = rows * F;
  return launch(ipd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true, si, sj, n, F,
                mode, out);
}

// ---- directional_feats ----
// stft [B][M][F][T] c64, steer [Bs][M][F] c128 (Bs = 1 or B), pairs [P][2] or null (all i < j),
// out [B][T][F] f64
__global__ void dirfeat_kernel(const float2* __restrict__ stft, const double2* __restrict__ steer,
                               int steer_batched, const int* __restrict__ pairs, int P, int B, int M,
                               int F, int T, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * F * T) return;
  const int t = (int)(i % T);
  const int f = (int)((i / T) % F);
  const int b = (int)(i / ((long long)T * F));
  float as[SETK_MAX_CHANNELS];
  double at[SETK_MAX_CHANNELS];
  const double2* sv = steer + (steer_batched ? (long long)b * M * F : 0);
  for (int m = 0; m < M; ++m) {
    as[m] = angle_f(stft[(((long long)b * M + m) * F + f) * T + t]);
    const double2 s = sv[(long long)m * F + f];
    at[m] = atan2(s.y, s.x);
  }
  double acc = 0.0;
  int cnt = 0;
  if (pairs) {
    for (int p = 0; p < P; ++p) {
      const int a = pairs[2 * p], c = pairs[2 * p + 1];
      acc += cos((double)(as[a] - as[c]) - (at[a] - at[c]));
    }
    cnt = P;
  } else {
    for (int a = 0; a < M; ++a)
      for (int c = a + 1; c < M; ++c) {
        acc += cos((double)(as[a] - as[c]) - (at[a] - at[c]));
        ++cnt;
      }
  }
  out[((long long)b * T + t) * F + f] = acc / (double)cnt;
}

cudaError_t run_dirfeat(const float2* stft, const double2* steer, int steer_batched, const int* pairs,
                        int P, int B, int M, int F, int T, double* out, void* stream) {
  const long long n = (long long)B * F * T;
  return launch(dirfeat_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, stream, true, stft,
                steer, steer_batched, pairs, P, B, M, F, T, out);
}

// ---- shared small reductions ----
// max |x| over n doubles -> bits of a non-negative double (ordered like the value);
// a NaN anywhere makes the result NaN like np.max
__global__ void absmax_f64_kernel(const double* __restrict__ x, long long n,
                                  unsigned long long* __restrict__ bits) {
  __shared__ double s_max[256];
  __shared__ int s_nan[256];
  double m = 0.0;
  int has_nan = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const double v = fabs(x[i]);
    if (v != v) has_nan = 1;
    else if (v > m) m = v;
  }
  s_max[threadIdx.x] = m;
  s_nan[threadIdx.x] = has_nan;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
      if (s_max[threadIdx.x + o] > s_max[threadIdx.x]) s_max[threadIdx.x] = s_max[threadIdx.x + o];
      s_nan[threadIdx.x] |= s_nan[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    // NaN sorts above every finite value as an unsigned pattern (0x7ff8...)
    const double r = s_nan[0] ? nan("") : s_max[0];
    atomicMax(bits, (unsigned long long)__double_as_longlong(r));
  }
}

// ---- gcc_phat ----
// table[f][d] = exp(-j omega_f tau_d)
__global__ void gcc_table_kernel(const double* __restrict__ omega, const double* __restrict__ tau, int F,
                                 int D, double2* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * D) return;
  const int f = i / D, d = i - f * D;
  double s, c;
  sincos(omega[f] * tau[d], &s, &c);
  table[i] = make_double2(c, -s);
}

// raw[t][d] = Re( sum_f exp(j (angle si - angle sj))[t][f] * table[f][d] ); one CTA per frame
__global__ void gcc_spectrum_kernel(const float2* __restrict__ si, const float2* __restrict__ sj,
                                    const double2* __restrict__ table, int F, int D,
                                    double* __restrict__ raw) {
  SETK_DYN_SMEM(double2, s_coh);
  const int t = blockIdx.x;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    // np.exp(1j * float32) is evaluated in complex64
    const float d = angle_f(si[(long long)t * F + f]) - angle_f(sj[(long long)t * F + f]);
    s_coh[f] = make_double2((double)cosf(d), (double)sinf(d));
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    double acc = 0.0;
    for (int f = 0; f < F; ++f) {
      const double2 c = s_coh[f];
      const double2 w = table[(long long)f * D + d];
      acc += c.x * w.x - c.y * w.y;
    }
    raw[(long long)t * D + d] = acc;
  }
}

// out (+)= floor(raw / max(max|raw|, eps))
__global__ void gcc_finish_kernel(const double* __restrict__ raw, long long n,
                                  const unsigned long long* __restrict__ maxbits, int normalize,
                                  int apply_floor, int accumulate, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double v = raw[i];
  if (normalize) {
    const double mx = __longlong_as_double((long long)*maxbits);
    v = v / (mx != mx ? mx : fmax(mx, SETK_EPS32_D));
  }
  if (apply_floor) v = (v != v) ? v : fmax(v, 0.0);      // np.maximum propagates NaN
  out[i] = accumulate ? out[i] + v : v;
}

size_t gcc_phat_work_doubles(int T, int F, int D) { return (size_t)2 * F * D + (size_t)T * D + 2; }

cudaError_t run_gcc_phat(const float2* si, const float2* sj, int T, int F, const double* omega,
                         const double* tau, int D, int normalize, int apply_floor, int accumulate,
                         double* work, double* out, void* stream) {
  double2* table = reinterpret_cast<double2*>(work);
  double* raw = work + (size_t)2 * F * D;
  unsigned long long* maxbits = reinterpret_cast<unsigned long long*>(raw + (size_t)T * D);
  cudaError_t e = cudaMemsetAsync(maxbits, 0, sizeof(unsigned long long), static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return e;
  e = launch(gcc_table_kernel, dim3((unsigned)((F * D + 255) / 256)), dim3(256), 0, stream, true, omega,
             tau, F, D, table);
  if (e != cudaSuccess) return e;
  e = launch(gcc_spectrum_kernel, dim3(T), dim3(128), sizeof(double2) * (size_t)F, stream, false, si, sj,
             (const double2*)table, F, D, raw);
  if (e != cudaSuccess) return e;
  const long long n = (long long)T * D;
  if (normalize) {
    e = launch(absmax_f64_kernel, dim3(64), dim3(256), 0, stream, false, (const double*)raw, n, maxbits);
    if (e != cudaSuccess) return e;
  }
  return launch(gcc_finish_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
                (const double*)raw, n, (const unsigned long long*)maxbits, normalize, apply_floor,
                accumulate, out);
}

// ---- msc ----
// spec [N][T][F] c64.  Per (t, f): numerator[a][c] = mean over the frame context of
// Y_a conj(Y_c) (frames clamped to [0, T-1]); icc = |numerator / sqrt(dig_a dig_c)|.
// s[t][f] = sum_{a,c} icc; the reference then adds the GRAND TOTAL of the diagonal
// terms (np.sum without an axis, spatial.py:153) to every cell: block partials of
// that total go to diag_part[block] and are added in fixed order by msc_finish.
#define SETK_MSC_MAXCTX 8
__global__ void msc_kernel(const float2* __restrict__ spec, int N, int T, int F, int context,
                           double* __restrict__ s_out, double* __restrict__ diag_part) {
  __shared__ double s_red[128];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double diag_local = 0.0;
  if (i < (long long)T * F) {
    const int t = (int)(i / F), f = (int)(i - (long long)t * F);
    const int K = 2 * context + 1;
    double dig[SETK_MAX_CHANNELS];
    for (int a = 0; a < N; ++a) {
      double acc = 0.0;
      for (int k = -context; k <= context; ++k) {
        const int s = imin(imax(t + k, 0), T - 1);
        const float2 y = spec[((long long)a * T + s) * F + f];
        acc += (double)y.x * (double)y.x + (double)y.y * (double)y.y;
      }
      dig[a] = fabs(acc / (double)K);
    }
    double sum = 0.0;
    for (int a = 0; a < N; ++a) {
      for (int c = 0; c < N; ++c) {
        double re = 0.0, im = 0.0;
        for (int k = -context; k <= context; ++k) {
          const int s = imin(imax(t + k, 0), T - 1);
          const float2 ya = spec[((long long)a * T + s) * F + f];
          const float2 yc = spec[((long long)c * T + s) * F + f];
          re += (double)ya.x * (double)yc.x + (double)ya.y * (double)yc.y;
          im += (double)ya.y * (double)yc.x - (double)ya.x * (double)yc.y;
        }
        re /= (double)K; im /= (double)K;
        const double den = sqrt(dig[a] * dig[c]);
        const double qr = re / den, qi = im / den;          // complex / real
        const double icc = hypot(qr, qi);
        sum += icc;
        if (a == c) diag_local += icc;
      }
    }
    s_out[i] = sum;
  }
  s_red[threadIdx.x] = diag_local;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) diag_part[blockIdx.x] = s_red[0];
}

// total = sum of the block partials (fixed order); coh = (total + s) / (N (N - 1))
__global__ void msc_total_kernel(const double* __restrict__ diag_part, int n_blocks,
                                 double* __restrict__ total) {
  __shared__ double s_red[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_blocks; i += blockDim.x) acc += diag_part[i];
  s_red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_red[0];
}
__global__ void msc_combine_kernel(const double* __restrict__ s, long long n,
                                   const double* __restrict__ total, int N, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (*total + s[i]) / (double)(N * (N - 1));
}
__global__ void scale_by_absmax_kernel(double* __restrict__ x, long long n,
                                       const unsigned long long* __restrict__ maxbits) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = x[i] / __longlong_as_double((long long)*maxbits);
}

static int msc_blocks(int T, int F) { return (int)(((long long)T * F + 127) / 128); }
size_t msc_work_doubles(int T, int F) { return (size_t)T * F + (size_t)msc_blocks(T, F) + 2; }

cudaError_t run_msc(const float2* spec, int N, int T, int F, int context, int normalize, double* work,
                    double* out, void* stream) {
  const long long n = (long long)T * F;
  const int nb = msc_blocks(T, F);
  double* s = work;
  double* part = work + n;
  double* total = part + nb;
  unsigned long long* maxbits = reinterpret_cast<unsigned long long*>(total + 1);
  cudaError_t e = cudaMemsetAsync(maxbits, 0, sizeof(unsigned long long), static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return e;
  e = launch(msc_kernel, dim3(nb), dim3(128), 0, stream, false, spec, N, T, F, context, s, part);
  if (e != cudaSuccess) return e;
  e = launch(msc_total_kernel, dim3(1), dim3(256), 0, stream, false, (const double*)part, nb, total);
  if (e != cudaSuccess) return e;
  e = launch(msc_combine_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true,
             (const double*)s, n, (const double*)total, N, out);
  if (e != cudaSuccess || !normalize) return e;
  e = launch(absmax_f64_kernel, dim3(64), dim3(256), 0, stream, false, (const double*)out, n, maxbits);
  if (e != cudaSuccess) return e;
  return launch(scale_by_absmax_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, true, out,
                n, (const unsigned long long*)maxbits);
}

}  // namespace setk

// sound source localisation (setk_ssl): its kernels build in this translation unit
#include "ssl.cuh"
