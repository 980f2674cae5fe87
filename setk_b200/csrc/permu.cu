// permu.cu -- frequency permutation alignment of K-class TF masks, the device form of
//   scripts/sptk/libs/cluster.py:48-91   permu_aligner
// One CTA per utterance.  The features are the masks normalised over the utterance's own frames;
// for every (iters, lo, hi) row of the sub-band plan, up to `iters` times:
//   the K x T centroid = mean over bins [lo, hi) of the features, normalised   (warp per (k, t))
//   every bin of the band scores its K classes against it, K x K, and takes the best of the K!
//   permutations                                                                (thread per bin)
// until no bin moved.  Within one iteration the bins depend only on the centroid, so they run in
// parallel; the iterations run in series.  The class order of each bin is an index table ord[k][f]
// (source class of slot k), and the features are read through it: no data move until the output,
// which gathers the float32 masks through the table.  fp64 throughout, as the reference aligns
// float64 masks.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

struct PermuRows { int n; int r[SETK_PERMU_MAX_ROWS][3]; };   // by value: no copy of the host plan

// the K! permutations of 0..K-1 in itertools.permutations order
__constant__ unsigned char c_perm2[2][2] = {{0, 1}, {1, 0}};
__constant__ unsigned char c_perm3[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
__constant__ unsigned char c_perm4[24][4] = {
    {0, 1, 2, 3}, {0, 1, 3, 2}, {0, 2, 1, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}, {0, 3, 2, 1},
    {1, 0, 2, 3}, {1, 0, 3, 2}, {1, 2, 0, 3}, {1, 2, 3, 0}, {1, 3, 0, 2}, {1, 3, 2, 0},
    {2, 0, 1, 3}, {2, 0, 3, 1}, {2, 1, 0, 3}, {2, 1, 3, 0}, {2, 3, 0, 1}, {2, 3, 1, 0},
    {3, 0, 1, 2}, {3, 0, 2, 1}, {3, 1, 0, 2}, {3, 1, 2, 0}, {3, 2, 0, 1}, {3, 2, 1, 0}};

template <int K>
__device__ __forceinline__ int perm_at(int p, int k) {
  if constexpr (K == 2) return c_perm2[p][k];
  else if constexpr (K == 3) return c_perm3[p][k];
  else return c_perm4[p][k];
}

constexpr int PERMU_THREADS = 256;
constexpr size_t PERMU_SMEM_MAX = 200 * 1024;

// shared memory of the per-bin tables: s1, s12 [K][F] f64, cn [4] f64, ord [K][F] i32, flag
static size_t permu_table_bytes(int K, int F) {
  return sizeof(double) * (2 * (size_t)K * F + 4) + sizeof(int) * ((size_t)K * F + 1);
}
static bool permu_cen_shared(int K, int T, int F) {
  return permu_table_bytes(K, F) + sizeof(double) * (size_t)K * T <= PERMU_SMEM_MAX;
}

template <int K>
__global__ void __launch_bounds__(PERMU_THREADS) permu_align_kernel(PermuArgs a, PermuRows rows, double* cen_g,
                                                                    float* out, int* mapping) {
  SETK_DYN_SMEM(double, sm);
  const int F = a.F, T = a.T, ld = a.ld;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  double* s1 = sm;                  // [K][F] 1 / max(|m_k(f)|, eps): feature = m s1 (cluster.py:61)
  double* s12 = s1 + K * F;         // [K][F] the feature normalised again, as the score does (cluster.py:77)
  double* cn = s12 + K * F;         // [K] max(|centroid_k|, eps)
  double* cen = cen_g ? cen_g + (size_t)b * K * T : cn + 4;       // [K][T]
  int* ord = reinterpret_cast<int*>(cen_g ? cn + 4 : cen + (size_t)K * T);   // [K][F]
  int* moved = ord + K * F;
  int Tb;
  if (a.n_frames) {
    Tb = a.n_frames[b];
  } else {
    Tb = frames_of(a.n_samples ? a.n_samples[b] : a.N, a.g.n_fft, a.g.hop, a.g.pad);
  }
  Tb = Tb < 0 ? 0 : (Tb > T ? T : Tb);
  const double* m = a.m + (size_t)b * K * T * ld;
  for (int q = tid; q < K * F; q += blockDim.x) {
    const int k = q / F, f = q - k * F;
    const double* x = m + (size_t)k * T * ld + f;
    double ss = 0.0;
    for (int t = 0; t < Tb; ++t) ss += x[(size_t)t * ld] * x[(size_t)t * ld];
    const double d1 = fmax(sqrt(ss), SETK_EPS32_D);
    double ss2 = 0.0;
    for (int t = 0; t < Tb; ++t) { const double v = x[(size_t)t * ld] / d1; ss2 += v * v; }
    s1[q] = 1.0 / d1;
    s12[q] = 1.0 / (d1 * fmax(sqrt(ss2), SETK_EPS32_D));
    ord[q] = k;
  }
  if (tid == 0) *moved = 0;
  __syncthreads();
  for (int r = 0; r < rows.n; ++r) {
    const int iters = rows.r[r][0], lo = rows.r[r][1], hi = rows.r[r][2];
    for (int it = 0; it < iters; ++it) {
      // centroid, K x T: mean over the band of the features, slot k of bin f read as class ord[k][f]
      for (int row = warp; row < K * Tb; row += nwarp) {
        const int k = row / Tb, t = row - k * Tb;
        double s = 0.0;
        for (int f = lo + lane; f < hi; f += 32) {
          const int j = ord[k * F + f];
          s += m[((size_t)j * T + t) * ld + f] * s1[j * F + f];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) cen[(size_t)k * T + t] = s / (double)(hi - lo);
      }
      __syncthreads();
      if (warp < K) {
        double ss = 0.0;
        for (int t = lane; t < Tb; t += 32) ss += cen[(size_t)warp * T + t] * cen[(size_t)warp * T + t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if (lane == 0) cn[warp] = fmax(sqrt(ss), SETK_EPS32_D);
      }
      if (tid == 0) *moved = 0;     // every thread read the last iteration's flag before the barrier above
      __syncthreads();
      for (int f = lo + tid; f < hi; f += blockDim.x) {
        int src[K];
        double sc[K], acc[K][K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
          src[j] = ord[j * F + f];
          sc[j] = s12[src[j] * F + f];
#pragma unroll
          for (int i = 0; i < K; ++i) acc[i][j] = 0.0;
        }
        for (int t = 0; t < Tb; ++t) {
          double x[K];
#pragma unroll
          for (int j = 0; j < K; ++j) x[j] = m[((size_t)src[j] * T + t) * ld + f] * sc[j];
#pragma unroll
          for (int i = 0; i < K; ++i) {
            const double c = cen[(size_t)i * T + t];
#pragma unroll
            for (int j = 0; j < K; ++j) acc[i][j] += c * x[j];
          }
        }
#pragma unroll
        for (int i = 0; i < K; ++i)
#pragma unroll
          for (int j = 0; j < K; ++j) acc[i][j] /= cn[i];
        // best of the K! permutations; a later one replaces the best only by more than 1e-15
        // (_best_permutation of setk_b200.libs.cluster), so exact ties stay on the identity
        constexpr int NP = K == 2 ? 2 : (K == 3 ? 6 : 24);
        int best = 0;
        double best_val = -INFINITY;
        for (int p = 0; p < NP; ++p) {
          double v = 0.0;
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const int pk = perm_at<K>(p, k);
            double e = acc[k][0];
#pragma unroll
            for (int j = 1; j < K; ++j) e = pk == j ? acc[k][j] : e;
            v += e;
          }
          if (v > best_val + 1e-15) { best = p; best_val = v; }
        }
        if (best != 0) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const int pk = perm_at<K>(best, k);
            int s = src[0];
#pragma unroll
            for (int j = 1; j < K; ++j) s = pk == j ? src[j] : s;
            ord[k * F + f] = s;
          }
          *moved = 1;
        }
      }
      __syncthreads();
      if (!*moved) break;
    }
  }
  float* o = out + (size_t)b * K * T * F;
  for (size_t q = tid; q < (size_t)K * T * F; q += blockDim.x) {
    const int f = (int)(q % F);
    const size_t kt = q / F;
    const int k = (int)(kt / T), t = (int)(kt - (size_t)k * T);
    o[q] = t < Tb ? (float)m[((size_t)ord[k * F + f] * T + t) * ld + f] : 0.f;
  }
  if (mapping)
    for (int q = tid; q < K * F; q += blockDim.x) mapping[(size_t)b * K * F + q] = ord[q];
}

long long permu_scratch_bytes(int B, int K, int T, int F) {
  if (permu_table_bytes(K, F) > PERMU_SMEM_MAX) return -1;
  return permu_cen_shared(K, T, F) ? 0 : (long long)sizeof(double) * B * K * T;
}

template <int K>
static cudaError_t permu_t(const PermuArgs& a, int B, const PermuRows& rows, double* scratch, float* out,
                           int* mapping, void* stream) {
  const bool shared = permu_cen_shared(K, a.T, a.F);
  const size_t smem = permu_table_bytes(K, a.F) + (shared ? sizeof(double) * (size_t)K * a.T : 0);
#ifndef SETK_EMU
  cudaError_t e = cudaFuncSetAttribute(permu_align_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
#endif
  return launch(permu_align_kernel<K>, dim3(B), dim3(PERMU_THREADS), smem, stream, false, a, rows,
                shared ? nullptr : scratch, out, mapping);
}

cudaError_t run_permu_align(const PermuArgs& a, int B, const int* rows_host, int R, double* scratch,
                            float* out, int* mapping, void* stream) {
  if (R < 0 || R > SETK_PERMU_MAX_ROWS || permu_scratch_bytes(B, a.K, a.T, a.F) < 0) return cudaErrorInvalidValue;
  PermuRows rows;
  rows.n = R;
  for (int r = 0; r < R; ++r)
    for (int c = 0; c < 3; ++c) rows.r[r][c] = rows_host[3 * r + c];
  switch (a.K) {
    case 2: return permu_t<2>(a, B, rows, scratch, out, mapping, stream);
    case 3: return permu_t<3>(a, B, rows, scratch, out, mapping, stream);
    case 4: return permu_t<4>(a, B, rows, scratch, out, mapping, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
