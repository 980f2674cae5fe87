// weights_coop.cu -- per-bin beamformer weights for C > 4 by a GROUP of threads
// per (utterance, bin), matrices in shared memory.
//
// weights.cu gives every bin to one thread; above C = 4 its matrices live in
// local memory and a batch offers only B*F threads (config 5, C = 16: 8 224
// threads, 10.9 ms per 32 utterances).  Here Coop<C>::GS (8 / 16) threads share
// a bin: the warp-cooperative Jacobi of jacobi_coop.cuh, and row- / column-
// parallel LU (partial pivoting), Cholesky and triangular solves with the same
// operation order per element as hermitian_solve.cuh.
//
// Kinds: MVDR (beamformer.py:527-539), MPDR (555-573), GEVD / PEVD (31-63, 674-682), with BAN
// (14-28).  MPDR-whiten, PMWF and the rank-1 options stay on weights.cu.
#include "jacobi_coop.cuh"
#include "launchers.cuh"
#include "lu_coop.cuh"
#include "weights_args.cuh"

namespace setk {

// The CPU execution model (tests/emu) launches the same CTAs: several warps' groups share one CTA's
// shared memory there too, and its warps run unsynchronised like the device's.  Inside one warp the
// groups run in lock step, so a group that wrote past its slot would only reach a neighbour's A once
// that A is dead; across warps it can land while the neighbour still uses it.  Whether it does
// depends on how the warps interleave, on the device and on the emulator's threads alike, which is
// why tests/solve_cases.py's batch-invariance check alternates fast and slow warps.
template <int C> struct WCfg { static constexpr int THREADS = C <= 8 ? 128 : 64; };

__device__ __forceinline__ cd load_c(const void* base, int dtype, long long i) {
  if (dtype == SETK_C128) {
    const double* p = reinterpret_cast<const double*>(base) + 2 * i;
    return cd_make(p[0], p[1]);
  }
  const float* p = reinterpret_cast<const float*>(base) + 2 * i;
  return cd_make((double)p[0], (double)p[1]);
}

// Hermitian matrix from the LOWER triangle of global R (LAPACK UPLO='L'), into A.
template <int C>
__device__ __forceinline__ void load_lower_hermitian(const void* R, int dtype, long long idx, cd* A, int r) {
  constexpr int LD = Coop<C>::LD;
  for (int j = 0; j <= r; ++j) {
    cd v = load_c(R, dtype, idx * (C * C) + r * C + j);
    if (j == r) v.y = 0.0;
    A[r * LD + j] = v;
    if (j != r) A[j * LD + r] = cd_conj(v);
  }
}

// principal eigenvector of the (diagonalised) A with eigenvectors V, library convention:
// unit norm, component 0 real >= 0.  Returns this thread's component.
template <int C>
__device__ __forceinline__ cd principal_component(const cd* A, const cd* V, int r, bool row) {
  constexpr int LD = Coop<C>::LD, GS = Coop<C>::GS;
  int best = 0;
  double lam = A[0].x;
  for (int i = 1; i < C; ++i)
    if (A[i * LD + i].x > lam) { lam = A[i * LD + i].x; best = i; }
  cd v = row ? V[r * LD + best] : cd_make(0.0, 0.0);
  const double n2 = group_sum<GS>(cd_abs2(v));
  const double inv = n2 > 0.0 ? 1.0 / sqrt(n2) : 0.0;
  const cd v0 = V[best];                                  // component 0 (row 0)
  const double m0 = sqrt(cd_abs2(v0));
  const cd ph = m0 > 0.0 ? cd_make(v0.x / m0, -v0.y / m0) : cd_make(1.0, 0.0);
  v = cd_scale(cd_mul(v, ph), inv);
  if (r == 0 && m0 > 0.0) v.y = 0.0;
  return v;
}

// Lower Cholesky factor in place (rows owned by threads, same operation order as
// cholesky_lower()).  Returns false (uniformly) if not positive definite.
template <int C>
__device__ __forceinline__ bool cholesky_coop(cd* L, int r, bool row, int lane_base) {
  constexpr int LD = Coop<C>::LD;
  bool ok = true;
  for (int j = 0; j < C; ++j) {
    double d = 0.0;
    if (row && r == j) {
      d = L[j * LD + j].x;
      for (int k = 0; k < j; ++k) d -= cd_abs2(L[j * LD + k]);
    }
    d = __shfl_sync(0xffffffffu, d, lane_base + j);
    if (!(d > 0.0)) { ok = false; d = 1.0; }
    const double l = sqrt(d);
    if (row && r == j) L[j * LD + j] = cd_make(l, 0.0);
    if (row && r > j) {
      cd s = L[r * LD + j];
      for (int k = 0; k < j; ++k) s = cd_sub(s, cd_mulc(L[r * LD + k], L[j * LD + k]));
      L[r * LD + j] = cd_scale(s, 1.0 / l);
    }
    if (row && r < j) L[r * LD + j] = cd_make(0.0, 0.0);
    __syncwarp();
  }
  return ok;
}

// B <- L^-1 B, thread c owns column c of B
template <int C>
__device__ __forceinline__ void forward_subst_coop(const cd* L, cd* B, int c, bool col) {
  constexpr int LD = Coop<C>::LD;
  if (col) {
    for (int i = 0; i < C; ++i) {
      cd s = B[i * LD + c];
      for (int k = 0; k < i; ++k) s = cd_sub(s, cd_mul(L[i * LD + k], B[k * LD + c]));
      B[i * LD + c] = cd_scale(s, 1.0 / L[i * LD + i].x);
    }
  }
  __syncwarp();
}

SETK_HD inline bool coop_two_matrices(const WeightsArgs& a) {
  return a.kind == SETK_BF_MVDR || a.kind == SETK_BF_MPDR || (a.kind == SETK_BF_PEVD && a.Rn == nullptr);
}
// Pitch between the groups' matrices, in cd (16 bytes = one bank group of a 128-byte wavefront).
// C = 4: a quarter-warp is two groups x four rows and rows sit 5 cd apart ({0, 5, 2, 7} mod 8), so
// the second group must start 4 (mod 8) later ({4, 1, 6, 3}): conflict-free rows AND columns.
// Otherwise an odd pitch (a group of 8 or 16 lanes fills its quarter-warps by itself).
template <int C>
SETK_HD inline int coop_group_pitch(bool two) {
  const int base = (two ? 2 : 3) * Coop<C>::MAT + C;
  if (Coop<C>::GS == 4) return base + ((4 - base % 8) + 8) % 8;
  return base | 1;
}

template <int C>
__global__ void __launch_bounds__(WCfg<C>::THREADS) weights_coop_kernel(WeightsArgs a) {
  using K = Coop<C>;
  constexpr int GS = K::GS, LD = K::LD, MAT = K::MAT, MPB = WCfg<C>::THREADS / GS;
  // cd per group: A, V, M, w.  The eigenvector kinds (MVDR, MPDR, PEVD of Rs) are done with A when
  // they fill M, so M lives on A: a third less shared memory = a third more problems resident.
  // The pitch staggers the groups of a warp over the 16-byte bank groups (coop_group_pitch).
  const bool two = coop_two_matrices(a);
  const int PER = coop_group_pitch<C>(two);
  SETK_DYN_SMEM(double, sm);
  const int tid = threadIdx.x;
  const int grp = tid / GS, r = tid - grp * GS;
  const int lane_base = (tid & 31) - r;            // first lane of this group in its warp
  cd* A = reinterpret_cast<cd*>(sm) + (size_t)grp * PER;
  cd* V = A + MAT;
  cd* M = two ? A : V + MAT;
  cd* wv = (two ? V : M) + MAT;
  double* rot = sm + (size_t)MPB * PER * 2 + grp * K::ROT;
  const long long idx = (long long)blockIdx.x * MPB + grp;
  const bool active = idx < (long long)a.B * a.F;
  const bool row = active && r < C;
  const int b = active ? (int)(idx / a.F) : 0;
  unsigned st = 0;
  const bool have_rn = a.Rn != nullptr;
  cd w = cd_make(0.0, 0.0);

  if (a.kind == SETK_BF_MVDR || a.kind == SETK_BF_MPDR || (a.kind == SETK_BF_PEVD && !have_rn)) {
    if (row) load_lower_hermitian<C>(a.Rs, a.r_dtype, idx, A, r);
    __syncwarp();
    if (!jacobi_coop<C>(A, V, rot, r, active)) st |= SETK_ST_NO_CONVERGE;
    const cd d = principal_component<C>(A, V, r, row);
    if (a.kind == SETK_BF_PEVD) {
      w = d;
    } else {
      // denominator matrix: Rn for MVDR, Ry (all-ones mask) for MPDR (beamformer.py:555-573)
      const void* D = a.kind == SETK_BF_MPDR ? a.Ry : a.Rn;
      __syncwarp();                                    // every lane has read A and V: M may overwrite A
      if (row) {
        for (int j = 0; j < C; ++j) M[r * LD + j] = load_c(D, a.r_dtype, idx * (C * C) + r * C + j);
        M[r * LD + C] = d;
      }
      __syncwarp();
      bool singular = false;
      const cd n = lu_solve_coop<C>(M, r, row, &singular);
      if (singular) st |= SETK_ST_SINGULAR;
      const cd t = row ? cd_mulc(n, d) : cd_make(0.0, 0.0);      // conj(d) n  (cd_mulc(a, b) = a conj(b))
      const cd den = cd_make(group_sum<GS>(t.x), group_sum<GS>(t.y));
      w = cd_div(n, den);
    }
  } else {  // SETK_BF_GEVD, or PEVD with Rn: principal generalised eigenvector
    double tr = 0.0;
    if (row) tr = load_c(a.Rn, a.r_dtype, idx * (C * C) + r * C + r).x;
    tr = group_sum<GS>(tr);
    // diagonal loading retries as in gev_principal(); the groups of a warp take the
    // same number of trips (the factorisation synchronises the whole warp)
    bool ok = !active;
    double load = 0.0;
    for (int attempt = 0; attempt < 6; ++attempt) {
      const bool need = active && !ok && (attempt == 0 || tr > 0.0);
      int any = need ? 1 : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) any |= __shfl_xor_sync(0xffffffffu, any, o);
      if (!any) break;
      if (row && need) {
        for (int j = 0; j <= r; ++j) M[r * LD + j] = load_c(a.Rn, a.r_dtype, idx * (C * C) + r * C + j);
        M[r * LD + r].x += load * tr / C;
      }
      __syncwarp();
      const bool fact = cholesky_coop<C>(M, r, row && need, lane_base);
      if (need) {
        ok = fact;
        if (attempt > 0) st |= SETK_ST_REGULARIZED;
      }
      load = attempt == 0 ? 1e-10 : load * 100.0;
    }
    if (active && !ok) st |= SETK_ST_NOT_PD;
    if (row) load_lower_hermitian<C>(a.Rs, a.r_dtype, idx, A, r);
    __syncwarp();
    forward_subst_coop<C>(M, A, r, row);              // X = L^-1 Rs
    if (row) for (int j = 0; j < C; ++j) V[r * LD + j] = cd_conj(A[j * LD + r]);   // X^H
    __syncwarp();
    forward_subst_coop<C>(M, V, r, row);              // Y = L^-1 X^H
    if (row) {
      for (int j = 0; j <= r; ++j) {                  // M' = (Y^H + Y) / 2, Hermitian
        const cd m = cd_scale(cd_add(cd_conj(V[j * LD + r]), V[r * LD + j]), 0.5);
        A[r * LD + j] = j == r ? cd_make(m.x, 0.0) : m;
        if (j != r) A[j * LD + r] = cd_conj(m);
      }
    }
    __syncwarp();
    if (!jacobi_coop<C>(A, V, rot, r, active)) st |= SETK_ST_NO_CONVERGE;
    const cd y = principal_component<C>(A, V, r, row);
    if (row) M[r * LD + C] = y;
    __syncwarp();
    for (int i = C - 1; i >= 0; --i) {                // L^H w = y, column-oriented
      if (row && r == i) { w = cd_scale(M[i * LD + C], 1.0 / M[i * LD + i].x); M[i * LD + C] = w; }
      __syncwarp();
      if (row && r < i) M[r * LD + C] = cd_sub(M[r * LD + C], cd_mul(cd_conj(M[i * LD + r]), M[i * LD + C]));
      __syncwarp();
    }
  }

  if (a.ban && have_rn) {                             // do_ban, beamformer.py:14-28
    if (row) wv[r] = w;
    __syncwarp();
    cd u = cd_make(0.0, 0.0);
    if (row) for (int j = 0; j < C; ++j) u = cd_add(u, cd_mul(load_c(a.Rn, a.r_dtype, idx * (C * C) + r * C + j), wv[j]));
    __syncwarp();
    if (row) wv[r] = u;
    __syncwarp();
    cd v = cd_make(0.0, 0.0);
    if (row) for (int j = 0; j < C; ++j) v = cd_add(v, cd_mul(load_c(a.Rn, a.r_dtype, idx * (C * C) + r * C + j), wv[j]));
    const cd tn = row ? cd_mul(cd_conj(w), v) : cd_make(0.0, 0.0);
    const cd td = row ? cd_mul(cd_conj(w), u) : cd_make(0.0, 0.0);
    const double nx = group_sum<GS>(tn.x), ny = group_sum<GS>(tn.y), dx = group_sum<GS>(td.x);
    const double g = sqrt(sqrt(nx * nx + ny * ny)) / fmax(dx, SETK_EPS32_D);
    w = cd_scale(w, g);
  }
  int bad = (row && !(isfinite(w.x) && isfinite(w.y))) ? 1 : 0;
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) bad |= __shfl_xor_sync(0xffffffffu, bad, o);
  if (bad) st |= SETK_ST_NONFINITE;
  if (row) {
    if (a.w_dtype == SETK_C128) {
      double* p = reinterpret_cast<double*>(a.w) + (idx * C + r) * 2;
      p[0] = w.x; p[1] = w.y;
    } else {
      float* p = reinterpret_cast<float*>(a.w) + (idx * C + r) * 2;
      p[0] = (float)w.x; p[1] = (float)w.y;
    }
    if (r == 0 && st) atomicOr(a.status + b, st);
  }
}

bool weights_coop_supported(const WeightsArgs& a, int C) {
  if (C <= 4) {
    // C = 4: four threads per bin for the eigenvector kinds (the one-thread solve is a single long fp64
    // dependency chain per bin that fills few warp slots); the Cholesky kinds and C < 4 keep the
    // register-resident one-thread solve.
    if (C != 4 || !coop_two_matrices(a)) return false;
  }
  if (a.rank1 != SETK_RANK1_NONE) return false;
  return a.kind == SETK_BF_MVDR || a.kind == SETK_BF_MPDR || a.kind == SETK_BF_GEVD ||
         a.kind == SETK_BF_PEVD;
}

template <int C>
static cudaError_t weights_coop_t(const WeightsArgs& a, void* stream) {
  using K = Coop<C>;
  constexpr int MPB = WCfg<C>::THREADS / K::GS;
  const size_t smem = sizeof(double) * ((size_t)MPB * coop_group_pitch<C>(coop_two_matrices(a)) * 2 +
                                        (size_t)MPB * K::ROT);
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(weights_coop_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem);
  if (ea != cudaSuccess) return ea;
#endif
  const long long n = (long long)a.B * a.F;
  return launch(weights_coop_kernel<C>, dim3((unsigned)((n + MPB - 1) / MPB)), dim3(WCfg<C>::THREADS), smem,
                stream, false, a);
}

cudaError_t weights_coop_launch(const WeightsArgs& a, int C, void* stream) {
  switch (C) {
#define SETK_CASE(k) case k: return weights_coop_t<k>(a, stream);
    SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8) SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12)
    SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
