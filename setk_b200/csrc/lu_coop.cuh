// lu_coop.cuh -- linear solve of a small complex system by a group of threads of one
// warp, the matrix in shared memory (rows owned by threads).  Same pivoting rule
// (|re| + |im|, first index on ties, like LAPACK's izamax) and per-element
// operation order as lu_factor / lu_solve_vec of hermitian_solve.cuh.
// Used by the beamformer weights for C > 4 (weights_coop.cu) and by AuxIVA for
// N > 4 (auxiva.cuh).
#pragma once
#include "jacobi_coop.cuh"

namespace setk {

// sum over the GS lanes of an aligned group (every lane gets the sum)
template <int GS>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
  for (int o = GS / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// In-place LU with partial pivoting of the augmented [M | b] (b in column C of the
// padded rows), rows owned by threads; forward elimination of b rides along.
// Then back substitution; returns x_r.  *singular set on an exactly zero pivot.
template <int C>
__device__ __forceinline__ cd lu_solve_coop(cd* M, int r, bool row, bool* singular) {
  constexpr int LD = Coop<C>::LD, GS = Coop<C>::GS;
  const unsigned full = 0xffffffffu;
  for (int k = 0; k < C; ++k) {
    double m = (row && r >= k) ? fabs(M[r * LD + k].x) + fabs(M[r * LD + k].y) : -1.0;
    int piv = r;
#pragma unroll
    for (int o = GS / 2; o > 0; o >>= 1) {          // arg max, first index on ties (like izamax)
      const double m2 = __shfl_xor_sync(full, m, o);
      const int p2 = __shfl_xor_sync(full, piv, o);
      if (m2 > m || (m2 == m && p2 < piv)) { m = m2; piv = p2; }
    }
    if (piv != k && row) {                          // swap rows k, piv: thread j owns column j
      cd t = M[k * LD + r]; M[k * LD + r] = M[piv * LD + r]; M[piv * LD + r] = t;
      if (r == 0) { t = M[k * LD + C]; M[k * LD + C] = M[piv * LD + C]; M[piv * LD + C] = t; }
    }
    __syncwarp();
    if (m == 0.0) *singular = true;                 // (no early exit: the barriers below are warp-wide)
    if (row && r > k && m != 0.0) {
      const cd inv = cd_div(cd_make(1.0, 0.0), M[k * LD + k]);
      const cd l = cd_mul(M[r * LD + k], inv);
      M[r * LD + k] = l;
      for (int j = k + 1; j <= C; ++j) M[r * LD + j] = cd_sub(M[r * LD + j], cd_mul(l, M[k * LD + j]));
    }
    __syncwarp();
  }
  cd x = cd_make(0.0, 0.0);
  for (int i = C - 1; i >= 0; --i) {                // column-oriented back substitution
    if (row && r == i) { x = cd_div(M[i * LD + C], M[i * LD + i]); M[i * LD + C] = x; }
    __syncwarp();
    if (row && r < i) M[r * LD + C] = cd_sub(M[r * LD + C], cd_mul(M[r * LD + i], M[i * LD + C]));
    __syncwarp();
  }
  return x;
}

}  // namespace setk
