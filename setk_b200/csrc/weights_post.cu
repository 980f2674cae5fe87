// weights_post.cu -- the two stand-alone per-bin helpers of the reference's
// beamformer library, as kernels of their own so that the Python mirror of
// libs/beamformer.py never has to leave the GPU:
//   setk_ban    do_ban(weight, Rn)             beamformer.py:14-28
//   setk_rank1  rank1_constraint(Rs, Rn=None)  beamformer.py:66-84
// (inside the weight solve both are applied in registers by weights.cu).
#include "common.cuh"
#include "hermitian_solve.cuh"
#include "launchers.cuh"

namespace setk {

struct PostArgs {
  int mode;                 // 0: BAN, 1: rank-1 approximation
  const void* A;            // BAN: weight [B][F][C]; rank1: Rs [B][F][C][C]
  const void* Rn;           // [B][F][C][C] (may be null for rank1)
  int dtype;
  int B, F;
  void* out;                // BAN: weight; rank1: R1 [B][F][C][C]
  unsigned* status;
};

template <int C>
__device__ inline void load_matp(const void* base, int dtype, long long idx, CMat<C>& M) {
  SETK_UNROLL_C
  for (int i = 0; i < C; ++i) {
    SETK_UNROLL_C
    for (int j = 0; j < C; ++j) {
      const long long e = idx * (long long)(C * C) + i * C + j;
      if (dtype == SETK_C128) {
        const double* p = reinterpret_cast<const double*>(base) + 2 * e;
        M.a[i][j] = cd_make(p[0], p[1]);
      } else {
        const float* p = reinterpret_cast<const float*>(base) + 2 * e;
        M.a[i][j] = cd_make((double)p[0], (double)p[1]);
      }
    }
  }
}

__device__ inline void store_c(void* base, int dtype, long long e, cd v) {
  if (dtype == SETK_C128) {
    double* p = reinterpret_cast<double*>(base) + 2 * e;
    p[0] = v.x; p[1] = v.y;
  } else {
    float* p = reinterpret_cast<float*>(base) + 2 * e;
    p[0] = (float)v.x; p[1] = (float)v.y;
  }
}

template <int C>
__global__ void __launch_bounds__(128) post_kernel(PostArgs a) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.B * a.F) return;
  const int b = (int)(idx / a.F);
  if (a.mode == 0) {
    CMat<C> Rn;
    load_matp<C>(a.Rn, a.dtype, idx, Rn);
    CVec<C> w, u, v;
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) {
      const long long e = idx * C + i;
      if (a.dtype == SETK_C128) {
        const double* p = reinterpret_cast<const double*>(a.A) + 2 * e;
        w.v[i] = cd_make(p[0], p[1]);
      } else {
        const float* p = reinterpret_cast<const float*>(a.A) + 2 * e;
        w.v[i] = cd_make((double)p[0], (double)p[1]);
      }
    }
    matvec<C>(Rn, w, u);
    matvec<C>(Rn, u, v);
    const cd num = dotc<C>(w, v), den = dotc<C>(w, u);
    const double g = sqrt(sqrt(num.x * num.x + num.y * num.y)) / fmax(den.x, SETK_EPS32_D);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) store_c(a.out, a.dtype, idx * C + i, cd_scale(w.v[i], g));
  } else {
    unsigned st = 0;
    CMat<C> Rs;
    load_matp<C>(a.A, a.dtype, idx, Rs);
    double tr = 0.0;
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) tr += Rs.a[i][i].x;
    CVec<C> p;
    if (a.Rn == nullptr) {
      if (!principal_eigvec<C>(Rs, p)) st |= SETK_ST_NO_CONVERGE;
    } else {
      CMat<C> Rn, Bm;
      load_matp<C>(a.Rn, a.dtype, idx, Rn);
      Bm = Rn;
      CVec<C> g;
      st |= gev_principal<C>(Rs, Bm, g);
      matvec<C>(Rn, g, p);
    }
    double tr1 = 0.0;
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) tr1 += cd_abs2(p.v[i]);
    const double scale = tr / fmax(tr1, SETK_EPS32_D);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) {
      SETK_UNROLL_C
      for (int j = 0; j < C; ++j)
        store_c(a.out, a.dtype, idx * (long long)(C * C) + i * C + j,
                cd_scale(cd_mulc(p.v[i], p.v[j]), scale));
    }
    if (st && a.status) atomicOr(a.status + b, st);
  }
}

cudaError_t post_run(int mode, const void* A, const void* Rn, int dtype, int B, int F, int C, void* out,
                     unsigned* status, void* stream) {
  PostArgs a;
  a.mode = mode; a.A = A; a.Rn = Rn; a.dtype = dtype; a.B = B; a.F = F; a.out = out; a.status = status;
  const long long n = (long long)B * F;
  dim3 block(128), grid((unsigned)((n + 127) / 128));
  switch (C) {
#define SETK_CASE(k) case k: return launch(post_kernel<k>, grid, block, 0, stream, true, a);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
