// weights.cu -- per-(utterance, bin) beamformer weight solve in fp64.
//
// One thread owns one C x C problem: bytes are negligible (Rs,Rn in, w out),
// the work is latency/ALU bound, so the kernel is judged by its share of the
// step, not by an HBM roofline (DESIGN.md "K3").
//
// Reference semantics reproduced (scripts/sptk/libs/beamformer.py):
//   solve_pevd 31-63, do_ban 14-28, rank1_constraint 66-84,
//   MvdrBeamformer.weight 527-539, MpdrBeamformer.weight 555-573,
//   PmwfBeamformer.weight/_snr 620-659, GevdBeamformer.weight 674-682.
#include "common.cuh"
#include "hermitian_solve.cuh"
#include "launchers.cuh"
#include "weights_args.cuh"

namespace setk {



template <int C>
__device__ inline void load_mat(const void* base, int dtype, long long idx, CMat<C>& M) {
  if (dtype == SETK_C128) {
    const double* p = reinterpret_cast<const double*>(base) + idx * (2LL * C * C);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i)
      SETK_UNROLL_C
      for (int j = 0; j < C; ++j) M.a[i][j] = cd_make(p[2 * (i * C + j)], p[2 * (i * C + j) + 1]);
  } else {
    const float* p = reinterpret_cast<const float*>(base) + idx * (2LL * C * C);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i)
      SETK_UNROLL_C
      for (int j = 0; j < C; ++j)
        M.a[i][j] = cd_make((double)p[2 * (i * C + j)], (double)p[2 * (i * C + j) + 1]);
  }
}

template <int C>
__device__ inline void store_vec(void* base, int dtype, long long idx, const CVec<C>& v) {
  if (dtype == SETK_C128) {
    double* p = reinterpret_cast<double*>(base) + idx * (2LL * C);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) { p[2 * i] = v.v[i].x; p[2 * i + 1] = v.v[i].y; }
  } else {
    float* p = reinterpret_cast<float*>(base) + idx * (2LL * C);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) { p[2 * i] = (float)v.v[i].x; p[2 * i + 1] = (float)v.v[i].y; }
  }
}

// do_ban, beamformer.py:14-28 (as written: w^H Rn Rn w, no transposes)
template <int C>
__device__ inline void apply_ban(CVec<C>& w, const CMat<C>& Rn) {
  CVec<C> u, v;
  matvec<C>(Rn, w, u);
  matvec<C>(Rn, u, v);
  cd num = dotc<C>(w, v);
  cd den = dotc<C>(w, u);
  double g = sqrt(sqrt(num.x * num.x + num.y * num.y)) / fmax(den.x, SETK_EPS32_D);
  for (int i = 0; i < C; ++i) w.v[i] = cd_scale(w.v[i], g);
}

// rank1_constraint, beamformer.py:66-84.  Rs replaced by its rank-1 model.
template <int C>
__device__ inline unsigned rank1_approx(CMat<C>& Rs, const CMat<C>& Rn, bool gev) {
  unsigned st = 0;
  CVec<C> p;
  double tr = 0.0;
  SETK_UNROLL_C
  for (int i = 0; i < C; ++i) tr += Rs.a[i][i].x;
  if (!gev) {
    CMat<C> A = Rs;
    if (!principal_eigvec<C>(A, p)) st |= SETK_ST_NO_CONVERGE;
  } else {
    CMat<C> A = Rs, Bm = Rn;
    CVec<C> g;
    st |= gev_principal<C>(A, Bm, g);
    matvec<C>(Rn, g, p);
  }
  double tr1 = 0.0;
  SETK_UNROLL_C
  for (int i = 0; i < C; ++i) tr1 += cd_abs2(p.v[i]);
  double scale = tr / fmax(tr1, SETK_EPS32_D);
  for (int i = 0; i < C; ++i)
    SETK_UNROLL_C
    for (int j = 0; j < C; ++j) Rs.a[i][j] = cd_scale(cd_mulc(p.v[i], p.v[j]), scale);
  return st;
}

template <int C>
__device__ inline bool all_finite(const CVec<C>& v) {
  bool ok = true;
  SETK_UNROLL_C
  for (int i = 0; i < C; ++i) ok = ok && isfinite(v.v[i].x) && isfinite(v.v[i].y);
  return ok;
}

// resident CTAs of 128 threads per SM the register allocation must allow (2 -> 255 registers)
#ifndef SETK_W_MINBLOCKS
#define SETK_W_MINBLOCKS 2
#endif

// KIND >= 0: an instantiation for ONE beamformer kind (the branches of the others fold away, and
// with them their registers: MVDR at C = 4 drops from 255 to <= 128 registers, i.e. from 8 to 16
// resident warps per SM for a kernel that is nothing but fp64 latency chains); KIND = -1: any kind.
template <int C, int KIND, int MINB>
__global__ void __launch_bounds__(128, MINB) weights_kernel(WeightsArgs a0) {
  WeightsArgs a = a0;
  if (KIND >= 0) { a.kind = KIND; if (KIND != SETK_BF_PMWF) a.rank1 = SETK_RANK1_NONE; }
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.B * a.F) return;
  int b = (int)(idx / a.F);
  unsigned st = 0;
  CMat<C> Rs, Rn;
  CVec<C> w;
  load_mat<C>(a.Rs, a.r_dtype, idx, Rs);
  const bool have_rn = a.Rn != nullptr;
  if (have_rn) load_mat<C>(a.Rn, a.r_dtype, idx, Rn);

  if (a.kind == SETK_BF_PEVD) {
    if (!have_rn) {
      CMat<C> A = Rs;
      if (!principal_eigvec<C>(A, w)) st |= SETK_ST_NO_CONVERGE;
    } else {
      CMat<C> A = Rs, Bm = Rn;
      st |= gev_principal<C>(A, Bm, w);
    }
  } else if (a.kind == SETK_BF_GEVD) {
    CMat<C> A = Rs, Bm = Rn;
    st |= gev_principal<C>(A, Bm, w);
  } else if (a.kind == SETK_BF_MVDR || a.kind == SETK_BF_MPDR || a.kind == SETK_BF_MPDR_WHITEN) {
    CVec<C> d;
    if (a.kind == SETK_BF_MPDR_WHITEN) {
      CMat<C> A = Rs, Bm = Rn;
      CVec<C> g;
      st |= gev_principal<C>(A, Bm, g);
      matvec<C>(Rn, g, d);
    } else {
      CMat<C> A = Rs;
      if (!principal_eigvec<C>(A, d)) st |= SETK_ST_NO_CONVERGE;
    }
    CMat<C> D;   // denominator matrix: Rn for MVDR, Ry for MPDR
    if (a.kind == SETK_BF_MVDR) D = Rn; else load_mat<C>(a.Ry, a.r_dtype, idx, D);
    int perm[C];
    if (!lu_factor<C>(D, perm)) st |= SETK_ST_SINGULAR;
    CVec<C> n = d;
    lu_solve_vec<C>(D, perm, n);
    cd den = dotc<C>(d, n);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) w.v[i] = cd_div(n.v[i], den);
  } else {  // SETK_BF_PMWF
    if (a.rank1 == SETK_RANK1_EIG) st |= rank1_approx<C>(Rs, Rn, false);
    if (a.rank1 == SETK_RANK1_GEV) st |= rank1_approx<C>(Rs, Rn, true);
    CMat<C> LU = Rn;
    int perm[C];
    if (!lu_factor<C>(LU, perm)) st |= SETK_ST_SINGULAR;
    CMat<C> G;   // Rn^-1 Rs, column by column
    cd tr = cd_make(0.0, 0.0);
    SETK_UNROLL_C
    for (int c = 0; c < C; ++c) {
      CVec<C> col;
      SETK_UNROLL_C
      for (int i = 0; i < C; ++i) col.v[i] = Rs.a[i][c];
      lu_solve_vec<C>(LU, perm, col);
      SETK_UNROLL_C
      for (int i = 0; i < C; ++i) G.a[i][c] = col.v[i];
      tr = cd_add(tr, col.v[c]);
    }
    cd den = cd_make(a.beta + tr.x, tr.y);
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i)
      SETK_UNROLL_C
      for (int j = 0; j < C; ++j) G.a[i][j] = cd_div(G.a[i][j], den);
    if (a.ref_channel >= 0) {
      int ref = a.ref_channel < C ? a.ref_channel : 0;
      if (a.ref_channel >= C) st |= SETK_ST_BAD_REF;
      for (int i = 0; i < C; ++i) w.v[i] = G.a[i][ref];
      if (a.ref_used && idx % a.F == 0) a.ref_used[b] = ref;
    } else {
      // defer: store W and the per-channel signal / noise powers of this bin
      double* Wp = a.Wfull + idx * (2LL * C * C);
      SETK_UNROLL_C
      for (int i = 0; i < C; ++i)
        SETK_UNROLL_C
        for (int j = 0; j < C; ++j) { Wp[2 * (i * C + j)] = G.a[i][j].x; Wp[2 * (i * C + j) + 1] = G.a[i][j].y; }
      double* pp = a.pows + idx * (2LL * C);
      SETK_UNROLL_C
      for (int c = 0; c < C; ++c) {
        CVec<C> wc, u;
        SETK_UNROLL_C
        for (int i = 0; i < C; ++i) wc.v[i] = G.a[i][c];
        matvec<C>(Rs, wc, u);
        pp[2 * c] = dotc<C>(wc, u).x;
        matvec<C>(Rn, wc, u);
        pp[2 * c + 1] = dotc<C>(wc, u).x;
      }
      if (st) atomicOr(a.status + b, st);
      return;
    }
  }
  if (a.ban && have_rn) apply_ban<C>(w, Rn);
  if (!all_finite<C>(w)) st |= SETK_ST_NONFINITE;
  store_vec<C>(a.w, a.w_dtype, idx, w);
  if (st) atomicOr(a.status + b, st);
}

// PMWF with ref_channel < 0: per utterance, pick argmax_c of
// sum_f Re(w_c^H Rs w_c) / max(eps, sum_f Re(w_c^H Rn w_c))  (beamformer.py:620-630,
// 650-653; first maximum like np.argmax), then gather that column.
template <int C>
__global__ void __launch_bounds__(128) pmwf_select_kernel(WeightsArgs a) {
  __shared__ double s_snr[SETK_MAX_CHANNELS];
  __shared__ int s_ref;
  const int b = blockIdx.x;
  if ((int)threadIdx.x < C) {
    const int c = threadIdx.x;
    double ps = 0.0, pn = 0.0;
    const double* pp = a.pows + ((long long)b * a.F) * (2LL * C);
    SETK_NOUNROLL
    for (int f = 0; f < a.F; ++f) { ps += pp[(long long)f * 2 * C + 2 * c]; pn += pp[(long long)f * 2 * C + 2 * c + 1]; }
    s_snr[c] = ps / fmax(SETK_EPS32_D, pn);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int ref = 0;
    SETK_UNROLL_C
    for (int c = 1; c < C; ++c) if (s_snr[c] > s_snr[ref]) ref = c;
    s_ref = ref;
    if (a.ref_used) a.ref_used[b] = ref;
  }
  __syncthreads();
  const int ref = s_ref;
  unsigned st = 0;
  SETK_NOUNROLL
  for (int f = threadIdx.x; f < a.F; f += blockDim.x) {
    long long idx = (long long)b * a.F + f;
    const double* Wp = a.Wfull + idx * (2LL * C * C);
    CVec<C> w;
    SETK_UNROLL_C
    for (int i = 0; i < C; ++i) w.v[i] = cd_make(Wp[2 * (i * C + ref)], Wp[2 * (i * C + ref) + 1]);
    if (a.ban) {
      CMat<C> Rn;
      load_mat<C>(a.Rn, a.r_dtype, idx, Rn);
      apply_ban<C>(w, Rn);
    }
    if (!all_finite<C>(w)) st |= SETK_ST_NONFINITE;
    store_vec<C>(a.w, a.w_dtype, idx, w);
  }
  if (st) atomicOr(a.status + b, st);
}

template <int C>
static cudaError_t launch_weights(const WeightsArgs& a, void* stream) {
  if (weights_coop_supported(a, C)) return weights_coop_launch(a, C, stream);
  long long n = (long long)a.B * a.F;
  const int bs = 128;
  dim3 block(bs), grid((unsigned)((n + bs - 1) / bs));
  cudaError_t e;
  if (C <= 4 && a.kind == SETK_BF_MVDR)
    e = launch(weights_kernel<(C <= 4 ? C : 1), SETK_BF_MVDR, 4>, grid, block, 0, stream, true, a);
  else if (C <= 4 && a.kind == SETK_BF_GEVD)
    e = launch(weights_kernel<(C <= 4 ? C : 1), SETK_BF_GEVD, 4>, grid, block, 0, stream, true, a);
  else
    e = launch(weights_kernel<C, -1, SETK_W_MINBLOCKS>, grid, block, 0, stream, /*barrier_free=*/true, a);
  if (e != cudaSuccess) return e;
  if (a.kind == SETK_BF_PMWF && a.ref_channel < 0)
    e = launch(pmwf_select_kernel<C>, dim3(a.B), dim3(128), 0, stream, /*barrier_free=*/false, a);
  return e;
}

static cudaError_t weights_dispatch(const WeightsArgs& a, int C, void* stream) {
  switch (C) {
#define SETK_CASE(n) case n: return launch_weights<n>(a, stream);
    SETK_CASE(1) SETK_CASE(2) SETK_CASE(3) SETK_CASE(4) SETK_CASE(5) SETK_CASE(6) SETK_CASE(7) SETK_CASE(8)
    SETK_CASE(9) SETK_CASE(10) SETK_CASE(11) SETK_CASE(12) SETK_CASE(13) SETK_CASE(14) SETK_CASE(15) SETK_CASE(16)
#undef SETK_CASE
    default: return cudaErrorInvalidValue;
  }
}

// Scratch of the PMWF automatic reference selection: allocated per call on the caller's
// stream (cudaMallocAsync / cudaFreeAsync, like the plan-free entry points of api.cu), so calls on
// different streams or devices never share it.
cudaError_t weights_run(int kind, double beta, int ref_channel, int rank1, int ban, const void* Rs,
                        const void* Rn, const void* Ry, int r_dtype, int B, int F, int C, void* w,
                        int w_dtype, unsigned* status, int* ref_used, void* stream) {
  WeightsArgs a;
  a.kind = kind; a.rank1 = rank1; a.ban = ban; a.ref_channel = ref_channel; a.beta = beta;
  a.Rs = Rs; a.Rn = Rn; a.Ry = Ry; a.r_dtype = r_dtype; a.B = B; a.F = F;
  a.w = w; a.w_dtype = w_dtype; a.status = status; a.ref_used = ref_used;
  a.Wfull = nullptr; a.pows = nullptr;
  double* ws = nullptr;
  if (kind == SETK_BF_PMWF && ref_channel < 0) {
    const size_t nW = (size_t)B * F * C * C * 2, nP = (size_t)B * F * C * 2;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&ws), sizeof(double) * (nW + nP),
                                    static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return e;
    a.Wfull = ws;
    a.pows = ws + nW;
  }
  cudaError_t e = weights_dispatch(a, C, stream);
  if (ws) {
    cudaError_t e2 = cudaFreeAsync(ws, static_cast<cudaStream_t>(stream));
    if (e == cudaSuccess) e = e2;
  }
  return e;
}

}  // namespace setk
