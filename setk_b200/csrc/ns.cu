// ns.cu -- single-channel noise suppression: the iMCRA noise estimator and the OM-LSA gain of
// scripts/sptk/libs/ns.py:212-387 (iMCRA.run, Cohen 2003), for every utterance of a batch
// (setk_ns_imcra).
//
// The recursion runs strictly in order over frames and in parallel over bins.  One CTA per
// utterance of at most 512 threads; thread i owns bins i, i + NT, ... (K = ceil(F / 512) of them).
// Each bin carries its own state from frame to frame: lambda_d_hat, gh1, var_s, var_s_hat and two
// running minima in registers, the two sub-window minima in shared memory (private to the owning
// thread, like xi_hat and v carried from one phase of the frame to the next).  Within a frame the bins meet only in np.convolve(., w_m, "same") with
// 2 w_mcra + 1 taps, three times:
//   * on obs_power[t]: depends only on the input, read from the staged tile;
//   * on indicator and obs_power * indicator: depend on the state, exchanged through two
//     double-buffered shared arrays, one barrier per frame.
// The STFT [B][F][T] is staged through shared memory TT frames at a time, read coalesced along T;
// enh = gain * X goes back through the same tile.  gain [B][T][F] is written row by row.
//
// Sub-window minima: every V frames ns.py:370-380 takes the min over the last U PER-FRAME values of
// var_s_min_sw (and _hat).  Those never increase within a sub-window, so that min is the min of the
// current value and the ends of the R = floor((U - 1) / V) sub-windows before it; a ring of R ends
// per bin (global scratch, touched once per sub-window) replaces the U-frame history.  R = 0 for
// U <= V (the default 8 <= 15).
//
// fp64 after the complex64 input.  No atomics: two calls give bit-identical results.  E1 is
// ns_expint below; at v == 0 it returns what the reference's quad returns (37.1912...), not +inf.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

struct NsArgs {
  double alpha, alpha_s, alpha_d, b_min_inv, gamma0, gamma1, zeta0, xi_min, log_gain_min, beta, eps;
  double w[2 * SETK_NS_MAX_W + 1];   // w_m of iMCRA.__init__
  int w_mcra, V, R;
  const float2* X;                   // [B][F][T]
  const int* n_frames;               // [B] or null
  int B, F, T, TT;
  double* gain;                      // [B][T][F] or null
  float2* enh;                       // [B][F][T] or null
  double* ring;                      // [B][R][2][F] or null (R == 0)
};

// quad(lambda t: exp(-t) / t, 0, inf) of the reference (ns.py:259-260), finite where E1(0) is not
#define SETK_NS_E1_AT_ZERO 37.191280375549404
#define SETK_EULER_GAMMA 0.57721566490153286061

// (-1)^(k+1) / (k k!), k = 1..26: the power series of E1(v) + gamma + ln v
__constant__ double kE1Series[26] = {
  1.0, -0.25, 0.05555555555555555, -0.010416666666666666, 0.0016666666666666668,
  -0.0002314814814814815, 2.834467120181406e-05, -3.1001984126984127e-06, 3.0619243582206544e-07,
  -2.755731922398589e-08, 2.27746439867652e-09, -1.7397297489890083e-10, 1.2353110643708935e-11,
  -8.193389712664089e-13, 5.0981091545465446e-14, -2.9871733327421158e-15, 1.6537983849091297e-16,
  -8.677337204770125e-18, 4.326650129802279e-19, -2.0551588116560825e-20, 9.32044812542441e-22,
  -4.0439960874775335e-23, 1.6818131176655147e-24, -6.715573212900493e-26, 2.5787801137537893e-27,
  -9.53690870471076e-29};

// Exponential integral E1(v), v >= 0, fp64.  v <= 2: -gamma - ln v + the series above by Horner (26
// FMAs, no division).  v > 2: e^-v over the continued fraction v + 1 - 1/(v + 3 - 4/(v + 5 - ...))
// by its forward (Wallis) recurrence -- FMAs only, one division at the end -- stopped when two
// convergents agree to 1e-17 (52 steps at v = 2, 7 at v = 50), at most 96 steps.  E1 underflows
// to 0 past v ~ 745.  Agrees with scipy.special.exp1 to ~1e-14 relative over [1e-300, 700].
__device__ __forceinline__ double ns_expint(double v) {
  if (v == 0.0) return SETK_NS_E1_AT_ZERO;
  if (v <= 2.0) {
    double s = kE1Series[25];
#pragma unroll
    for (int k = 24; k >= 0; --k) s = fma(s, v, kE1Series[k]);
    return s * v - SETK_EULER_GAMMA - log(v);
  }
  if (v > 746.0) return 0.0;
  double a1 = 1.0, a0 = v + 1.0, b1 = 0.0, b0 = 1.0;
  for (int n = 1; n <= 96; ++n) {
    const double an = -(double)(n * n), bn = v + (double)(2 * n + 1);
    const double a2 = fma(bn, a0, an * a1), b2 = fma(bn, b0, an * b1);
    a1 = a0; a0 = a2; b1 = b0; b0 = b2;
    if (fabs(a0 * b1 - a1 * b0) <= 1e-17 * fabs(a0 * b1)) break;
    if (fabs(a0) > 1e150) { a0 *= 1e-150; a1 *= 1e-150; b0 *= 1e-150; b1 *= 1e-150; }
  }
  return exp(-v) * (b0 / a0);
}

// np.minimum / np.maximum: a NaN operand wins
__device__ __forceinline__ double nmin(double a, double b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ double nmax(double a, double b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ double abs2d(float2 x) { return (double)x.x * x.x + (double)x.y * x.y; }

constexpr int kNsThreads = 512;   // most threads of a CTA: bins per thread K = ceil(F / 512)

inline int ns_tile_frames(int F) { return F <= 1025 ? 16 : 4; }
// the tile [F][TT + 1] float2, then [2][F] doubles each of oi, xi_hat / v, and the sub-window minima
inline size_t ns_smem_bytes(int F, int TT) {
  return sizeof(float2) * (size_t)F * (TT + 1) + sizeof(double) * 6 * (size_t)F;
}

template <int K>
__global__ void __launch_bounds__(kNsThreads, 1) ns_imcra_kernel(NsArgs a) {
  SETK_DYN_SMEM(double, sm);
  const int F = a.F, T = a.T, TT = a.TT, P = TT + 1, NT = blockDim.x, tid = threadIdx.x;
  const int b = blockIdx.x;
  float2* xs = reinterpret_cast<float2*>(sm);              // [F][P]  the tile: X, then enh
  double* oi = sm + (size_t)F * P;                         // [2][F]  obs_power where indicator, else -1
  double* xiv = oi + 2 * (size_t)F;                        // [2][F]  xi_hat, v of the frame
  double* msw = xiv + 2 * (size_t)F;                       // [2][F]  var_s_min_sw, var_s_min_sw_hat
  __shared__ double w[2 * SETK_NS_MAX_W + 1];
  if (tid < 2 * SETK_NS_MAX_W + 1) w[tid] = a.w[tid];
  const int Tb = a.n_frames ? imin(imax(a.n_frames[b], 0), T) : T;
  const float2* X = a.X + (size_t)b * F * T;
  const int wm = a.w_mcra, taps = 2 * wm + 1;
  const double as = a.alpha_s, ad = a.alpha_d, at = a.alpha, bmin = a.b_min_inv, eps = a.eps;

  double lam[K], gh1[K], vs[K], vsh[K], vmin[K], vminh[K];
#pragma unroll
  for (int k = 0; k < K; ++k) gh1[k] = 1.0;

  int prev_t0 = -1, prev_n = 0;
  for (int t0 = 0; t0 < T; t0 += TT) {
    const int n = imin(TT, T - t0);
    __syncthreads();                                       // the previous tile's frames are done
    if (a.enh && prev_t0 >= 0)
      for (int q = tid; q < F * TT; q += NT) {
        const int f = q / TT, u = q - f * TT;
        if (u < prev_n) a.enh[((size_t)b * F + f) * T + prev_t0 + u] = xs[f * P + u];
      }
    for (int q = tid; q < F * TT; q += NT) {              // same (f, u) -> same thread as the store
      const int f = q / TT, u = q - f * TT;
      if (u < n) xs[f * P + u] = t0 + u < Tb ? X[(size_t)f * T + t0 + u] : make_float2(0.f, 0.f);
    }
    __syncthreads();
    for (int u = 0; u < n; ++u) {
      const int t = t0 + u;
      if (t >= Tb) {                                       // past the utterance: gain 0, enh 0 (staged)
        if (a.gain)
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const int f = tid + k * NT;
            if (f < F) a.gain[((size_t)b * T + t) * F + f] = 0.0;
          }
        continue;
      }
      double* oib = oi + (t & 1) * F;
      // ---- phase 1: everything up to the indicator (ns.py:269-307) ----
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int f = tid + k * NT;
        if (f >= F) continue;
        const double o = abs2d(xs[f * P + u]);
        if (t == 0) lam[k] = o;
        const double gamma = o / nmax(lam[k] * a.beta, eps);
        double x = at * (gh1[k] * gh1[k] * gamma) + (1 - at) * nmax(gamma - 1, 0.0);
        x = nmax(x, a.xi_min);
        const double v = gamma * x / (1 + x);
        gh1[k] = x / (1 + x) * exp(0.5 * ns_expint(v));
        double vsf = 0.0;                                  // np.convolve(obs_power[t], w_m, "same")
        for (int j = 0; j < taps; ++j) {
          const int fi = f + wm - j;
          if (fi >= 0 && fi < F) vsf += w[j] * abs2d(xs[fi * P + u]);
        }
        if (t == 0) {
          vs[k] = vsh[k] = vmin[k] = msw[f] = vsf;
        } else {
          vs[k] = as * vs[k] + (1 - as) * vsf;
          vmin[k] = nmin(vmin[k], vs[k]);
          msw[f] = nmin(msw[f], vs[k]);
        }
        const double den = nmax(vmin[k], eps);
        const bool ind_on = (o * bmin / den < a.gamma0) && (vsf * bmin / den < a.zeta0);
        oib[f] = ind_on ? o : -1.0;
        xiv[f] = x;
        xiv[F + f] = v;
      }
      __syncthreads();                                     // indicators of frame t are complete
      // ---- phase 2: smoothed minima, speech presence, noise update and gain (ns.py:311-384) ----
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int f = tid + k * NT;
        if (f >= F) continue;
        double ic = 0.0, oc = 0.0;
        for (int j = 0; j < taps; ++j) {
          const int fi = f + wm - j;
          const double e = fi >= 0 && fi < F ? oib[fi] : -1.0;
          if (e >= 0) {
            ic += w[j];
            oc += w[j] * e;
          }
        }
        const double vsfh = ic > 0 ? oc / ic : vsh[k];     // var_sf_hat from the PREVIOUS var_s_hat
        if (t == 0) {
          vminh[k] = vs[k];
          msw[F + f] = vs[k];                              // var_sf, equal to var_s at t = 0
        } else {
          vsh[k] = as * vsh[k] + (1 - as) * vsfh;
          vminh[k] = nmin(vminh[k], vsh[k]);
          msw[F + f] = nmin(msw[F + f], vsh[k]);
        }
        const float2 xv = xs[f * P + u];
        const double o = abs2d(xv), x = xiv[f], v = xiv[F + f];
        const double denh = nmax(vminh[k], eps);
        const double gmh = o * bmin / denh, zh = vs[k] * bmin / denh;
        double p = 0.0;
        if (gmh > 1 && gmh < a.gamma1 && zh < a.zeta0) {
          const double q = (a.gamma1 - gmh) / (a.gamma1 - 1);
          p = 1 / (1 + q * (1 + x) / (1 - q) * exp(-v));
        }
        if (gmh >= a.gamma1 && zh >= a.zeta0) p = 1.0;
        const double adh = ad + (1 - ad) * p;
        lam[k] = adh * lam[k] + (1 - adh) * o;
        if ((t + 1) % a.V == 0) {                          // end of a sub-window
          double m = msw[f], mh = msw[F + f];
          if (a.R > 0) {
            const int kw = (t + 1) / a.V - 1;              // this sub-window
            double* ring = a.ring + (size_t)b * a.R * 2 * F + f;
            for (int j = 1; j <= imin(kw, a.R); ++j) {
              const int s = (kw - j) % a.R;
              m = nmin(m, ring[(size_t)(2 * s) * F]);
              mh = nmin(mh, ring[(size_t)(2 * s + 1) * F]);
            }
            const int s = kw % a.R;
            ring[(size_t)(2 * s) * F] = msw[f];
            ring[(size_t)(2 * s + 1) * F] = msw[F + f];
          }
          vmin[k] = m;
          vminh[k] = mh;
          msw[f] = vs[k];
          msw[F + f] = vsh[k];
        }
        // gh1^p gain_min^(1-p) as one exp (gh1 > 0; p == 0 gives gain_min even for gh1 = inf)
        const double g = exp((p > 0 ? p * log(gh1[k]) : 0.0) + (1 - p) * a.log_gain_min);
        if (a.gain) a.gain[((size_t)b * T + t) * F + f] = g;
        xs[f * P + u] = make_float2((float)(g * (double)xv.x), (float)(g * (double)xv.y));
      }
    }
    prev_t0 = t0;
    prev_n = n;
  }
  __syncthreads();
  if (a.enh && prev_t0 >= 0)
    for (int q = tid; q < F * TT; q += NT) {
      const int f = q / TT, u = q - f * TT;
      if (u < prev_n) a.enh[((size_t)b * F + f) * T + prev_t0 + u] = xs[f * P + u];
    }
}

size_t ns_ring_bytes(const setk_imcra_config_t& cfg, int B, int F) {
  const int R = (cfg.U - 1) / cfg.V;
  return sizeof(double) * (size_t)B * R * 2 * F;
}

template <int K>
static cudaError_t ns_launch(const NsArgs& a, void* stream) {
  const int NT = ((a.F + K - 1) / K + 31) / 32 * 32;   // <= kNsThreads
  const size_t smem = ns_smem_bytes(a.F, a.TT);
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(ns_imcra_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (ea != cudaSuccess) return ea;
#endif
  return launch(ns_imcra_kernel<K>, dim3(a.B), dim3(NT), smem, stream, false, a);
}

cudaError_t run_ns_imcra(const setk_imcra_config_t& cfg, const float2* X, const int* n_frames, int B, int F,
                         int T, double* ring, double* gain, float2* enh, void* stream) {
  NsArgs a;
  a.alpha = cfg.alpha; a.alpha_s = cfg.alpha_s; a.alpha_d = cfg.alpha_d;
  a.b_min_inv = 1 / cfg.b_min;                             // ns.py:240
  a.gamma0 = cfg.gamma0; a.gamma1 = cfg.gamma1; a.zeta0 = cfg.zeta0;
  a.xi_min = pow(10.0, cfg.xi_min_db / 10);                // ns.py:241
  a.log_gain_min = log(pow(10.0, cfg.gmin_db / 10));       // ln of gain_min, ns.py:242
  a.beta = cfg.beta; a.eps = cfg.eps;
  for (int j = 0; j < 2 * SETK_NS_MAX_W + 1; ++j) a.w[j] = j < 2 * cfg.w_mcra + 1 ? cfg.window_host[j] : 0.0;
  a.w_mcra = cfg.w_mcra; a.V = cfg.V; a.R = (cfg.U - 1) / cfg.V;
  a.X = X; a.n_frames = n_frames;
  a.B = B; a.F = F; a.T = T; a.TT = ns_tile_frames(F);
  a.gain = gain; a.enh = enh; a.ring = ring;
  switch ((F + kNsThreads - 1) / kNsThreads) {
    case 1: return ns_launch<1>(a, stream);
    case 2: return ns_launch<2>(a, stream);
    case 3: return ns_launch<3>(a, stream);
    case 4: return ns_launch<4>(a, stream);
    case 5: return ns_launch<5>(a, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace setk
