// rir.cu -- image-method room impulse responses (setk_rir_image): RirGenerator::GenerateRir of the
// reference's include/rir-generator.cc:108-192 (Habets' RIR-Generator, what rir-simulate runs) for a
// batch of problems b = (room, beta, source), each with M receivers.
//
// One CTA of kRirThreads per (segment, receiver m, problem b).  A segment is kRirSeg output samples
// [s0, s1); L <= kRirSeg is one segment.  The CTA walks the whole image lattice of its channel:
//   * rows (x, y) of the lattice go to the warps round robin; a row whose nearest image (over q, j)
//     is already past the segment's reach is skipped as a whole;
//   * the 8 (2 nz + 1) candidates (z, q, j, k) of a row go to the lanes, 32 at a time.  A lane
//     computes its image in fp64 -- distance, floor(dist), frac, the order test, the segment
//     overlap test, the reflection factor from per-axis tables of beta^|.| in shared memory (no
//     pow per image) and the gain -- and stages a surviving image in the warp's shared slots;
//   * the warp then spreads each staged image's Tw taps over its lanes: lane l owns taps
//     l, l + 32, ..., so one image writes consecutive shared addresses.
// Taps are float32.  The window's cosine comes from angle addition with per-lane constants and the
// sinc's sine from sin(pi (k - frac)) = -(-1)^k sin(pi frac), so a tap costs no transcendental.
//
// Determinism: the segment accumulates in shared memory as 64-bit fixed point, 2^-44 per unit
// (resolution 5.7e-14, range +-2^19 = +-524288), with integer atomicAdd.  Integer addition is
// associative, so the sum is bit-identical whatever the order of the images and however the work
// is split.  A tap that is not finite or of magnitude >= kRirTapMax, or an addition that leaves the
// signed 64-bit range, sets SETK_ST_NONFINITE for the problem (the tap is dropped); nothing wraps
// silently.
//
// High-pass filter (rir-generator.cc:180-190): fp64, one thread's recurrence over the channel.  One
// segment: fused at the end of the CTA.  Several segments: the CTAs write fp64 sums to scratch and
// a second kernel, one thread per channel, filters them into the output.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

#ifndef SETK_RIR_SEG
#define SETK_RIR_SEG 8192   // output samples per CTA: 64 KB of accumulator (the CPU tier also tests 256)
#endif
constexpr int kRirSeg = SETK_RIR_SEG;
constexpr int kRirThreads = 256;
constexpr int kRirWarps = kRirThreads / 32;
constexpr float kRirFix = 17592186044416.0f;            // 2^44: fixed-point units per unit
constexpr double kRirUnfix = 1.0 / 17592186044416.0;    // 2^-44
constexpr float kRirTapMax = 4096.0f;                   // |tap| >= 2^12: out of range

struct RirArgs {
  const double* room;      // [B][3] metres
  const double* beta;      // [B][6]
  const double* src;       // [B][3]
  const double* rcv;       // [B][M][3]
  int B, M, L, Tw, nseg, order, hp, max_n;   // max_n: the tables' capacity per axis (host-checked)
  double cts;              // c / fs: metres per sample
  double rho, ux, uy, uz;  // polar pattern: rho + (1 - rho) u . dir (u = 0 for omni)
  double hp_b1, hp_b2, hp_a1, hp_r1;
  float* rir;              // [B][M][L]
  double* ws;              // [B][M][L] fp64 sums (several segments with the filter) or null
  unsigned* status;        // [B] or null
};

// n of the lattice x in [-n, n] along one axis (rir-generator.cc:127-129), T the room in samples
SETK_HD inline int rir_axis_n(int L, double T) { return (int)ceil((double)L / (2.0 * T)); }

double rir_lattice_half(int L, double room, double cts) { return ceil((double)L / (2.0 * (room / cts))); }

int rir_window_taps(double fs) { return 2 * (int)(0.004 * fs + 0.5); }   // rir-generator.cc:119

__device__ __forceinline__ unsigned rir_ballot(bool p) {
#ifdef SETK_EMU
  unsigned m = p ? 1u << (threadIdx.x & 31) : 0u;
  for (int o = 1; o < 32; o <<= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
  return m;
#else
  return __ballot_sync(0xffffffffu, p);
#endif
}

__device__ __forceinline__ long long rir_to_fixed(float v) {
#ifdef SETK_EMU
  return llrintf(v * kRirFix);
#else
  return __float2ll_rn(v * kRirFix);
#endif
}

// 2-pole high-pass of rir-generator.cc:180-190 in fp64: y0 = b1 y1 + b2 y2 + x; out = y0 + a1 y1 + r1 y2
struct RirHp {
  double y1 = 0, y2 = 0;
  __device__ __forceinline__ double step(const RirArgs& a, double x) {
    const double y0 = a.hp_b1 * y1 + a.hp_b2 * y2 + x;
    const double out = y0 + a.hp_a1 * y1 + a.hp_r1 * y2;
    y2 = y1;
    y1 = y0;
    return out;
  }
};

size_t rir_smem_bytes(int L, int max_n) {
  const int seg = imin(L, kRirSeg);
  return sizeof(unsigned long long) * seg + sizeof(double) * 6 * (size_t)(max_n + 2) +
         (sizeof(int) + 5 * sizeof(float)) * kRirThreads;
}

// TPL: taps per lane, ceil(Tw / 32) rounded up to a power of two (Tw = 128 at 16 kHz: 4)
template <int TPL>
__global__ void __launch_bounds__(kRirThreads, TPL <= 8 ? 2 : 1) rir_image_kernel(RirArgs a) {
  SETK_DYN_SMEM(unsigned long long, acc);
  const int seg = blockIdx.x, m = blockIdx.y, b = blockIdx.z;
  const int L = a.L, Tw = a.Tw, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s0 = seg * kRirSeg, s1 = imin(L, s0 + kRirSeg), len = s1 - s0;
  const int cap = a.max_n + 2;
  double* tab = reinterpret_cast<double*>(acc + imin(L, kRirSeg));   // [3 axes][2][cap]
  int* st_pos = reinterpret_cast<int*>(tab + 6 * (size_t)cap);         // [warp][32] staged images
  float* st_frac = reinterpret_cast<float*>(st_pos + kRirThreads);
  float* st_cph = st_frac + kRirThreads;
  float* st_sph = st_cph + kRirThreads;
  float* st_gs = st_sph + kRirThreads;
  float* st_g = st_gs + kRirThreads;

  const double cts = a.cts;
  double T[3], S[3], R[3];
  int n[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    T[d] = a.room[(size_t)b * 3 + d] / cts;
    S[d] = a.src[(size_t)b * 3 + d] / cts;
    R[d] = a.rcv[((size_t)b * a.M + m) * 3 + d] / cts;
    n[d] = rir_axis_n(L, T[d]);
  }
  // tab[d][0][k] = beta[2d]^k, tab[d][1][k] = beta[2d+1]^k, k = 0 .. n[d] + 1 (pow(0, 0) = 1)
  for (int d = 0; d < 3; ++d)
    for (int i = tid; i < 2 * (n[d] + 2); i += kRirThreads) {
      const int w = i / (n[d] + 2), k = i - w * (n[d] + 2);
      tab[(size_t)(2 * d + w) * cap + k] = pow(a.beta[(size_t)b * 6 + 2 * d + w], (double)k);
    }
  for (int i = tid; i < len; i += kRirThreads) acc[i] = 0ull;

  // per-lane tap constants: taps n = lane + 32 i, cos / sin of 2 pi (n + 1) / Tw, (-1)^(n + 1 - Tw/2)
  float ca[TPL], sa[TPL], kf[TPL], sg[TPL];
#pragma unroll
  for (int i = 0; i < TPL; ++i) {
    const int nt = lane + 32 * i, k = nt + 1 - Tw / 2;
    double s, c;
    sincospi(2.0 * (nt + 1) / Tw, &s, &c);
    ca[i] = (float)c;
    sa[i] = (float)s;
    kf[i] = (float)k;
    sg[i] = (k & 1) ? -1.f : 1.f;
  }
  __syncthreads();

  // an image's taps reach samples floor(dist) - Tw/2 + 1 .. floor(dist) + Tw/2: it can touch the
  // segment only when lo <= floor(dist) < hi (and floor(dist) < L, rir-generator.cc:158)
  const int lo = imax(0, s0 - Tw / 2), hi = imin(L, s1 + Tw / 2 - 1);
  const double reach2 = ((double)hi + 1) * ((double)hi + 1);
  const double pre_lo2 = lo > 1 ? ((double)lo - 1) * ((double)lo - 1) : 0.0;
  const int Nx = 2 * n[0] + 1, Ny = 2 * n[1] + 1, Nz = 2 * n[2] + 1, per_row = 8 * Nz;
  const double* tx = tab;
  const double* ty = tab + 2 * (size_t)cap;
  const double* tz = tab + 4 * (size_t)cap;
  const int order = a.order;
  const double gain_den = 4.0 * M_PI * cts;
  bool bad = false;
  int* wpos = st_pos + warp * 32;
  float *wfrac = st_frac + warp * 32, *wcph = st_cph + warp * 32, *wsph = st_sph + warp * 32;
  float *wgs = st_gs + warp * 32, *wg = st_g + warp * 32;

  for (int row = warp; row < Nx * Ny; row += kRirWarps) {
    const int x = row / Ny - n[0], y = row % Ny - n[1];
    // (1 - 2q) S - R + 2 x T, for q = 0, 1 (rir-generator.cc:132-149)
    const double dx0 = S[0] - R[0] + 2 * x * T[0], dx1 = -S[0] - R[0] + 2 * x * T[0];
    const double dy0 = S[1] - R[1] + 2 * y * T[1], dy1 = -S[1] - R[1] + 2 * y * T[1];
    if (fmin(dx0 * dx0, dx1 * dx1) + fmin(dy0 * dy0, dy1 * dy1) >= reach2) continue;   // warp-uniform
    const int ax = x < 0 ? -x : x, ay = y < 0 ? -y : y;
    for (int c0 = 0; c0 < per_row; c0 += 32) {
      const int c = c0 + lane;
      bool keep = false;
      int pos = 0;
      float frac = 0.f, cph = 0.f, sph = 0.f, gs = 0.f, g = 0.f;
      if (c < per_row) {
        const int z = (c >> 3) - n[2], q = (c >> 2) & 1, j = (c >> 1) & 1, k = c & 1;
        const int az = z < 0 ? -z : z;
        const int ord = abs(2 * x - q) + abs(2 * y - j) + abs(2 * z - k);
        const double px = q ? dx1 : dx0, py = j ? dy1 : dy0;
        const double pz = (1 - 2 * k) * S[2] - R[2] + 2 * z * T[2];
        const double d2 = px * px + py * py + pz * pz;
        if ((order == -1 || ord <= order) && d2 < reach2 && d2 >= pre_lo2) {
          const double dist = sqrt(d2), fd = floor(dist);
          const int ifd = (int)fd;
          if (ifd >= lo && ifd < hi) {
            const double refl = (tx[abs(x - q)] * tx[cap + ax]) * (ty[abs(y - j)] * ty[cap + ay]) *
                                (tz[abs(z - k)] * tz[cap + az]);
            if (refl != 0.0) {
              const double mic = a.rho + (a.ux * px + a.uy * py + a.uz * pz) / dist;   // MicrophoneSim
              const double gd = mic * refl / (gain_den * dist);
              const double fr = dist - fd;
              float s_pf, c_pf, s_ph, c_ph;
              sincospif((float)fr, &s_pf, &c_pf);
              sincospif((float)(2.0 * fr / Tw), &s_ph, &c_ph);
              keep = true;
              pos = ifd - Tw / 2 + 1;
              frac = (float)fr;
              cph = c_ph;
              sph = s_ph;
              g = (float)gd;
              gs = (float)(-gd * (double)s_pf / M_PI);
            }
          }
        }
      }
      const unsigned mask = rir_ballot(keep);
      if (keep) {
        const int slot = __popc(mask & ((1u << lane) - 1u));
        wpos[slot] = pos; wfrac[slot] = frac; wcph[slot] = cph; wsph[slot] = sph; wgs[slot] = gs; wg[slot] = g;
      }
      __syncwarp();
      const int cnt = __popc(mask);
      for (int e = 0; e < cnt; ++e) {
        const int p = wpos[e];
        const float fr = wfrac[e], cp = wcph[e], sp = wsph[e], gse = wgs[e], ge = wg[e];
#pragma unroll
        for (int i = 0; i < TPL; ++i) {
          const int nt = lane + 32 * i, t = p + nt;
          if (nt < Tw && t >= s0 && t < s1) {
            const float win = 0.5f - 0.5f * fmaf(ca[i], cp, sa[i] * sp);   // 0.5 (1 - cos(2 pi (n+1-frac)/Tw))
            const float den = kf[i] - fr;
            const float v = den != 0.f ? win * (sg[i] * gse) / den : win * ge;
            if (!(fabsf(v) < kRirTapMax)) {
              bad = true;
              continue;
            }
            const long long fx = rir_to_fixed(v);
            const unsigned long long old = atomicAdd(&acc[t - s0], (unsigned long long)fx);
            const long long o = (long long)old, nw = (long long)(old + (unsigned long long)fx);
            if (((o ^ nw) & (fx ^ nw)) < 0) bad = true;   // signed overflow of the running sum
          }
        }
      }
      __syncwarp();
    }
  }
  if (bad && a.status) atomicOr(&a.status[b], SETK_ST_NONFINITE);
  __syncthreads();

  const size_t ch = ((size_t)b * a.M + m) * L;
  if (a.hp && a.nseg == 1) {
    if (tid == 0) {
      RirHp f;
      for (int t = 0; t < L; ++t) a.rir[ch + t] = (float)f.step(a, (double)(long long)acc[t] * kRirUnfix);
    }
  } else if (a.ws) {
    for (int i = tid; i < len; i += kRirThreads) a.ws[ch + s0 + i] = (double)(long long)acc[i] * kRirUnfix;
  } else {
    for (int i = tid; i < len; i += kRirThreads) a.rir[ch + s0 + i] = (float)((double)(long long)acc[i] * kRirUnfix);
  }
}

// several segments with the filter: one thread per channel runs the recurrence over the fp64 sums
__global__ void __launch_bounds__(128) rir_hp_kernel(RirArgs a) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= a.B * a.M) return;
  const size_t o = (size_t)ch * a.L;
  RirHp f;
  for (int t = 0; t < a.L; ++t) a.rir[o + t] = (float)f.step(a, a.ws[o + t]);
}

template <int TPL>
static cudaError_t rir_launch(const RirArgs& a, size_t smem, void* stream) {
#ifndef SETK_EMU
  cudaError_t ea = cudaFuncSetAttribute(rir_image_kernel<TPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (ea != cudaSuccess) return ea;
#endif
  return launch(rir_image_kernel<TPL>, dim3(a.nseg, a.M, a.B), dim3(kRirThreads), smem, stream, false, a);
}

int rir_segments(int L) { return (L + kRirSeg - 1) / kRirSeg; }

cudaError_t run_rir_image(const setk_rir_config_t& cfg, const double* room, const double* beta,
                          const double* source, const double* receivers, int B, int M, int max_n, float* rir,
                          double* ws, unsigned* status, void* stream) {
  RirArgs a;
  a.room = room; a.beta = beta; a.src = source; a.rcv = receivers;
  a.B = B; a.M = M; a.L = cfg.n_samples; a.Tw = rir_window_taps(cfg.samp_frequency);
  a.nseg = rir_segments(a.L); a.order = cfg.order; a.hp = cfg.hp_filter != 0; a.max_n = max_n;
  a.cts = cfg.sound_velocity / cfg.samp_frequency;
  static const double kRho[5] = {1.0, 0.75, 0.5, 0.25, 0.0};   // rir-generator.cc:196-212
  a.rho = kRho[cfg.mic_type];
  // rho + (1 - rho) (sin(pi/2 - el) sin(theta) cos(az - phi) + cos(pi/2 - el) cos(theta))
  // = rho + (1 - rho) u . p / |p| with u = (cos el cos az, cos el sin az, sin el)
  const double w = 1.0 - a.rho;
  a.ux = w * cos(cfg.elevation) * cos(cfg.azimuth);
  a.uy = w * cos(cfg.elevation) * sin(cfg.azimuth);
  a.uz = w * sin(cfg.elevation);
  const double W = 2 * M_PI * 100 / cfg.samp_frequency;   // rir-generator.cc:120-121
  a.hp_r1 = exp(-W);
  a.hp_b1 = 2 * a.hp_r1 * cos(W);
  a.hp_b2 = -a.hp_r1 * a.hp_r1;
  a.hp_a1 = -1 - a.hp_r1;
  a.rir = rir;
  a.ws = ws;
  a.status = status;
  const size_t smem = rir_smem_bytes(a.L, max_n);
  const int tpl = (a.Tw + 31) / 32;
  cudaError_t e = tpl <= 1 ? rir_launch<1>(a, smem, stream)
                : tpl <= 2 ? rir_launch<2>(a, smem, stream)
                : tpl <= 4 ? rir_launch<4>(a, smem, stream)
                : tpl <= 8 ? rir_launch<8>(a, smem, stream)
                           : rir_launch<16>(a, smem, stream);
  if (e != cudaSuccess || !ws) return e;
  return launch(rir_hp_kernel, dim3((B * M + 127) / 128), dim3(128), 0, stream, true, a);
}

}  // namespace setk
