// api.cu -- the C-ABI of libsetk_b200.so (include/setk_b200.h): argument
// checking, plan / workspace management and dispatch to the kernels.
#include "common.cuh"
#include "launchers.cuh"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <cmath>
#include <vector>

namespace setk {

std::atomic<long long> g_launch_count{0};

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
static int cuda_fail(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof(g_err), "%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
  return (int)e;
}
// the return of every entry point: SETK_OK, or the CUDA error reported as `who`
static int done(cudaError_t e, const char* who) { return e == cudaSuccess ? SETK_OK : cuda_fail(e, who); }

// grow-only device workspace
template <class T>
static cudaError_t ensure(T** ptr, size_t* have, size_t want) {
  if (*have >= want && *ptr) return cudaSuccess;
  if (*ptr) cudaFree(*ptr);
  *ptr = nullptr; *have = 0;
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(ptr), want);
  if (e == cudaSuccess) *have = want;
  return e;
}

static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// Tile STFT of the batch into the plan's bin-major workspace d_stft_ws [B][T][C][bin_pitch(F)]
// (stft_spill.cu), with max|x| per utterance into maxabs_bits unless that is null.  A failure is
// reported as ws_what when the workspace cannot grow, as run_what when the launch fails.
static int stft_to_bin_major(setk_plan* pl, const float* audio, const int32_t* n_samples, int B, int N, int T,
                             unsigned* maxabs_bits, void* stream, const char* ws_what, const char* run_what) {
  const Geometry& g = pl->geo;
  cudaError_t e = ensure(&pl->d_stft_ws, &pl->stft_ws_bytes, stft_spill_bytes(g, B, T));
  if (e != cudaSuccess) return cuda_fail(e, ws_what);
  const int groups = (g.C + 3) / 4;   // the kernels take channels in groups of <= 4
  e = run_stft_spill(pl, audio, n_samples, B, N, T, stft_cov_pick_chunks(pl, B * groups, T), pl->d_stft_ws,
                     maxabs_bits, stream);
  return done(e, run_what);
}

// Runs run(scratch) with `bytes` of scratch allocated on the caller's stream (cudaMallocAsync /
// cudaFreeAsync), so that the plan-free entry points share no memory between calls on different
// streams or devices.  A failed free is reported only when the run itself succeeded.
template <class Run>
static int with_scratch(size_t bytes, void* stream, const char* alloc_what, const char* run_what, Run run) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* ws = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&ws), bytes, st);
  if (e != cudaSuccess) return cuda_fail(e, alloc_what);
  e = run(ws);
  const cudaError_t ef = cudaFreeAsync(ws, st);
  if (e == cudaSuccess) e = ef;
  return done(e, run_what);
}

// with_scratch with the host table `table` copied to its head on the stream (256-byte aligned): runs
// run(device table, the `bytes` of scratch after it)
template <class Run>
static int with_host_table(const std::vector<int>& table, size_t bytes, void* stream, const char* alloc_what,
                           const char* run_what, Run run) {
  const size_t table_bytes = up256(sizeof(int) * table.size());
  return with_scratch(table_bytes + bytes, stream, alloc_what, run_what, [&](char* ws) {
    const cudaError_t e = cudaMemcpyAsync(ws, table.data(), sizeof(int) * table.size(), cudaMemcpyHostToDevice,
                                          static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? run(reinterpret_cast<const int*>(ws), ws + table_bytes) : e;
  });
}

// with_scratch holding the bin-major copy X [B][T][C][P = bin_pitch(F)] of a [B][C][F][T] STFT, then
// (256-byte aligned) `bytes` of workspace: runs run(X, P, workspace) once the copy is enqueued
template <class Run>
static int with_bin_major(const void* stft, int B, int C, int F, int T, size_t bytes, void* stream,
                          const char* alloc_what, const char* run_what, Run run) {
  const int P = bin_pitch(F);
  const size_t x_bytes = sizeof(float2) * (size_t)B * T * C * P;
  return with_scratch(x_bytes + bytes + 256, stream, alloc_what, run_what, [&](char* ws) {
    float2* X = reinterpret_cast<float2*>(ws);
    const cudaError_t e = run_bcft_to_spill(static_cast<const float2*>(stft), B, C, F, T, P, X, stream);
    return e == cudaSuccess ? run(X, P, reinterpret_cast<double*>(ws + up256(x_bytes))) : e;
  });
}

}  // namespace setk

using namespace setk;

extern "C" {

int setk_version(void) { return SETK_VERSION; }
#ifdef SETK_EMU
// present only in the CPU test tier's build (tests/emu): lets the Python layer
// tell the two apart so that the product library never sees host pointers
int setk_emulated(void) { return 1; }
#endif
const char* setk_last_error_string(void) { return g_err; }
int64_t setk_launch_count(void) { return (int64_t)g_launch_count.load(); }

int setk_plan_create(const setk_config_t* cfg, setk_plan_t** plan_out) {
  if (!cfg || !plan_out) return fail(SETK_EINVAL, "setk_plan_create: null argument");
  *plan_out = nullptr;
  if (cfg->num_channels < 1 || cfg->num_channels > SETK_MAX_CHANNELS)
    return fail(SETK_EINVAL, "num_channels %d outside [1, %d]", cfg->num_channels, SETK_MAX_CHANNELS);
  if (cfg->frame_len < 1 || cfg->frame_hop < 1)
    return fail(SETK_EINVAL, "frame_len %d / frame_hop %d must be positive", cfg->frame_len, cfg->frame_hop);
  if (cfg->n_fft < cfg->frame_len)
    return fail(SETK_EINVAL, "n_fft %d smaller than frame_len %d", cfg->n_fft, cfg->frame_len);
  // powers of two run the FFT kernels; any other EVEN size (--round-power-of-two false,
  // utils.py:115) the direct-DFT path of the generic kernels (librosa's istft itself derives
  // n_fft = 2 (F - 1), i.e. it only round-trips even sizes)
  if (cfg->n_fft < 32 || cfg->n_fft > 4096 || (cfg->n_fft & 1))
    return fail(SETK_EUNSUPPORTED, "n_fft %d: only even sizes in [32, 4096] are supported", cfg->n_fft);
  if (!cfg->window_host) return fail(SETK_EINVAL, "window_host is null");
  if (cfg->max_batch < 1 || cfg->max_samples < 1)
    return fail(SETK_EINVAL, "max_batch / max_samples must be positive");

  setk_plan* pl = static_cast<setk_plan*>(calloc(1, sizeof(setk_plan)));
  if (!pl) return fail(SETK_ENOMEM, "out of host memory");
  pl->cfg = *cfg;
  pl->cfg.window_host = nullptr;
  Geometry& g = pl->geo;
  g.C = cfg->num_channels;
  g.n_fft = cfg->n_fft;
  g.log2n = 0;
  while ((1 << g.log2n) < g.n_fft) ++g.log2n;
  if (!is_pow2(g.n_fft)) g.log2n = -1;     // marks the direct-DFT route
  g.hop = cfg->frame_hop;
  g.pad = cfg->center ? g.n_fft / 2 : 0;
  g.F = g.n_fft / 2 + 1;

  // librosa.util.pad_center: left pad (n_fft - frame_len) // 2
  std::vector<float> win(g.n_fft, 0.f), wsq(g.n_fft, 0.f);
  const int lpad = (g.n_fft - cfg->frame_len) / 2;
  for (int i = 0; i < cfg->frame_len; ++i) {
    const double w = cfg->window_host[i];
    win[lpad + i] = (float)w;
    wsq[lpad + i] = (float)(w * w);
  }
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&pl->d_window), sizeof(float) * g.n_fft);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&pl->d_wsq), sizeof(float) * g.n_fft);
  if (e == cudaSuccess) e = cudaMemcpy(pl->d_window, win.data(), sizeof(float) * g.n_fft, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(pl->d_wsq, wsq.data(), sizeof(float) * g.n_fft, cudaMemcpyHostToDevice);
  int dev = 0;
  if (e == cudaSuccess) e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&pl->sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) {
    setk_plan_destroy(pl);
    return cuda_fail(e, "setk_plan_create");
  }
  *plan_out = pl;
  return SETK_OK;
}

int setk_plan_destroy(setk_plan_t* pl) {
  if (!pl) return SETK_OK;
  if (pl->d_window) cudaFree(pl->d_window);
  if (pl->d_wsq) cudaFree(pl->d_wsq);
  if (pl->d_partials) cudaFree(pl->d_partials);
  if (pl->d_wave_ws) cudaFree(pl->d_wave_ws);
  if (pl->d_stft_ws) cudaFree(pl->d_stft_ws);
  if (pl->d_enh_ws) cudaFree(pl->d_enh_ws);
  if (pl->d_frames_ws) cudaFree(pl->d_frames_ws);
  if (pl->d_cgmm_ws) cudaFree(pl->d_cgmm_ws);
  if (pl->d_peak) cudaFree(pl->d_peak);
  if (pl->d_tile_prefix) cudaFree(pl->d_tile_prefix);
  if (pl->d_mel) cudaFree(pl->d_mel);
  free(pl);
  return SETK_OK;
}

int setk_num_frames(const setk_plan_t* pl, int32_t n_samples) {
  if (!pl) return fail(SETK_EINVAL, "null plan");
  const int T = frames_of(n_samples, pl->geo.n_fft, pl->geo.hop, pl->geo.pad);
  return T > 0 ? T : -1;
}

int setk_istft_length(const setk_plan_t* pl, int32_t num_frames) {
  if (!pl) return fail(SETK_EINVAL, "null plan");
  if (num_frames < 1) return -1;
  return pl->geo.hop * (num_frames - 1) + pl->geo.n_fft - 2 * pl->geo.pad;
}

int setk_num_bins(const setk_plan_t* pl) { return pl ? pl->geo.F : fail(SETK_EINVAL, "null plan"); }

static int check_batch(const setk_plan_t* pl, int B, int N, const char* who) {
  if (!pl) return fail(SETK_EINVAL, "%s: null plan", who);
  if (B < 1 || B > pl->cfg.max_batch) return fail(SETK_ESHAPE, "%s: batch %d outside [1, max_batch=%d]", who, B, pl->cfg.max_batch);
  if (N < 1 || N > pl->cfg.max_samples) return fail(SETK_ESHAPE, "%s: N=%d outside [1, max_samples=%d]", who, N, pl->cfg.max_samples);
  if (frames_of(N, pl->geo.n_fft, pl->geo.hop, pl->geo.pad) < 1)
    return fail(SETK_ESHAPE, "%s: N=%d too short for n_fft=%d", who, N, pl->geo.n_fft);
  return SETK_OK;
}

int setk_stft(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
              void* stft_out, void* stream) {
  int rc = check_batch(pl, B, N, "setk_stft");
  if (rc) return rc;
  if (!audio || !stft_out) return fail(SETK_EINVAL, "setk_stft: null buffer");
  const Geometry& g = pl->geo;
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  cudaError_t e;
  if (stft_spill_supported(g) && (long long)B * g.C <= 65535) {
    // tile STFT into the bin-major workspace, then one transposing copy
    rc = stft_to_bin_major(pl, audio, n_samples, B, N, T, nullptr, stream, "setk_stft(workspace)", "setk_stft");
    if (rc) return rc;
    e = run_spill_to_bcft(pl, pl->d_stft_ws, B, T, static_cast<float2*>(stft_out), stream);
  } else {
    e = run_stft_generic(pl, audio, n_samples, B, N, T, static_cast<float2*>(stft_out), stream);
  }
  return done(e, "setk_stft");
}

int setk_plan_set_mel(setk_plan_t* pl, int32_t num_mel, const float* mel_host) {
  if (!pl) return fail(SETK_EINVAL, "setk_plan_set_mel: null plan");
  if (num_mel < 0 || num_mel > 1024) return fail(SETK_EINVAL, "setk_plan_set_mel: num_mel %d outside [0, 1024]", num_mel);
  if (num_mel > 0 && !mel_host) return fail(SETK_EINVAL, "setk_plan_set_mel: null mel_host");
  const int F = pl->geo.F;
  // [num_mel][4] {first bin, bins, weight offset, 0}, then the weights of every band
  std::vector<int> band(4 * (size_t)num_mel, 0);
  std::vector<float> w;
  for (int m = 0; m < num_mel; ++m) {
    int lo = -1, hi = -1;
    for (int k = 0; k < F; ++k) {
      const float v = mel_host[(size_t)m * F + k];
      if (!std::isfinite(v) || v < 0.f)
        return fail(SETK_EINVAL, "setk_plan_set_mel: weight [%d][%d] = %g is not finite and >= 0", m, k, (double)v);
      if (v > 0.f) { if (lo < 0) lo = k; hi = k; }
    }
    band[4 * m] = lo < 0 ? 0 : lo;
    band[4 * m + 1] = lo < 0 ? 0 : hi - lo + 1;
    band[4 * m + 2] = (int)w.size();
    for (int k = lo; lo >= 0 && k <= hi; ++k) w.push_back(mel_host[(size_t)m * F + k]);
  }
  if (pl->d_mel) cudaFree(pl->d_mel);
  pl->d_mel = nullptr; pl->num_mel = 0; pl->mel_weights = 0;
  if (num_mel == 0) return SETK_OK;
  const size_t band_bytes = sizeof(int) * band.size();
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&pl->d_mel), band_bytes + sizeof(float) * w.size());
  if (e == cudaSuccess) e = cudaMemcpy(pl->d_mel, band.data(), band_bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && !w.empty())
    e = cudaMemcpy(pl->d_mel + band.size(), w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (pl->d_mel) cudaFree(pl->d_mel);
    pl->d_mel = nullptr;
    return cuda_fail(e, "setk_plan_set_mel");
  }
  pl->num_mel = num_mel;
  pl->mel_weights = (int)w.size();
  return SETK_OK;
}

int setk_spectral_feats(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                        uint32_t flags, float sample_scale, float* out, void* stream) {
  int rc = check_batch(pl, B, N, "setk_spectral_feats");
  if (rc) return rc;
  if (!audio || !out) return fail(SETK_EINVAL, "setk_spectral_feats: null buffer");
  if (flags & ~(SETK_FEAT_POW | SETK_FEAT_MEL | SETK_FEAT_LOG))
    return fail(SETK_EINVAL, "setk_spectral_feats: unknown flags 0x%x", flags);
  if ((flags & SETK_FEAT_MEL) && !pl->d_mel)
    return fail(SETK_EINVAL, "setk_spectral_feats: SETK_FEAT_MEL without a mel table (setk_plan_set_mel)");
  if (!std::isfinite(sample_scale) || !(sample_scale > 0.f))
    return fail(SETK_EINVAL, "setk_spectral_feats: sample_scale %g must be finite and > 0", (double)sample_scale);
  if (B > 65535) return fail(SETK_ESHAPE, "setk_spectral_feats: batch %d > 65535", B);
  const Geometry& g = pl->geo;
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  if (feats_fused_supported(g))
    return done(run_feats_fused(pl, audio, n_samples, B, N, T, flags, sample_scale, out, stream),
                "setk_spectral_feats");
  cudaError_t e = ensure(&pl->d_stft_ws, &pl->stft_ws_bytes, sizeof(float2) * (size_t)B * g.C * g.F * T);
  if (e != cudaSuccess) return cuda_fail(e, "setk_spectral_feats(workspace)");
  e = run_stft_generic(pl, audio, n_samples, B, N, T, pl->d_stft_ws, stream);
  if (e == cudaSuccess) e = run_feats_stft(pl, pl->d_stft_ws, n_samples, B, N, T, flags, sample_scale, out, stream);
  return done(e, "setk_spectral_feats");
}

int setk_cov(const void* stft, const float* mask, uint32_t flags, int32_t B, int32_t C, int32_t F,
             int32_t T, void* R, void* stream) {
  if (!stft || !mask || !R) return fail(SETK_EINVAL, "setk_cov: null buffer");
  if (B < 1 || F < 1 || T < 1 || C < 1 || C > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_cov: bad shape B=%d C=%d F=%d T=%d", B, C, F, T);
  if (B > 65535) return fail(SETK_ESHAPE, "setk_cov: batch %d > 65535", B);
  cudaError_t e = run_cov_generic(static_cast<const float2*>(stft), mask, flags, B, C, F, T,
                                  static_cast<float2*>(R), stream);
  return done(e, "setk_cov");
}

int setk_stft_cov(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                  const float* mask_s, const float* mask_n, uint32_t flags, void* Rs, void* Rn,
                  float* maxabs, void* stream) {
  int rc = check_batch(pl, B, N, "setk_stft_cov");
  if (rc) return rc;
  if (!audio || !mask_s || !Rs || !Rn) return fail(SETK_EINVAL, "setk_stft_cov: null buffer");
  const Geometry& g = pl->geo;
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  cudaError_t e = ensure(&pl->d_peak, &pl->peak_bytes, sizeof(unsigned) * 2 * (size_t)pl->cfg.max_batch);
  if (e != cudaSuccess) return cuda_fail(e, "setk_stft_cov(workspace)");
  unsigned* maxabs_bits = nullptr;
  if (maxabs) {
    maxabs_bits = pl->d_peak + pl->cfg.max_batch;   // second half: audio max|x|
    e = cudaMemsetAsync(maxabs_bits, 0, sizeof(unsigned) * B, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return cuda_fail(e, "setk_stft_cov(memset)");
  }
  if (stft_cov_fused_supported(g)) {
    e = ensure(&pl->d_partials, &pl->partials_bytes, stft_cov_partial_bytes(pl, B, T));
    if (e == cudaSuccess && n_samples)
      e = ensure(&pl->d_tile_prefix, &pl->tile_prefix_bytes, sizeof(int) * ((size_t)pl->cfg.max_batch + 1));
    if (e != cudaSuccess) return cuda_fail(e, "setk_stft_cov(workspace)");
    e = run_stft_cov_fused(pl, audio, n_samples, B, N, T, mask_s, mask_n, flags, pl->d_tile_prefix,
                           pl->d_partials, maxabs_bits, static_cast<float2*>(Rs),
                           static_cast<float2*>(Rn), maxabs, stream);
    return done(e, "setk_stft_cov");
  }
  if (stft_spill_supported(g)) {
    // many-channel route (C > 4 at n_fft = 512, any C at n_fft = 1024): fast STFT
    // into a bin-major workspace, then a streaming covariance kernel (stft_spill.cu)
    // >= 16 short fp32 runs per utterance, combined in double by the finalize kernel
    const int chunks = cov_spill_chunks(pl, B, T);
    e = ensure(&pl->d_partials, &pl->partials_bytes, cov_spill_partial_bytes(g, B, chunks));
    if (e != cudaSuccess) return cuda_fail(e, "setk_stft_cov(workspace)");
    rc = stft_to_bin_major(pl, audio, n_samples, B, N, T, maxabs_bits, stream, "setk_stft_cov(workspace)",
                           "setk_stft_cov(spill)");
    if (rc) return rc;
    e = run_cov_spill(pl, pl->d_stft_ws, mask_s, mask_n, flags, n_samples, B, N, T, chunks, pl->d_partials,
                      static_cast<float2*>(Rs), static_cast<float2*>(Rn), stream);
    if (e == cudaSuccess && maxabs) e = run_bits_to_float(maxabs_bits, B, maxabs, stream);
    return done(e, "setk_stft_cov(spill)");
  }
  // shape-generic route: explicit STFT in workspace, then two covariance passes
  const size_t want = sizeof(float2) * (size_t)B * g.C * g.F * T;
  e = ensure(&pl->d_stft_ws, &pl->stft_ws_bytes, want);
  if (e != cudaSuccess) return cuda_fail(e, "setk_stft_cov(workspace)");
  e = run_stft_generic(pl, audio, n_samples, B, N, T, pl->d_stft_ws, stream);
  if (e == cudaSuccess)
    e = run_cov_generic(pl->d_stft_ws, mask_s, flags, B, g.C, g.F, T, static_cast<float2*>(Rs), stream);
  if (e == cudaSuccess) {
    if (mask_n)
      e = run_cov_generic(pl->d_stft_ws, mask_n, flags & ~SETK_F_CLIP_MASK, B, g.C, g.F, T,
                          static_cast<float2*>(Rn), stream);
    else
      e = run_cov_generic(pl->d_stft_ws, mask_s, flags | SETK_F_ONE_MINUS_INTERNAL, B, g.C, g.F, T,
                          static_cast<float2*>(Rn), stream);
  }
  if (e == cudaSuccess && maxabs)
    e = maxabs_generic(audio, n_samples, B, g.C, N, maxabs_bits, maxabs, stream);
  return done(e, "setk_stft_cov(generic)");
}

int setk_weights(int32_t kind, double beta, int32_t ref_channel, int32_t rank1, int32_t ban,
                 const void* Rs, const void* Rn, const void* Ry, int32_t r_dtype, int32_t B, int32_t F,
                 int32_t C, void* w, int32_t w_dtype, uint32_t* status, int32_t* ref_used, void* stream) {
  if (!Rs || !w || !status) return fail(SETK_EINVAL, "setk_weights: null buffer");
  if (B < 1 || F < 1 || C < 1 || C > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_weights: bad shape B=%d F=%d C=%d", B, F, C);
  if (kind < SETK_BF_MVDR || kind > SETK_BF_PEVD) return fail(SETK_EINVAL, "setk_weights: unknown kind %d", kind);
  if ((r_dtype != SETK_C64 && r_dtype != SETK_C128) || (w_dtype != SETK_C64 && w_dtype != SETK_C128))
    return fail(SETK_EINVAL, "setk_weights: bad dtype");
  const bool need_rn = kind == SETK_BF_MVDR || kind == SETK_BF_MPDR_WHITEN || kind == SETK_BF_GEVD ||
                       kind == SETK_BF_PMWF;
  if (need_rn && !Rn) return fail(SETK_EINVAL, "setk_weights: Rn required for kind %d", kind);
  if ((kind == SETK_BF_MPDR || kind == SETK_BF_MPDR_WHITEN) && !Ry)
    return fail(SETK_EINVAL, "setk_weights: Ry required for MPDR");
  if (ban && !Rn) return fail(SETK_EINVAL, "setk_weights: BAN needs Rn");
  if (rank1 < SETK_RANK1_NONE || rank1 > SETK_RANK1_GEV) return fail(SETK_EINVAL, "setk_weights: bad rank1 %d", rank1);
  cudaError_t e = weights_run(kind, beta, ref_channel, rank1, ban, Rs, Rn, Ry, r_dtype, B, F, C, w, w_dtype,
                              status, ref_used, stream);
  return done(e, "setk_weights");
}

int setk_ban(const void* w_in, const void* Rn, int32_t dtype, int32_t B, int32_t F, int32_t C,
             void* w_out, void* stream) {
  if (!w_in || !Rn || !w_out) return fail(SETK_EINVAL, "setk_ban: null buffer");
  if (B < 1 || F < 1 || C < 1 || C > SETK_MAX_CHANNELS) return fail(SETK_ESHAPE, "setk_ban: bad shape");
  if (dtype != SETK_C64 && dtype != SETK_C128) return fail(SETK_EINVAL, "setk_ban: bad dtype");
  cudaError_t e = post_run(0, w_in, Rn, dtype, B, F, C, w_out, nullptr, stream);
  return done(e, "setk_ban");
}

int setk_rank1(const void* Rs, const void* Rn, int32_t dtype, int32_t B, int32_t F, int32_t C,
               void* R1_out, uint32_t* status, void* stream) {
  if (!Rs || !R1_out) return fail(SETK_EINVAL, "setk_rank1: null buffer");
  if (B < 1 || F < 1 || C < 1 || C > SETK_MAX_CHANNELS) return fail(SETK_ESHAPE, "setk_rank1: bad shape");
  if (dtype != SETK_C64 && dtype != SETK_C128) return fail(SETK_EINVAL, "setk_rank1: bad dtype");
  cudaError_t e = post_run(1, Rs, Rn, dtype, B, F, C, R1_out, status, stream);
  return done(e, "setk_rank1");
}

int setk_apply(const void* stft, const void* w, int32_t w_dtype, const float* post_mask, int32_t B,
               int32_t C, int32_t F, int32_t T, void* enh, void* stream) {
  if (!stft || !w || !enh) return fail(SETK_EINVAL, "setk_apply: null buffer");
  if (B < 1 || F < 1 || T < 1 || C < 1 || C > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_apply: bad shape B=%d C=%d F=%d T=%d", B, C, F, T);
  cudaError_t e = run_apply_generic(static_cast<const float2*>(stft), w, w_dtype, post_mask, B, C, F, T,
                                    static_cast<float2*>(enh), stream);
  return done(e, "setk_apply");
}

int setk_istft(setk_plan_t* pl, const void* enh, int32_t B, int32_t T, int32_t n_out, const float* norm,
               float* wave, void* stream) {
  if (!pl || !enh || !wave) return fail(SETK_EINVAL, "setk_istft: null argument");
  if (B < 1 || B > pl->cfg.max_batch || T < 1 || n_out < 1)
    return fail(SETK_ESHAPE, "setk_istft: bad shape B=%d T=%d n_out=%d", B, T, n_out);
  const Geometry& g = pl->geo;
  const int T_used = imin(T, istft_frame_cap(g, n_out));
  cudaError_t e = ensure(&pl->d_frames_ws, &pl->frames_ws_bytes, sizeof(float) * (size_t)B * T_used * g.n_fft);
  if (e == cudaSuccess) e = ensure(&pl->d_peak, &pl->peak_bytes, sizeof(unsigned) * 2 * (size_t)pl->cfg.max_batch);
  if (e != cudaSuccess) return cuda_fail(e, "setk_istft(workspace)");
  unsigned* peak = norm ? pl->d_peak : nullptr;
  if (peak) {
    e = cudaMemsetAsync(peak, 0, sizeof(unsigned) * B, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return cuda_fail(e, "setk_istft(memset)");
  }
  e = run_istft_generic(pl, static_cast<const float2*>(enh), B, T, T_used, n_out, nullptr, pl->d_frames_ws,
                        wave, peak, stream);
  if (e == cudaSuccess && norm) e = run_peak_scale(wave, B, n_out, norm, peak, stream);
  return done(e, "setk_istft");
}

// wave != null: float output (+ norm rescale in place); pcm != null: the float wave goes to a plan
// workspace and the rescale pass writes PCM-16 instead
static int apply_istft_impl(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B,
                            int32_t N, const void* w, int32_t w_dtype, const float* post_mask,
                            int32_t n_out, const float* norm, float* wave, int16_t* pcm, void* stream) {
  int rc = check_batch(pl, B, N, "setk_apply_istft");
  if (rc) return rc;
  if (!audio || !w || (!wave && !pcm)) return fail(SETK_EINVAL, "setk_apply_istft: null buffer");
  if (n_out < 1) return fail(SETK_ESHAPE, "setk_apply_istft: n_out=%d", n_out);
  const Geometry& g = pl->geo;
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  const int T_used = imin(T, istft_frame_cap(g, n_out));   // the workspace routes' iSTFT
  cudaError_t e = ensure(&pl->d_peak, &pl->peak_bytes, sizeof(unsigned) * 2 * (size_t)pl->cfg.max_batch);
  if (e == cudaSuccess && pcm) {
    e = ensure(&pl->d_wave_ws, &pl->wave_ws_bytes, sizeof(float) * (size_t)B * n_out);
    wave = pl->d_wave_ws;
  }
  if (e != cudaSuccess) return cuda_fail(e, "setk_apply_istft(workspace)");
  unsigned* peak = norm ? pl->d_peak : nullptr;
  if (peak) {
    e = cudaMemsetAsync(peak, 0, sizeof(unsigned) * B, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return cuda_fail(e, "setk_apply_istft(memset)");
  }
  if (apply_istft_fused_supported(g)) {
    if (n_samples)
      e = ensure(&pl->d_tile_prefix, &pl->tile_prefix_bytes, sizeof(int) * ((size_t)pl->cfg.max_batch + 1));
    if (e != cudaSuccess) return cuda_fail(e, "setk_apply_istft(workspace)");
    e = run_apply_istft_fused(pl, audio, n_samples, B, N, T, w, w_dtype, post_mask, n_out,
                              pl->d_tile_prefix, wave, peak, stream);
  } else if (stft_spill_supported(g)) {
    // tile STFT into the bin-major workspace, y = w^H x over it, then the
    // frame-wise inverse FFT + overlap-add reading Y[b][t][f] in place
    const long long pitch = bin_pitch(g.F);
    e = ensure(&pl->d_enh_ws, &pl->enh_ws_bytes, apply_spill_bytes(g, B, T));
    if (e == cudaSuccess)
      e = ensure(&pl->d_frames_ws, &pl->frames_ws_bytes, sizeof(float) * (size_t)B * T_used * g.n_fft);
    if (e != cudaSuccess) return cuda_fail(e, "setk_apply_istft");
    rc = stft_to_bin_major(pl, audio, n_samples, B, N, T, nullptr, stream, "setk_apply_istft", "setk_apply_istft");
    if (rc) return rc;
    e = run_apply_spill(pl, pl->d_stft_ws, w, w_dtype, post_mask, B, T, pl->d_enh_ws, stream);
    if (e == cudaSuccess)
      e = run_istft_strided(pl, pl->d_enh_ws, (long long)T * pitch, 1, pitch, B, T_used, n_out, n_samples,
                            pl->d_frames_ws, wave, peak, stream);
  } else {
    e = ensure(&pl->d_stft_ws, &pl->stft_ws_bytes, sizeof(float2) * (size_t)B * g.C * g.F * T);
    if (e == cudaSuccess) e = ensure(&pl->d_enh_ws, &pl->enh_ws_bytes, sizeof(float2) * (size_t)B * g.F * T);
    if (e == cudaSuccess)
      e = ensure(&pl->d_frames_ws, &pl->frames_ws_bytes, sizeof(float) * (size_t)B * T_used * g.n_fft);
    if (e == cudaSuccess) e = run_stft_generic(pl, audio, n_samples, B, N, T, pl->d_stft_ws, stream);
    if (e == cudaSuccess)
      e = run_apply_generic(pl->d_stft_ws, w, w_dtype, post_mask, B, g.C, g.F, T, pl->d_enh_ws, stream);
    if (e == cudaSuccess)
      e = run_istft_generic(pl, pl->d_enh_ws, B, T, T_used, n_out, n_samples, pl->d_frames_ws, wave, peak,
                            stream);
  }
  if (e == cudaSuccess && pcm) e = run_peak_scale_pcm16(wave, B, n_out, norm, peak, pcm, stream);
  else if (e == cudaSuccess && norm) e = run_peak_scale(wave, B, n_out, norm, peak, stream);
  return done(e, "setk_apply_istft");
}

int setk_apply_istft(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                     const void* w, int32_t w_dtype, const float* post_mask, int32_t n_out,
                     const float* norm, float* wave, void* stream) {
  if (!wave) return fail(SETK_EINVAL, "setk_apply_istft: null buffer");
  return apply_istft_impl(pl, audio, n_samples, B, N, w, w_dtype, post_mask, n_out, norm, wave, nullptr,
                          stream);
}

int setk_apply_istft_pcm16(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B,
                           int32_t N, const void* w, int32_t w_dtype, const float* post_mask,
                           int32_t n_out, const float* norm, int16_t* pcm, void* stream) {
  if (!pcm) return fail(SETK_EINVAL, "setk_apply_istft_pcm16: null buffer");
  return apply_istft_impl(pl, audio, n_samples, B, N, w, w_dtype, post_mask, n_out, norm, nullptr, pcm,
                          stream);
}

int setk_cgmm_masks(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                    int32_t num_classes, int32_t num_iters, const float* init_gamma, int32_t update_alpha,
                    float* masks, uint32_t* status, void* stream) {
  int rc = check_batch(pl, B, N, "setk_cgmm_masks");
  if (rc) return rc;
  if (!audio || !masks) return fail(SETK_EINVAL, "setk_cgmm_masks: null buffer");
  if (num_classes < 2 || num_classes > 4)
    return fail(SETK_EINVAL, "setk_cgmm_masks: num_classes %d outside 2..4", num_classes);
  if (!init_gamma && num_classes != 2)
    return fail(SETK_EINVAL, "setk_cgmm_masks: %d classes need init_gamma (the reference's start is random)",
                num_classes);
  if (num_iters < 0) return fail(SETK_EINVAL, "setk_cgmm_masks: num_iters %d", num_iters);
  const Geometry& g = pl->geo;
  if (!stft_spill_supported(g))
    return fail(SETK_EUNSUPPORTED, "setk_cgmm_masks: needs n_fft 512 or 1024 (got %d, hop %d)", g.n_fft, g.hop);
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  if (T < 1) return fail(SETK_ESHAPE, "setk_cgmm_masks: no frame in %d samples", N);
  const int P = bin_pitch(g.F);
  CgCtx ctx;
  ctx.geo = g; ctx.sm_count = pl->sm_count;
  cudaError_t e = ensure(&pl->d_cgmm_ws, &pl->cgmm_ws_bytes, cgmm_workspace_bytes(&ctx, B, T, num_classes, P));
  if (e != cudaSuccess) return cuda_fail(e, "setk_cgmm_masks(workspace)");
  rc = stft_to_bin_major(pl, audio, n_samples, B, N, T, nullptr, stream, "setk_cgmm_masks(workspace)",
                         "setk_cgmm_masks");
  if (rc) return rc;
  e = run_cgmm(&ctx, pl->d_stft_ws, P, pl->d_cgmm_ws, n_samples, B, N, T, num_classes, num_iters, init_gamma,
               update_alpha, masks, status, stream);
  return done(e, "setk_cgmm_masks");
}

int setk_cgmm_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t num_classes,
                   int32_t num_iters, const float* init_gamma, int32_t update_alpha, float* masks,
                   uint32_t* status, void* stream) {
  if (!stft || !masks) return fail(SETK_EINVAL, "setk_cgmm_stft: null buffer");
  if (B < 1 || B > 65535 || F < 1 || T < 1 || C < 1 || C > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_cgmm_stft: bad shape B=%d C=%d F=%d T=%d", B, C, F, T);
  if (num_classes < 2 || num_classes > 4)
    return fail(SETK_EINVAL, "setk_cgmm_stft: num_classes %d outside 2..4", num_classes);
  if (!init_gamma && num_classes != 2)
    return fail(SETK_EINVAL, "setk_cgmm_stft: %d classes need init_gamma (the reference's start is random)",
                num_classes);
  if (num_iters < 0) return fail(SETK_EINVAL, "setk_cgmm_stft: num_iters %d", num_iters);
  CgCtx ctx;
  // frames are given, not derived from samples: a geometry whose frame count never limits
  ctx.geo.C = C; ctx.geo.F = F; ctx.geo.n_fft = 2; ctx.geo.log2n = 1; ctx.geo.hop = 1; ctx.geo.pad = 0;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx.sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return cuda_fail(e, "setk_cgmm_stft(device)");
  return with_bin_major(stft, B, C, F, T, cgmm_workspace_bytes(&ctx, B, T, num_classes, bin_pitch(F)), stream,
                        "setk_cgmm_stft(workspace)", "setk_cgmm_stft", [&](float2* X, int P, double* ws) {
    return run_cgmm(&ctx, X, P, ws, nullptr, B, /*N=*/T + 1, T, num_classes, num_iters, init_gamma, update_alpha,
                    masks, status, stream);
  });
}

// plan rows (iterations, lo, hi) of the permutation aligner: 0 <= lo < hi <= F, iterations >= 0;
// NULL or R = 0 (no alignment) only when `required` is false
static int check_permu_plan(const char* who, const int32_t* plan, int R, int F, bool required) {
  if (!plan || R == 0) return required ? fail(SETK_EINVAL, "%s: empty alignment plan", who) : SETK_OK;
  if (R < 0 || R > SETK_PERMU_MAX_ROWS)
    return fail(SETK_EINVAL, "%s: %d plan rows outside [1, %d]", who, R, SETK_PERMU_MAX_ROWS);
  for (int r = 0; r < R; ++r) {
    const int it = plan[3 * r], lo = plan[3 * r + 1], hi = plan[3 * r + 2];
    if (it < 0 || lo < 0 || lo >= hi || hi > F)
      return fail(SETK_EINVAL, "%s: plan row %d (%d, %d, %d) needs iterations >= 0 and 0 <= lo < hi <= F = %d",
                  who, r, it, lo, hi, F);
  }
  return SETK_OK;
}

// the checks every CACGMM / alignment entry point shares: class count, start, plan rows over F bins
static int check_cacgmm(const char* who, int C, int K, int num_iters, const double* init_gamma, int cgmm_init,
                        const int32_t* plan, int R, int F) {
  if (K < 2 || K > 4) return fail(SETK_EINVAL, "%s: num_classes %d outside 2..4", who, K);
  if (C < 2) return fail(SETK_EINVAL, "%s: %d channel(s), the CACGMM needs 2 or more", who, C);
  if (num_iters < 0) return fail(SETK_EINVAL, "%s: num_iters %d", who, num_iters);
  if (!init_gamma && !(cgmm_init && K == 2))
    return fail(SETK_EINVAL, "%s: a NULL init_gamma needs cgmm_init with 2 classes", who);
  return check_permu_plan(who, plan, R, F, false);
}

int setk_cacgmm_masks(setk_plan_t* pl, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                      int32_t num_classes, int32_t num_iters, const double* init_gamma, int32_t cgmm_init,
                      int32_t update_alpha, const int32_t* permu_plan, int32_t R, float* masks, uint32_t* status,
                      void* stream) {
  int rc = check_batch(pl, B, N, "setk_cacgmm_masks");
  if (rc) return rc;
  if (!audio || !masks) return fail(SETK_EINVAL, "setk_cacgmm_masks: null buffer");
  const Geometry& g = pl->geo;
  rc = check_cacgmm("setk_cacgmm_masks", g.C, num_classes, num_iters, init_gamma, cgmm_init, permu_plan, R, g.F);
  if (rc) return rc;
  if (!stft_spill_supported(g))
    return fail(SETK_EUNSUPPORTED, "setk_cacgmm_masks: needs n_fft 512 or 1024 (got %d, hop %d)", g.n_fft, g.hop);
  const int T = frames_of(N, g.n_fft, g.hop, g.pad);
  if (T < 1) return fail(SETK_ESHAPE, "setk_cacgmm_masks: no frame in %d samples", N);
  if (permu_plan && R > 0 && permu_scratch_bytes(B, num_classes, T, g.F) < 0)
    return fail(SETK_EUNSUPPORTED, "setk_cacgmm_masks: %d bins exceed the aligner's shared memory", g.F);
  const int P = bin_pitch(g.F);
  CgCtx ctx;
  ctx.geo = g; ctx.sm_count = pl->sm_count;
  cudaError_t e = ensure(&pl->d_cgmm_ws, &pl->cgmm_ws_bytes, cacgmm_workspace_bytes(&ctx, B, T, num_classes, P));
  if (e != cudaSuccess) return cuda_fail(e, "setk_cacgmm_masks(workspace)");
  rc = stft_to_bin_major(pl, audio, n_samples, B, N, T, nullptr, stream, "setk_cacgmm_masks(workspace)",
                         "setk_cacgmm_masks");
  if (rc) return rc;
  e = run_cacgmm(&ctx, pl->d_stft_ws, P, pl->d_cgmm_ws, n_samples, B, N, T, num_classes, num_iters, init_gamma,
                 cgmm_init, update_alpha, permu_plan, permu_plan ? R : 0, masks, status, stream);
  return done(e, "setk_cacgmm_masks");
}

int setk_cacgmm_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t num_classes,
                     int32_t num_iters, const double* init_gamma, int32_t cgmm_init, int32_t update_alpha,
                     const int32_t* permu_plan, int32_t R, float* masks, uint32_t* status, void* stream) {
  if (!stft || !masks) return fail(SETK_EINVAL, "setk_cacgmm_stft: null buffer");
  if (B < 1 || B > 65535 || F < 1 || T < 1 || C < 1 || C > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_cacgmm_stft: bad shape B=%d C=%d F=%d T=%d", B, C, F, T);
  int rc = check_cacgmm("setk_cacgmm_stft", C, num_classes, num_iters, init_gamma, cgmm_init, permu_plan, R, F);
  if (rc) return rc;
  if (permu_plan && R > 0 && permu_scratch_bytes(B, num_classes, T, F) < 0)
    return fail(SETK_EUNSUPPORTED, "setk_cacgmm_stft: %d bins exceed the aligner's shared memory", F);
  CgCtx ctx;
  // frames are given, not derived from samples: a geometry whose frame count never limits
  ctx.geo.C = C; ctx.geo.F = F; ctx.geo.n_fft = 2; ctx.geo.log2n = 1; ctx.geo.hop = 1; ctx.geo.pad = 0;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx.sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return cuda_fail(e, "setk_cacgmm_stft(device)");
  return with_bin_major(stft, B, C, F, T, cacgmm_workspace_bytes(&ctx, B, T, num_classes, bin_pitch(F)), stream,
                        "setk_cacgmm_stft(workspace)", "setk_cacgmm_stft", [&](float2* X, int P, double* ws) {
    return run_cacgmm(&ctx, X, P, ws, nullptr, B, /*N=*/T + 1, T, num_classes, num_iters, init_gamma, cgmm_init,
                      update_alpha, permu_plan, permu_plan ? R : 0, masks, status, stream);
  });
}

int setk_permu_align(const double* masks, const int32_t* n_frames, int32_t B, int32_t K, int32_t T, int32_t F,
                     const int32_t* plan, int32_t R, float* out, int32_t* mapping, void* stream) {
  if (!masks || !out) return fail(SETK_EINVAL, "setk_permu_align: null buffer");
  if (K < 2 || K > 4) return fail(SETK_EINVAL, "setk_permu_align: num_classes %d outside 2..4", K);
  if (B < 1 || T < 1 || F < 1) return fail(SETK_EINVAL, "setk_permu_align: bad shape B=%d T=%d F=%d", B, T, F);
  int rc = check_permu_plan("setk_permu_align", plan, R, F, true);
  if (rc) return rc;
  const long long sb = permu_scratch_bytes(B, K, T, F);
  if (sb < 0) return fail(SETK_EUNSUPPORTED, "setk_permu_align: %d bins exceed the aligner's shared memory", F);
  PermuArgs a;
  a.m = masks; a.ld = F; a.n_frames = n_frames; a.n_samples = nullptr; a.N = T + 1;
  a.g.C = 1; a.g.F = F; a.g.n_fft = 2; a.g.log2n = 1; a.g.hop = 1; a.g.pad = 0;   // T frames unless n_frames
  a.K = K; a.T = T; a.F = F;
  return with_scratch((size_t)sb + 256, stream, "setk_permu_align(scratch)", "setk_permu_align", [&](char* ws) {
    return run_permu_align(a, B, plan, R, reinterpret_cast<double*>(ws), out, mapping, stream);
  });
}

static int wpe_entry(const char* who, const void* stft, const void* lambda_enh, int32_t B, int32_t C, int32_t F,
                     int32_t T, int32_t taps, int32_t delay, int32_t context, int32_t num_iters, void* out,
                     float* inv_lambda, uint32_t* status, void* stream) {
  if (!stft || !out) return fail(SETK_EINVAL, "%s: null buffer", who);
  if (B < 1 || F < 1 || T < 1 || C < 1 || C > SETK_MAX_CHANNELS || (long long)B * F > 2000000000LL)
    return fail(SETK_ESHAPE, "%s: bad shape B=%d C=%d F=%d T=%d", who, B, C, F, T);
  if (taps < 1 || delay < 0 || context < 0 || num_iters < 1)
    return fail(SETK_EINVAL, "%s: taps=%d delay=%d context=%d num_iters=%d", who, taps, delay, context,
                num_iters);
  if (!wpe_supported(C, T, taps, delay, context))
    return fail(SETK_EUNSUPPORTED, "%s: %d channels x %d taps (context %d) exceeds the kernels' "
                "shared-memory budget", who, C, taps, context);
  return with_bin_major(stft, B, C, F, T, wpe_workspace_bytes(B, C, F, taps), stream, who, who,
                        [&](float2* X, int P, double* ws) {
    return run_wpe(X, P, B, C, F, T, taps, delay, context, num_iters, ws, static_cast<float2*>(out), status,
                   static_cast<const float2*>(lambda_enh), inv_lambda, stream);
  });
}

int setk_wpe_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t taps, int32_t delay,
                  int32_t context, int32_t num_iters, void* out, uint32_t* status, void* stream) {
  return wpe_entry("setk_wpe_stft", stft, nullptr, B, C, F, T, taps, delay, context, num_iters, out, nullptr,
                   status, stream);
}

int setk_wpe_step(const void* stft, const void* lambda_enh, int32_t B, int32_t C, int32_t F, int32_t T,
                  int32_t taps, int32_t delay, int32_t context, void* out, float* inv_lambda,
                  uint32_t* status, void* stream) {
  return wpe_entry("setk_wpe_step", stft, lambda_enh, B, C, F, T, taps, delay, context, 1, out, inv_lambda,
                   status, stream);
}

int setk_float_to_pcm16(const float* wave, int64_t n, int16_t* pcm, void* stream) {
  if (!wave || !pcm || n < 0) return fail(SETK_EINVAL, "setk_float_to_pcm16: bad argument");
  if (n == 0) return SETK_OK;
  cudaError_t e = run_float_to_pcm16(wave, n, pcm, stream);
  return done(e, "setk_float_to_pcm16");
}

int setk_pcm16_to_float(const int16_t* pcm, int64_t n, float* wave, void* stream) {
  if (!wave || !pcm || n < 0) return fail(SETK_EINVAL, "setk_pcm16_to_float: bad argument");
  if (n == 0) return SETK_OK;
  cudaError_t e = run_pcm16_to_float(pcm, n, wave, stream);
  return done(e, "setk_pcm16_to_float");
}

int setk_cm_masks(const uint8_t* blobs, int64_t slot_bytes, int32_t B, int32_t T, int32_t F, float* out,
                  int32_t* status, void* stream) {
  if (!blobs || !out || !status || B < 0 || T < 0 || F < 0 || slot_bytes < 16 || (slot_bytes & 15) ||
      (reinterpret_cast<uintptr_t>(blobs) & 15))
    return fail(SETK_EINVAL, "setk_cm_masks: bad argument");
  cudaError_t e = run_cm_masks(blobs, slot_bytes, B, T, F, out, status, stream);
  return done(e, "setk_cm_masks");
}

// ---- spatial features (spatial.cu) ----
int setk_ipd(const void* si, const void* sj, int64_t rows, int32_t F, int32_t mode, float* out,
             void* stream) {
  if (!si || !sj || !out) return fail(SETK_EINVAL, "setk_ipd: null buffer");
  if (rows < 1 || F < 1) return fail(SETK_ESHAPE, "setk_ipd: rows=%lld F=%d", (long long)rows, F);
  if (mode < 0 || mode > 2) return fail(SETK_EINVAL, "setk_ipd: mode %d outside 0..2", mode);
  cudaError_t e = run_ipd(static_cast<const float2*>(si), static_cast<const float2*>(sj), rows, F, mode,
                          out, stream);
  return done(e, "setk_ipd");
}

int setk_directional_feats(const void* stft, const void* steer, int32_t steer_batched,
                           const int32_t* pairs, int32_t n_pairs, int32_t B, int32_t M, int32_t F,
                           int32_t T, double* out, void* stream) {
  if (!stft || !steer || !out) return fail(SETK_EINVAL, "setk_directional_feats: null buffer");
  if (B < 1 || F < 1 || T < 1 || M < 2 || M > SETK_MAX_CHANNELS)
    return fail(SETK_ESHAPE, "setk_directional_feats: bad shape B=%d M=%d F=%d T=%d", B, M, F, T);
  if (pairs && n_pairs < 1) return fail(SETK_EINVAL, "setk_directional_feats: empty pair list");
  cudaError_t e = run_dirfeat(static_cast<const float2*>(stft), static_cast<const double2*>(steer),
                              steer_batched, pairs, n_pairs, B, M, F, T, out, stream);
  return done(e, "setk_directional_feats");
}

int64_t setk_gcc_phat_work_doubles(int32_t T, int32_t F, int32_t D) {
  if (T < 1 || F < 1 || D < 1) return -1;
  return (int64_t)gcc_phat_work_doubles(T, F, D);
}

int setk_gcc_phat(const void* si, const void* sj, int32_t T, int32_t F, const double* omega,
                  const double* tau, int32_t D, int32_t normalize, int32_t apply_floor,
                  int32_t accumulate, double* work, double* out, void* stream) {
  if (!si || !sj || !omega || !tau || !work || !out) return fail(SETK_EINVAL, "setk_gcc_phat: null buffer");
  if (T < 1 || F < 1 || D < 1) return fail(SETK_ESHAPE, "setk_gcc_phat: T=%d F=%d D=%d", T, F, D);
  if ((size_t)F * sizeof(double2) > 48 * 1024)
    return fail(SETK_EUNSUPPORTED, "setk_gcc_phat: F=%d too large (<= 3072 bins)", F);
  cudaError_t e = run_gcc_phat(static_cast<const float2*>(si), static_cast<const float2*>(sj), T, F, omega,
                               tau, D, normalize, apply_floor, accumulate, work, out, stream);
  return done(e, "setk_gcc_phat");
}

int64_t setk_msc_work_doubles(int32_t T, int32_t F) {
  if (T < 1 || F < 1) return -1;
  return (int64_t)msc_work_doubles(T, F);
}

int setk_msc(const void* spec, int32_t N, int32_t T, int32_t F, int32_t context, int32_t normalize,
             double* work, double* out, void* stream) {
  if (!spec || !work || !out) return fail(SETK_EINVAL, "setk_msc: null buffer");
  if (N < 2 || N > SETK_MAX_CHANNELS || T < 1 || F < 1)
    return fail(SETK_ESHAPE, "setk_msc: bad shape N=%d T=%d F=%d", N, T, F);
  if (context < 0) return fail(SETK_EINVAL, "setk_msc: context %d < 0", context);
  cudaError_t e = run_msc(static_cast<const float2*>(spec), N, T, F, context, normalize, work, out, stream);
  return done(e, "setk_msc");
}

// ---- sound source localisation (ssl.cuh, built in spatial.cu) ----
int setk_ssl(int32_t backend, const void* stft, int32_t B, int32_t M, int32_t F, int32_t T, const void* steer,
             int32_t A, int32_t steer_F, const float* mask, int32_t N, const int32_t* windows_host, int32_t W,
             const int32_t* pairs_host, int32_t P, double compression, double eps, int32_t normalize,
             double* scores, int32_t* index, void* stream) {
  if (!stft || !steer || !windows_host || !scores || !index) return fail(SETK_EINVAL, "setk_ssl: null buffer");
  if (backend < SETK_SSL_ML || backend > SETK_SSL_MUSIC) return fail(SETK_EINVAL, "setk_ssl: unknown backend %d", backend);
  if (M < 1 || M > SETK_MAX_CHANNELS) return fail(SETK_EINVAL, "setk_ssl: M=%d outside [1, %d]", M, SETK_MAX_CHANNELS);
  if (A < 1) return fail(SETK_EINVAL, "setk_ssl: A=%d directions", A);
  if (B < 1 || F < 1 || T < 1 || W < 1 || B > 65535)
    return fail(SETK_ESHAPE, "setk_ssl: bad shape B=%d F=%d T=%d W=%d", B, F, T, W);
  if (steer_F != F) return fail(SETK_ESHAPE, "setk_ssl: steering table has %d bins, the STFT %d", steer_F, F);
  if (N < 1 || N > SETK_SSL_MAX_MASKS || (!mask && N != 1))
    return fail(SETK_EINVAL, "setk_ssl: N=%d masks (1..%d, 1 without a mask)", N, SETK_SSL_MAX_MASKS);
  if (N > 1 && backend != SETK_SSL_ML) return fail(SETK_EINVAL, "setk_ssl: N=%d masks need the ML backend", N);
  if (backend == SETK_SSL_SRP) {
    if (!pairs_host || P < 1) return fail(SETK_EINVAL, "setk_ssl: SRP needs microphone pairs");
    for (int p = 0; p < 2 * P; ++p)
      if (pairs_host[p] < 0 || pairs_host[p] >= M)
        return fail(SETK_EINVAL, "setk_ssl: pair index %d outside [0, %d)", pairs_host[p], M);
  } else {
    P = 0;
  }
  for (long long i = 0; i < (long long)B * W; ++i) {
    const int s = windows_host[2 * i], e = windows_host[2 * i + 1];
    if (s < 0 || e > T || s >= e)
      return fail(SETK_EINVAL, "setk_ssl: window [%d, %d) of utterance %lld outside [0, %d] or empty", s, e,
                  i / W, T);
  }
  return with_scratch(ssl_scratch_bytes(backend, B, N, M, F, T, A, W, P), stream, "setk_ssl(workspace)", "setk_ssl",
                      [&](char* ws) {
    return run_ssl(backend, static_cast<const float2*>(stft), B, M, F, T, static_cast<const double2*>(steer), A,
                   mask, N, windows_host, W, pairs_host, P, compression, eps, normalize, ws, scores, index, stream);
  });
}

// ---- AuxIVA blind source separation (auxiva.cuh, built in wpe.cu) ----
int setk_auxiva_stft(const void* stft, int32_t B, int32_t N, int32_t F, int32_t T, int32_t num_epochs,
                     void* out, uint32_t* status, void* stream) {
  if (!stft || !out) return fail(SETK_EINVAL, "setk_auxiva_stft: null buffer");
  if (N < 2 || N > SETK_MAX_CHANNELS)
    return fail(SETK_EINVAL, "setk_auxiva_stft: N=%d outside [2, %d]", N, SETK_MAX_CHANNELS);
  if (num_epochs < 0) return fail(SETK_EINVAL, "setk_auxiva_stft: num_epochs=%d", num_epochs);
  if (B < 1 || F < 1 || T < 1 || B > 65535 || (long long)B * F > 2000000000LL)
    return fail(SETK_EINVAL, "setk_auxiva_stft: bad shape B=%d F=%d T=%d", B, F, T);
  return with_scratch(auxiva_scratch_bytes(B, N, F, T), stream, "setk_auxiva_stft(workspace)", "setk_auxiva_stft",
                      [&](char* ws) {
    return run_auxiva(static_cast<const float2*>(stft), B, N, F, T, num_epochs, ws, static_cast<double2*>(out),
                      status, stream);
  });
}

// ---- iMCRA / OM-LSA noise suppression (ns.cu) ----
int setk_ns_imcra(const setk_imcra_config_t* cfg, const void* stft, const int32_t* n_frames, int32_t B,
                  int32_t F, int32_t T, double* gain, void* enh, void* stream) {
  if (!cfg || !cfg->window_host || !stft) return fail(SETK_EINVAL, "setk_ns_imcra: null argument");
  if (!gain && !enh) return fail(SETK_EINVAL, "setk_ns_imcra: gain and enh are both null");
  if (B < 1 || F < 1 || T < 1 || F > SETK_NS_MAX_BINS || B > 65535)
    return fail(SETK_EINVAL, "setk_ns_imcra: bad shape B=%d F=%d T=%d (F <= %d)", B, F, T, SETK_NS_MAX_BINS);
  if (cfg->w_mcra < 0 || cfg->w_mcra > SETK_NS_MAX_W)
    return fail(SETK_EINVAL, "setk_ns_imcra: w_mcra=%d outside [0, %d]", cfg->w_mcra, SETK_NS_MAX_W);
  if (F < 2 * cfg->w_mcra + 1)
    return fail(SETK_EINVAL, "setk_ns_imcra: F=%d bins < %d smoothing taps", F, 2 * cfg->w_mcra + 1);
  if (cfg->V < 1) return fail(SETK_EINVAL, "setk_ns_imcra: V=%d < 1", cfg->V);
  if (cfg->U < 1 || cfg->U > SETK_NS_MAX_U)
    return fail(SETK_EINVAL, "setk_ns_imcra: U=%d outside [1, %d]", cfg->U, SETK_NS_MAX_U);
  const float2* X = static_cast<const float2*>(stft);
  float2* out = static_cast<float2*>(enh);
  const size_t ring = ns_ring_bytes(*cfg, B, F);
  if (ring == 0) {
    cudaError_t e = run_ns_imcra(*cfg, X, n_frames, B, F, T, nullptr, gain, out, stream);
    return done(e, "setk_ns_imcra");
  }
  return with_scratch(ring, stream, "setk_ns_imcra(workspace)", "setk_ns_imcra", [&](char* ws) {
    return run_ns_imcra(*cfg, X, n_frames, B, F, T, reinterpret_cast<double*>(ws), gain, out, stream);
  });
}

// ---- image-method room impulse responses (rir.cu) ----
int setk_rir_image(const setk_rir_config_t* cfg, const double* room, const double* beta, const double* source,
                   const double* receivers, int32_t B, int32_t M, float* rir, uint32_t* status, void* stream) {
  if (!cfg || !room || !beta || !source || !receivers || !rir) return fail(SETK_EINVAL, "setk_rir_image: null argument");
  const int L = cfg->n_samples;
  if (B < 1 || M < 1 || L < 1 || B > 65535 || M > 65535)
    return fail(SETK_EINVAL, "setk_rir_image: bad shape B=%d M=%d L=%d", B, M, L);
  if (!(cfg->sound_velocity >= 1) || !(cfg->samp_frequency >= 1))
    return fail(SETK_EINVAL, "setk_rir_image: c=%g and fs=%g must be >= 1", cfg->sound_velocity, cfg->samp_frequency);
  if (cfg->order < -1) return fail(SETK_EINVAL, "setk_rir_image: order=%d < -1", cfg->order);
  if (cfg->mic_type < SETK_MIC_OMNI || cfg->mic_type > SETK_MIC_BIDIRECTIONAL)
    return fail(SETK_EINVAL, "setk_rir_image: unknown mic_type %d", cfg->mic_type);
  const int Tw = rir_window_taps(cfg->samp_frequency);
  if (Tw > SETK_RIR_MAX_TW)
    return fail(SETK_EUNSUPPORTED, "setk_rir_image: fs=%g gives Tw=%d > %d taps", cfg->samp_frequency, Tw,
                SETK_RIR_MAX_TW);
  std::vector<double> dims((size_t)B * 3);
  cudaError_t e = cudaMemcpyAsync(dims.data(), room, sizeof(double) * dims.size(), cudaMemcpyDeviceToHost,
                                  static_cast<cudaStream_t>(stream));
  if (e == cudaSuccess) e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return cuda_fail(e, "setk_rir_image(room)");
  const double cts = cfg->sound_velocity / cfg->samp_frequency;
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    double cand = 8;
    for (int d = 0; d < 3; ++d) {
      const double r = dims[(size_t)b * 3 + d];
      if (!(r > 0) || !std::isfinite(r))
        return fail(SETK_EINVAL, "setk_rir_image: problem %d: room dimension %d is %g, not > 0", b, d, r);
      const double n = rir_lattice_half(L, r, cts);
      if (n > SETK_RIR_MAX_HALF)
        return fail(SETK_EUNSUPPORTED, "setk_rir_image: problem %d: lattice half-width %.0f > %d along axis %d",
                    b, n, SETK_RIR_MAX_HALF, d);
      max_n = imax(max_n, (int)n);
      cand *= 2 * n + 1;
    }
    if (cand > SETK_RIR_MAX_CANDIDATES)
      return fail(SETK_EUNSUPPORTED, "setk_rir_image: problem %d: %.3g images per channel > %.3g", b, cand,
                  SETK_RIR_MAX_CANDIDATES);
  }
  if (rir_segments(L) == 1 || !cfg->hp_filter) {
    e = run_rir_image(*cfg, room, beta, source, receivers, B, M, max_n, rir, nullptr, status, stream);
    return done(e, "setk_rir_image");
  }
  return with_scratch(sizeof(double) * (size_t)B * M * L, stream, "setk_rir_image(workspace)", "setk_rir_image",
                      [&](char* ws) {
    return run_rir_image(*cfg, room, beta, source, receivers, B, M, max_n, rir, reinterpret_cast<double*>(ws),
                         status, stream);
  });
}

// ---- long convolution and mixture simulation (simu.cu) ----
int setk_convolve(const float* x, int32_t Sx, const float* h, int32_t Lh, int32_t B, int32_t M,
                  const int32_t* s_len_host, const int32_t* h_len_host, const int32_t* n_out_host, float* y,
                  int32_t Ny, void* stream) {
  if (!x || !h || !y) return fail(SETK_EINVAL, "setk_convolve: null argument");
  if (B < 1 || M < 1 || Sx < 1 || Lh < 1 || Ny < 1 || B > 65535 || M > 65535)
    return fail(SETK_EINVAL, "setk_convolve: bad shape B=%d M=%d Sx=%d Lh=%d Ny=%d", B, M, Sx, Lh, Ny);
  if (Sx > SETK_CONV_MAX_LEN || Lh > SETK_CONV_MAX_LEN || Ny > SETK_CONV_MAX_LEN)
    return fail(SETK_EUNSUPPORTED, "setk_convolve: Sx=%d Lh=%d Ny=%d: each must be <= %d", Sx, Lh, Ny,
                SETK_CONV_MAX_LEN);
  std::vector<int> len((size_t)B * 3);
  for (int b = 0; b < B; ++b) {
    const int S = s_len_host ? s_len_host[b] : Sx, L = h_len_host ? h_len_host[b] : Lh;
    const int n = n_out_host ? n_out_host[b] : Ny;
    if (S < 1 || S > Sx || L < 1 || L > Lh || n < 1 || n > Ny)
      return fail(SETK_EINVAL, "setk_convolve: problem %d: S=%d L=%d n_out=%d outside [1, %d], [1, %d], [1, %d]", b,
                  S, L, n, Sx, Lh, Ny);
    len[3 * (size_t)b] = S;
    len[3 * (size_t)b + 1] = L;
    len[3 * (size_t)b + 2] = n;
  }
  return with_host_table(len, conv_spectra_bytes(B, M, Lh, Ny), stream, "setk_convolve(workspace)", "setk_convolve",
                         [&](const int* d_len, char* ws) {
    return run_convolve(x, Sx, h, Lh, B, M, d_len, y, Ny, ws, stream);
  });
}

int setk_simulate_mix(const float* pool, int64_t pool_len, const setk_simu_mix_t* mixes_host, int32_t B,
                      const setk_simu_term_t* terms_host, int32_t n_terms, int32_t M, int32_t K, int32_t n_pitch,
                      int32_t pcm16, void* mix, void* spk, void* noise, double* factor, void* stream) {
  if (!pool || !mixes_host || !terms_host || !mix) return fail(SETK_EINVAL, "setk_simulate_mix: null argument");
  if (B < 1 || n_terms < 1 || M < 1 || K < 1 || n_pitch < 1 || B > 65535 || pool_len < 1)
    return fail(SETK_EINVAL, "setk_simulate_mix: bad shape B=%d terms=%d M=%d K=%d n_pitch=%d pool=%lld", B,
                n_terms, M, K, n_pitch, (long long)pool_len);
  for (int b = 0; b < B; ++b) {
    const setk_simu_mix_t& mx = mixes_host[b];
    if (mx.n_terms > SETK_SIMU_MAX_TERMS)
      return fail(SETK_EUNSUPPORTED, "setk_simulate_mix: mixture %d has %d terms > %d", b, mx.n_terms,
                  SETK_SIMU_MAX_TERMS);
    if (mx.first_term < 0 || mx.n_terms < 1 || mx.first_term > n_terms - mx.n_terms)
      return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d: terms [%d, +%d) outside the table of %d", b,
                  mx.first_term, mx.n_terms, n_terms);
    if (mx.n_samples < 1 || mx.n_samples > n_pitch || mx.n_channels < 1 || mx.n_channels > M)
      return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d: n_samples=%d n_channels=%d outside [1, %d], [1, %d]",
                  b, mx.n_samples, mx.n_channels, n_pitch, M);
    int n_spk = 0, last_kind = SETK_SIMU_SPEAKER;
    for (int i = 0; i < mx.n_terms; ++i) {
      const setk_simu_term_t& t = terms_host[mx.first_term + i];
      if (t.kind < SETK_SIMU_SPEAKER || t.kind > SETK_SIMU_ISOTROPIC || t.kind < last_kind ||
          (i > 0 && t.kind == SETK_SIMU_ISOTROPIC && last_kind == SETK_SIMU_ISOTROPIC))
        return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d term %d: kind %d out of order", b, i, t.kind);
      last_kind = t.kind;
      n_spk += t.kind == SETK_SIMU_SPEAKER;
      if (t.n_channels != 1 && (t.n_channels != mx.n_channels || t.kind == SETK_SIMU_ISOTROPIC))
        return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d term %d: %d channels for a %d-channel mixture", b,
                    i, t.n_channels, mx.n_channels);
      if (t.begin < 0 || t.length < 0 || t.begin > mx.n_samples - t.length)
        return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d term %d: samples [%d, +%d) outside [0, %d)", b, i,
                    t.begin, t.length, mx.n_samples);
      const int64_t reach = (int64_t)(t.n_channels - 1) * t.pitch + (t.repeat ? 1 : t.length);
      if (t.src < 0 || t.pitch < 0 || t.src + reach > pool_len || t.power_begin < 0 ||
          t.power_end <= t.power_begin || t.src + t.power_end > pool_len)
        return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d term %d: image or power range outside the pool",
                    b, i);
    }
    if (n_spk < 1 || n_spk > K)
      return fail(SETK_EINVAL, "setk_simulate_mix: mixture %d has %d speakers, want [1, %d]", b, n_spk, K);
  }
  return with_scratch(simu_scratch_bytes(B, n_terms, n_pitch), stream, "setk_simulate_mix(workspace)",
                      "setk_simulate_mix", [&](char* ws) {
    return run_simulate_mix(pool, B, n_terms, M, K, n_pitch, pcm16, ws, mixes_host, terms_host, mix, spk, noise,
                            factor, stream);
  });
}

// ---- separation metrics (sep_eval.cu) ----
// n_b of every utterance into `len` (checked against [1, S])
static int sep_lengths(const char* who, const int32_t* n_samples_host, int B, int S, std::vector<int>& len) {
  len.resize((size_t)B);
  for (int b = 0; b < B; ++b) {
    len[b] = n_samples_host ? n_samples_host[b] : S;
    if (len[b] < 1 || len[b] > S)
      return fail(SETK_EINVAL, "%s: utterance %d has %d samples, want [1, %d]", who, b, len[b], S);
  }
  return SETK_OK;
}

int64_t setk_bss_eval_scratch_bytes(int32_t B, int32_t N, int32_t S, int32_t L) {
  if (B < 1 || N < 1 || S < 1 || L < 1 || B > 65535 || N > SETK_SEP_MAX_SOURCES || L > SETK_SEP_MAX_FLEN ||
      N * L > SETK_SEP_MAX_COLS || S > SETK_SEP_MAX_SAMPLES)
    return -1;
  // what setk_bss_eval's with_host_table allocates: the B lengths, then the kernels' scratch
  return (int64_t)(up256(sizeof(int) * B) + sep_eval_scratch_bytes(B, N, S, L));
}

int setk_bss_eval(const float* est, const float* ref, const int32_t* n_samples_host, int32_t B, int32_t N, int32_t S,
                  int32_t L, double* crit, int32_t* dropped, uint32_t* status, void* stream) {
  if (!est || !ref || !crit || !status) return fail(SETK_EINVAL, "setk_bss_eval: null argument");
  if (B < 1 || N < 1 || S < 1 || L < 1 || B > 65535)
    return fail(SETK_EINVAL, "setk_bss_eval: bad shape B=%d N=%d S=%d L=%d", B, N, S, L);
  if (N > SETK_SEP_MAX_SOURCES || L > SETK_SEP_MAX_FLEN || N * L > SETK_SEP_MAX_COLS || S > SETK_SEP_MAX_SAMPLES)
    return fail(SETK_EUNSUPPORTED, "setk_bss_eval: N=%d L=%d S=%d: want N <= %d, L <= %d, N L <= %d, S <= %d", N, L, S,
                SETK_SEP_MAX_SOURCES, SETK_SEP_MAX_FLEN, SETK_SEP_MAX_COLS, SETK_SEP_MAX_SAMPLES);
  std::vector<int> len;
  const int rc = sep_lengths("setk_bss_eval", n_samples_host, B, S, len);
  if (rc != SETK_OK) return rc;
  return with_host_table(len, sep_eval_scratch_bytes(B, N, S, L), stream, "setk_bss_eval(workspace)", "setk_bss_eval",
                         [&](const int* d_len, char* ws) {
    return run_bss_eval(est, ref, d_len, B, N, S, L, ws, crit, dropped, status, stream);
  });
}

int setk_si_snr(const float* est, const float* ref, const int32_t* n_samples_host, int32_t B, int32_t N, int32_t S,
                int32_t remove_dc, double eps, double* out, void* stream) {
  if (!est || !ref || !out) return fail(SETK_EINVAL, "setk_si_snr: null argument");
  if (B < 1 || N < 1 || S < 1 || B > 65535 || !(eps >= 0) || !std::isfinite(eps))
    return fail(SETK_EINVAL, "setk_si_snr: bad argument B=%d N=%d S=%d eps=%g", B, N, S, eps);
  if (N > SETK_SEP_MAX_SOURCES || S > SETK_SEP_MAX_SAMPLES)
    return fail(SETK_EUNSUPPORTED, "setk_si_snr: N=%d S=%d: want N <= %d, S <= %d", N, S, SETK_SEP_MAX_SOURCES,
                SETK_SEP_MAX_SAMPLES);
  std::vector<int> len;
  const int rc = sep_lengths("setk_si_snr", n_samples_host, B, S, len);
  if (rc != SETK_OK) return rc;
  return with_host_table(len, 0, stream, "setk_si_snr(workspace)", "setk_si_snr", [&](const int* d_len, char*) {
    return run_si_snr(est, ref, d_len, B, N, S, remove_dc, eps, out, stream);
  });
}

}  // extern "C"
