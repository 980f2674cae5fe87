// launchers.cuh -- every host function of libsetk_b200 that one translation unit calls in another,
// declared once, grouped by the file that defines it.  The defining file and every caller include
// this header, so a definition and its callers cannot disagree about a signature.
#pragma once
#include "common.cuh"

namespace setk {

struct TileSched;      // stft_tile.cuh
struct StftCovArgs;    // stft_cov_args.cuh
struct CovSpillArgs;   // cov_spill_args.cuh
struct WeightsArgs;    // weights_args.cuh

// ---- generic.cu: shape-generic STFT / covariance / apply / iSTFT and the element-wise passes ----
cudaError_t run_stft_generic(const setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                             float2* out, void* stream);
cudaError_t run_cov_generic(const float2* stft, const float* mask, unsigned flags, int B, int C, int F, int T,
                            float2* R, void* stream);
cudaError_t run_apply_generic(const float2* stft, const void* w, int w_dtype, const float* post_mask, int B, int C,
                              int F, int T, float2* enh, void* stream);
cudaError_t run_istft_strided(const setk_plan* pl, const float2* enh, long long sb, long long sf, long long st,
                              int B, int T_used, int n_out, const int* n_samples, float* frames_ws, float* wave,
                              unsigned* peak, void* stream);
cudaError_t run_istft_generic(const setk_plan* pl, const float2* enh, int B, int T, int T_used, int n_out,
                              const int* n_samples, float* frames_ws, float* wave, unsigned* peak, void* stream);
cudaError_t run_peak_scale(float* wave, int B, int n_out, const float* norm, const unsigned* peak, void* stream);
cudaError_t run_peak_scale_pcm16(const float* wave, int B, int n_out, const float* norm, const unsigned* peak,
                                 int16_t* pcm, void* stream);
cudaError_t run_bits_to_float(const unsigned* bits, int n, float* out, void* stream);
cudaError_t maxabs_generic(const float* audio, const int* n_samples, int B, int C, int N, unsigned* bits,
                           float* out, void* stream);
cudaError_t run_float_to_pcm16(const float* wave, long long n, int16_t* pcm, void* stream);
cudaError_t run_pcm16_to_float(const int16_t* pcm, long long n, float* wave, void* stream);

// ---- stft_cov_fused.cu: fused STFT + covariance (n_fft 512, C <= 4) and the persistent schedule ----
bool stft_cov_fused_supported(const Geometry& g);
size_t stft_cov_partial_bytes(const setk_plan* pl, int B, int T);
int stft_cov_pick_chunks(const setk_plan* pl, int B, int T);
cudaError_t fused_schedule(const setk_plan* pl, int B, int T, int TT, int T_cap, const int* n_samples,
                           int* tile_prefix, void* stream, TileSched* sched, int* n_ctas, int* slots);
cudaError_t run_stft_cov_fused(setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                               const float* mask_s, const float* mask_n, unsigned flags, int* tile_prefix,
                               float* partials, unsigned* maxabs_bits, float2* Rs, float2* Rn, float* maxabs,
                               void* stream);

// ---- stft_cov_ws.cu: the warp-specialised C = 4 build of the fused pass ----
cudaError_t run_stft_cov_ws(const StftCovArgs& a, int n_ctas, void* stream);

// ---- apply_istft_fused.cu: fused apply + iSTFT (n_fft 512) ----
bool apply_istft_fused_supported(const Geometry& g);
cudaError_t run_apply_istft_fused(setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                                  const void* w, int w_dtype, const float* post_mask, int n_out, int* tile_prefix,
                                  float* wave, unsigned* peak, void* stream);

// ---- stft_spill.cu: tile STFT into the bin-major workspace and the passes over it ----
bool stft_spill_supported(const Geometry& g);
size_t stft_spill_bytes(const Geometry& g, int B, int T);
size_t apply_spill_bytes(const Geometry& g, int B, int T);
cudaError_t run_stft_spill(setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                           int n_chunks, float2* xws, unsigned* maxabs_bits, void* stream);
int cov_spill_chunks(const setk_plan* pl, int B, int T);
size_t cov_spill_partial_bytes(const Geometry& g, int B, int n_chunks);
cudaError_t run_cov_spill(setk_plan* pl, const float2* xws, const float* mask_s, const float* mask_n,
                          unsigned flags, const int* n_samples, int B, int N, int T, int n_chunks,
                          float* partials, float2* Rs, float2* Rn, void* stream);
cudaError_t run_spill_to_bcft(const setk_plan* pl, const float2* xws, int B, int T, float2* out, void* stream);
cudaError_t run_apply_spill(setk_plan* pl, const float2* xws, const void* w, int w_dtype, const float* post_mask,
                            int B, int T, float2* yws, void* stream);

// ---- feats.cu: spectral features (magnitude / power / mel / log) ----
bool feats_fused_supported(const Geometry& g);
cudaError_t run_feats_fused(const setk_plan* pl, const float* audio, const int* n_samples, int B, int N, int T,
                            unsigned flags, float scale, float* out, void* stream);
cudaError_t run_feats_stft(const setk_plan* pl, const float2* stft, const int* n_samples, int B, int N, int T,
                           unsigned flags, float scale, float* out, void* stream);

// ---- cov_mma.cu: tensor-core covariance over the workspace (C >= 5) ----
int cov_mma_bins_per_cta(int C);
cudaError_t run_cov_mma(const CovSpillArgs& a, int B, void* stream);

// ---- weights.cu, weights_coop.cu, weights_post.cu: per-bin solves ----
cudaError_t weights_run(int kind, double beta, int ref_channel, int rank1, int ban, const void* Rs,
                        const void* Rn, const void* Ry, int r_dtype, int B, int F, int C, void* w, int w_dtype,
                        unsigned* status, int* ref_used, void* stream);
bool weights_coop_supported(const WeightsArgs& a, int C);
cudaError_t weights_coop_launch(const WeightsArgs& a, int C, void* stream);
cudaError_t post_run(int mode, const void* A, const void* Rn, int dtype, int B, int F, int C, void* out,
                     unsigned* status, void* stream);

// ---- cgmm.cu: CGMM mask estimation over a bin-major STFT ----
struct CgCtx { Geometry geo; int sm_count; };   // what the CGMM passes need of a plan
cudaError_t run_bcft_to_spill(const float2* in, int B, int C, int F, int T, int P, float2* xws, void* stream);
size_t cgmm_workspace_bytes(const CgCtx* pl, int B, int T, int K, int P);
cudaError_t run_cgmm(const CgCtx* pl, const float2* X, int P, double* ws, const int* n_samples, int B, int N,
                     int T, int K, int num_iters, const float* init_gamma, int update_alpha, float* masks,
                     unsigned* status, void* stream);
size_t cacgmm_workspace_bytes(const CgCtx* pl, int B, int T, int K, int P);
cudaError_t run_cacgmm(const CgCtx* pl, const float2* X, int P, double* ws, const int* n_samples, int B, int N,
                       int T, int K, int num_iters, const double* init_gamma, int cgmm_init, int update_alpha,
                       const int* permu_rows, int R, float* masks, unsigned* status, void* stream);

// ---- permu.cu: frequency permutation alignment of K-class masks ----
struct PermuArgs {
  const double* m; int ld;       // posteriors [B][K][T][ld], bins [0, F) of each row
  const int* n_frames;           // [B] frames per utterance, or null: from n_samples / N and g
  const int* n_samples; int N; Geometry g;
  int K, T, F;
};
// bytes of global centroid scratch a call needs (0 when the centroids fit in shared memory); -1 when
// the per-bin tables alone exceed shared memory
long long permu_scratch_bytes(int B, int K, int T, int F);
cudaError_t run_permu_align(const PermuArgs& a, int B, const int* rows_host, int R, double* scratch,
                            float* out, int* mapping, void* stream);

// ---- wpe.cu (with auxiva.cuh): fp64 per-bin iterative front ends ----
bool wpe_supported(int C, int T, int taps, int delay, int ctx);
size_t wpe_workspace_bytes(int B, int C, int F, int taps);
cudaError_t run_wpe(const float2* X, int P, int B, int C, int F, int T, int taps, int delay, int ctx,
                    int num_iters, double* ws, float2* out, unsigned* status, const float2* lam_src,
                    float* linv_out, void* stream);
size_t auxiva_scratch_bytes(int B, int N, int F, int T);
cudaError_t run_auxiva(const float2* X, int B, int N, int F, int T, int epochs, char* ws, double2* out,
                       unsigned* status, void* stream);

// ---- spatial.cu (with ssl.cuh): spatial features and sound source localisation ----
cudaError_t run_ipd(const float2* si, const float2* sj, long long rows, int F, int mode, float* out,
                    void* stream);
cudaError_t run_dirfeat(const float2* stft, const double2* steer, int steer_batched, const int* pairs, int P,
                        int B, int M, int F, int T, double* out, void* stream);
size_t gcc_phat_work_doubles(int T, int F, int D);
cudaError_t run_gcc_phat(const float2* si, const float2* sj, int T, int F, const double* omega,
                         const double* tau, int D, int normalize, int apply_floor, int accumulate,
                         double* work, double* out, void* stream);
size_t msc_work_doubles(int T, int F);
cudaError_t run_msc(const float2* spec, int N, int T, int F, int context, int normalize, double* work,
                    double* out, void* stream);
size_t ssl_scratch_bytes(int backend, int B, int N, int M, int F, int T, int A, int W, int P);
cudaError_t run_ssl(int backend, const float2* stft, int B, int M, int F, int T, const double2* sv, int A,
                    const float* mask, int N, const int* windows_host, int W, const int* pairs_host, int P,
                    double compression, double eps, int normalize, char* ws, double* scores, int* index,
                    void* stream);

// ---- ns.cu: iMCRA noise estimation and the OM-LSA gain ----
size_t ns_ring_bytes(const setk_imcra_config_t& cfg, int B, int F);
cudaError_t run_ns_imcra(const setk_imcra_config_t& cfg, const float2* X, const int* n_frames, int B, int F,
                         int T, double* ring, double* gain, float2* enh, void* stream);

// ---- rir.cu: image-method room impulse responses ----
double rir_lattice_half(int L, double room, double cts);
int rir_window_taps(double fs);
int rir_segments(int L);
cudaError_t run_rir_image(const setk_rir_config_t& cfg, const double* room, const double* beta,
                          const double* source, const double* receivers, int B, int M, int max_n, float* rir,
                          double* ws, unsigned* status, void* stream);

// ---- simu.cu: long convolution and mixture simulation ----
int conv_block();
size_t conv_spectra_bytes(int B, int M, int Lh, int Ny);
cudaError_t run_convolve(const float* x, int Sx, const float* h, int Lh, int B, int M, const int* len, float* y,
                         int Ny, char* ws, void* stream);
size_t simu_scratch_bytes(int B, int n_terms, int n_pitch);
cudaError_t run_simulate_mix(const float* pool, int B, int n_terms, int M, int K, int n_pitch, int pcm16,
                             char* ws, const setk_simu_mix_t* mixes_host, const setk_simu_term_t* terms_host,
                             void* mix, void* spk, void* noise, double* factor, void* stream);

// ---- sep_eval.cu: BSS-Eval and SI-SNR separation metrics ----
size_t sep_eval_scratch_bytes(int B, int N, int S, int L);
cudaError_t run_bss_eval(const float* est, const float* ref, const int* len, int B, int N, int S, int L, char* ws,
                         double* crit, int* dropped, unsigned* status, void* stream);
cudaError_t run_si_snr(const float* est, const float* ref, const int* len, int B, int N, int S, int remove_dc,
                       double eps, double* out, void* stream);

// ---- cm_mask.cu: Kaldi compressed-matrix masks ----
cudaError_t run_cm_masks(const unsigned char* blobs, long long slot_bytes, int B, int T, int F, float* out,
                         int* status, void* stream);

}  // namespace setk
