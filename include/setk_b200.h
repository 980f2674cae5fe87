/*
 * setk_b200.h -- C-ABI of libsetk_b200.so: the B200-native (sm_100a) mask-based
 * adaptive-beamformer hot path of funcwj/setk.
 *
 *   multichannel STFT -> mask-weighted spatial covariance -> MVDR / MPDR / GEV /
 *   PMWF weight solve (+BAN, rank-1) -> beamform apply -> iSTFT (+peak norm)
 *
 * and the front ends around it: CGMM masks, WPE / WPD, spatial features, sound
 * source localisation, AuxIVA blind source separation, iMCRA / OM-LSA
 * noise suppression, image-method room impulse responses, mixture simulation,
 * the separation metrics (BSS-Eval SDR / SIR / SAR, SI-SNR) and spectral features
 * (magnitude / power / log spectrogram, log-mel filterbank).
 *
 * Every entry point below replaces one reference interface; the citation is
 * the reference file:line (paths relative to the reference tree).  The Python
 * mirror of the reference's operator API (setk_b200/libs/{utils,stft,
 * beamformer}.py) binds these with ctypes; INTEGRATION.md shows the stub a
 * reference maintainer would add.
 *
 * Conventions
 *   - all data pointers are DEVICE pointers unless the name ends in _host;
 *   - every call is asynchronous on the caller's `stream` (a cudaStream_t passed
 *     as void*), re-entrant, and keeps no global state besides the last error
 *     string (thread local); setk_rir_image alone synchronises its stream (it
 *     reads the room sizes back to size the launch);
 *   - arrays are dense, row-major, the reference's axis order:
 *       audio  f32 [B][C][N]          (read_wav: C x N, utils.py:65-92)
 *       mask   f32 [B][T][F]          (T x F, beamformer.py:89)
 *       stft   c64 [B][C][F][T]       (N x F x T, data_handler.py:502-503)
 *       R      c64|c128 [B][F][C][C]  (F x N x N, beamformer.py:93)
 *       weight c64|c128 [B][F][C]     (F x N,     beamformer.py:18)
 *       enh    c64 [B][F][T]          (F x T,     beamformer.py:226)
 *       wave   f32 [B][N_out]
 *     complex = interleaved (re, im);
 *   - ragged batches: `n_samples` (i32[B], device) gives each utterance's true
 *     length (<= N); NULL means every utterance has N samples.  Frames past an
 *     utterance's own frame count are skipped (covariance) / written as zero;
 *   - return value: 0 ok, < 0 bad argument (SETK_E*), > 0 a cudaError_t.
 *     Numerical failures (singular Rn, non-PD Rn for GEV, ...) never fail the
 *     call: they set bits in the per-utterance `status` word, which the Python
 *     layer maps to numpy.linalg.LinAlgError per key like the reference CLI's
 *     per-utterance try/except (apply_adaptive_beamformer.py:160-172).
 */
#ifndef SETK_B200_H_
#define SETK_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SETK_VERSION 100 /* 0.1.0 */

#define SETK_MAX_CHANNELS 16

/* ---- error codes (negative) ---- */
#define SETK_OK 0
#define SETK_EINVAL -1      /* bad argument / unsupported configuration        */
#define SETK_ENOMEM -2      /* host allocation failed                           */
#define SETK_ESHAPE -3      /* shape inconsistent with the plan                 */
#define SETK_EUNSUPPORTED -4

/* ---- per-utterance status bits written by setk_weights ---- */
#define SETK_ST_SINGULAR 1u     /* exactly singular pivot in a linear solve (np.linalg.solve -> LinAlgError) */
#define SETK_ST_NOT_PD 2u       /* Rn not positive definite in the GEV reduction (scipy eigh(a,b) -> LinAlgError) */
#define SETK_ST_NO_CONVERGE 4u  /* Jacobi eigen-iteration hit its sweep limit  */
#define SETK_ST_NONFINITE 8u    /* NaN/Inf in the result                       */
#define SETK_ST_BAD_REF 16u     /* PMWF reference channel >= C (RuntimeError, beamformer.py:656-658) */
#define SETK_ST_REGULARIZED 32u /* WARNING only: Rn was numerically not PD in a GEV reduction and its
                                   diagonal was loaded (the reference falls back to a non-Hermitian eig
                                   there, beamformer.py:55-58) */
#define SETK_ST_SILENT 64u      /* a reference or estimate is all zeros (mir_eval's ValueError, setk_bss_eval) */

/* ---- beamformer kinds: apply_adaptive_beamformer.py:22,92-110 ---- */
#define SETK_BF_MVDR 0          /* beamformer.py:527-539 */
#define SETK_BF_MPDR 1          /* beamformer.py:555-573 (Ry in place of Rn)   */
#define SETK_BF_MPDR_WHITEN 2   /* beamformer.py:566-568 */
#define SETK_BF_GEVD 3          /* beamformer.py:674-682 */
#define SETK_BF_PMWF 4          /* beamformer.py:632-659 */
#define SETK_BF_PEVD 5          /* bare solve_pevd(Rs) / solve_pevd(Rs,Rn) when Rn != NULL (beamformer.py:31-63) */

/* ---- rank-1 approximation of Rs for PMWF: beamformer.py:66-84,641-645 ---- */
#define SETK_RANK1_NONE 0
#define SETK_RANK1_EIG 1
#define SETK_RANK1_GEV 2

/* ---- flags for setk_stft_cov / setk_cov ---- */
#define SETK_F_CLIP_MASK 1u     /* mask <- min(mask, 1): apply_adaptive_beamformer.py:142 */
#define SETK_F_MASK_FT 2u       /* masks are stored [B][F][T] and transposed on the fly (ibid. 149-152) */

/* ---- element types of R / weight buffers ---- */
#define SETK_C64 0              /* complex<float>  */
#define SETK_C128 1             /* complex<double> */

typedef struct setk_plan setk_plan_t;

/*
 * STFT geometry of one plan.  Mirrors StftParser (libs/opts.py:21-49) and the
 * keyword arguments of forward_stft / inverse_stft (libs/utils.py:96-105,
 * 142-150).  n_fft = nextpow2(frame_len) when round_power_of_two, else
 * frame_len (utils.py:114); only power-of-two n_fft in [32, 4096] is supported
 * (SETK_EUNSUPPORTED otherwise).
 */
typedef struct setk_config {
  int32_t num_channels;      /* C, 1..SETK_MAX_CHANNELS                                   */
  int32_t frame_len;         /* window length (--frame-len)                               */
  int32_t n_fft;             /* FFT size >= frame_len                                     */
  int32_t frame_hop;         /* --frame-hop                                               */
  int32_t center;            /* --center: reflect-pad n_fft/2 both sides                  */
  int32_t max_batch;         /* largest B any call will pass (workspace sizing)           */
  int32_t max_samples;       /* largest N any call will pass                              */
  int32_t reserved;
  const double* window_host; /* HOST pointer, frame_len analysis-window values
                                (scipy.signal.get_window(window, frame_len, fftbins=True),
                                or hann**0.5 for "sqrthann": utils.py:116-117)            */
} setk_config_t;

/* -------------------------------------------------------------------------- */
int setk_version(void);
/* thread-local description of the last non-zero return */
const char* setk_last_error_string(void);

/* Plan: window tables, synthesis-normalisation tables, partial-sum and STFT
 * workspace.  One per (C, frame_len, n_fft, hop, center, max_batch, max_samples).
 * Replaces the per-call window construction of librosa.stft/istft reached from
 * utils.py:123-128,159-164 and stft.h:75-154 (ShortTimeFTComputer). */
int setk_plan_create(const setk_config_t* cfg, setk_plan_t** plan_out);
int setk_plan_destroy(setk_plan_t* plan);

/* Integer bookkeeping, bit-exact with librosa 0.8.1 (SURVEY.md App. A) and
 * stft.h:143-153 (NumFrames / NumSamples):
 *   T     = 1 + (N + 2*(n_fft/2)*center - n_fft) / hop      (or -1 if too short)
 *   N_out = hop*(T-1) + n_fft - 2*(n_fft/2)*center */
int setk_num_frames(const setk_plan_t* plan, int32_t n_samples);
int setk_istft_length(const setk_plan_t* plan, int32_t num_frames);
int setk_num_bins(const setk_plan_t* plan);

/* forward_stft x C + np.stack: utils.py:96-138, data_handler.py:492-503;
 * C++ twin ShortTimeFTComputer::Compute (stft.cc:28-66,108).
 * stft_out c64 [B][C][F][T], T = setk_num_frames(plan, N). */
int setk_stft(setk_plan_t* plan, const float* audio, const int32_t* n_samples,
              int32_t B, int32_t N, void* stft_out, void* stream);

/* Spectral features, compute_spectrogram.py:19-40 and compute_fbank.py:22-61: forward_stft with
 * apply_abs (utils.py:130-135; cmat_abs, utils.py:30-42), then per flag, in this order,
 *   SETK_FEAT_POW  the rounded magnitude squared               (np.power(., 2), utils.py:132-133)
 *   SETK_FEAT_MEL  np.dot(mel, .) with the plan's mel table    (compute_fbank.py:49-51)
 *   SETK_FEAT_LOG  log(max(., FLT_EPSILON))                    (utils.py:134-135, compute_fbank.py:52-53)
 * sample_scale multiplies the magnitude before those steps: for a power of two this equals scaling
 * the samples, bit for bit (x / 32768 with scale 32768 gives the features of the raw int16 values,
 * read_wav(normalize=False), utils.py:65-92).
 *   out  f32 [B][C][T][D], T = setk_num_frames(plan, N), D = setk_num_bins(plan), or num_mel under
 *        SETK_FEAT_MEL; frames past an utterance's own count are zero rows.
 * n_fft 512 (even hop) and 1024 (hop % 4 == 0) run fused from the audio: the STFT stays on chip.  Other
 * geometries run the generic STFT into the plan's workspace, then the same tail.
 * SETK_EINVAL: null plan / audio / out, SETK_FEAT_MEL without a table (setk_plan_set_mel), unknown
 * flag bits, sample_scale not finite and > 0.  SETK_ESHAPE: the batch checks of setk_stft, B > 65535. */
#define SETK_FEAT_POW 1u
#define SETK_FEAT_MEL 2u
#define SETK_FEAT_LOG 4u
int setk_spectral_feats(setk_plan_t* plan, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                        uint32_t flags, float sample_scale, float* out, void* stream);

/* The plan's mel filterbank for setk_spectral_feats: librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax,
 * htk=True) as compute_fbank.py:45-48 builds it (setk_b200.libs.filters.mel restates it on the host).
 *   mel_host  f32 [num_mel][F] host matrix, F = setk_num_bins(plan): finite, >= 0.  Each row keeps the
 *             bins from its first to its last non-zero weight (the exact zeros outside are skipped);
 *             an all-zero row gives zero features.  num_mel = 0 clears the table.
 * Synchronous (uploads like setk_plan_create's window).  SETK_EINVAL: null plan, mel_host null with
 * num_mel > 0, num_mel outside [0, 1024], a negative or non-finite weight. */
int setk_plan_set_mel(setk_plan_t* plan, int32_t num_mel, const float* mel_host);

/* THE METRIC KERNEL.  Fused multichannel STFT + mask-weighted spatial
 * covariance: data_handler.py:502-503 -> beamformer.py:279-281 -> 87-103
 * (SupervisedBeamformer.run computing Rn then Rs), C++ twin EstimatePsd
 * (beamformer.cc:91-120).  The STFT is never written to HBM.
 *   mask_s  f32 [B][T][F]  target mask
 *   mask_n  f32 [B][T][F] or NULL -> 1 - mask_s (beamformer.py:279)
 *   Rs, Rn  c64 [B][F][C][C]: sum_t m x x^H / max(sum_t m, 1e-6)
 *   maxabs  f32 [B] or NULL: max |sample| over all channels
 *           (SpectrogramReader.maxabs, data_handler.py:398-400) -- the `norm`
 *           later handed to inverse_stft (apply_adaptive_beamformer.py:133,176) */
int setk_stft_cov(setk_plan_t* plan, const float* audio, const int32_t* n_samples,
                  int32_t B, int32_t N, const float* mask_s, const float* mask_n,
                  uint32_t flags, void* Rs, void* Rn, float* maxabs, void* stream);

/* compute_covar on an explicit STFT: beamformer.py:87-103.  Plan-free.
 *   stft c64 [B][C][F][T], mask f32 [B][T][F], R c64 [B][F][C][C] */
int setk_cov(const void* stft, const float* mask, uint32_t flags, int32_t B,
             int32_t C, int32_t F, int32_t T, void* R, void* stream);

/* Per-bin weight solve, fp64 internally, one thread-resident problem per
 * (utterance, bin).  Replaces solve_pevd / do_ban / rank1_constraint /
 * {Mvdr,Mpdr,Gevd,Pmwf}Beamformer.weight (beamformer.py:14-84,527-682) and the
 * C++ twins EstimateSteerVector / ComputeMvdrBeamWeights /
 * ComputeGevdBeamWeights (beamformer.cc:128-204).
 *   kind         SETK_BF_*
 *   beta         PMWF beta (0: pmwf-0, 1: pmwf-1)
 *   ref_channel  PMWF reference channel, < 0: pick argmax of the estimated
 *                output SNR (beamformer.py:620-630,650-653)
 *   rank1        SETK_RANK1_* (PMWF only)
 *   ban          != 0: blind analytical normalisation with Rn (beamformer.py:14-28)
 *   Rs, Rn, Ry   [B][F][C][C] of r_dtype (Ry only for MPDR kinds; Rn may be
 *                NULL for SETK_BF_PEVD and for SETK_BF_MPDR without ban)
 *   w            [B][F][C] of w_dtype
 *   status       u32 [B], OR-ed SETK_ST_* bits (caller zeroes it)
 *   ref_used     i32 [B] or NULL: PMWF reference channel actually used
 * Eigenvector convention (the reference's is LAPACK-defined up to a sign, see
 * SURVEY.md finding 4): principal eigenvector has unit 2-norm and component 0
 * real and >= 0; GEV: Rn = L L^H, y principal of L^-1 Rs L^-H with the same
 * convention, w = L^-H y (so w^H Rn w = 1, scipy.linalg.eigh(a, b)). */
int setk_weights(int32_t kind, double beta, int32_t ref_channel, int32_t rank1,
                 int32_t ban, const void* Rs, const void* Rn, const void* Ry,
                 int32_t r_dtype, int32_t B, int32_t F, int32_t C, void* w,
                 int32_t w_dtype, uint32_t* status, int32_t* ref_used, void* stream);

/* do_ban(weight, Rn): beamformer.py:14-28.  w_in / w_out [B][F][C], Rn [B][F][C][C],
 * all of `dtype` (SETK_C64 / SETK_C128). */
int setk_ban(const void* w_in, const void* Rn, int32_t dtype, int32_t B, int32_t F, int32_t C,
             void* w_out, void* stream);

/* rank1_constraint(Rs, Rn=None): beamformer.py:66-84.  Rn == NULL: principal
 * eigenvector of Rs; else Rn * (principal generalised eigenvector of (Rs, Rn)).
 * R1_out [B][F][C][C] = v v^H * tr(Rs) / max(tr(v v^H), eps32).  status u32[B] or NULL. */
int setk_rank1(const void* Rs, const void* Rn, int32_t dtype, int32_t B, int32_t F, int32_t C,
               void* R1_out, uint32_t* status, void* stream);

/* Beamformer.beamform on an explicit STFT: beamformer.py:220-234, C++ twin
 * Beamform (beamformer.cc:215-230).  enh[b][f][t] = sum_c conj(w[b][f][c]) x[b][c][f][t]
 *   post_mask f32 [B][T][F] or NULL: enh *= mask^T (apply_adaptive_beamformer.py:174-175) */
int setk_apply(const void* stft, const void* w, int32_t w_dtype, const float* post_mask,
               int32_t B, int32_t C, int32_t F, int32_t T, void* enh, void* stream);

/* inverse_stft: utils.py:142-173 (librosa.istft + peak normalisation), C++ twin
 * InverseShortTimeFT (stft.cc:154-198).
 *   enh     c64 [B][F][T]
 *   n_out   output samples per utterance: setk_istft_length(plan, T) when the
 *           reference passes nsamps=None, else nsamps (fix_length semantics)
 *   norm    f32 [B] or NULL: if given, wave <- wave * norm / (max|wave| + eps32)
 *           (utils.py:166-168)
 *   wave    f32 [B][n_out] */
int setk_istft(setk_plan_t* plan, const void* enh, int32_t B, int32_t T, int32_t n_out,
               const float* norm, float* wave, void* stream);

/* Fused beamform-apply + iSTFT from the multichannel AUDIO (the STFT is
 * recomputed on chip, never read from HBM): beamformer.py:283 ->
 * apply_adaptive_beamformer.py:174-176 -> utils.py:159-168.
 *   w        [B][F][C] of w_dtype
 *   post_mask, norm, wave, n_out as above */
int setk_apply_istft(setk_plan_t* plan, const float* audio, const int32_t* n_samples,
                     int32_t B, int32_t N, const void* w, int32_t w_dtype,
                     const float* post_mask, int32_t n_out, const float* norm,
                     float* wave, void* stream);

/* The same, through to the wav writer: the pass that applies inverse_stft's `norm`
 * rescale (utils.py:166-168) also performs WaveWriter.write -> write_wav's float ->
 * PCM-16 conversion (data_handler.py:600-605, utils.py:45-62; soundfile's default
 * subtype = floor(y * 32768) clipped, SURVEY.md finding 3), so the float wave is
 * never written out: bit-identical to setk_apply_istft + setk_float_to_pcm16.
 *   norm  f32 [B] or NULL (no rescale)      pcm  i16 [B][n_out] */
int setk_apply_istft_pcm16(setk_plan_t* plan, const float* audio, const int32_t* n_samples,
                           int32_t B, int32_t N, const void* w, int32_t w_dtype,
                           const float* post_mask, int32_t n_out, const float* norm,
                           int16_t* pcm, void* stream);

/*
 * CGMM time-frequency mask estimation from audio: the tile STFT, then
 * CgmmTrainer(stft, num_classes, gamma=init, update_alpha=...).train(num_iters)
 * (scripts/sptk/libs/cluster.py:396-465 with 94-130, 187-287) for every utterance
 * of the batch, and the CLI's transpose (scripts/sptk/estimate_cgmm_masks.py:36-60).
 * fp64 arithmetic after the complex64 STFT, like the reference.
 *
 *   num_classes  2..4.  init_gamma == NULL needs num_classes == 2 (the reference's
 *                deterministic start R_0 = sum_t y y^H / T, R_1 = I; for more classes
 *                it draws numpy random posteriors -- pass them in).
 *   init_gamma   f32 [B][K][T][F] starting posteriors or NULL
 *   update_alpha nonzero: the priors follow mean_t gamma (cluster.py:251-252)
 *   masks        f32 [B][K][T][F]  (the reference writes masks[0] when K == 2)
 *   status       u32 [B] or NULL, OR-ed SETK_ST_NO_CONVERGE (caller zeroes it)
 * Needs n_fft 512 or 1024 (the tile STFT); SETK_EUNSUPPORTED otherwise.
 */
int setk_cgmm_masks(setk_plan_t* plan, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                    int32_t num_classes, int32_t num_iters, const float* init_gamma, int32_t update_alpha,
                    float* masks, uint32_t* status, void* stream);

/*
 * The same estimator for a caller that brings its own STFT -- the reference's
 * CgmmTrainer(obs, num_classes, gamma, update_alpha).train(num_iters) signature
 * (cluster.py:401-466).  Plan-free; scratch is stream-ordered (cudaMallocAsync).
 *   stft   c64 [B][C][F][T]  (forward_stft with transpose=False, stacked over channels)
 *   other arguments as for setk_cgmm_masks; any F, T >= 1.
 */
int setk_cgmm_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t num_classes,
                   int32_t num_iters, const float* init_gamma, int32_t update_alpha, float* masks,
                   uint32_t* status, void* stream);

#define SETK_PERMU_MAX_ROWS 64   /* rows of a permutation-alignment sub-band plan */

/*
 * CACGMM speaker-mask estimation from audio: the tile STFT, then
 * CacgmmTrainer(stft, num_classes, gamma=init, cgmm_init=..., update_alpha=...).train(num_iters)
 * (scripts/sptk/libs/cluster.py:468-535 with 39-45, 94-136, 290-393) for every utterance of the
 * batch, then, when permu_plan is given, permu_aligner (cluster.py:48-91) on the fp64 posteriors,
 * and the CLI's transpose (scripts/sptk/estimate_cacgmm_masks.py:40-63).  fp64 arithmetic after
 * the complex64 STFT, on the observations normalised over channels.
 *
 *   num_classes  2..4
 *   init_gamma   f64 [B][K][T][F] starting posteriors (the reference's numpy draw, or a given
 *                mask), or NULL with cgmm_init && num_classes == 2
 *   cgmm_init    nonzero with num_classes == 2: the start B_0 = sum_t z z^H / T, B_1 = I and one
 *                E-step (cluster.py:495-506); otherwise the start is init_gamma, no E-step
 *   update_alpha nonzero: the priors follow mean_t gamma (cluster.py:364-365)
 *   permu_plan   host i32 [R][3] rows (iterations, first bin, end bin), 0 <= lo < hi <= F,
 *                R <= SETK_PERMU_MAX_ROWS, or NULL / R = 0: no alignment
 *   masks        f32 [B][K][T][F], 0 past each utterance's frames
 *   status       u32 [B] or NULL, OR-ed SETK_ST_NO_CONVERGE (caller zeroes it)
 * num_iters = 0 returns the start.  SETK_EINVAL for a null buffer, K outside 2..4, C < 2,
 * num_iters < 0, a NULL start without cgmm_init && K == 2, or a bad plan row; SETK_EUNSUPPORTED
 * unless n_fft is 512 or 1024 (the tile STFT).
 */
int setk_cacgmm_masks(setk_plan_t* plan, const float* audio, const int32_t* n_samples, int32_t B, int32_t N,
                      int32_t num_classes, int32_t num_iters, const double* init_gamma, int32_t cgmm_init,
                      int32_t update_alpha, const int32_t* permu_plan, int32_t R, float* masks, uint32_t* status,
                      void* stream);

/*
 * The same estimator for a caller that brings its own STFT -- the reference's
 * CacgmmTrainer(obs, num_classes, gamma, cgmm_init, update_alpha).train(num_iters) signature
 * (cluster.py:468-535).  Plan-free; scratch is stream-ordered (cudaMallocAsync).
 *   stft   c64 [B][C][F][T]; other arguments as for setk_cacgmm_masks; any F, T >= 1.
 */
int setk_cacgmm_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t num_classes,
                     int32_t num_iters, const double* init_gamma, int32_t cgmm_init, int32_t update_alpha,
                     const int32_t* permu_plan, int32_t R, float* masks, uint32_t* status, void* stream);

/*
 * permu_aligner(masks) (cluster.py:48-91) for a batch of fp64 masks: per utterance, the features
 * are the masks normalised over its own frames; every plan row (iters, lo, hi) re-orders the
 * classes of each bin in [lo, hi) to the best permutation against the band's centroid, up to
 * `iters` times or until no bin moves.  Exact score ties keep the current order.
 *   masks    f64 [B][K][T][F]        n_frames  i32 [B] device, or NULL (every utterance has T)
 *   plan     host i32 [R][3] as for setk_cacgmm_masks, 1 <= R <= SETK_PERMU_MAX_ROWS
 *   out      f32 [B][K][T][F] the masks gathered through the mapping, 0 past each n_frames
 *   mapping  i32 [B][K][F] or NULL: source class of slot k in bin f
 * Plan-free.  SETK_EINVAL for a null buffer, K outside 2..4, B, T or F < 1, or a bad plan row;
 * SETK_EUNSUPPORTED when F is too large for the per-bin tables in shared memory.
 */
int setk_permu_align(const double* masks, const int32_t* n_frames, int32_t B, int32_t K, int32_t T, int32_t F,
                     const int32_t* plan, int32_t R, float* out, int32_t* mapping, void* stream);

/*
 * WPE dereverberation of a multichannel STFT: libs/wpe.py wpe(reverb, taps, delay,
 * context, num_iters) (scripts/sptk/libs/wpe.py:82-110 with 14-79; driven by
 * apply_wpe.py:36-52) for every utterance of the batch.  Plan-free; scratch is
 * stream-ordered.  fp64 arithmetic (the reference computes in complex64 for
 * complex64 input).
 *   stft   c64 [B][C][F][T]   (the reference's F x N x T per utterance, channel-major here)
 *   out    c64 [B][C][F][T]   dereverberated
 *   status u32 [B] or NULL, SETK_ST_SINGULAR when solve(R, r) hits an exactly singular
 *          matrix (numpy.linalg.LinAlgError in the reference, caught per utterance by its CLI)
 * channels x taps <= 128 and the bin's time series must fit shared memory
 * (SETK_EUNSUPPORTED otherwise; 8 ch x 10 taps x 10 s at hop 256 does).
 */
int setk_wpe_stft(const void* stft, int32_t B, int32_t C, int32_t F, int32_t T, int32_t taps, int32_t delay,
                  int32_t context, int32_t num_iters, void* out, uint32_t* status, void* stream);

/* One WPE step with a caller-supplied variance: the dereverberation stage of facted_wpd
 * (libs/wpe.py:113-177; wpe_step 58-77 with lambda from the previous WPD output, 150-153).
 *   stft        c64 [B][C][F][T]
 *   lambda_enh  c64 [B][F][T] or NULL: lambda = max(|lambda_enh|^2, eps32); NULL: compute_lambda(stft, context)
 *               (then the call equals setk_wpe_stft with num_iters = 1)
 *   out         c64 [B][C][F][T]   dereverberated observations
 *   inv_lambda  f32 [B][T][F] or NULL: 1 / lambda, the frame weights of Rd (wpe.py:165) in the layout
 *               setk_cov takes as a mask
 *   status      u32 [B] or NULL (SETK_ST_SINGULAR like setk_wpe_stft) */
int setk_wpe_step(const void* stft, const void* lambda_enh, int32_t B, int32_t C, int32_t F, int32_t T,
                  int32_t taps, int32_t delay, int32_t context, void* out, float* inv_lambda,
                  uint32_t* status, void* stream);

/* ---- spatial features on explicit STFTs: scripts/sptk/libs/spatial.py (SURVEY.md 8f rank 3) ---- */

/* ipd(si, sj, cos, sin): spatial.py:163-181.  si, sj c64 [rows][F] (rows = B*T);
 *   mode 0: np.mod(angle(si) - angle(sj) + pi, 2 pi) - pi   -> out f32 [rows][F]
 *   mode 1: cos(angle(si) - angle(sj))                      -> out f32 [rows][F]
 *   mode 2: [cos | sin]                                     -> out f32 [rows][2F] */
int setk_ipd(const void* si, const void* sj, int64_t rows, int32_t F, int32_t mode, float* out,
             void* stream);

/* directional_feats(spectrogram, steer_vector, df_pair): spatial.py:184-208.
 *   stft   c64  [B][M][F][T]
 *   steer  c128 [M][F] (steer_batched == 0) or [B][M][F]
 *   pairs  i32  [n_pairs][2] or NULL (all i < j)
 *   out    f64  [B][T][F] = mean over pairs of cos((arg x_i - arg x_j) - (arg d_i - arg d_j)) */
int setk_directional_feats(const void* stft, const void* steer, int32_t steer_batched,
                           const int32_t* pairs, int32_t n_pairs, int32_t B, int32_t M, int32_t F,
                           int32_t T, double* out, void* stream);

/* gcc_phat_linear / gcc_phat_diag: spatial.py:37-92 (the caller supplies the TDOA grid that
 * linear_tdoa_grid, 11-34, or the circular-array formula, 78-80, produce).
 *   si, sj c64 [T][F];  omega f64 [F] (rad/s);  tau f64 [D] (s)
 *   spectrum = Re(exp(j (angle si - angle sj)) @ exp(-j outer(omega, tau)))      [T][D]
 *   normalize:   spectrum /= max(max |spectrum|, eps32);  apply_floor: max(spectrum, 0)
 *   accumulate != 0: out += spectrum (srp_phat_linear, 95-123, sums the pairs) else out = spectrum
 *   work   f64 [setk_gcc_phat_work_doubles(T, F, D)] scratch;  out f64 [T][D] */
int64_t setk_gcc_phat_work_doubles(int32_t T, int32_t F, int32_t D);
int setk_gcc_phat(const void* si, const void* sj, int32_t T, int32_t F, const double* omega,
                  const double* tau, int32_t D, int32_t normalize, int32_t apply_floor,
                  int32_t accumulate, double* work, double* out, void* stream);

/* msc(spectrogram, context, normalize): spatial.py:126-160, as written (the diagonal terms
 * enter as their grand total, np.sum without an axis at :153).
 *   spec c64 [N][T][F];  work f64 [setk_msc_work_doubles(T, F)];  out f64 [T][F] */
int64_t setk_msc_work_doubles(int32_t T, int32_t F);
int setk_msc(const void* spec, int32_t N, int32_t T, int32_t F, int32_t context, int32_t normalize,
             double* work, double* out, void* stream);

/* ---- sound source localisation on explicit STFTs: scripts/sptk/libs/ssl.py, do_ssl.py ---- */
#define SETK_SSL_ML 0           /* ml_ssl    ssl.py:12-43 (do_ssl.py:34 passes compression=-1, eps=EPSILON) */
#define SETK_SSL_SRP 1          /* srp_ssl   ssl.py:46-77 */
#define SETK_SSL_MUSIC 2        /* music_ssl ssl.py:80-110 */
#define SETK_SSL_MAX_MASKS 8

/*
 * DoA scores and their arg-extreme for every (utterance, mask, frame window, direction).
 *   backend      SETK_SSL_*
 *   stft         c64 [B][M][F][T]     (the reference's M x T x F per utterance, bins before frames here)
 *   steer        c128 [A][M][steer_F] steering vectors as np.load gives them (compute_steer_vector.py:44-51,
 *                do_ssl.py:49); ML normalises them over microphones (ssl.py:27), MUSIC uses them as given
 *   steer_F      bins of the steering table: SETK_ESHAPE unless it equals F
 *   mask         f32 [B][N][T][F] or NULL (ssl.py:24-25,58-61,91-92: all ones); N > 1 is the 3-D mask of
 *                ml_ssl (ssl.py:41-42), ML only, N <= SETK_SSL_MAX_MASKS; N must be 1 when mask is NULL
 *   windows_host i32 [B][W][2] HOST array of frame ranges [s, e), 0 <= s < e <= T: [0, T) offline, the
 *                chunks [max(t - look_back, 0), t + chunk_len) of do_ssl.py's online mode (:103-111)
 *   pairs_host   i32 [P][2] HOST array of microphone pairs (l, r), SRP only (srp_pair, ssl.py:62; do_ssl.py:70-74)
 *   compression  ML: <= 0 -> -log(max(delta, eps)), else -delta**compression (ssl.py:34-37)
 *   eps          ML: floor of delta and of |x| for normalize, delta = ssh - ssv / (1 + eps) (ssl.py:29,33)
 *   normalize    ML: x / max(|x|, eps) first (norm=True, ssl.py:28-29)
 *   scores       f64 [B][N][W][A]: ML the masked log-likelihood sum (ssl.py:39-42), SRP the masked mean
 *                pair response (:71-76), MUSIC sum_f |s^H (I - u u^H) s| (:93-109)
 *   index        i32 [B][N][W]: numpy's argmax of the scores (ML, SRP) or argmin (MUSIC) -- the first
 *                extreme, or the first NaN when there is one
 * Plan-free; scratch is stream-ordered.  SETK_EINVAL for an unknown backend, N > 1 with SRP or MUSIC, a
 * pair index outside [0, M), A < 1, a window outside [0, T] or empty, M > SETK_MAX_CHANNELS.
 */
int setk_ssl(int32_t backend, const void* stft, int32_t B, int32_t M, int32_t F, int32_t T, const void* steer,
             int32_t A, int32_t steer_F, const float* mask, int32_t N, const int32_t* windows_host, int32_t W,
             const int32_t* pairs_host, int32_t P, double compression, double eps, int32_t normalize,
             double* scores, int32_t* index, void* stream);

/*
 * AuxIVA: scripts/sptk/apply_auxiva.py:24-57 for every utterance of the batch.  Plan-free; scratch is
 * stream-ordered.  fp64 after the complex64 input.
 *   stft    c64  [B][N][F][T]   (the reference's N x T x F per utterance, bins before frames here)
 *   out     c128 [B][N][F][T]   separated sources Y (the reference returns complex128)
 *   status  u32 [B] or NULL     SETK_ST_SINGULAR / SETK_ST_NONFINITE (-> numpy.linalg.LinAlgError per key;
 *                               caller zeroes it)
 * 2 <= N <= SETK_MAX_CHANNELS, num_epochs >= 0 (0 returns X), F, T >= 1; SETK_EINVAL otherwise.
 */
int setk_auxiva_stft(const void* stft, int32_t B, int32_t N, int32_t F, int32_t T, int32_t num_epochs,
                     void* out, uint32_t* status, void* stream);

/* ---- single-channel noise suppression: scripts/sptk/libs/ns.py iMCRA, apply_ns.py ---- */
#define SETK_NS_MAX_W 8         /* w_mcra <= 8: at most 17 smoothing taps */
#define SETK_NS_MAX_U 64        /* U <= 64 frames of sub-window minima */
#define SETK_NS_MAX_BINS 2049   /* F <= 2049 (n_fft 4096) */

typedef struct setk_imcra_config {   /* iMCRA.__init__ keywords, ns.py:221-245, and run(eps), ns.py:247 */
  double alpha, alpha_s, alpha_d, b_min, gamma0, gamma1, zeta0, xi_min_db, gmin_db, beta, eps;
  int32_t w_mcra, V, U, reserved;
  const double* window_host;         /* HOST pointer, 2*w_mcra+1 values of
                                        scipy.signal.get_window(h_mcra, 2*w_mcra+1) (ns.py:243) */
} setk_imcra_config_t;

/*
 * iMCRA noise estimation + OM-LSA gain: iMCRA(**cfg).run(stft, eps) (ns.py:247-387) for every
 * utterance of the batch; apply_ns.py:41-42 multiplies the gain into the STFT.  Plan-free; scratch (only
 * when U > V) is stream-ordered.  fp64 after the complex64 input.
 *   stft      c64 [B][F][T]   (the reference's T x F per utterance, bins before frames here: what a
 *                              one-channel setk_stft writes)
 *   n_frames  i32 [B] or NULL (= T): utterance b runs over its first n_frames[b] frames; later frames
 *                              get gain 0 and enh 0
 *   gain      f64 [B][T][F] or NULL   the reference's T x F gain (ns.py:383-387)
 *   enh       c64 [B][F][T] or NULL   gain * stft (apply_ns.py:42), ready for setk_istft
 * Per frame (ns.py line by line): lambda_d = beta lambda_d_hat (269); gamma (272, NOT floored); xi_hat
 * (275-280); v, gh1 = xi/(1+xi) exp(E1(v)/2) (283-284); var_sf = conv(|x|^2, w_m, "same") (288);
 * var_s and its minima (291-301); indicator (304-307); var_sf_hat from the previous var_s_hat (311-317);
 * var_s_hat and its minima (320-329); q_hat, p_hat (332-358); lambda_d_hat (362-367); every V frames
 * the minima over the last U per-frame sub-window minima (370-380); gain = gh1^p gmin^(1-p) (383).
 * E1(0) is the 37.191280375549404 the reference's quad returns there, not +inf.
 * SETK_EINVAL: a null cfg, window or stft; gain and enh both NULL; B, F or T < 1;
 * F > SETK_NS_MAX_BINS; w_mcra outside [0, SETK_NS_MAX_W]; F < 2*w_mcra+1 (np.convolve would swap
 * its operands, ns.py:288); V < 1; U outside [1, SETK_NS_MAX_U].
 */
int setk_ns_imcra(const setk_imcra_config_t* cfg, const void* stft, const int32_t* n_frames, int32_t B,
                  int32_t F, int32_t T, double* gain, void* enh, void* stream);

/* ---- room impulse responses: include/rir-generator.{h,cc} (rir-simulate), rir_generate_{1d,2d}.py ---- */
#define SETK_MIC_OMNI 0                /* rho = 1     rir-generator.cc:196-212 */
#define SETK_MIC_SUBCARDIOID 1         /* rho = 0.75 */
#define SETK_MIC_CARDIOID 2            /* rho = 0.5  */
#define SETK_MIC_HYPERCARDIOID 3       /* rho = 0.25 */
#define SETK_MIC_BIDIRECTIONAL 4       /* rho = 0    */
#define SETK_RIR_MAX_TW 512            /* window taps Tw <= 512: fs < 64125 Hz */
#define SETK_RIR_MAX_HALF 2048         /* lattice half-width n = ceil(L / (2 T)) <= 2048 per axis */
#define SETK_RIR_MAX_CANDIDATES 4294967296.0   /* 8 (2nx+1)(2ny+1)(2nz+1) <= 2^32 images per channel */

typedef struct setk_rir_config {
  double sound_velocity, samp_frequency;         /* c, fs; both >= 1 (rir-generator.cc:29-30) */
  double azimuth, elevation;                     /* receiver orientation, radians (only for non-omni) */
  int32_t n_samples, order, mic_type, hp_filter; /* L >= 1; order >= -1 (-1: every order); SETK_MIC_* */
} setk_rir_config_t;

/*
 * Image-method room impulse responses: RirGenerator::GenerateRir (rir-generator.cc:108-192, with
 * MicrophoneSim 194-223 and Sinc, rir-generator.h:156) for B problems b = (room, beta, source), each
 * with M receivers.  Plan-free; scratch (several segments with the filter) is stream-ordered.  The
 * call reads `room` back to the host to check it and size the launch, so it synchronises `stream`.
 *   room       f64 [B][3]     room dimensions, metres
 *   beta       f64 [B][6]     reflection coefficients of the walls x=0, x=Lx, y=0, y=Ly, z=0, z=Lz
 *                             (a T60 becomes these on the host: setk_b200.plan.rir_beta,
 *                             rir-generator.cc:78-92)
 *   source     f64 [B][3]     metres
 *   receivers  f64 [B][M][3]  metres
 *   rir        f32 [B][M][L]  the response, written whole
 *   status     u32 [B] or NULL  SETK_ST_NONFINITE when a tap is not finite or |tap| >= 4096, or a
 *                             sample leaves the accumulator's range (caller zeroes it)
 * Per image (x, y, z in [-n, n], q, j, k in {0, 1}): distance in samples from (1-2q)S - R + 2xT,
 * reflection factor beta0^|x-q| beta1^|x| beta2^|y-j| beta3^|y| beta4^|z-k| beta5^|z|, kept when
 * |2x-q| + |2y-j| + |2z-k| <= order (or order == -1) and floor(dist) < L; Tw = 2 int(0.004 fs + 0.5)
 * Hann-windowed sinc taps from floor(dist) - Tw/2 + 1, gain mic * refl / (4 pi dist c/fs), taps
 * outside [0, L) dropped; then the 100 Hz high-pass (180-190) when hp_filter != 0.
 * Differences from the reference: distances, floor and frac are fp64 (the reference's float32
 * geometry is most of its own error), taps float32, the sum 64-bit fixed point (2^-44 per unit) so
 * two calls are bit-identical, the high-pass fp64.
 * SETK_EINVAL: a null pointer; B, M or L < 1; B or M > 65535; c or fs < 1; order < -1; an unknown
 * mic_type; a room dimension <= 0 (the reference divides by it).
 * SETK_EUNSUPPORTED: Tw > SETK_RIR_MAX_TW; a lattice half-width > SETK_RIR_MAX_HALF; more than
 * SETK_RIR_MAX_CANDIDATES images per channel (a 1 m cube at 16 kHz reaches it at L = 38 119, 2.4 s).
 */
int setk_rir_image(const setk_rir_config_t* cfg, const double* room, const double* beta, const double* source,
                   const double* receivers, int32_t B, int32_t M, float* rir, uint32_t* status, void* stream);

/* ---- speech + RIR + noise mixture simulation (scripts/sptk/wav_simulate.py; csrc/simu.cu) ---- */
#define SETK_CONV_MAX_LEN (1 << 24)   /* Sx, Lh and Ny each <= 2^24 samples (17 min at 16 kHz) */
#define SETK_SIMU_MAX_TERMS 64        /* terms per mixture */

/*
 * Batched long linear convolution: ss.convolve(spk[None], rir)[..., :S] of add_room_response
 * (wav_simulate.py:29-54, minus the power) for B problems, each a mono source and an M-channel filter:
 *   y[b][m][n] = sum_k x[b][n - k] h[b][m][k],  n < n_out_b;  y[b][m][n] = 0 for n_out_b <= n < Ny.
 *   x  f32 [B][Sx]     source b is x[b][0 .. S_b)
 *   h  f32 [B][M][Lh]  filter b is h[b][m][0 .. L_b)
 *   y  f32 [B][M][Ny]  written whole
 *   s_len_host, h_len_host, n_out_host  i32 [B] on the host, or NULL for Sx, Lh and Ny; n_out_b = S_b
 *   is the reference's truncation, S_b + L_b - 1 the full convolution (any n_out_b in [1, Ny] is accepted).
 * Uniformly partitioned overlap-save, 1024-sample blocks, fp32 FFTs in shared memory with exact twiddles;
 * deterministic (a problem gives the same bits alone and inside a batch).  Scratch (the spectra,
 * 8 (P + 1) B (ceil(Ny / P) + M ceil(Lh / P)) bytes) is stream-ordered.
 * SETK_EINVAL: a null pointer; B, M, Sx, Lh or Ny < 1; B or M > 65535; S_b, L_b or n_out_b outside
 * [1, Sx], [1, Lh], [1, Ny].  SETK_EUNSUPPORTED: Sx, Lh or Ny > SETK_CONV_MAX_LEN.
 */
int setk_convolve(const float* x, int32_t Sx, const float* h, int32_t Lh, int32_t B, int32_t M,
                  const int32_t* s_len_host, const int32_t* h_len_host, const int32_t* n_out_host, float* y,
                  int32_t Ny, void* stream);

#define SETK_SIMU_SPEAKER 0
#define SETK_SIMU_POINT_NOISE 1
#define SETK_SIMU_ISOTROPIC 2

typedef struct setk_simu_term {
  int64_t src;                     /* offset (floats) of the image's channel 0 in `pool` */
  int32_t kind;                    /* SETK_SIMU_* */
  int32_t n_channels;              /* 1 (added to every channel) or the mixture's channel count */
  int32_t pitch;                   /* floats between the image's channels */
  int32_t begin, length;           /* the image lands on mixture samples [begin, begin + length) */
  int32_t repeat;                  /* 1: image sample 0 is added at every one of those samples */
  int32_t power_begin, power_end;  /* the image's channel-0 samples its power is taken over */
  int32_t reserved;
  double level_db;                 /* SDR of a speaker after the first, SNR of a noise */
} setk_simu_term_t;

typedef struct setk_simu_mix {
  int32_t first_term, n_terms;     /* its terms: speakers, then point noises, then at most one isotropic */
  int32_t n_samples, n_channels;   /* mix_nsamps (<= n_pitch) and N (<= M) */
  double norm_factor;
} setk_simu_mix_t;

/*
 * Mixing and normalisation of run_simu (wav_simulate.py:166-312) for B mixtures whose images (the
 * convolved or raw sources and noises, float32) lie in `pool`:
 *   - power of every image on its channel 0 over [power_begin, power_end), fp64 (add_room_response :54,
 *     add_speaker :72, add_point_noise :124, isotropic :295);
 *   - speaker 0 has coefficient 1, speaker k coeff_snr(P_k, P_0, sdr_k) (:87-92);
 *   - P_spk = mean over n_samples of the scaled speakers' channel-0 sum (:252-255);
 *   - every noise coeff_snr(P_noise, P_spk, snr) (:141, :296);
 *   - mix = (sum of speakers + sum of point noises) + isotropic, per channel and sample, terms added in
 *     table order in fp64; an image of one channel is added to every channel;
 *   - factor = norm_factor / (max |mix| + EPSILON) over every channel (:304), and the outputs
 *       mix    [B][M][n_pitch]  mix times factor (channels >= N and samples >= n_samples are 0),
 *       spk    [B][K][n_pitch]  channel 0 of each scaled speaker times factor, or NULL,
 *       noise  [B][n_pitch]     channel 0 of point noises + isotropic times factor, or NULL,
 *       factor f64 [B]          or NULL,
 *     float32, or with pcm16 != 0 int16 floor(y * 32768) clipped (write_wav's PCM-16).
 * The term tables are host arrays, copied on `stream`; nothing synchronises the host.
 * SETK_EINVAL: a null pointer (pool, tables, mix); B, n_terms, M, K or n_pitch < 1; a mixture with no
 * speaker, more than K speakers, terms out of order, more than one isotropic term, a term range outside
 * the table, n_samples outside [1, n_pitch] or n_channels outside [1, M]; a term whose n_channels is
 * neither 1 nor the mixture's (an isotropic term must have 1), whose samples fall outside
 * [0, n_samples), whose image or power range falls outside the pool, or an empty power range.
 * SETK_EUNSUPPORTED: more than SETK_SIMU_MAX_TERMS terms in one mixture.
 */
int setk_simulate_mix(const float* pool, int64_t pool_len, const setk_simu_mix_t* mixes_host, int32_t B,
                      const setk_simu_term_t* terms_host, int32_t n_terms, int32_t M, int32_t K, int32_t n_pitch,
                      int32_t pcm16, void* mix, void* spk, void* noise, double* factor, void* stream);

/* ---- separation metrics (scripts/sptk/compute_sdr.py, compute_si_snr.py, libs/metric.py; csrc/sep_eval.cu) ---- */
#define SETK_SEP_MAX_SOURCES 8          /* N in [1, 8] */
#define SETK_SEP_MAX_FLEN 512           /* L in [1, 512] (mir_eval's bss_eval_sources uses 512) */
#define SETK_SEP_MAX_COLS 4096          /* N * L <= 4096: the least-squares system is N L square */
#define SETK_SEP_MAX_SAMPLES (1 << 24)  /* S <= 2^24 samples (17 min at 16 kHz) */

/*
 * BSS-Eval v3 sources criteria: what mir_eval.separation.bss_eval_sources(ref, sep) computes for
 * compute_sdr.py:63-80 (its _bss_decomp_mtifilt, _project and _bss_source_crit), for every (estimate j,
 * reference i) pair of B utterances, with the filter length L:
 *   est, ref   f32 [B][N][S]     utterance b is [.][.][0 .. n_b)
 *   n_samples_host  i32 [B] on the host, or NULL for S; each n_b in [1, S]
 *   crit       f64 [B][3][N][N]  SDR, SIR, SAR of estimate j against reference i at [b][k][j][i]
 *   dropped    i32 [B] or NULL   columns of the N L square least-squares system found dependent
 *   status     u32 [B]           written: SETK_ST_SILENT when a reference or estimate is all zeros (the
 *                                criteria are then meaningless), SETK_ST_NONFINITE for a NaN criterion
 * With A_i the delayed copies s_i[n - a], a < L, of reference i over n < n_b + L - 1, P_all(j) is
 * estimate j's least-squares projection onto every A_i and P_spat(j, i) onto A_i alone:
 *   SDR = 10 log10(|P_spat|^2 / |e_j - P_spat|^2), SIR = 10 log10(|P_spat|^2 / |P_all - P_spat|^2),
 *   SAR = 10 log10(|P_all|^2 / |e_j - P_all|^2), +inf when the denominator is 0.
 * Differences from mir_eval: the correlations are direct fp64 sums, not float64 FFTs; the normal
 * equations are solved by Cholesky, and a column whose pivot is <= 1e-10 of its original diagonal is
 * dropped, so dependent references (where numpy.linalg.solve is ill-posed) still give the least-squares
 * projection; the residual energies come from the signals.  The permutation search is the caller's
 * (setk_b200.libs.metric).  Deterministic: an utterance gives the same bits alone as inside a batch.
 * Scratch, setk_bss_eval_scratch_bytes(B, N, S, L): about 8 B (N L)^2 bytes for the system plus
 * 8 B (N L (4 N + 2) + 24 N (N + 1) (S + L) / 256) bytes; it is stream-ordered.
 * SETK_EINVAL: a null pointer (est, ref, crit, status); B, N, S or L < 1; B > 65535; an n_b outside
 * [1, S].  SETK_EUNSUPPORTED: N > SETK_SEP_MAX_SOURCES, L > SETK_SEP_MAX_FLEN, N L > SETK_SEP_MAX_COLS,
 * S > SETK_SEP_MAX_SAMPLES.
 */
int setk_bss_eval(const float* est, const float* ref, const int32_t* n_samples_host, int32_t B, int32_t N, int32_t S,
                  int32_t L, double* crit, int32_t* dropped, uint32_t* status, void* stream);
/* Bytes of device scratch setk_bss_eval allocates for these sizes (callers that split a batch to bound
 * it ask here); -1 when setk_bss_eval would reject the sizes. */
int64_t setk_bss_eval_scratch_bytes(int32_t B, int32_t N, int32_t S, int32_t L);

/*
 * SI-SNR of every (estimate j, reference i) pair: si_snr(x, s, eps, remove_dc) of libs/metric.py:13-34,
 * as compute_si_snr.py:82-106 and permute_si_snr (:37-60) call it:
 *   20 log10(|t| / (|x' - t| + eps) + eps),  t = <x', s'> s' / (|s'|^2 + eps),
 * x', s' the estimate and reference less their means when remove_dc != 0.
 *   est, ref   f32 [B][N][S]; n_samples_host as for setk_bss_eval
 *   out        f64 [B][N][N]     at [b][j][i]
 * fp64 throughout (the reference computes in float32); |x' - t| is taken from the residual's samples.
 * SETK_EINVAL: a null pointer; B, N or S < 1; B > 65535; eps < 0 or not finite; an n_b outside [1, S].
 * SETK_EUNSUPPORTED: N > SETK_SEP_MAX_SOURCES, S > SETK_SEP_MAX_SAMPLES.
 */
int setk_si_snr(const float* est, const float* ref, const int32_t* n_samples_host, int32_t B, int32_t N, int32_t S,
                int32_t remove_dc, double eps, double* out, void* stream);

/* floor(y * 32768) clipped to int16: the PCM_16 conversion of
 * WaveWriter.write -> write_wav -> soundfile (data_handler.py:600-605,
 * utils.py:45-62; SURVEY.md finding 3).  wave f32 [n], pcm i16 [n]. */
int setk_float_to_pcm16(const float* wave, int64_t n, int16_t* pcm, void* stream);
/* int16 / 32768 -> float32: read_wav (utils.py:80-92). */
int setk_pcm16_to_float(const int16_t* pcm, int64_t n, float* wave, void* stream);

/* Kaldi CompressedMatrix masks, format "CM" (per-column percentile headers + one byte per element),
 * expanded on the device: kaldi_io.py:248-281 uncompress() as reached by the mask ScriptReader of
 * apply_adaptive_beamformer.py:139-142 (--mask-format kaldi), same float32 operations, bit-identical.
 *   blobs  u8  [B][slot_bytes]  one matrix per slot exactly as it lies in the archive behind the "CM "
 *                               token: {f32 min, f32 range, i32 rows, i32 cols}, cols x 4 u16,
 *                               cols x rows u8 (column major); slot_bytes a multiple of 16
 *   out    f32 [B][T][F]        rows t < rows_b decoded, the rest zero (ragged batches)
 *   status i32 [B]              set to 1 where a header is inconsistent (cols != F, rows > T, the
 *                               matrix does not fit its slot); that matrix decodes to zeros */
int setk_cm_masks(const uint8_t* blobs, int64_t slot_bytes, int32_t B, int32_t T, int32_t F, float* out,
                  int32_t* status, void* stream);

/* How many kernels of this library have been launched by this process
 * (for bench.py's "gpu_launches"). */
int64_t setk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* SETK_B200_H_ */
