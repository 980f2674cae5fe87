"""
setk_b200.plan -- Python handle on a libsetk_b200 STFT plan plus the plan-free
entry points, operating on torch tensors (device memory, streams) and calling
the CUDA kernels through the C-ABI.  PyTorch is plumbing here: it owns the
buffers and the stream; every arithmetic step is a kernel of libsetk_b200.

Layouts are the reference's (scripts/sptk/libs): audio (B,C,N) f32, mask
(B,T,F) f32, stft (B,C,F,T) c64, R (B,F,C,C), weight (B,F,C), enhanced
(B,F,T) c64, wave (B,N_out) f32.
"""
import contextlib
import ctypes
import math

import numpy as np
import scipy.signal
import torch

from . import _lib

EPSILON = float(np.finfo(np.float32).eps)  # libs/utils.py:16


def nextpow2(window_size):
    """libs/utils.py:25-27"""
    return 2**math.ceil(math.log2(window_size))


def make_window(window, frame_len):
    """
    Analysis window, float64, length frame_len: librosa's
    get_window(window, frame_len, fftbins=True); "sqrthann" as in
    libs/utils.py:116-117.
    """
    if isinstance(window, str):
        if window == "sqrthann":
            return scipy.signal.get_window("hann", frame_len, fftbins=True)**0.5
        return scipy.signal.get_window(window, frame_len, fftbins=True)
    if isinstance(window, torch.Tensor):
        window = window.detach().cpu().numpy()
    window = np.ascontiguousarray(window, dtype=np.float64)
    if window.shape != (frame_len,):
        raise ValueError(f"Window size mismatch: {window.shape} vs {frame_len}")
    return window


def _dtype_code(t):
    if t.dtype == torch.complex64:
        return _lib.C64
    if t.dtype == torch.complex128:
        return _lib.C128
    raise TypeError(f"expected a complex64/complex128 tensor, got {t.dtype}")


def _arg(t, dev, dtype, shape, what):
    """
    A tensor input of a C-ABI call: `t` as a contiguous tensor on `dev` (None: where it is) of `dtype`
    (None: its own), or None for None.  `shape` None takes any shape; else every entry that is not None
    must match, or ValueError names `what`.  Reads metadata only, so it never synchronises the host.
    """
    if t is None:
        return None
    t = torch.as_tensor(t, dtype=dtype, device=dev).contiguous()
    if shape is not None and (t.dim() != len(shape) or any(s is not None and s != n for s, n in zip(shape, t.shape))):
        want = ", ".join("*" if s is None else str(s) for s in shape)
        raise ValueError(f"{what} must be ({want}), got {tuple(t.shape)}")
    return t


def _out(t, dev, dtype, shape, what):
    """A caller's output buffer: the kernel writes it in place, so it is never converted and must already
    be a contiguous `dtype` tensor of `shape` on `dev` (ValueError naming `what` otherwise)."""
    if t.dtype != dtype or tuple(t.shape) != tuple(shape) or t.device != dev or not t.is_contiguous():
        raise ValueError(f"{what} must be a contiguous {dtype} {tuple(shape)} tensor on {dev}, got {t.dtype} "
                         f"{tuple(t.shape)} on {t.device}, contiguous={t.is_contiguous()}")
    return t


def _host_i32(v, shape=None):
    """
    A host table for a C-ABI `const int32_t*` argument: (v as a C-contiguous int32 array, broadcast to
    `shape` when given; the pointer the call takes, which keeps the array alive), or (None, None) for None.
    """
    if v is None:
        return None, None
    a = np.asarray(v, dtype=np.int32)
    a = np.ascontiguousarray(a if shape is None else np.broadcast_to(a, shape))
    return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def _ctx(device):
    return torch.cuda.device(device) if device.type == "cuda" else contextlib.nullcontext()


def _launch(dev, name, *args):
    """libsetk_b200's `name`(*args, stream) on `dev`, on the current stream of `dev`; raises on an error."""
    with _ctx(dev):
        _lib.check(getattr(_lib.library(), name)(*args, _lib.current_stream(dev)))


class StftPlan(object):
    """
    One STFT geometry (mirrors StftParser, libs/opts.py:21-49, and the keyword
    arguments of forward_stft / inverse_stft, libs/utils.py:96-105,142-150).
    """

    def __init__(self, num_channels, frame_len=512, frame_hop=256, center=True,
                 round_power_of_two=True, window="hann", max_batch=1,
                 max_samples=160000, device=None):
        self.device = torch.device(device if device is not None else (
            "cuda" if torch.cuda.is_available() else "cpu"))
        if self.device.type != "cuda" and not _lib.emulated():
            raise RuntimeError("StftPlan needs a CUDA device (setk_b200 has no CPU fallback)")
        self.num_channels = int(num_channels)
        self.frame_len = int(frame_len)
        self.frame_hop = int(frame_hop)
        self.center = bool(center)
        self.n_fft = nextpow2(frame_len) if round_power_of_two else int(frame_len)
        self.num_bins = self.n_fft // 2 + 1
        self.num_mel = 0
        self.max_batch = int(max_batch)
        self.max_samples = int(max_samples)
        win = make_window(window, self.frame_len)
        self._win = np.ascontiguousarray(win, dtype=np.float64)
        cfg = _lib.SetkConfig(
            num_channels=self.num_channels, frame_len=self.frame_len,
            n_fft=self.n_fft, frame_hop=self.frame_hop, center=int(self.center),
            max_batch=self.max_batch, max_samples=self.max_samples, reserved=0,
            window_host=self._win.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
        handle = ctypes.c_void_p()
        with _ctx(self.device):
            _lib.check(_lib.library().setk_plan_create(ctypes.byref(cfg), ctypes.byref(handle)))
        self._h = handle

    # ------------------------------------------------------------------ misc
    def close(self):
        if getattr(self, "_h", None):
            try:
                with _ctx(self.device):
                    _lib.library().setk_plan_destroy(self._h)
            finally:
                self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def num_frames(self, nsamps):
        T = _lib.library().setk_num_frames(self._h, int(nsamps))
        if T < 1:
            raise ValueError(f"{nsamps} samples are too short for n_fft={self.n_fft}")
        return T

    def istft_length(self, num_frames):
        return _lib.library().setk_istft_length(self._h, int(num_frames))

    def _check_audio(self, audio):
        return _arg(audio, self.device, torch.float32, (None, self.num_channels, None), "audio")

    # --------------------------------------------------------------- kernels
    def stft(self, audio, n_samples=None):
        """audio (B,C,N) -> (B,C,F,T) complex64.  forward_stft per channel."""
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        out = torch.empty((B, C, self.num_bins, T), dtype=torch.complex64, device=self.device)
        _launch(self.device, "setk_stft", self._h, _lib.ptr(audio), _lib.ptr(ns), B, N, _lib.ptr(out))
        return out

    def stft_cov(self, audio, mask_s, mask_n=None, n_samples=None, clip_mask=False,
                 mask_ft=False, want_maxabs=True):
        """
        Fused STFT + mask-weighted covariance.  Returns (Rs, Rn, maxabs):
        Rs, Rn (B,F,C,C) complex64; maxabs (B,) float32 or None.
        """
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        F = self.num_bins
        mshape = (B, F, T) if mask_ft else (B, T, F)
        mask_s = _arg(mask_s, self.device, torch.float32, mshape, "mask")
        mask_n = _arg(mask_n, self.device, torch.float32, mshape, "mask_n")
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        Rs = torch.empty((B, F, C, C), dtype=torch.complex64, device=self.device)
        Rn = torch.empty_like(Rs)
        maxabs = torch.empty((B,), dtype=torch.float32, device=self.device) if want_maxabs else None
        flags = (_lib.F_CLIP_MASK if clip_mask else 0) | (_lib.F_MASK_FT if mask_ft else 0)
        _launch(self.device, "setk_stft_cov", self._h, _lib.ptr(audio), _lib.ptr(ns), B, N, _lib.ptr(mask_s),
                _lib.ptr(mask_n), flags, _lib.ptr(Rs), _lib.ptr(Rn), _lib.ptr(maxabs))
        return Rs, Rn, maxabs

    def set_mel(self, weights):
        """
        The mel filterbank of spectral_feats(mel=True): weights (M, F) float32 on the host, finite and
        >= 0, 1 <= M <= 1024 (setk_b200.libs.filters.mel builds the reference's); None clears it.
        """
        if weights is None:
            _lib.check(_lib.library().setk_plan_set_mel(self._h, 0, None))
            self.num_mel = 0
            return
        if isinstance(weights, torch.Tensor):
            weights = weights.detach().cpu().numpy()
        w = np.ascontiguousarray(weights, dtype=np.float32)
        if w.ndim != 2 or w.shape[1] != self.num_bins or not 1 <= w.shape[0] <= _lib.FEAT_MAX_MEL:
            raise ValueError(f"mel weights must be (M, {self.num_bins}) with 1 <= M <= {_lib.FEAT_MAX_MEL}, "
                             f"got {w.shape}")
        if not (np.all(np.isfinite(w)) and np.all(w >= 0)):
            raise ValueError("mel weights must be finite and >= 0")
        with _ctx(self.device):
            _lib.check(_lib.library().setk_plan_set_mel(self._h, w.shape[0], w.ctypes.data_as(ctypes.c_void_p)))
        self.num_mel = w.shape[0]

    def spectral_feats(self, audio, n_samples=None, apply_pow=False, mel=False, apply_log=False,
                       sample_scale=1.0):
        """
        audio (B,C,N) -> (B,C,T,D) float32: |STFT| * sample_scale, then squared (apply_pow), projected
        on the mel filters of set_mel (mel, D = M; else D = F) and log(max(., EPSILON)) (apply_log).
        Frames past an utterance's n_samples are zero rows.
        """
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        if mel and not self.num_mel:
            raise ValueError("spectral_feats(mel=True) needs set_mel() first")
        scale = float(sample_scale)
        if not (math.isfinite(scale) and scale > 0):
            raise ValueError(f"sample_scale must be finite and > 0, got {sample_scale}")
        D = self.num_mel if mel else self.num_bins
        out = torch.empty((B, C, T, D), dtype=torch.float32, device=self.device)
        flags = (_lib.FEAT_POW if apply_pow else 0) | (_lib.FEAT_MEL if mel else 0) | \
            (_lib.FEAT_LOG if apply_log else 0)
        _launch(self.device, "setk_spectral_feats", self._h, _lib.ptr(audio), _lib.ptr(ns), B, N, flags, scale,
                _lib.ptr(out))
        return out

    def cgmm_masks(self, audio, num_classes=2, num_iters=20, init_gamma=None, update_alpha=False,
                   n_samples=None):
        """
        CGMM mask estimation from audio (STFT + CgmmTrainer(...).train(num_iters),
        cluster.py:396-465).  init_gamma (B,K,T,F) or None (2 classes only).
        Returns (masks (B,K,T,F) float32, status (B,) int32).
        """
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        F = self.num_bins
        K = int(num_classes)
        init_gamma = _arg(init_gamma, self.device, torch.float32, (B, K, T, F), "init_gamma")
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        masks = torch.empty((B, K, T, F), dtype=torch.float32, device=self.device)
        status = torch.zeros((B,), dtype=torch.int32, device=self.device)
        _launch(self.device, "setk_cgmm_masks", self._h, _lib.ptr(audio), _lib.ptr(ns), B, N, K, int(num_iters),
                _lib.ptr(init_gamma), 1 if update_alpha else 0, _lib.ptr(masks), _lib.ptr(status))
        return masks, status

    def cacgmm_masks(self, audio, num_classes=2, num_iters=50, init_gamma=None, cgmm_init=False,
                     update_alpha=True, permu_plan=None, n_samples=None):
        """
        CACGMM mask estimation from audio (STFT + CacgmmTrainer(...).train(num_iters), cluster.py:468-535),
        then permu_aligner (cluster.py:48-91) on the fp64 posteriors when `permu_plan` rows (iterations,
        first bin, end bin) are given (PERMU_PLANS[F] is the reference's).  init_gamma (B,K,T,F) float64, or
        None with cgmm_init and 2 classes.  Returns (masks (B,K,T,F) float32, status (B,) int32).
        """
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        F = self.num_bins
        K, rows, rows_p, R = _cacgmm_checks(C, num_classes, num_iters, init_gamma, cgmm_init, permu_plan, F)
        init_gamma = _arg(init_gamma, self.device, torch.float64, (B, K, T, F), "init_gamma")
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        masks = torch.empty((B, K, T, F), dtype=torch.float32, device=self.device)
        status = torch.zeros((B,), dtype=torch.int32, device=self.device)
        _launch(self.device, "setk_cacgmm_masks", self._h, _lib.ptr(audio), _lib.ptr(ns), B, N, K, int(num_iters),
                _lib.ptr(init_gamma), int(bool(cgmm_init)), int(bool(update_alpha)), rows_p, R, _lib.ptr(masks),
                _lib.ptr(status))
        return masks, status

    def istft(self, enh, n_out=None, norm=None):
        """enh (B,F,T) complex64 -> wave (B,n_out) float32 (inverse_stft)."""
        enh = _arg(enh, self.device, torch.complex64, (None, self.num_bins, None), "enh")
        B, F, T = enh.shape
        if n_out is None:
            n_out = self.istft_length(T)
        norm = _arg(norm, self.device, torch.float32, (B,), "norm")
        wave = torch.empty((B, int(n_out)), dtype=torch.float32, device=self.device)
        _launch(self.device, "setk_istft", self._h, _lib.ptr(enh), B, T, int(n_out), _lib.ptr(norm), _lib.ptr(wave))
        return wave

    def apply_istft(self, audio, weight, post_mask=None, n_out=None, norm=None, n_samples=None,
                    pcm16=False):
        """Fused beamform + iSTFT from audio.  weight (B,F,C) complex.
        pcm16=True: the `norm` rescale pass writes what WaveWriter would put in the wav file
        (int16 = floor(y * 32768) clipped, utils.py:45-62) instead of float32."""
        audio = self._check_audio(audio)
        B, C, N = audio.shape
        T = self.num_frames(N)
        F = self.num_bins
        weight = _arg(weight, self.device, None, (B, F, C), "weight")
        post_mask = _arg(post_mask, self.device, torch.float32, (B, T, F), "post_mask")
        if n_out is None:
            n_out = self.istft_length(T)
        norm = _arg(norm, self.device, torch.float32, (B,), "norm")
        ns = _arg(n_samples, self.device, torch.int32, (B,), "n_samples")
        wave = torch.empty((B, int(n_out)), dtype=torch.int16 if pcm16 else torch.float32,
                           device=self.device)
        _launch(self.device, "setk_apply_istft_pcm16" if pcm16 else "setk_apply_istft", self._h, _lib.ptr(audio),
                _lib.ptr(ns), B, N, _lib.ptr(weight), _dtype_code(weight), _lib.ptr(post_mask), int(n_out),
                _lib.ptr(norm), _lib.ptr(wave))
        return wave


# ---------------------------------------------------------------- plan-free ---
def cgmm_from_stft(stft, num_classes=2, num_iters=20, init_gamma=None, update_alpha=False):
    """
    CgmmTrainer(obs, K, gamma, update_alpha).train(num_iters) batched (cluster.py:396-465).
    stft (B,C,F,T) complex64; init_gamma (B,K,T,F) or None (2 classes only).
    Returns (masks (B,K,T,F) float32, status (B,) int32).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    K = int(num_classes)
    init_gamma = _arg(init_gamma, stft.device, torch.float32, (B, K, T, F), "init_gamma")
    masks = torch.empty((B, K, T, F), dtype=torch.float32, device=stft.device)
    status = torch.zeros((B,), dtype=torch.int32, device=stft.device)
    _launch(stft.device, "setk_cgmm_stft", _lib.ptr(stft), B, C, F, T, K, int(num_iters), _lib.ptr(init_gamma),
            1 if update_alpha else 0, _lib.ptr(masks), _lib.ptr(status))
    return masks, status


# frequency sub-band schedule of the permutation aligner, per number of bins: rows of (iterations,
# first bin, end bin) (cluster.py:29-36)
PERMU_PLANS = {
    257: [(20, 70, 170), (2, 90, 190), (2, 50, 150), (2, 110, 210), (2, 30, 130), (2, 130, 230),
          (2, 0, 110), (2, 150, 257)],
    513: [(20, 100, 200), (2, 120, 220), (2, 80, 180), (2, 140, 240), (2, 60, 160), (2, 160, 260),
          (2, 40, 140), (2, 180, 280), (2, 0, 120)] +
         [(2, lo, lo + 100) for lo in range(200, 400, 20)] + [(2, 400, 513)],
}


def _permu_rows(plan, F):
    """plan rows as a host int32 (R, 3) table: (array, pointer, R); ValueError unless 0 <= lo < hi <= F,
    iterations >= 0 and 1 <= R <= 64 (SETK_PERMU_MAX_ROWS)."""
    rows = np.asarray(plan, dtype=np.int64).reshape(-1, 3) if np.size(plan) else np.zeros((0, 3), np.int64)
    if not 1 <= rows.shape[0] <= 64:
        raise ValueError(f"an alignment plan has 1..64 rows, got {rows.shape[0]}")
    bad = (rows[:, 0] < 0) | (rows[:, 1] < 0) | (rows[:, 1] >= rows[:, 2]) | (rows[:, 2] > F)
    if bad.any():
        raise ValueError(f"alignment plan row {tuple(rows[bad][0])}: needs iterations >= 0 and "
                         f"0 <= lo < hi <= F = {F}")
    a, p = _host_i32(rows)
    return a, p, rows.shape[0]


def _cacgmm_checks(C, num_classes, num_iters, init_gamma, cgmm_init, permu_plan, F):
    """The arguments setk_cacgmm_* refuse, as ValueError: returns (K, plan table, its pointer, R)."""
    K = int(num_classes)
    if not 2 <= K <= 4:
        raise ValueError(f"CACGMM: num_classes {K} outside 2..4")
    if C < 2:
        raise ValueError(f"CACGMM: {C} channel(s), needs 2 or more")
    if int(num_iters) < 0:
        raise ValueError(f"CACGMM: num_iters {num_iters} < 0")
    if init_gamma is None and not (cgmm_init and K == 2):
        raise ValueError("CACGMM: starting posteriors init_gamma are needed unless cgmm_init with 2 classes")
    if permu_plan is None:
        return K, None, None, 0
    return (K, *_permu_rows(permu_plan, F))


def cacgmm_from_stft(stft, num_classes=2, num_iters=50, init_gamma=None, cgmm_init=False, update_alpha=True,
                     permu_plan=None):
    """
    CacgmmTrainer(obs, K, gamma, cgmm_init=..., update_alpha=...).train(num_iters) batched (cluster.py:468-535),
    then permu_aligner on the fp64 posteriors when `permu_plan` is given.  stft (B,C,F,T) complex64;
    init_gamma (B,K,T,F) float64 or None (cgmm_init with 2 classes).
    Returns (masks (B,K,T,F) float32, status (B,) int32).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    K, rows, rows_p, R = _cacgmm_checks(C, num_classes, num_iters, init_gamma, cgmm_init, permu_plan, F)
    init_gamma = _arg(init_gamma, stft.device, torch.float64, (B, K, T, F), "init_gamma")
    masks = torch.empty((B, K, T, F), dtype=torch.float32, device=stft.device)
    status = torch.zeros((B,), dtype=torch.int32, device=stft.device)
    _launch(stft.device, "setk_cacgmm_stft", _lib.ptr(stft), B, C, F, T, K, int(num_iters), _lib.ptr(init_gamma),
            int(bool(cgmm_init)), int(bool(update_alpha)), rows_p, R, _lib.ptr(masks), _lib.ptr(status))
    return masks, status


def permu_align(masks, n_frames=None, plan=None):
    """
    permu_aligner(masks) (cluster.py:48-91) on the device: masks K x T x F (or a batch B x K x T x F),
    aligned in float64; n_frames (B,) frames of each utterance of a batch (None: T); plan the sub-band
    rows (None: PERMU_PLANS[F], ValueError for another F, as the reference).  Returns (the masks gathered
    through the mapping, float32, same shape; the mapping K x F (B x K x F) int32, source class of slot k).
    """
    masks = torch.as_tensor(masks)
    if masks.dim() not in (3, 4):
        raise RuntimeError("Expect 3D TF-masks, K x T x F or K x F x T")
    single = masks.dim() == 3
    masks = _arg(masks[None] if single else masks, None, torch.float64, (None,) * 4, "masks")
    B, K, T, F = masks.shape
    if plan is None:
        if F not in PERMU_PLANS:
            raise ValueError(f"Unsupported num_bins: {F}")
        plan = PERMU_PLANS[F]
    if not 2 <= K <= 4:
        raise ValueError(f"permu_align: {K} classes outside 2..4")
    rows, rows_p, R = _permu_rows(plan, F)
    nf = _arg(n_frames, masks.device, torch.int32, (B,), "n_frames")
    out = torch.empty((B, K, T, F), dtype=torch.float32, device=masks.device)
    mapping = torch.empty((B, K, F), dtype=torch.int32, device=masks.device)
    _launch(masks.device, "setk_permu_align", _lib.ptr(masks), _lib.ptr(nf), B, K, T, F, rows_p, R, _lib.ptr(out),
            _lib.ptr(mapping))
    return (out[0], mapping[0]) if single else (out, mapping)


def wpe_from_stft(stft, taps=10, delay=3, context=1, num_iters=3):
    """
    wpe(reverb, taps, delay, context, num_iters) batched (libs/wpe.py:82-110).
    stft (B,C,F,T) complex64 -> (dereverberated (B,C,F,T) complex64, status (B,) int32).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    out = torch.empty_like(stft)
    status = torch.zeros((B,), dtype=torch.int32, device=stft.device)
    _launch(stft.device, "setk_wpe_stft", _lib.ptr(stft), B, C, F, T, int(taps), int(delay), int(context),
            int(num_iters), _lib.ptr(out), _lib.ptr(status))
    return out, status


def wpe_step(stft, lambda_enh=None, taps=10, delay=3, context=1, want_inv_lambda=True):
    """
    One WPE step with the variance of facted_wpd (libs/wpe.py:147-155): stft (B,C,F,T) complex64,
    lambda_enh (B,F,T) complex64 or None (first iteration: compute_lambda of the observations).
    Returns (dereverberated (B,C,F,T) complex64, 1/lambda (B,T,F) float32 or None, status (B,) int32).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    lambda_enh = _arg(lambda_enh, stft.device, torch.complex64, (B, F, T), "lambda_enh")
    out = torch.empty_like(stft)
    inv = torch.empty((B, T, F), dtype=torch.float32, device=stft.device) if want_inv_lambda else None
    status = torch.zeros((B,), dtype=torch.int32, device=stft.device)
    _launch(stft.device, "setk_wpe_step", _lib.ptr(stft), _lib.ptr(lambda_enh), B, C, F, T, int(taps), int(delay),
            int(context), _lib.ptr(out), _lib.ptr(inv), _lib.ptr(status))
    return out, inv, status


def covariance(stft, mask, clip_mask=False, mask_ft=False):
    """compute_covar batched: stft (B,C,F,T) c64, mask (B,T,F) (or (B,F,T) with mask_ft) -> (B,F,C,C) c64."""
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    mask = _arg(mask, stft.device, torch.float32, (B, F, T) if mask_ft else (B, T, F), "mask")
    R = torch.empty((B, F, C, C), dtype=torch.complex64, device=stft.device)
    flags = (_lib.F_CLIP_MASK if clip_mask else 0) | (_lib.F_MASK_FT if mask_ft else 0)
    _launch(stft.device, "setk_cov", _lib.ptr(stft), _lib.ptr(mask), flags, B, C, F, T, _lib.ptr(R))
    return R


def _square(Rs):
    """Rs through _arg as a (B,F,C,C) stack of square matrices, dtype kept."""
    Rs = _arg(Rs, None, None, (None,) * 4, "Rs")
    if Rs.shape[3] != Rs.shape[2]:
        raise ValueError(f"Rs must be (B, F, C, C), got {tuple(Rs.shape)}")
    return Rs


def weights(kind, Rs, Rn=None, Ry=None, beta=0.0, ref_channel=-1, rank1=_lib.RANK1_NONE,
            ban=False, out_dtype=None):
    """
    Per-bin weight solve.  Rs/Rn/Ry (B,F,C,C) complex64|complex128 (same dtype).
    Returns (w (B,F,C), status (B,) int32 tensor, ref_used (B,) int32 tensor).
    """
    Rs = _square(Rs)
    B, F, C, _ = Rs.shape
    dt = _dtype_code(Rs)
    Rn, Ry = (_arg(m, Rs.device, None, (B, F, C, C), what) for m, what in ((Rn, "Rn"), (Ry, "Ry")))
    if any(m is not None and m.dtype != Rs.dtype for m in (Rn, Ry)):
        raise ValueError("Rs / Rn / Ry must share dtype and shape")
    out_dtype = Rs.dtype if out_dtype is None else out_dtype
    w = torch.empty((B, F, C), dtype=out_dtype, device=Rs.device)
    status = torch.zeros((B,), dtype=torch.int32, device=Rs.device)
    ref_used = torch.full((B,), -1, dtype=torch.int32, device=Rs.device)
    _launch(Rs.device, "setk_weights", int(kind), float(beta), int(ref_channel), int(rank1), int(bool(ban)),
            _lib.ptr(Rs), _lib.ptr(Rn), _lib.ptr(Ry), dt, B, F, C, _lib.ptr(w), _dtype_code(w), _lib.ptr(status),
            _lib.ptr(ref_used))
    return w, status, ref_used


def ban(weight, Rn):
    """do_ban batched: weight (B,F,C), Rn (B,F,C,C); weight is taken in Rn's complex dtype."""
    weight = _arg(weight, None, None, (None,) * 3, "weight")
    B, F, C = weight.shape
    Rn = _arg(Rn, weight.device, None, (B, F, C, C), "Rn")
    weight = weight.to(Rn.dtype)
    out = torch.empty_like(weight)
    _launch(weight.device, "setk_ban", _lib.ptr(weight), _lib.ptr(Rn), _dtype_code(Rn), B, F, C, _lib.ptr(out))
    return out


def rank1(Rs, Rn=None):
    """rank1_constraint batched.  Returns (R1 (B,F,C,C), status (B,))."""
    Rs = _square(Rs)
    B, F, C, _ = Rs.shape
    Rn = _arg(Rn, Rs.device, Rs.dtype, (B, F, C, C), "Rn")
    out = torch.empty_like(Rs)
    status = torch.zeros((B,), dtype=torch.int32, device=Rs.device)
    _launch(Rs.device, "setk_rank1", _lib.ptr(Rs), _lib.ptr(Rn), _dtype_code(Rs), B, F, C, _lib.ptr(out),
            _lib.ptr(status))
    return out, status


def apply_weights(stft, weight, post_mask=None):
    """Beamformer.beamform batched: (B,C,F,T) x (B,F,C) [x post_mask (B,T,F)] -> (B,F,T) complex64."""
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, C, F, T = stft.shape
    weight = _arg(weight, stft.device, None, (B, F, C), "weight")
    post_mask = _arg(post_mask, stft.device, torch.float32, (B, T, F), "post_mask")
    enh = torch.empty((B, F, T), dtype=torch.complex64, device=stft.device)
    _launch(stft.device, "setk_apply", _lib.ptr(stft), _lib.ptr(weight), _dtype_code(weight), _lib.ptr(post_mask),
            B, C, F, T, _lib.ptr(enh))
    return enh


def float_to_pcm16(wave):
    wave = _arg(wave, None, torch.float32, None, "wave")
    pcm = torch.empty(wave.shape, dtype=torch.int16, device=wave.device)
    _launch(wave.device, "setk_float_to_pcm16", _lib.ptr(wave), wave.numel(), _lib.ptr(pcm))
    return pcm


def pcm16_to_float(pcm):
    pcm = _arg(pcm, None, None, None, "pcm")
    if pcm.dtype != torch.int16:
        raise ValueError(f"pcm16_to_float: pcm must be int16, got {pcm.dtype}")
    wave = torch.empty(pcm.shape, dtype=torch.float32, device=pcm.device)
    _launch(pcm.device, "setk_pcm16_to_float", _lib.ptr(pcm), pcm.numel(), _lib.ptr(wave))
    return wave


def cm_masks(blobs, T, F, out=None):
    """
    Kaldi "CM" compressed matrices -> float32 masks [B][T][F] on the device (kaldi_io.py:248-281).
    blobs: uint8 [B][slot_bytes] device tensor, one matrix per slot as it lies in the archive behind
    the "CM " token (slot_bytes a multiple of 16).  Returns (masks, status int32 [B]).
    """
    blobs = _arg(blobs, None, None, None, "blobs")
    if blobs.dtype != torch.uint8 or blobs.dim() != 2:
        raise ValueError("cm_masks: blobs must be uint8 [B][slot_bytes]")
    B = blobs.shape[0]
    if out is None:
        out = torch.empty((B, T, F), dtype=torch.float32, device=blobs.device)
    else:
        out = _out(out, blobs.device, torch.float32, (B, T, F), "cm_masks: out")
    status = torch.zeros((B,), dtype=torch.int32, device=blobs.device)
    _launch(blobs.device, "setk_cm_masks", _lib.ptr(blobs), blobs.shape[1], B, T, F, _lib.ptr(out), _lib.ptr(status))
    return out, status


# ---------------------------------------------------------------------------
# spatial features on explicit STFTs (libs/spatial.py of the reference; csrc/spatial.cu)
# ---------------------------------------------------------------------------
def ipd(si, sj, mode=0):
    """spatial.ipd: si, sj (..., T, F) complex64 -> float32 (..., T, F) (mode 0/1) or (..., T, 2F)."""
    si = _arg(si, None, torch.complex64, None, "ipd: si")
    if si.dim() < 2:
        raise ValueError(f"ipd: si must be (..., T, F), got {tuple(si.shape)}")
    sj = _arg(sj, si.device, torch.complex64, si.shape, "ipd: sj")
    F = si.shape[-1]
    rows = si.numel() // F
    shape = list(si.shape)
    if mode == 2:
        shape[-1] = 2 * F
    out = torch.empty(shape, dtype=torch.float32, device=si.device)
    _launch(si.device, "setk_ipd", _lib.ptr(si), _lib.ptr(sj), rows, F, int(mode), _lib.ptr(out))
    return out


def directional_feats(stft, steer, pairs=None):
    """
    spatial.directional_feats batched: stft (B,M,F,T) complex64, steer (M,F) or (B,M,F)
    complex -> (B,T,F) float64.  pairs: list of (i, j) or None (all i < j).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, M, F, T = stft.shape
    batched = np.ndim(steer) == 3
    steer = _arg(steer, stft.device, torch.complex128, (B, M, F) if batched else (M, F), "steer vector")
    p_t = _arg(pairs, stft.device, torch.int32, None, "df_pair")
    n_pairs = 0
    if p_t is not None:
        p_t = p_t.reshape(-1, 2)
        n_pairs = p_t.shape[0]
        if n_pairs == 0 or int(p_t.min()) < 0 or int(p_t.max()) >= M:
            raise ValueError(f"df_pair entries must lie in [0, {M})")
    out = torch.empty((B, T, F), dtype=torch.float64, device=stft.device)
    _launch(stft.device, "setk_directional_feats", _lib.ptr(stft), _lib.ptr(steer), int(batched), _lib.ptr(p_t),
            n_pairs, B, M, F, T, _lib.ptr(out))
    return out


def gcc_phat(si, sj, omega, tau, normalize=True, apply_floor=True, out=None):
    """
    One microphone pair of gcc_phat_linear / gcc_phat_diag: si, sj (T,F) complex64, omega (F,)
    and tau (D,) float64 -> (T,D) float64.  With `out` given the pair is ADDED to it
    (srp_phat_linear).
    """
    si = _arg(si, None, torch.complex64, (None, None), "gcc_phat: si")
    T, F = si.shape
    dev = si.device
    sj = _arg(sj, dev, torch.complex64, (T, F), "gcc_phat: sj")
    omega = _arg(omega, dev, torch.float64, (F,), "gcc_phat: omega")
    tau = _arg(tau, dev, torch.float64, (None,), "gcc_phat: tau")
    D = tau.shape[0]
    work = torch.empty((int(_lib.library().setk_gcc_phat_work_doubles(T, F, D)),), dtype=torch.float64, device=dev)
    accumulate = out is not None
    if accumulate:
        out = _out(out, dev, torch.float64, (T, D), "gcc_phat: out")
    else:
        out = torch.empty((T, D), dtype=torch.float64, device=dev)
    _launch(dev, "setk_gcc_phat", _lib.ptr(si), _lib.ptr(sj), T, F, _lib.ptr(omega), _lib.ptr(tau), D,
            int(bool(normalize)), int(bool(apply_floor)), int(accumulate), _lib.ptr(work), _lib.ptr(out))
    return out


def msc(spec, context=1, normalize=True):
    """spatial.msc: spec (N,T,F) complex64 -> (T,F) float64."""
    spec = _arg(spec, None, torch.complex64, (None,) * 3, "msc: spectrogram")
    N, T, F = spec.shape
    work = torch.empty((int(_lib.library().setk_msc_work_doubles(T, F)),), dtype=torch.float64, device=spec.device)
    out = torch.empty((T, F), dtype=torch.float64, device=spec.device)
    _launch(spec.device, "setk_msc", _lib.ptr(spec), N, T, F, int(context), int(bool(normalize)), _lib.ptr(work),
            _lib.ptr(out))
    return out


# ---------------------------------------------------------------------------
# sound source localisation on explicit STFTs (libs/ssl.py of the reference; csrc/ssl.cuh)
# ---------------------------------------------------------------------------
_SSL_BACKENDS = {"ml": _lib.SSL_ML, "srp": _lib.SSL_SRP, "music": _lib.SSL_MUSIC}


def ssl(stft, steer, backend="ml", mask=None, windows=None, pairs=None, compression=0.0, eps=1e-8,
        normalize=False):
    """
    DoA scores and indices, batched.  stft (B,M,F,T) complex64; steer (A,M,F) complex128;
    mask (B,N,T,F) float32 or None; windows: (B,W,2) frame ranges [s, e) or None (one window
    [0, T)); pairs: list of (l, r) microphone pairs (SRP).
    Returns (scores (B,N,W,A) float64, index (B,N,W) int32), N = 1 without a mask.
    """
    if backend not in _SSL_BACKENDS:
        raise ValueError(f"unknown SSL backend {backend!r}")
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, M, F, T = stft.shape
    dev = stft.device
    steer = _arg(steer, dev, torch.complex128, (None, M, None), "steer vector")   # its bins: setk_ssl checks
    A = steer.shape[0]
    mask = _arg(mask, dev, torch.float32, (B, None, T, F), "mask")
    N = 1 if mask is None else mask.shape[1]
    win, win_p = _host_i32(np.reshape([[0, T]] * B if windows is None else windows, (B, -1, 2)))
    pr, pr_p = _host_i32(None if pairs is None else np.reshape(pairs, (-1, 2)))
    W, P = win.shape[1], 0 if pr is None else pr.shape[0]
    scores = torch.empty((B, N, W, A), dtype=torch.float64, device=dev)
    index = torch.empty((B, N, W), dtype=torch.int32, device=dev)
    _launch(dev, "setk_ssl", _SSL_BACKENDS[backend], _lib.ptr(stft), B, M, F, T, _lib.ptr(steer), A, steer.shape[2],
            _lib.ptr(mask), N, win_p, W, pr_p, P, float(compression), float(eps), int(bool(normalize)),
            _lib.ptr(scores), _lib.ptr(index))
    return scores, index


# ---------------------------------------------------------------------------
# AuxIVA blind source separation on explicit STFTs (apply_auxiva.py of the reference; csrc/auxiva.cuh)
# ---------------------------------------------------------------------------
def auxiva_from_stft(stft, num_epochs=20):
    """
    auxiva(X, epochs) batched (apply_auxiva.py:24-57).
    stft (B,N,F,T) complex64 -> (separated sources (B,N,F,T) complex128, status (B,) int32).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 4, "stft")
    B, N, F, T = stft.shape
    out = torch.empty((B, N, F, T), dtype=torch.complex128, device=stft.device)
    status = torch.zeros((B,), dtype=torch.int32, device=stft.device)
    _launch(stft.device, "setk_auxiva_stft", _lib.ptr(stft), B, N, F, T, int(num_epochs), _lib.ptr(out),
            _lib.ptr(status))
    return out, status


# ---------------------------------------------------------------------------
# iMCRA / OM-LSA noise suppression on explicit STFTs (libs/ns.py, apply_ns.py of the reference; csrc/ns.cu)
# ---------------------------------------------------------------------------
IMCRA_DEFAULTS = dict(alpha=0.92, alpha_s=0.9, alpha_d=0.85, b_min=1.66, gamma0=4.6, gamma1=3, zeta0=1.67,
                      xi_min_db=-18, gmin_db=-10, w_mcra=1, h_mcra="hann", beta=1.47, V=15, U=8)


def imcra_config(config=None, eps=1e-7):
    """
    setk_imcra_config_t from iMCRA keywords (ns.py:221-245; missing ones take the reference's
    defaults) and run(eps).  Returns (config, window): keep `window` alive while the config is used.
    """
    conf = dict(IMCRA_DEFAULTS, **(config or {}))
    unknown = set(conf) - set(IMCRA_DEFAULTS)
    if unknown:
        raise TypeError(f"unknown iMCRA keywords: {sorted(unknown)}")
    w_mcra = int(conf["w_mcra"])
    if w_mcra < 0 or w_mcra > _lib.NS_MAX_W:
        raise ValueError(f"w_mcra={w_mcra} outside [0, {_lib.NS_MAX_W}]")
    window = np.ascontiguousarray(scipy.signal.get_window(conf["h_mcra"], 2 * w_mcra + 1), dtype=np.float64)
    cfg = _lib.ImcraConfig(
        alpha=conf["alpha"], alpha_s=conf["alpha_s"], alpha_d=conf["alpha_d"], b_min=conf["b_min"],
        gamma0=conf["gamma0"], gamma1=conf["gamma1"], zeta0=conf["zeta0"], xi_min_db=conf["xi_min_db"],
        gmin_db=conf["gmin_db"], beta=conf["beta"], eps=float(eps), w_mcra=w_mcra, V=int(conf["V"]),
        U=int(conf["U"]), reserved=0, window_host=window.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
    return cfg, window


def ns_from_stft(stft, n_frames=None, config=None, gain=True, enh=True, eps=1e-7):
    """
    iMCRA(**config).run(stft, eps) batched (ns.py:247-387), and gain * stft (apply_ns.py:42).
    stft (B,F,T) complex64; n_frames (B,) int or None (every utterance has T frames).
    Returns (gain (B,T,F) float64 or None, enh (B,F,T) complex64 or None).
    """
    stft = _arg(stft, None, torch.complex64, (None,) * 3, "stft")
    if not (gain or enh):
        raise ValueError("ns_from_stft: ask for the gain, the enhanced STFT or both")
    B, F, T = stft.shape
    dev = stft.device
    nf = _arg(n_frames, dev, torch.int32, (B,), "n_frames")
    g = torch.empty((B, T, F), dtype=torch.float64, device=dev) if gain else None
    e = torch.empty((B, F, T), dtype=torch.complex64, device=dev) if enh else None
    cfg, window = imcra_config(config, eps)
    _launch(dev, "setk_ns_imcra", ctypes.byref(cfg), _lib.ptr(stft), _lib.ptr(nf), B, F, T, _lib.ptr(g), _lib.ptr(e))
    del window
    return g, e


# ---------------------------------------------------------------------------
# Image-method room impulse responses (include/rir-generator.cc, rir_generate_{1d,2d}.py; csrc/rir.cu)
# ---------------------------------------------------------------------------
def rir_beta(room, rt60_or_refl, c=340):
    """
    Reflection coefficients (6,) float64 for one room: six coefficients pass through; one T60 (a
    number or a one-element sequence) becomes sqrt(1 - alpha) on every wall, alpha = 24 V ln10 /
    (c S T60), and T60 = 0 gives 0 (rir-generator.cc:78-92, in float64).  ValueError when alpha > 1.
    """
    refl = np.atleast_1d(np.asarray(rt60_or_refl, dtype=np.float64))
    if refl.shape == (6,):
        return refl.copy()
    if refl.shape != (1,):
        raise ValueError(f"beta must be one T60 or six reflection coefficients, got {refl.shape[0]} values")
    t60 = float(refl[0])
    lx, ly, lz = (float(v) for v in np.asarray(room, dtype=np.float64).reshape(3))
    if t60 == 0:
        return np.zeros(6)
    V, S = lx * ly * lz, 2 * (lx * ly + lx * lz + ly * lz)
    alpha = 24 * V * math.log(10.0) / (c * S * t60)
    if alpha > 1:
        raise ValueError(f"{alpha} > 1: The reflection coefficients cannot be calculated using the current "
                         "room parameters, i.e. room size and reverberation time.")
    return np.full(6, math.sqrt(1 - alpha))


def rir_image(room, beta, source, receivers, n_samples, sr=16000, c=340, order=-1, mic_type="omnidirectional",
              orientation=(0, 0), hp_filter=True, device=None):
    """
    Image-method RIRs (rir-generator.cc:108-223) for B problems b = (room, beta, source) with M
    receivers each: room (B,3), beta (B,6) reflection coefficients (rir_beta turns a T60 into them),
    source (B,3), receivers (B,M,3), all metres; one problem may drop the leading B.  Returns
    (B, M, n_samples) float32 on `device` (default: the inputs' device, else cuda).  A problem whose
    response leaves the accumulator's range raises ValueError naming it.
    """
    if mic_type not in _lib.MIC_TYPES:
        raise ValueError(f"unknown mic_type {mic_type!r}: one of {_lib.MIC_TYPES}")
    if device is None:
        device = next((t.device for t in (room, beta, source, receivers) if isinstance(t, torch.Tensor)),
                      "cuda" if torch.cuda.is_available() else "cpu")
    dev = torch.device(device)

    def f64(t, shape, what):      # one problem (B = 1) may drop the leading B
        single = np.ndim(t) == len(shape) - 1 and shape[0] in (None, 1)
        t = _arg(t, dev, torch.float64, shape[1:] if single else shape, what)
        return t[None] if single else t

    room = f64(room, (None, 3), "room")
    B = room.shape[0]
    beta, source = f64(beta, (B, 6), "beta"), f64(source, (B, 3), "source")
    receivers = f64(receivers, (B, None, 3), "receivers")
    M, L = receivers.shape[1], int(n_samples)
    out = torch.empty((B, M, max(L, 0)), dtype=torch.float32, device=dev)
    status = torch.zeros(B, dtype=torch.int32, device=dev)
    az, el = (float(v) for v in orientation)
    cfg = _lib.RirConfig(sound_velocity=float(c), samp_frequency=float(sr), azimuth=az, elevation=el,
                         n_samples=L, order=int(order), mic_type=_lib.MIC_TYPES.index(mic_type),
                         hp_filter=int(bool(hp_filter)))
    _launch(dev, "setk_rir_image", ctypes.byref(cfg), _lib.ptr(room), _lib.ptr(beta), _lib.ptr(source),
            _lib.ptr(receivers), B, M, _lib.ptr(out), _lib.ptr(status))
    bad = torch.nonzero(status).flatten().tolist()
    if bad:
        raise ValueError(f"rir_image: the response of problem {bad[0]} is not finite or out of range "
                         f"(status {int(status[bad[0]])}; {len(bad)} problem(s) in all)")
    return out


# ---------------------------------------------------------------------------
# Speech + RIR + noise mixtures (wav_simulate.py of the reference; csrc/simu.cu, setk_b200/simu.py)
# ---------------------------------------------------------------------------
def convolve(x, h, n_out=None, s_len=None, h_len=None, out=None):
    """
    ss.convolve(x[None], h)[..., :n_out] of add_room_response (wav_simulate.py:29-54, without the
    power) for B problems: x (B,S) float32 sources, h (B,M,L) float32 filters; one problem may drop
    the leading B (x (S,), h (M,L) or (L,)).  n_out: None gives S (the reference's truncation), S + L - 1
    is the full convolution; an int or (B,) per problem.  s_len / h_len: (B,) true lengths of a ragged
    batch (None: S and L).  Returns y (B,M,Ny) float32, Ny = max n_out, zero past each problem's n_out
    (or writes `out`, a contiguous (B,M,Ny) float32 tensor).
    """
    x, h = torch.as_tensor(x), torch.as_tensor(h)
    single = x.dim() == 1
    if single:
        x = x[None]
        h = h.reshape(1, 1, -1) if h.dim() == 1 else h[None]
    dev = h.device if h.device.type != "cpu" else x.device
    x = _arg(x, dev, torch.float32, (None, None), "convolve: x")
    B, Sx = x.shape
    h = _arg(h, dev, torch.float32, (B, None, None), "convolve: h")
    M, Lh = h.shape[1], h.shape[2]
    _, s_p = _host_i32(s_len, (B,))
    _, h_p = _host_i32(h_len, (B,))
    if n_out is None:
        n_out = Sx if s_len is None else s_len
    n_l, n_p = _host_i32(n_out, (B,))
    Ny = int(n_l.max()) if B else 0
    if out is None:
        out = torch.empty((B, M, max(Ny, 0)), dtype=torch.float32, device=dev)
    else:
        out = _out(out, dev, torch.float32, (B, M, Ny), "convolve: out")
    _launch(dev, "setk_convolve", _lib.ptr(x), Sx, _lib.ptr(h), Lh, B, M, s_p, h_p, n_p, _lib.ptr(out), Ny)
    return out[0] if single else out


def simulate_mix(pool, mixes, terms, n_channels, n_speakers, n_samples, pcm16=False, spk=True, noise=True):
    """
    Mixing and normalisation of run_simu (wav_simulate.py:166-312) for B mixtures whose images lie in
    `pool` (a flat float32 tensor).  mixes: B dicts of setk_simu_mix_t (first_term, n_terms, n_samples,
    n_channels, norm_factor); terms: dicts of setk_simu_term_t (src, kind, n_channels, pitch, begin,
    length, repeat, power_begin, power_end, level_db).  n_channels, n_speakers, n_samples: the output
    shape M, K, n_pitch.  Returns (mix (B,M,n_pitch), spk (B,K,n_pitch) or None, noise (B,n_pitch) or
    None, factor (B,) float64), float32 or, with pcm16, int16 as write_wav stores them.
    """
    # the pool holds every image of the batch: it is refused rather than converted, since a silent
    # float32 copy would double the largest buffer of the call
    pool = pool.reshape(-1)
    if pool.dtype != torch.float32 or not pool.is_contiguous():
        raise ValueError("simulate_mix: pool must be a contiguous float32 tensor")
    dev = pool.device
    B, T = len(mixes), len(terms)
    mx = (_lib.SimuMix * max(B, 1))(*[_lib.SimuMix(**m) for m in mixes])
    tm = (_lib.SimuTerm * max(T, 1))(*[_lib.SimuTerm(**t) for t in terms])
    M, K, N = int(n_channels), int(n_speakers), int(n_samples)
    dt = torch.int16 if pcm16 else torch.float32
    mix = torch.empty((B, M, max(N, 0)), dtype=dt, device=dev)
    s = torch.empty((B, K, max(N, 0)), dtype=dt, device=dev) if spk else None
    nz = torch.empty((B, max(N, 0)), dtype=dt, device=dev) if noise else None
    factor = torch.empty((B,), dtype=torch.float64, device=dev)
    _launch(dev, "setk_simulate_mix", _lib.ptr(pool), pool.numel(), ctypes.cast(mx, ctypes.c_void_p), B,
            ctypes.cast(tm, ctypes.c_void_p), T, M, K, N, int(bool(pcm16)), _lib.ptr(mix), _lib.ptr(s), _lib.ptr(nz),
            _lib.ptr(factor))
    return mix, s, nz, factor


# ---------------------------------------------------------------------------
# Separation metrics (compute_sdr.py / compute_si_snr.py / libs/metric.py of the reference; csrc/sep_eval.cu)
# ---------------------------------------------------------------------------
SEP_SCRATCH_BYTES = 4 << 30   # bss_eval splits a batch so that one call's scratch stays under this (4 GiB)


def _sep_inputs(est, ref, n_samples, who):
    est, ref = torch.as_tensor(est), torch.as_tensor(ref)
    dev = ref.device if ref.device.type != "cpu" else est.device
    est = _arg(est, dev, torch.float32, (None,) * 3, f"{who}: est")
    ref = _arg(ref, dev, torch.float32, est.shape, f"{who}: ref")
    B, N, S = est.shape
    lens = None
    if n_samples is not None:
        lens = np.broadcast_to(np.asarray(n_samples, dtype=np.int64), (B,))   # checked before the int32 cast
        if lens.size and (lens.min() < 1 or lens.max() > S):
            raise ValueError(f"{who}: n_samples must lie in [1, {S}]")
    return est, ref, lens, dev


def bss_eval_batch_step(B, N, S, flen=512):
    """utterances per setk_bss_eval call that bss_eval uses for a (B, N, S) batch: all B when the call's
    scratch (setk_bss_eval_scratch_bytes) fits SEP_SCRATCH_BYTES, else the most that fit (at least 1)"""
    lib = _lib.library()
    total = lib.setk_bss_eval_scratch_bytes(B, N, S, int(flen))
    if total < 0 or total <= SEP_SCRATCH_BYTES:
        return B   # sizes setk_bss_eval rejects are reported by the call itself
    step = max(1, B * SEP_SCRATCH_BYTES // total)
    while step > 1 and lib.setk_bss_eval_scratch_bytes(step, N, S, int(flen)) > SEP_SCRATCH_BYTES:
        step -= 1
    return step


def bss_eval(est, ref, n_samples=None, flen=512):
    """
    BSS-Eval v3 sources criteria (mir_eval.separation.bss_eval_sources before its permutation search) of
    every (estimate j, reference i) pair: est, ref (B, N, S) float32, n_samples (B,) true lengths of a
    ragged batch (None: S), flen the filter length L.  Returns (crit (B, 3, N, N) float64 with
    crit[b, k, j, i] the SDR / SIR / SAR (k = 0, 1, 2) of estimate j against reference i, dropped (B,)
    int32 dependent columns of the least-squares system, status (B,) int32 SETK_ST_* bits).
    """
    est, ref, lens, dev = _sep_inputs(est, ref, n_samples, "bss_eval")
    B, N, S = est.shape
    L = int(flen)
    crit = torch.empty((B, 3, N, N), dtype=torch.float64, device=dev)
    dropped = torch.zeros((B,), dtype=torch.int32, device=dev)
    status = torch.zeros((B,), dtype=torch.int32, device=dev)
    step = bss_eval_batch_step(B, N, S, L)
    for b0 in range(0, B, step):
        b1 = min(B, b0 + step)
        _, lens_p = _host_i32(None if lens is None else lens[b0:b1])
        _launch(dev, "setk_bss_eval", _lib.ptr(est[b0:b1]), _lib.ptr(ref[b0:b1]), lens_p, b1 - b0, N, S, L,
                _lib.ptr(crit[b0:b1]), _lib.ptr(dropped[b0:b1]), _lib.ptr(status[b0:b1]))
    return crit, dropped, status


def si_snr(est, ref, n_samples=None, remove_dc=True, eps=1e-8):
    """
    si_snr(x, s, eps, remove_dc) of libs/metric.py for every (estimate j, reference i) pair in fp64: est,
    ref (B, N, S) float32, n_samples (B,) true lengths (None: S).  Returns (B, N, N) float64, [b, j, i].
    """
    est, ref, lens, dev = _sep_inputs(est, ref, n_samples, "si_snr")
    B, N, S = est.shape
    out = torch.empty((B, N, N), dtype=torch.float64, device=dev)
    _launch(dev, "setk_si_snr", _lib.ptr(est), _lib.ptr(ref), _host_i32(lens)[1], B, N, S, int(bool(remove_dc)),
            float(eps), _lib.ptr(out))
    return out
