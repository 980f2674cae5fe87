"""
setk_b200._lib -- ctypes binding of libsetk_b200.so (include/setk_b200.h).

The library is the product: hand-written sm_90a CUDA kernels behind a C-ABI.
There is NO fallback: if the shared object is missing, or a call reports an
error, this module raises.  (`use_library()` exists so the CPU test tier can
point the same host code at tests/emu/libsetk_b200_emu.so -- the kernels'
sources compiled for a CPU execution model -- it is never called by the
package itself.)
"""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32,
                    c_int64, c_uint32, c_void_p)

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIBRARY = os.path.join(_HERE, "libsetk_b200.so")

# ---- constants mirrored from include/setk_b200.h ----
SETK_MAX_CHANNELS = 16
SETK_EINVAL, SETK_ENOMEM, SETK_ESHAPE, SETK_EUNSUPPORTED = -1, -2, -3, -4
ST_SINGULAR, ST_NOT_PD, ST_NO_CONVERGE, ST_NONFINITE, ST_BAD_REF = 1, 2, 4, 8, 16
ST_REGULARIZED = 32          # warning only
ST_SILENT = 64               # setk_bss_eval: a reference or estimate is all zeros
SEP_MAX_SOURCES, SEP_MAX_FLEN, SEP_MAX_COLS, SEP_MAX_SAMPLES = 8, 512, 4096, 1 << 24
ST_ERROR_MASK = 31
BF_MVDR, BF_MPDR, BF_MPDR_WHITEN, BF_GEVD, BF_PMWF, BF_PEVD = 0, 1, 2, 3, 4, 5
RANK1_NONE, RANK1_EIG, RANK1_GEV = 0, 1, 2
F_CLIP_MASK, F_MASK_FT = 1, 2
FEAT_POW, FEAT_MEL, FEAT_LOG = 1, 2, 4
FEAT_MAX_MEL = 1024
C64, C128 = 0, 1
SSL_ML, SSL_SRP, SSL_MUSIC = 0, 1, 2
SSL_MAX_MASKS = 8
NS_MAX_W, NS_MAX_U, NS_MAX_BINS = 8, 64, 2049
MIC_TYPES = ("omnidirectional", "subcardioid", "cardioid", "hypercardioid", "bidirectional")  # SETK_MIC_*


class SetkConfig(Structure):
    _fields_ = [("num_channels", c_int32), ("frame_len", c_int32),
                ("n_fft", c_int32), ("frame_hop", c_int32),
                ("center", c_int32), ("max_batch", c_int32),
                ("max_samples", c_int32), ("reserved", c_int32),
                ("window_host", POINTER(c_double))]


class ImcraConfig(Structure):
    _fields_ = [("alpha", c_double), ("alpha_s", c_double), ("alpha_d", c_double), ("b_min", c_double),
                ("gamma0", c_double), ("gamma1", c_double), ("zeta0", c_double), ("xi_min_db", c_double),
                ("gmin_db", c_double), ("beta", c_double), ("eps", c_double),
                ("w_mcra", c_int32), ("V", c_int32), ("U", c_int32), ("reserved", c_int32),
                ("window_host", POINTER(c_double))]


class RirConfig(Structure):
    _fields_ = [("sound_velocity", c_double), ("samp_frequency", c_double), ("azimuth", c_double),
                ("elevation", c_double), ("n_samples", c_int32), ("order", c_int32), ("mic_type", c_int32),
                ("hp_filter", c_int32)]


CONV_MAX_LEN, SIMU_MAX_TERMS = 1 << 24, 64
SIMU_SPEAKER, SIMU_POINT_NOISE, SIMU_ISOTROPIC = 0, 1, 2


class SimuTerm(Structure):
    _fields_ = [("src", c_int64), ("kind", c_int32), ("n_channels", c_int32), ("pitch", c_int32),
                ("begin", c_int32), ("length", c_int32), ("repeat", c_int32), ("power_begin", c_int32),
                ("power_end", c_int32), ("reserved", c_int32), ("level_db", c_double)]


class SimuMix(Structure):
    _fields_ = [("first_term", c_int32), ("n_terms", c_int32), ("n_samples", c_int32), ("n_channels", c_int32),
                ("norm_factor", c_double)]


class SetkError(RuntimeError):
    """A libsetk_b200 call failed (bad argument or CUDA error)."""

    def __init__(self, code, message):
        super().__init__(f"libsetk_b200 error {code}: {message}")
        self.code = code


_PROTOTYPES = {
    "setk_version": (c_int, []),
    "setk_last_error_string": (c_char_p, []),
    "setk_launch_count": (c_int64, []),
    "setk_plan_create": (c_int, [POINTER(SetkConfig), POINTER(c_void_p)]),
    "setk_plan_destroy": (c_int, [c_void_p]),
    "setk_num_frames": (c_int, [c_void_p, c_int32]),
    "setk_istft_length": (c_int, [c_void_p, c_int32]),
    "setk_num_bins": (c_int, [c_void_p]),
    "setk_stft": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                          c_void_p, c_void_p]),
    "setk_stft_cov": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                              c_void_p, c_void_p, c_uint32, c_void_p, c_void_p,
                              c_void_p, c_void_p]),
    "setk_spectral_feats": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_uint32, c_float,
                                    c_void_p, c_void_p]),
    "setk_plan_set_mel": (c_int, [c_void_p, c_int32, c_void_p]),
    "setk_cov": (c_int, [c_void_p, c_void_p, c_uint32, c_int32, c_int32,
                         c_int32, c_int32, c_void_p, c_void_p]),
    "setk_weights": (c_int, [c_int32, c_double, c_int32, c_int32, c_int32,
                             c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                             c_int32, c_int32, c_void_p, c_int32, c_void_p,
                             c_void_p, c_void_p]),
    "setk_ban": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                         c_void_p, c_void_p]),
    "setk_rank1": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                           c_void_p, c_void_p, c_void_p]),
    "setk_apply": (c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_int32,
                           c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "setk_istft": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32,
                           c_void_p, c_void_p, c_void_p]),
    "setk_apply_istft": (c_int, [c_void_p, c_void_p, c_void_p, c_int32,
                                 c_int32, c_void_p, c_int32, c_void_p, c_int32,
                                 c_void_p, c_void_p, c_void_p]),
    "setk_apply_istft_pcm16": (c_int, [c_void_p, c_void_p, c_void_p, c_int32,
                                       c_int32, c_void_p, c_int32, c_void_p, c_int32,
                                       c_void_p, c_void_p, c_void_p]),
    "setk_cgmm_masks": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                c_int32, c_int32, c_void_p, c_int32, c_void_p,
                                c_void_p, c_void_p]),
    "setk_cgmm_stft": (c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32,
                               c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "setk_cacgmm_masks": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                  c_void_p, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_void_p,
                                  c_void_p]),
    "setk_cacgmm_stft": (c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                 c_void_p, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_void_p,
                                 c_void_p]),
    "setk_permu_align": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                 c_int32, c_void_p, c_void_p, c_void_p]),
    "setk_wpe_stft": (c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                              c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "setk_wpe_step": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                              c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "setk_ipd": (c_int, [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p]),
    "setk_directional_feats": (c_int, [c_void_p, c_void_p, c_int32, c_void_p, c_int32, c_int32,
                                       c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    "setk_gcc_phat_work_doubles": (c_int64, [c_int32, c_int32, c_int32]),
    "setk_gcc_phat": (c_int, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_int32,
                              c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "setk_msc_work_doubles": (c_int64, [c_int32, c_int32]),
    "setk_msc": (c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                         c_void_p]),
    "setk_float_to_pcm16": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "setk_pcm16_to_float": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "setk_cm_masks": (c_int, [c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    "setk_ssl": (c_int, [c_int32, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32,
                         c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_double, c_double, c_int32,
                         c_void_p, c_void_p, c_void_p]),
    "setk_auxiva_stft": (c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                                 c_void_p]),
    "setk_ns_imcra": (c_int, [POINTER(ImcraConfig), c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p,
                              c_void_p, c_void_p]),
    "setk_rir_image": (c_int, [POINTER(RirConfig), c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                               c_void_p, c_void_p, c_void_p]),
    "setk_convolve": (c_int, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_int32, c_void_p]),
    "setk_simulate_mix": (c_int, [c_void_p, c_int64, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32,
                                  c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "setk_bss_eval": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                              c_void_p, c_void_p]),
    "setk_bss_eval_scratch_bytes": (c_int64, [c_int32, c_int32, c_int32, c_int32]),
    "setk_si_snr": (c_int, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_double, c_void_p,
                            c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_PROTOTYPES)

_cdll = None
_path = None


def _bind(path):
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in _PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def use_library(path):
    """Bind a specific shared object (test tooling only)."""
    global _cdll, _path
    _cdll = _bind(path)
    _path = path
    return _cdll


def library():
    """The bound library; loads setk_b200/libsetk_b200.so on first use."""
    global _cdll, _path
    if _cdll is None:
        if not os.path.exists(DEFAULT_LIBRARY):
            raise ImportError(
                f"{DEFAULT_LIBRARY} not found: the CUDA extension is not built. "
                "Run `python -c 'import __graft_entry__ as g; g.build()'` or "
                "setk_b200/csrc/build.sh (nvcc, sm_90a). setk_b200 has no CPU "
                "fallback.")
        _cdll = _bind(DEFAULT_LIBRARY)
        _path = DEFAULT_LIBRARY
    return _cdll


def library_path():
    library()
    return _path


def check(rc):
    if rc != 0:
        msg = library().setk_last_error_string()
        raise SetkError(rc, msg.decode("utf-8", "replace") if msg else "")


def launch_count():
    return int(library().setk_launch_count())


def emulated():
    """True when the bound library is the CPU test tier's build (tests/emu)."""
    return hasattr(library(), "setk_emulated")


def ptr(t):
    """
    Raw data pointer of a torch tensor (None -> NULL).  The product library
    takes DEVICE pointers only: a host tensor is an error, not a slow path.
    """
    if t is None:
        return None
    if isinstance(t, np.ndarray):
        if not emulated():
            raise RuntimeError("libsetk_b200 needs device memory (no CPU fallback)")
        return c_void_p(t.ctypes.data)
    if not t.is_cuda and not emulated():
        raise RuntimeError("libsetk_b200 needs CUDA tensors (no CPU fallback); got a "
                           f"{t.device} tensor")
    return c_void_p(t.data_ptr())


def current_stream(device):
    """cudaStream_t of torch's current stream on `device` (NULL on CPU)."""
    import torch
    if device.type != "cuda":
        return None
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)
