"""
setk_b200.libs.ns -- GPU mirror of the reference's iMCRA noise suppressor
(scripts/sptk/libs/ns.py:212-387: iMCRA noise estimation + the OM-LSA gain, Cohen 2003).

    suppressor = iMCRA(alpha=0.92, ..., V=15, U=8)
    gain = suppressor.run(stft, eps=1e-7)        # T x F complex in, T x F float64 out

Same constructor keywords and defaults, method, argument and axes as the reference; the
arithmetic runs in libsetk_b200.so (setk_ns_imcra: one CTA per utterance, the recursion over
frames in fp64, csrc/ns.cu).  No CPU path.

Differences from the reference:
  * stft may be a torch tensor or a numpy array (the same kind comes back), with an optional
    leading batch axis (B x T x F);
  * E1 is a series / continued fraction (ns.py uses scipy.integrate.quad per cell); at v == 0 it is
    the 37.191280375549404 quad returns there, for 0 < v < 1e-12 the true E1 where quad is wrong;
  * |x|^2 is formed in fp64 (the reference squares in float32).
MCRA (ns.py:10-209) is not mirrored: no command line reaches it -- apply_ns.py is hard coded to
iMCRA (doc/ns/README.md).
"""
import numpy as np
import torch

from .. import plan as _plan
from .utils import default_device

__all__ = ["iMCRA"]


class iMCRA(object):
    """OM-LSA with iMCRA noise estimation (ns.py:212-245)."""

    def __init__(self, alpha=0.92, alpha_s=0.9, alpha_d=0.85, b_min=1.66, gamma0=4.6, gamma1=3, zeta0=1.67,
                 xi_min_db=-18, gmin_db=-10, w_mcra=1, h_mcra="hann", beta=1.47, V=15, U=8):
        self.conf = dict(alpha=alpha, alpha_s=alpha_s, alpha_d=alpha_d, b_min=b_min, gamma0=gamma0,
                         gamma1=gamma1, zeta0=zeta0, xi_min_db=xi_min_db, gmin_db=gmin_db, w_mcra=w_mcra,
                         h_mcra=h_mcra, beta=beta, V=V, U=U)
        _plan.imcra_config(self.conf)          # the window and the keyword values are checked here

    def run(self, stft, eps=1e-7):
        """
        Arguments:
            stft: complex STFT, T x F (or B x T x F)
        Return:
            gain: real array, T x F (or B x T x F), float64
        """
        was_numpy = not isinstance(stft, torch.Tensor)
        x = torch.as_tensor(np.asarray(stft) if was_numpy else stft)
        if not torch.is_complex(x) or x.dim() not in (2, 3):
            raise ValueError("iMCRA.run expects a complex STFT, T x F")
        batched = x.dim() == 3
        if not batched:
            x = x[None]
        dev = x.device if x.device.type == "cuda" else default_device()
        X = x.to(dev).to(torch.complex64).transpose(1, 2).contiguous()            # B x F x T
        gain, _ = _plan.ns_from_stft(X, config=self.conf, gain=True, enh=False, eps=eps)
        if not batched:
            gain = gain[0]
        return gain.cpu().numpy() if was_numpy else gain
