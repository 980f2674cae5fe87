"""
oracle/ns_oracle.py -- float64 restatement of iMCRA.__init__ / iMCRA.run of the reference's
scripts/sptk/libs/ns.py:212-387 (Cohen 2003: iMCRA noise estimation + the OM-LSA gain): the
contract of the noise-suppression kernel (csrc/ns.cu, setk_ns_imcra).

TEST INFRASTRUCTURE.  Vectorised over bins, one Python loop over frames, statements in the
reference's order.  Differences from the reference, none of which flips a threshold decision on
the stored fixtures (tests/golden/PINNING_ns.json):
  * |x|^2 is formed in float64 from the complex64 STFT (the reference squares in float32);
  * E1 is scipy.special.exp1, not scipy.integrate.quad through np.vectorize (ns.py:259-262).

Reference quirks kept as written:
  * E1(0): on an exactly zero cell (|x|^2 = 0, so v = 0) quad returns 37.191280375549404 (with an
    IntegrationWarning) where E1(0) is +inf; that finite value is used, so gh1 stays finite and the
    following frames do not become NaN.  For 0 < v < 1e-12 quad is wrong as well (at v = 1e-30 it
    returns 37.19 where E1 = 68.5); the true E1 is used there -- a documented deviation.
  * h_mcra = "hann" with w_mcra = 1 is the PERIODIC 3-point Hann window [0, .75, .75]: the "same"
    convolution averages bins f and f - 1 only, an asymmetric smoothing.
  * gamma is not floored (MCRA floors it, iMCRA does not); the eps floors sit where ns.py puts them.
  * var_sf_hat starts from the PREVIOUS var_s_hat; at t = 0 var_s_hat is not updated and
    var_s_min_hat = var_s.
  * every V frames the minima become the min over the last U PER-FRAME values of the sub-window
    minima (ns.py:370-380), not over U sub-window minima.
  * gain = gh1**p * gmin**(1 - p), in float64 (gh1 reaches ~1e6 after a silent frame).
"""
import numpy as np
import scipy.signal as ss
import scipy.special as sp

# what scipy.integrate.quad returns for the integral of exp(-t) / t over [0, inf) (ns.py:259-260)
E1_AT_ZERO = 37.191280375549404

DEFAULTS = dict(alpha=0.92, alpha_s=0.9, alpha_d=0.85, b_min=1.66, gamma0=4.6, gamma1=3, zeta0=1.67,
                xi_min_db=-18, gmin_db=-10, w_mcra=1, h_mcra="hann", beta=1.47, V=15, U=8)


def expint(v):
    """E1 as the reference's quad gives it at v == 0, scipy.special.exp1 elsewhere."""
    v = np.asarray(v, dtype=np.float64)
    out = sp.exp1(np.where(v == 0, 1.0, v))
    return np.where(v == 0, E1_AT_ZERO, out)


def mcra_window(h_mcra="hann", w_mcra=1):
    """self.w_m of iMCRA.__init__ (ns.py:243)."""
    return ss.get_window(h_mcra, w_mcra * 2 + 1)


class iMCRA(object):
    """iMCRA / OM-LSA with the reference's constructor (ns.py:221-245)."""

    def __init__(self, alpha=0.92, alpha_s=0.9, alpha_d=0.85, b_min=1.66, gamma0=4.6, gamma1=3, zeta0=1.67,
                 xi_min_db=-18, gmin_db=-10, w_mcra=1, h_mcra="hann", beta=1.47, V=15, U=8):
        self.alpha = {"s": alpha_s, "d": alpha_d, "t": alpha}
        self.beta = beta
        self.gamma0, self.gamma1 = gamma0, gamma1
        self.zeta0 = zeta0
        self.b_min = 1 / b_min
        self.xi_min = 10**(xi_min_db / 10)
        self.gain_min = 10**(gmin_db / 10)
        self.w_m = mcra_window(h_mcra, w_mcra)
        self.V = V
        self.U = U

    def run(self, stft, eps=1e-7):
        """stft: T x F complex -> gain T x F float64 (ns.py:247-387)."""
        stft = np.asarray(stft)
        T, F = stft.shape
        obs_power = stft.real.astype(np.float64)**2 + stft.imag.astype(np.float64)**2
        a_s, a_d, a_t = self.alpha["s"], self.alpha["d"], self.alpha["t"]

        def conv(x):
            return np.convolve(x, self.w_m, mode="same")

        lambda_d_hat = obs_power[0]
        gh1 = 1
        s_min_sw, s_min_sw_hat, G = [], [], []
        for t in range(T):
            lambda_d = lambda_d_hat * self.beta
            gamma = obs_power[t] / np.maximum(lambda_d, eps)
            gain = gh1**2 * gamma
            xi_hat = a_t * gain + (1 - a_t) * np.maximum(gamma - 1, 0)
            xi_hat = np.maximum(xi_hat, self.xi_min)
            v = gamma * xi_hat / (1 + xi_hat)
            gh1 = xi_hat / (1 + xi_hat) * np.exp(0.5 * expint(v))
            var_sf = conv(obs_power[t])
            if t == 0:
                var_s = var_s_hat = var_s_min = var_s_min_sw = var_sf
            else:
                var_s = a_s * var_s + (1 - a_s) * var_sf
                var_s_min = np.minimum(var_s_min, var_s)
                var_s_min_sw = np.minimum(var_s_min_sw, var_s)
            gamma_min = obs_power[t] * self.b_min / np.maximum(var_s_min, eps)
            zeta = var_sf * self.b_min / np.maximum(var_s_min, eps)
            indicator = np.logical_and(gamma_min < self.gamma0, zeta < self.zeta0)
            ind_conv = conv(indicator.astype(np.float64))
            ind_nz = ind_conv > 0
            obs_conv = conv(obs_power[t] * indicator)
            var_sf_hat = var_s_hat.copy()
            var_sf_hat[ind_nz] = obs_conv[ind_nz] / ind_conv[ind_nz]
            if t == 0:
                var_s_min_hat = var_s
                var_s_min_sw_hat = var_sf
            else:
                var_s_hat = a_s * var_s_hat + (1 - a_s) * var_sf_hat
                var_s_min_hat = np.minimum(var_s_min_hat, var_s_hat)
                var_s_min_sw_hat = np.minimum(var_s_min_sw_hat, var_s_hat)
            gamma_min_hat = obs_power[t] * self.b_min / np.maximum(var_s_min_hat, eps)
            zeta_hat = var_s * self.b_min / np.maximum(var_s_min_hat, eps)
            q_idx = (gamma_min_hat > 1) & (gamma_min_hat < self.gamma1) & (zeta_hat < self.zeta0)
            q_hat = np.zeros(F)
            q_hat[q_idx] = (self.gamma1 - gamma_min_hat[q_idx]) / (self.gamma1 - 1)
            p_hat = np.zeros(F)
            p_hat[q_idx] = 1 / (1 + q_hat[q_idx] * (1 + xi_hat[q_idx]) / (1 - q_hat[q_idx]) * np.exp(-v[q_idx]))
            p_hat[(gamma_min_hat >= self.gamma1) & (zeta_hat >= self.zeta0)] = 1
            alpha_d_hat = a_d + (1 - a_d) * p_hat
            lambda_d_hat = alpha_d_hat * lambda_d_hat + (1 - alpha_d_hat) * obs_power[t]
            s_min_sw.append(var_s_min_sw)
            s_min_sw_hat.append(var_s_min_sw_hat)
            if (t + 1) % self.V == 0:
                var_s_min = np.min(np.stack(s_min_sw[-self.U:]), 0)
                var_s_min_hat = np.min(np.stack(s_min_sw_hat[-self.U:]), 0)
                var_s_min_sw = var_s
                var_s_min_sw_hat = var_s_hat
            G.append(gh1**p_hat * self.gain_min**(1 - p_hat))
        return np.stack(G)


def ns_bft(stft, n_frames=None, eps=1e-7, **conf):
    """The layout of setk_ns_imcra: stft B x F x T -> (gain B x T x F float64, enh B x F x T complex128).
    Utterance b runs over its first n_frames[b] frames; later frames get gain 0 and enh 0."""
    stft = np.asarray(stft)
    B, F, T = stft.shape
    gain = np.zeros((B, T, F))
    enh = np.zeros((B, F, T), np.complex128)
    est = iMCRA(**conf)
    for b in range(B):
        Tb = T if n_frames is None else int(n_frames[b])
        if Tb <= 0:
            continue
        g = est.run(stft[b, :, :Tb].T)
        gain[b, :Tb] = g
        enh[b, :, :Tb] = g.T * stft[b, :, :Tb].astype(np.complex128)
    return gain, enh
