"""
oracle/auxiva_oracle.py -- float64 restatement of auxiva(X, epochs) of the reference's
scripts/sptk/apply_auxiva.py:24-57: the contract of the AuxIVA kernels (csrc/auxiva.cuh).

TEST INFRASTRUCTURE.  The reference already computes in complex128 (W starts as a complex128
identity and promotes everything it touches), so the float64 restatement IS the reference's dtype
flow; only BLAS summation orders differ.

Two quirks of the reference are kept as written:
  * the column update divides by w^H V w itself, not by sqrt(w^H V w) as the pyroomacoustics
    original does;
  * w^H V w is a complex number (its imaginary part is at the rounding level) and the division is a
    complex division, not a division by its real part.
"""
import numpy as np

EPSILON = float(np.finfo(np.float32).eps)   # libs/utils.py:16


def auxiva(X, epochs=20):
    """X: N x T x F (complex64 in the reference) -> Y: N x T x F complex128.
    Raises numpy.linalg.LinAlgError on an exactly singular W^H V, as the reference does."""
    X = np.asarray(X)
    N, T, F = X.shape
    Xf = np.ascontiguousarray(X.transpose(2, 1, 0)).astype(np.complex128)     # F x T x N
    W = np.tile(np.eye(N, dtype=np.complex128), (F, 1, 1))                    # F x N x N
    for _ in range(epochs):
        Y = np.einsum("ftn,fnx->ftx", Xf, W.conj())
        R = np.sqrt(np.sum(np.abs(Y)**2, axis=0))                             # T x N
        Gr = 1 / (R.T + EPSILON)                                              # N x T
        for f in range(F):
            x = Xf[f]                                                         # T x N
            for n in range(N):
                V = ((Gr[n][:, None] * x).T @ x.conj()) / T
                w = np.linalg.solve(W[f].conj().T @ V, np.eye(N)[n])
                W[f, :, n] = w / (w.conj() @ (V @ w))
    Y = np.einsum("ftn,fnx->ftx", Xf, W.conj())
    return np.ascontiguousarray(Y.transpose(2, 1, 0))


def auxiva_bnft(X, epochs=20):
    """The layout of setk_auxiva_stft: X B x N x F x T -> (Y B x N x F x T complex128, singular[B])."""
    X = np.asarray(X)
    Y = np.zeros(X.shape, np.complex128)
    bad = np.zeros(X.shape[0], bool)
    for b in range(X.shape[0]):
        try:
            Y[b] = auxiva(X[b].transpose(0, 2, 1), epochs).transpose(0, 2, 1)
        except np.linalg.LinAlgError:
            bad[b] = True
    return Y, bad
