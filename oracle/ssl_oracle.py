"""
oracle/ssl_oracle.py -- numpy restatement of the reference's sound source localisation
(scripts/sptk/libs/ssl.py ml_ssl / srp_ssl / music_ssl) and of do_ssl.py's host logic
(winner-take-all masks, direction labels, online chunk windows).

TEST INFRASTRUCTURE.  Every estimator returns (index, scores) and takes `flow`:
  * "reference": numpy's dtype promotion exactly as the reference meets it -- float32 ssh,
    float32 np.angle phases, and for MUSIC the covariance and eigh in complex64 when the mask
    is float32 (complex128 when it is absent, since np.ones is float64);
  * "float64": the arithmetic the CUDA kernels promise -- the float32 quantities the
    reference rounds once (ssh, the norm=True scaling, the SRP phases, taken as the
    correctly rounded angle) stay float32, everything downstream is float64, MUSIC's
    covariance and eigenvectors included.
"""
import numpy as np

EPSILON = float(np.finfo(np.float32).eps)


def _ssh_f32(stft):
    """|sum_m x conj(x)| of a complex64 M x T x F STFT: per channel re*re + im*im, added in
    channel order, every step rounded to float32 (what einsum does for complex64)."""
    acc = np.zeros(stft.shape[1:], dtype=np.float32)
    for x in stft:
        acc = acc + (x.real * x.real + x.imag * x.imag)
    return acc


def _normalise_f32(stft, eps):
    """stft / max(|stft|, eps) for complex64: numpy multiplies by the float32 reciprocal."""
    mag = np.sqrt(stft.real * stft.real + stft.imag * stft.imag)
    inv = np.float32(1) / np.maximum(mag, np.float32(eps))
    return (stft.real * inv + 1j * (stft.imag * inv)).astype(np.complex64)


def ml_ssl(stft, sv, compression=0, eps=1e-8, norm=False, mask=None, flow="reference"):
    stft = np.asarray(stft)
    _, T, F = stft.shape
    unit = sv / np.linalg.norm(sv, axis=1, keepdims=True)         # A x M x F
    if norm:
        stft = _normalise_f32(stft, eps)
    ssh = _ssh_f32(stft).astype(np.float64)                      # T x F
    proj = np.einsum("amf,mtf->atf", unit, np.conj(stft).astype(np.complex128))
    # |.|^2: the reference squares np.abs (a hypot); the kernels add the squared parts
    ssv = np.abs(proj)**2 if flow == "reference" else proj.real**2 + proj.imag**2
    delta = ssh[None] - ssv / (1 + eps)
    with np.errstate(invalid="ignore", divide="ignore"):
        ll = -np.log(np.maximum(delta, eps)) if compression <= 0 else -np.power(delta, compression)
    if mask is None:
        scores = ll.sum(axis=(1, 2))
    elif np.ndim(mask) == 2:
        scores = (np.asarray(mask)[None] * ll).sum(axis=(1, 2))
    else:
        scores = np.einsum("ntf,atf->na", np.asarray(mask), ll)
    return np.argmax(scores, axis=-1), scores


def _angle_rounded(z):
    return np.arctan2(z.imag.astype(np.float64), z.real.astype(np.float64)).astype(np.float32)


def srp_ssl(stft, sv, srp_pair=None, mask=None, flow="reference"):
    if srp_pair is None:
        raise ValueError("srp_pair cannot be None, (list, list)")
    stft = np.asarray(stft)
    left, right = (list(np.atleast_1d(p)) for p in srp_pair)
    pha = np.angle(stft) if flow == "reference" else _angle_rounded(stft)   # float32
    obs = pha[left] - pha[right]                                  # P x T x F, float32
    sv_pha = np.angle(sv)
    ora = sv_pha[:, left] - sv_pha[:, right]                      # A x P x F, float64
    resp = np.cos(obs[None] - ora[:, :, None, :]).mean(axis=1)    # A x T x F
    w = np.ones(stft.shape[1:]) if mask is None else np.asarray(mask)
    scores = (resp * w[None]).sum(axis=(1, 2))
    return np.argmax(scores), scores


def music_ssl(stft, sv, mask=None, flow="reference"):
    stft = np.asarray(stft)
    _, T, F = stft.shape
    w = np.ones((T, F)) if mask is None else np.asarray(mask)
    if flow == "float64":
        stft, w = stft.astype(np.complex128), w.astype(np.float64)
    # complex64 rounding depends on the contraction numpy picks: einsum, as in the reference
    y = np.transpose(stft * w, (2, 0, 1))                         # F x M x T
    cov = np.einsum("fit,fjt->fij", y, np.conj(y)) / T            # F x M x M
    _, vec = np.linalg.eigh(cov)                                  # ascending eigenvalues
    minor = vec[..., :-1]
    proj = np.einsum("fik,fjk->fij", minor, np.conj(minor))       # F x M x M
    s = np.transpose(sv, (2, 0, 1))                               # F x A x M
    quad = np.einsum("...i,...ij,...j->...", np.conj(s), proj[:, None], s)
    scores = np.abs(quad).sum(axis=0)
    return np.argmin(scores), scores


def add_wta(masks, eps=1e-4):
    """Winner-take-all over a list of masks: a cell keeps its value where it is the largest."""
    top = np.max(np.stack(masks, axis=-1), axis=-1)
    return [np.where(m == top, m, eps) for m in masks]


def doa_labels(lo, hi, num_doa, output):
    """The label of every direction index (do_ssl.py): linspace over A + 1 points."""
    if output == "radian":
        return np.linspace(lo * np.pi / 180, hi * np.pi / 180, num_doa + 1)
    return np.linspace(lo, hi, num_doa + 1)


def online_windows(T, chunk_len, look_back):
    """Frame ranges [max(t - look_back, 0), min(t + chunk_len, T)) for t = 0, chunk_len, ..."""
    return [(max(t - look_back, 0), min(t + chunk_len, T)) for t in range(0, T, chunk_len)]


def estimate(backend, stft, sv, mask=None, srp_pair=None, flow="reference"):
    """get_doa of do_ssl.py: the backend with do_ssl's arguments -> (index, scores)."""
    if backend == "srp":
        return srp_ssl(stft, sv, srp_pair=srp_pair, mask=mask, flow=flow)
    if backend == "ml":
        return ml_ssl(stft, sv, mask=mask, compression=-1, eps=EPSILON, flow=flow)
    return music_ssl(stft, sv, mask=mask, flow=flow)


# ---- inputs of tests/golden/ref_ssl.npz that are regenerated instead of stored ----------------
# The fixture keeps the PCM-16 audio, exact slices ("pins") of the reference's STFTs and steering
# tables, and the reference's results; the STFTs, steering tables and seeded masks are rebuilt here.
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)
FIXTURE_GEOMETRY = {
    "lin4": dict(kind="linear", topo=[0.0, 0.04, 0.08, 0.12], A=37, doa=60.0, n=8000, seed=11),
    "circ7": dict(kind="circular", radius=0.05, A=72, doa=200.0, n=6000, seed=12),
    "lin2": dict(kind="linear", topo=[0.0, 0.1], A=19, doa=120.0, n=6000, seed=13),
}
CLI_TOPO, CLI_NUM_DOA = [0.0, 0.04, 0.08, 0.12], 37


def fixture_stft(pcm):
    """M x T x F complex64 STFT of PCM-16 audio, as do_ssl.py's SpectrogramReader computes it."""
    from . import stft_oracle
    x = stft_oracle.float_from_pcm16(pcm)
    return np.stack([stft_oracle.forward_stft(np.ascontiguousarray(c), transpose=True, out_dtype=np.complex64, **STFT_KW)
                     for c in x])


def fixture_steering(bf, geo, num_bins=257):
    """A x M x F steering table of a fixture geometry; bf provides linear_/circular_steer_vector."""
    if geo["kind"] == "linear":
        sv = [bf.linear_steer_vector(np.array(geo["topo"]), d, num_bins, c=343)
              for d in np.linspace(0, 180, geo["A"])]
    else:
        sv = [bf.circular_steer_vector(geo["radius"], 6, d, num_bins, c=343, center=True)
              for d in np.arange(0, 360, 360 / geo["A"])]
    return np.ascontiguousarray(np.stack(sv).transpose(0, 2, 1))


def fixture_masks(seed, T, F):
    """(2-D mask, 3-D mask with N = 2, 2-D mask that is zero in every frame of bin 37), float32."""
    rng = np.random.default_rng(seed + 1000)
    mask = rng.uniform(0, 1, (T, F)).astype(np.float32)
    mask3 = rng.uniform(0, 1, (2, T, F)).astype(np.float32)
    zero = mask.copy()
    zero[:, 37] = 0
    return mask, mask3, zero


def cli_masks(k, T, F=257):
    """The three mask files of CLI utterance k: two T x F, the third stored F x T."""
    rng = np.random.default_rng(77 + k)
    m = [rng.uniform(0, 1, (T, F)).astype(np.float32) for _ in range(3)]
    m[2] = np.ascontiguousarray(m[2].T)
    return m


def expand_fixture(stored, bf):
    """The stored fixture plus its regenerated inputs (dict): <name>/{stft,sv,mask,mask3,
    mask_zero_bin}, cli/sv, cli/<key>/mask<j>.  Pins are checked: the regenerated arrays must equal
    the reference's exactly where the fixture stored them."""
    g = {k: stored[k] for k in stored.keys()}
    for name, geo in FIXTURE_GEOMETRY.items():
        S = fixture_stft(g[name + "/pcm16"])
        sv = fixture_steering(bf, geo)
        assert np.array_equal(S[:, :, ::16], g[name + "/stft_pin"]), name + ": STFT differs from the reference's"
        assert np.array_equal(sv[:, :, ::16], g[name + "/sv_pin"]), name + ": steering differs from the reference's"
        g[name + "/stft"], g[name + "/sv"] = S, sv
        g[name + "/mask"], g[name + "/mask3"], g[name + "/mask_zero_bin"] = fixture_masks(geo["seed"], *S.shape[1:])
        assert np.array_equal(g[name + "/mask"][0, :8], g[name + "/mask_head"]), name + ": mask stream"
    g["cli/sv"] = fixture_steering(bf, dict(kind="linear", topo=CLI_TOPO, A=CLI_NUM_DOA))
    assert np.array_equal(g["cli/sv"][:, :, ::16], g["cli/sv_pin"])
    for k in range(2):
        T = 1 + g[f"cli/utt{k}/pcm16"].shape[1] // STFT_KW["frame_hop"]
        for j, m in enumerate(cli_masks(k, T)):
            g[f"cli/utt{k}/mask{j}"] = m
    return g
