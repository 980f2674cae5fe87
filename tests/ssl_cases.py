"""
Shared cases of the sound-source-localisation tests (tests/test_ssl.py on the CPU execution
model, tests/test_gpu_ssl.py on the device): setk_ssl through setk_b200.plan.ssl against the
float64 oracle (oracle/ssl_oracle.py) and the reference fixtures (tests/golden/ref_ssl.npz).
"""
import os

import numpy as np
import torch

from script_runner import run_script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_ssl.npz")

from oracle import ssl_oracle as so  # noqa: E402
from oracle import stft_oracle  # noqa: E402

_FIXTURE = None


def load_fixture():
    """tests/golden/ref_ssl.npz with its regenerated inputs (STFTs, steering tables, masks)."""
    global _FIXTURE
    if _FIXTURE is None:
        from setk_b200.libs import beamformer
        _FIXTURE = so.expand_fixture(np.load(GOLD), beamformer)
    return _FIXTURE


# score tolerance against the float64 oracle, relative to max |score|
TOL_F64 = 1e-9
# against the reference's own results: ML shares every rounding; SRP's float32 phases and MUSIC's
# complex64 eigh (float32 masks) are where the reference and the port legitimately differ
# (tests/golden/PINNING_ssl.json */oracle_float64_scores_rel_to_max: <= 6.3e-9)
TOL_REF = {"ml": 1e-9, "srp": 2e-8, "music": 2e-8}


def synth(rng, B, M, F, T, A, planted=True):
    """Random STFTs with a planted direction per utterance and unit-modulus steering vectors."""
    sv = np.exp(1j * rng.uniform(0, 2 * np.pi, (A, M, F))) * rng.uniform(0.5, 1.5, (A, M, F))
    X = (rng.standard_normal((B, M, F, T)) + 1j * rng.standard_normal((B, M, F, T))) * 0.3
    if planted:
        for b in range(B):
            a = (7 * b + 3) % A
            src = rng.standard_normal((F, T)) + 1j * rng.standard_normal((F, T))
            X[b] += sv[a][:, :, None] * src[None]
    return X.astype(np.complex64), sv


def windows_for(B, T):
    """Offline, a ragged stop and overlapping online chunks: W = 3 windows per utterance."""
    return np.array([[(0, T), (0, T - 1 - b), (max(T // 2 - 3, 0), T // 2 + 4)] for b in range(B)], np.int32)


def oracle_window(backend, X, sv, mask, s, e, flow="float64", **kw):
    """The oracle on frames [s, e) of one utterance X (M x F x T), mask T x F / N x T x F / None."""
    S = np.ascontiguousarray(np.transpose(X[:, :, s:e], (0, 2, 1)))           # M x T x F
    m = None if mask is None else mask[..., s:e, :]
    if backend == "ml":
        return so.ml_ssl(S, sv, mask=m, flow=flow, **kw)
    if backend == "srp":
        return so.srp_ssl(S, sv, mask=m, flow=flow, **kw)
    return so.music_ssl(S, sv, mask=m, flow=flow)


def check_scores(got, want, idx_got, idx_want, tol, what):
    scale = np.max(np.abs(want))
    err = np.max(np.abs(got - want)) / scale
    assert err <= tol, f"{what}: scores off by {err:.3e} of max|score| (tol {tol:g})"
    order = np.sort(want)
    margin = (order[-1] - order[-2]) / scale if idx_want == np.argmax(want) else (order[1] - order[0]) / scale
    if margin > 1e-6:
        assert int(idx_got) == int(idx_want), f"{what}: index {idx_got} != {idx_want} (margin {margin:.2e})"
    return err


def run_parity(device, backend, B, M, F, T, A, mask_kind, rng, windows=None, **kw):
    """plan.ssl vs the float64 oracle for every (utterance, mask, window); returns the worst error."""
    from setk_b200 import plan
    X, sv = synth(rng, B, M, F, T, A)
    if mask_kind is None:
        mask = None
    else:
        N = 2 if mask_kind == "3d" else 1
        mask = rng.uniform(0, 1, (B, N, T, F)).astype(np.float32)
        if mask_kind == "zero_bin":
            mask[:, :, :, F // 2] = 0
    win = windows_for(B, T) if windows is None else windows
    pairs = kw.pop("pairs", None)
    scores, index = plan.ssl(torch.from_numpy(X).to(device), torch.from_numpy(sv).to(device), backend=backend,
                             mask=None if mask is None else torch.from_numpy(mask).to(device), windows=win,
                             pairs=pairs, **kw)
    scores, index = scores.cpu().numpy(), index.cpu().numpy()
    okw = dict(kw)
    if backend == "ml":
        okw = dict(compression=kw.get("compression", 0.0), eps=kw.get("eps", 1e-8), norm=kw.get("normalize", False))
    elif backend == "srp":
        okw = dict(srp_pair=([p[0] for p in pairs], [p[1] for p in pairs]))
    worst = 0.0
    for b in range(B):
        for w, (s, e) in enumerate(win[b]):
            if mask is None:
                masks = [None]
            elif mask_kind == "3d":
                masks = [mask[b]]
            else:
                masks = [mask[b, 0]]
            idx_o, sc_o = oracle_window(backend, X[b], sv, masks[0], s, e, **okw)
            sc_o = np.atleast_2d(sc_o)
            idx_o = np.atleast_1d(idx_o)
            for n in range(sc_o.shape[0]):
                worst = max(worst, check_scores(scores[b, n, w], sc_o[n], index[b, n, w], idx_o[n], TOL_F64,
                                                f"{backend} b={b} n={n} w={w}"))
    return worst


def fixture_runs(g, name):
    """(run, backend, kwargs of plan.ssl, mask) of every stored reference result of mixture `name`."""
    pairs = [tuple(p) for p in g[name + "/pairs"]]
    eps = so.EPSILON
    return [
        ("ml", "ml", dict(compression=-1, eps=eps), None),
        ("ml_mask", "ml", dict(compression=-1, eps=eps), g[name + "/mask"]),
        ("ml_norm", "ml", dict(normalize=True), g[name + "/mask"]),
        ("ml_mask3", "ml", dict(compression=-1, eps=eps), g[name + "/mask3"]),
        ("ml_pow", "ml", dict(compression=0.5), g[name + "/mask"]),
        ("srp", "srp", dict(pairs=pairs), None),
        ("srp_mask", "srp", dict(pairs=pairs), g[name + "/mask"]),
        ("music", "music", {}, None),
        ("music_mask", "music", {}, g[name + "/mask_zero_bin"]),
    ]


def run_fixtures(device):
    """The kernels on the reference's inputs; indices equal, scores within TOL_REF."""
    from setk_b200 import plan
    g = load_fixture()
    worst = {}
    for name in ("lin4", "circ7", "lin2"):
        S = g[name + "/stft"]                                                    # M x T x F
        X = torch.from_numpy(np.ascontiguousarray(np.transpose(S, (0, 2, 1)))[None]).to(device)
        sv = torch.from_numpy(g[name + "/sv"]).to(device)
        for run, backend, kw, mask in fixture_runs(g, name):
            m = None
            if mask is not None:
                m = torch.from_numpy(mask[None] if mask.ndim == 3 else mask[None, None]).to(device)
            scores, index = plan.ssl(X, sv, backend=backend, mask=m, **kw)
            got = scores[0, :, 0].cpu().numpy()
            want = np.atleast_2d(g[f"{name}/{run}/scores"])
            idx_want = np.atleast_1d(g[f"{name}/{run}/index"])
            for n in range(want.shape[0]):
                err = check_scores(got[n], want[n], index[0, n, 0].item(), idx_want[n], TOL_REF[backend],
                                   f"{name}/{run}")
                assert int(index[0, n, 0]) == int(idx_want[n]), f"{name}/{run}: index differs from the reference"
                worst[backend] = max(worst.get(backend, 0.0), err)
    return worst


def write_cli_inputs(tmp_path):
    """wav.scp, mask scripts and steering vectors of the stored do_ssl.py runs."""
    import scipy.io.wavfile as wavfile
    g = load_fixture()
    np.save(tmp_path / "sv.npy", g["cli/sv"])
    scp = {"wav.scp": [], "mask0.scp": [], "mask1.scp": [], "mask2.scp": []}
    for key in ("utt0", "utt1"):
        wavfile.write(str(tmp_path / f"{key}.wav"), 16000, g[f"cli/{key}/pcm16"].T)
        scp["wav.scp"].append(f"{key} {tmp_path / (key + '.wav')}")
        for j in range(3):
            np.save(tmp_path / f"{key}_m{j}.npy", g[f"cli/{key}/mask{j}"])
            scp[f"mask{j}.scp"].append(f"{key} {tmp_path / f'{key}_m{j}.npy'}")
    for name, lines in scp.items():
        (tmp_path / name).write_text("\n".join(lines) + "\n")
    return g


CLI_RUNS = ("ml", "ml_radian", "ml_index", "srp", "music", "ml_wta", "srp_mask", "music_mask", "ml_online",
            "ml_online_range")


def cli_argv(tmp_path, flags, out):
    import json
    argv = []
    for k, v in json.loads(flags).items():
        if k == "mask_scp":
            v = ",".join(str(tmp_path / s) for s in v.split(","))
        argv += ["--" + k.replace("_", "-"), str(v)]
    return argv + [str(tmp_path / "wav.scp"), str(tmp_path / "sv.npy"), str(out)]


def check_cli(tmp_path, library=None):
    g = write_cli_inputs(tmp_path)
    for run in CLI_RUNS:
        out = tmp_path / f"{run}.txt"
        run_script("do_ssl.py", cli_argv(tmp_path, str(g[f"cli/{run}/flags"]), out), library)
        assert out.read_text() == str(g[f"cli/{run}/doa_scp"]), f"do_ssl.py {run}: output differs"


def check_cli_online_mask(tmp_path, library=None):
    """Online mode with a mask (the reference fails there): every chunk equals the oracle run on the
    chunk's frames of the STFT and of the mask."""
    g = write_cli_inputs(tmp_path)
    out = tmp_path / "online_mask.txt"
    run_script("do_ssl.py", ["--chunk-len", "6", "--look-back", "9", "--mask-scp", str(tmp_path / "mask2.scp"),
                             "--doa-range", "0,180", str(tmp_path / "wav.scp"), str(tmp_path / "sv.npy"), str(out)],
               library)
    lines = dict(line.split("\t") for line in out.read_text().splitlines())
    labels = so.doa_labels(0, 180, g["cli/sv"].shape[0], "degree")
    for key in ("utt0", "utt1"):
        x = stft_oracle.float_from_pcm16(g[f"cli/{key}/pcm16"])
        S = stft_oracle.multichannel_stft(x, frame_len=512, frame_hop=256, window="hann", center=True,
                                          round_power_of_two=True, transpose=True)          # M x T x F
        mask = g[f"cli/{key}/mask2"].T                                                      # T x F
        want = []
        for s, e in so.online_windows(S.shape[1], 6, 9):
            idx, _ = so.ml_ssl(S[:, s:e], g["cli/sv"], mask=mask[s:e], compression=-1, eps=so.EPSILON)
            want.append(f"{labels[idx]:.4f}")
        assert lines[key] == " ".join(want), key
