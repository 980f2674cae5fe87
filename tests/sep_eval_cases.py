"""
Shared helpers of the separation-metric tests (tests/test_sep_eval.py, tests/test_gpu_sep_eval.py):
speech from the simulation fixture's inputs, deterministic estimates, the tolerance rule and a small
scp/wav corpus for the two command lines.
"""
import os

import numpy as np
import scipy.io.wavfile as wavfile
import scipy.signal

from oracle import sep_eval_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def speech():
    """spk1, spk2 and noise of the simulation fixture (the reference's doc/data_simu assets, 4 s), float32"""
    z = np.load(os.path.join(GOLDEN, "ref_simu.npz"))
    return [z[f"in/{f}"].astype(np.float32) / 32768 for f in ("spk1.wav", "spk2.wav", "noise.wav")]


def sources(N, S, offset=0):
    """N references of S samples cut from the fixture's speech and noise (sources i and i + 3 differ in offset)"""
    sp = speech()
    out = []
    for i in range(N):
        src = sp[i % 3]
        start = (offset + 4001 * (i // 3)) % (src.size - S)
        out.append(src[start:start + S])
    return np.stack(out).astype(np.float32)


def estimates(refs, seed=0, swap=False, noise=0.05):
    """short-FIR-filtered references with cross-talk and white noise (float32); swap reverses the order"""
    rng = np.random.default_rng(seed)
    N, S = refs.shape
    out = []
    for j in range(N):
        h = np.array([1.0, 0.3, -0.1], np.float64) * (1 + 0.1 * j)
        e = scipy.signal.lfilter(h, [1.0], refs[j].astype(np.float64))
        e += 0.2 * refs[(j + 1) % N] if N > 1 else 0.0
        e += noise * np.std(refs[j]) * rng.standard_normal(S)
        out.append(e)
    out = np.stack(out)
    return (out[::-1] if swap else out).astype(np.float32)


def delayed_pair(S, delay=3):
    """two references, the second an exact delay of the first (the first ends in `delay` zeros)"""
    s0 = sources(1, S)[0].copy()
    s0[S - delay:] = 0
    s1 = np.zeros_like(s0)
    s1[delay:] = s0[:S - delay]
    return np.stack([s0, s1])


def assert_criteria_close(got, want, what=""):
    """1e-4 dB up to 60 dB, 1e-2 dB above; +inf where both are infinite"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    both_inf = np.isinf(got) & np.isinf(want) & (np.sign(got) == np.sign(want))
    fin = ~both_inf
    assert np.all(np.isfinite(got[fin])) and np.all(np.isfinite(want[fin])), f"{what}: {got} vs {want}"
    tol = np.where(np.abs(want[fin]) <= 60, 1e-4, 1e-2)
    err = np.abs(got[fin] - want[fin])
    assert np.all(err <= tol), f"{what}: max error {err.max():.3g} dB\n{got}\n{want}"


def oracle_criteria(refs, ests, flen, explicit=False):
    return so.criteria(refs, ests, flen, project=so.explicit_projection if explicit else so._fft_project)


def write_corpus(tmp, utts, n_spk, tag):
    """utts: {key: (refs (N, S), ests (N, S'))}; PCM-16 wavs and one scp per speaker and side.
    Returns (sep_scp, ref_scp) comma-joined, and the PCM-rounded float arrays that were written."""
    os.makedirs(tmp, exist_ok=True)
    scps = {"sep": [], "ref": []}
    stored = {}
    for side in ("sep", "ref"):
        for k in range(n_spk):
            path = os.path.join(tmp, f"{tag}_{side}{k}.scp")
            with open(path, "w") as f:
                for key, (refs, ests) in utts.items():
                    x = (ests if side == "sep" else refs)[k]
                    pcm = np.clip(np.round(np.asarray(x, np.float64) * 32768), -32768, 32767).astype(np.int16)
                    wav = os.path.join(tmp, f"{tag}_{key}_{side}{k}.wav")
                    wavfile.write(wav, 16000, pcm.T if pcm.ndim > 1 else pcm)
                    f.write(f"{key}\t{wav}\n")
                    stored[(key, side, k)] = pcm.astype(np.float32) / 32768
            scps[side].append(path)
    return ",".join(scps["sep"]), ",".join(scps["ref"]), stored


def golden():
    return np.load(os.path.join(GOLDEN, "ref_sep_eval.npz"))


def golden_signals(z, name, key):
    """(refs, ests) of a fixture utterance as compute_sdr.py scores it: channel 0, truncated, float32"""
    n_spk = len([k for k in z.files if k.startswith(f"wav/{name}/ref") and k.endswith("/" + key)])
    r = [z[f"wav/{name}/ref{k}/{key}"] for k in range(n_spk)]
    e = [z[f"wav/{name}/sep{k}/{key}"] for k in range(n_spk)]
    r, e = ([(x[:, 0] if x.ndim > 1 else x).astype(np.float32) / 32768 for x in xs] for xs in (r, e))
    n = min(r[0].size, e[0].size)
    return np.stack([x[:n] for x in r]), np.stack([x[:n] for x in e])


def golden_keys(z, name):
    return sorted({k.split("/")[3] for k in z.files if k.startswith(f"wav/{name}/ref0/")})


def _numbers(text):
    import re
    parts = re.split(r"(-?\d+\.\d+)", text)
    return parts[0::2], [float(x) for x in parts[1::2]]


def assert_text_close(got, want, tol, what=""):
    """the same text with every decimal number within tol"""
    gw, gn = _numbers(got)
    ww, wn = _numbers(want)
    assert gw == ww, f"{what}: {got!r} vs {want!r}"
    assert np.all(np.abs(np.array(gn) - np.array(wn)) <= tol), f"{what}: {got!r} vs {want!r}"


def check_golden_run(z, run, run_script_fn, tmp, library=None, batch_size=None):
    """run `run` of the fixture with this repository's script and compare it with the reference's"""
    from oracle.make_golden_sep_eval import RUNS, run_args, write
    files = {k: z[k] for k in z.files if k.startswith("wav/")}
    scps = write(files, str(tmp))
    script, argv = run_args(run, scps, str(tmp), str(tmp))
    if batch_size is not None:
        argv += ["--batch-size", str(batch_size)]
    r = run_script_fn(script, argv, library=library)
    # SDR: two 2-decimal roundings of values within 1e-4 dB; SI-SNR: fp64 against the reference's float32
    tol = 0.0101
    with open(os.path.join(str(tmp), f"{run}.per_utt")) as f:
        assert_text_close(f.read(), str(z[f"out/{run}/per_utt"]), tol, f"{run} per_utt")
    if RUNS[run][4]:
        with open(os.path.join(str(tmp), f"{run}.ali")) as f:
            assert f.read() == str(z[f"out/{run}/ali"]), run
    assert_text_close(r.stdout, str(z[f"out/{run}/report"]), 0.0011, f"{run} report")
