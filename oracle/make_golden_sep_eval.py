"""
oracle/make_golden_sep_eval.py -- tests/golden/ref_sep_eval.npz and PINNING_sep_eval.json: the
reference's own scripts/sptk/compute_si_snr.py and compute_sdr.py, run unmodified under
oracle/ref_shim.py on a small corpus cut from doc/data_simu/asset.

Stubs the scripts need here:
  * editdistance (imported by libs/metric.py, used only by permute_ed, which no run reaches);
  * mir_eval.separation (not installed): bss_eval_sources is oracle/sep_eval_oracle.py's, mir_eval's
    FFT / Toeplitz / solve route.  No mir_eval run was available, so compute_sdr.py's runs pin the
    script's glue (channel 0, truncation, the mean, the formats, the report) to the reference's own
    code, and the BSS-Eval numbers are pinned separately to the definition through the explicit
    dense least-squares route (bss_explicit/*).

Corpus (PCM-16, 16 kHz), cut from spk1.wav, spk2.wav and noise.wav:
  two/     N = 2, keys u1 .. u4: FIR-filtered references with cross-talk and noise; u2's estimates
           swapped; u3's estimates 40 samples longer than its references; u4's speaker-0 estimate a
           two-channel file (channel 0 is the estimate); spk2class u1, u3 -> F, u2, u4 -> M;
  three/   N = 3, keys v1 (estimates a 3-cycle of the references) and v2.
The npz holds every file (wav/<set>/<side><k>/<key>), the spk2class table, each run's --per-utt,
--utt-ali and report (out/<run>/...), the reference's own float32 si_snr of every (estimate,
reference) pair (si_snr_ref/<set>/<key>, [j, i], on the truncated signals), and the explicit-route
criteria (bss_explicit/<set>/<key>, [k, j, i], L = 512).
Run from the repository root where the reference tree exists.
"""
import contextlib
import io
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import scipy.io.wavfile as wavfile
import scipy.signal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, sep_eval_oracle as so  # noqa: E402

ASSET = "/root/reference/doc/data_simu/asset"
FLEN = 512


def pcm(x):
    return np.clip(np.round(np.asarray(x, np.float64) * 32768), -32768, 32767).astype(np.int16)


def corpus():
    src = [wavfile.read(os.path.join(ASSET, f))[1].astype(np.float64) / 32768
           for f in ("spk1.wav", "spk2.wav", "noise.wav")]
    rng = np.random.default_rng(2024)

    def refs(N, S, off):
        return np.stack([src[i][off + 3000 * i:off + 3000 * i + S] for i in range(N)])

    def ests(r, order):
        N, S = r.shape
        out = []
        for j in range(N):
            e = scipy.signal.lfilter([1.0, 0.3 + 0.05 * j, -0.1], [1.0], r[j])
            e = e + 0.25 * r[(j + 1) % N] + 0.03 * np.std(r[j]) * rng.standard_normal(S)
            out.append(e)
        return np.stack(out)[list(order)]

    sets = {"two": {}, "three": {}}
    for key, S, off, order in (("u1", 8000, 16000, (0, 1)), ("u2", 6000, 24000, (1, 0)),
                               ("u3", 7000, 30000, (0, 1)), ("u4", 7500, 40000, (0, 1))):
        r = refs(2, S, off)
        e = ests(r, order)
        if key == "u3":
            e = np.concatenate([e, 0.01 * rng.standard_normal((2, 40))], axis=1)
        sets["two"][key] = (r, e)
    for key, S, off, order in (("v1", 6000, 20000, (1, 2, 0)), ("v2", 5000, 36000, (0, 1, 2))):
        r = refs(3, S, off)
        sets["three"][key] = (r, ests(r, order))
    files = {}
    for name, utts in sets.items():
        for key, (r, e) in utts.items():
            for k in range(r.shape[0]):
                files[f"wav/{name}/ref{k}/{key}"] = pcm(r[k])
                x = pcm(e[k])
                if name == "two" and key == "u4" and k == 0:   # a two-channel file: channel 0 is the estimate
                    x = np.stack([x, pcm(0.5 * r[1])], axis=1)
                files[f"wav/{name}/sep{k}/{key}"] = x
    return files


def write(files, tmp):
    """the wavs and one scp per (set, side, speaker); returns {set: (sep_scps, ref_scps)} comma-joined"""
    scps = {}
    for name in sorted({k.split("/")[1] for k in files}):
        n_spk = len({k.split("/")[2] for k in files if k.startswith(f"wav/{name}/ref")})
        sides = {}
        for side in ("sep", "ref"):
            paths = []
            for k in range(n_spk):
                prefix = f"wav/{name}/{side}{k}/"
                path = os.path.join(tmp, f"{name}_{side}{k}.scp")
                with open(path, "w") as f:
                    for fk in sorted(x for x in files if x.startswith(prefix)):
                        key = fk[len(prefix):]
                        wav = os.path.join(tmp, f"{name}_{side}{k}_{key}.wav")
                        wavfile.write(wav, 16000, files[fk])
                        f.write(f"{key}\t{wav}\n")
                paths.append(path)
            sides[side] = ",".join(paths)
        scps[name] = (sides["sep"], sides["ref"])
    return scps


SPK2CLASS = "u1\tF\nu2\tM\nu3\tF\nu4\tM\n"
RUNS = {   # run: (script, set, speakers (None: all), spk2class, want alignment)
    "sdr_two": ("compute_sdr.py", "two", None, True, True),
    "sdr_three": ("compute_sdr.py", "three", None, False, True),
    "si_two": ("compute_si_snr.py", "two", None, True, True),
    "si_three": ("compute_si_snr.py", "three", None, False, True),
    "si_single": ("compute_si_snr.py", "two", 1, False, False),
}


def run_args(run, scps, tmp, out_dir):
    script, name, spk, s2c, ali = RUNS[run]
    sep, ref = scps[name]
    if spk is not None:
        sep, ref = sep.split(",")[spk], ref.split(",")[spk]
    argv = [sep, ref, "--per-utt", os.path.join(out_dir, f"{run}.per_utt")]
    if ali:
        argv += ["--utt-ali", os.path.join(out_dir, f"{run}.ali")]
    if s2c:
        path = os.path.join(tmp, "spk2class")
        with open(path, "w") as f:
            f.write(SPK2CLASS)
        argv += ["--spk2class", path]
    return script, argv


def read(path):
    with open(path) as f:
        return f.read()


def main():
    ns = ref_shim.load_reference()
    sys.modules.setdefault("editdistance", types.ModuleType("editdistance"))
    mir, sep_mod = types.ModuleType("mir_eval"), types.ModuleType("mir_eval.separation")
    sep_mod.bss_eval_sources = so.bss_eval_sources
    mir.separation = sep_mod
    sys.modules["mir_eval"], sys.modules["mir_eval.separation"] = mir, sep_mod
    import importlib
    ref_metric = importlib.import_module("libs.metric")
    assert ns.data_handler is not None

    files = corpus()
    tmp = tempfile.mkdtemp()
    scps = write(files, tmp)
    store = dict(files)
    store["spk2class"] = np.array(SPK2CLASS)
    for run in RUNS:
        script, argv = run_args(run, scps, tmp, tmp)
        buf = io.StringIO()
        old = sys.argv
        sys.argv = [script] + argv
        try:
            with contextlib.redirect_stdout(buf):
                runpy.run_path(os.path.join(ref_shim.REFERENCE_SPTK, script), run_name="__main__")
        finally:
            sys.argv = old
        store[f"out/{run}/report"] = np.array(buf.getvalue())
        store[f"out/{run}/per_utt"] = np.array(read(os.path.join(tmp, f"{run}.per_utt")))
        if RUNS[run][4]:
            store[f"out/{run}/ali"] = np.array(read(os.path.join(tmp, f"{run}.ali")))
        print(run, buf.getvalue().replace("\n", " | "))

    pin = {"note": "no mir_eval run was available: compute_sdr.py ran with oracle/sep_eval_oracle.py's "
                   "FFT route as mir_eval.separation; the BSS-Eval numbers are pinned to the definition "
                   "through the explicit dense least-squares route",
           "si_snr_fp64_vs_reference_float32_db": {}, "fft_route_vs_explicit_db": {}}
    for name in ("two", "three"):
        keys = sorted({k.split("/")[3] for k in files if k.startswith(f"wav/{name}/ref0/")})
        n_spk = 2 if name == "two" else 3
        for key in keys:
            r = np.stack([files[f"wav/{name}/ref{k}/{key}"] for k in range(n_spk)]).astype(np.float32) / 32768
            e = [files[f"wav/{name}/sep{k}/{key}"] for k in range(n_spk)]
            e = [(x[:, 0] if x.ndim > 1 else x).astype(np.float32) / 32768 for x in e]
            n = min(r.shape[-1], e[0].size)
            r, e = r[:, :n], np.stack([x[:n] for x in e])
            m = np.array([[ref_metric.si_snr(e[j], r[i]) for i in range(n_spk)] for j in range(n_spk)])
            store[f"si_snr_ref/{name}/{key}"] = m
            m64 = np.array([[so.si_snr(e[j], r[i]) for i in range(n_spk)] for j in range(n_spk)])
            pin["si_snr_fp64_vs_reference_float32_db"][f"{name}/{key}"] = float(np.abs(m64 - m).max())
            exp = so.criteria(r, e, FLEN, project=so.explicit_projection)
            fft = so.criteria(r, e, FLEN)
            store[f"bss_explicit/{name}/{key}"] = exp
            pin["fft_route_vs_explicit_db"][f"{name}/{key}"] = float(np.abs(fft - exp).max())
            print(name, key, pin["si_snr_fp64_vs_reference_float32_db"][f"{name}/{key}"],
                  pin["fft_route_vs_explicit_db"][f"{name}/{key}"])
    out = os.path.join(ROOT, "tests", "golden", "ref_sep_eval.npz")
    np.savez_compressed(out, **store)
    with open(os.path.join(ROOT, "tests", "golden", "PINNING_sep_eval.json"), "w") as f:
        json.dump(pin, f, indent=1)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
