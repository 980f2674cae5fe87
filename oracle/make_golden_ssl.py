#!/usr/bin/env python
"""
oracle/make_golden_ssl.py -- generate tests/golden/ref_ssl.npz from the REFERENCE's own
libs/ssl.py, do_ssl.py and compute_steer_vector.py (imported under oracle/ref_shim.py), and
record in tests/golden/PINNING_ssl.json how oracle/ssl_oracle.py compares with them.

Run in the build container only (needs the reference tree):
    python -m oracle.make_golden_ssl

TEST INFRASTRUCTURE.  Three seeded mixtures with one clear source direction:
  lin4   4-mic linear array, A = 37 directions over 0..180 degrees, source at 60
  circ7  6-mic circular array (r = 5 cm) plus a centre mic, A = 72 over 0..355, source at 200
  lin2   2-mic linear array, A = 19, source at 120
(geometry, lengths and seeds: ssl_oracle.FIXTURE_GEOMETRY)
For each: the PCM-16 audio, and the index AND score vector of ml_ssl (no mask, 2-D mask, norm=True,
3-D mask, compression 0.5), srp_ssl (with and without a mask) and music_ssl (without a mask, and
with a mask that is zero in every frame of one bin).  The scores are caught by handing the
reference module a numpy proxy whose argmax / argmin remember their argument.
do_ssl.run(args) runs on a two-utterance wav.scp of the lin4 geometry: ML, SRP, MUSIC offline,
ML with two masks and winner-take-all, online ML without a mask, and all three --output kinds;
its doa_scp text is stored.  compute_steer_vector.run(args) output is stored for a linear and a
circular geometry.
The STFTs, steering tables and seeded masks are not stored: oracle/ssl_oracle.py regenerates them
(expand_fixture), and exact slices of the reference's STFTs and steering tables are stored to check
that the regenerated ones are the same arrays.
"""
import argparse
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np
import scipy.io.wavfile as wavfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle import ssl_oracle as so  # noqa: E402
from oracle import stft_oracle  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SR = 16000
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)


class _Recorder(types.ModuleType):
    """numpy, except that argmax / argmin keep the array they were given."""

    def __init__(self):
        super().__init__("numpy")
        self.seen = []

    def __getattr__(self, name):
        return getattr(np, name)

    def argmax(self, a, *args, **kw):
        self.seen.append(np.array(a))
        return np.argmax(a, *args, **kw)

    def argmin(self, a, *args, **kw):
        self.seen.append(np.array(a))
        return np.argmin(a, *args, **kw)


def _delayed(src, delays, n):
    """src delayed by `delays` seconds (one row per microphone), via the DFT."""
    L = 2 * n
    spec = np.fft.rfft(src, L)
    freqs = np.fft.rfftfreq(L, 1 / SR)
    return np.stack([np.fft.irfft(spec * np.exp(-2j * np.pi * freqs * d), L)[:n] for d in delays])


def mixture(rng, dist, n, snr_db=10.0):
    """One source whose steering vector matches plane_steer_vector(dist), plus white noise."""
    src = rng.standard_normal(n) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * np.arange(n) / SR))
    x = _delayed(src, np.asarray(dist) / 343.0, n)
    noise = rng.standard_normal(x.shape) * np.std(x) * 10**(-snr_db / 20)
    x = x + noise
    return (0.5 * x / np.max(np.abs(x))).astype(np.float32)


def pcm16(x):
    return stft_oracle.float_from_pcm16(stft_oracle.pcm16_from_float(x))


def ref_stft(ref, x):
    """The reference's M x T x F complex64 STFT of float32 audio (do_ssl.py's SpectrogramReader)."""
    return np.stack([ref.utils.forward_stft(np.ascontiguousarray(c), transpose=True, **STFT_KW) for c in x])


def cases(ref, ref_ssl, rec, report):
    """The estimators of the reference on the three mixtures; full inputs in `full`, stored form in `out`."""
    from setk_b200.libs import beamformer as mirror
    out, full = {}, {}
    for name, geo in so.FIXTURE_GEOMETRY.items():
        rng = np.random.default_rng(geo["seed"])
        sv = so.fixture_steering(ref.beamformer, geo)                    # A x M x F complex128
        assert np.array_equal(sv, so.fixture_steering(mirror, geo)), "steering mirror differs"
        if geo["kind"] == "linear":
            dist = np.cos(geo["doa"] * np.pi / 180) * np.array(geo["topo"])
            doas = np.linspace(0, 180, geo["A"])
        else:
            dirc = np.arange(6) * 2 * np.pi / 6
            dist = -np.concatenate([[0.0], np.cos(dirc - geo["doa"] * np.pi / 180) * geo["radius"]])
            doas = np.arange(0, 360, 360 / geo["A"])
        pcm = stft_oracle.pcm16_from_float(mixture(rng, dist, geo["n"]))
        S = ref_stft(ref, stft_oracle.float_from_pcm16(pcm))             # M x T x F complex64
        assert np.array_equal(S, so.fixture_stft(pcm)), "oracle STFT differs from the reference's"
        M, T, F = S.shape
        mask, mask3, mask_z = so.fixture_masks(geo["seed"], T, F)
        pairs = (list(range(M - 1)), list(range(1, M)))
        out[name + "/pcm16"] = pcm
        out[name + "/stft_pin"] = S[:, :, ::16]
        out[name + "/sv_pin"] = sv[:, :, ::16]
        out[name + "/mask_head"] = mask[0, :8]
        out[name + "/pairs"] = np.array(pairs, dtype=np.int32).T       # P x 2
        full.update({name + "/stft": S, name + "/sv": sv, name + "/mask": mask, name + "/mask3": mask3,
                     name + "/mask_zero_bin": mask_z})
        runs = {
            "ml": lambda: ref_ssl.ml_ssl(S, sv, compression=-1, eps=so.EPSILON),
            "ml_mask": lambda: ref_ssl.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, mask=mask),
            "ml_norm": lambda: ref_ssl.ml_ssl(S, sv, norm=True, mask=mask),
            "ml_mask3": lambda: ref_ssl.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, mask=mask3),
            "ml_pow": lambda: ref_ssl.ml_ssl(S, sv, compression=0.5, mask=mask),
            "srp": lambda: ref_ssl.srp_ssl(S, sv, srp_pair=pairs),
            "srp_mask": lambda: ref_ssl.srp_ssl(S, sv, srp_pair=pairs, mask=mask),
            "music": lambda: ref_ssl.music_ssl(S, sv),
            "music_mask": lambda: ref_ssl.music_ssl(S, sv, mask=mask_z),
        }
        for run, fn in runs.items():
            rec.seen.clear()
            idx = fn()
            out[f"{name}/{run}/index"] = np.asarray(idx)
            out[f"{name}/{run}/scores"] = rec.seen[-1]
        report[f"{name}/true_doa_index"] = int(np.argmin(np.abs(doas - geo["doa"])))
        report[f"{name}/ml_index"] = int(out[f"{name}/ml/index"])
    full.update(out)
    return out, full


def do_ssl_cases(ref, out, report):
    """do_ssl.run(args) of the reference on a tiny wav.scp; its output text."""
    do_ssl = importlib.import_module("do_ssl")
    rng = np.random.default_rng(77)
    topo = so.CLI_TOPO
    sv = so.fixture_steering(ref.beamformer, dict(kind="linear", topo=topo, A=so.CLI_NUM_DOA))
    tmp = tempfile.mkdtemp()
    sv_path = os.path.join(tmp, "sv.npy")
    np.save(sv_path, sv)
    scp = []
    masks = {0: [], 1: [], 2: []}
    for k, (doa, n) in enumerate(((45.0, 6000), (130.0, 5000))):
        x = mixture(rng, np.cos(doa * np.pi / 180) * np.array(topo), n)
        pcm = stft_oracle.pcm16_from_float(x)
        key = f"utt{k}"
        path = os.path.join(tmp, key + ".wav")
        wavfile.write(path, SR, pcm.T)
        scp.append(f"{key} {path}")
        out[f"cli/{key}/pcm16"] = pcm
        for j, m in enumerate(so.cli_masks(k, 1 + n // 256)):         # the third is F x T: do_ssl transposes it
            np.save(os.path.join(tmp, f"{key}_m{j}.npy"), m)
            masks[j].append(f"{key} {os.path.join(tmp, f'{key}_m{j}.npy')}")
    for name, lines in (("wav.scp", scp), ("mask0.scp", masks[0]), ("mask1.scp", masks[1]),
                        ("mask2.scp", masks[2])):
        with open(os.path.join(tmp, name), "w") as f:
            f.write("\n".join(lines) + "\n")
    out["cli/sv_pin"] = sv[:, :, ::16]
    runs = {
        "ml": dict(),
        "ml_radian": dict(output="radian"),
        "ml_index": dict(output="index"),
        "srp": dict(backend="srp", srp_pair="0,1;1,2;2,3"),
        "music": dict(backend="music"),
        "ml_wta": dict(mask_scp="mask0.scp,mask1.scp", mask_eps=0.01),
        "srp_mask": dict(backend="srp", srp_pair="0,3;1,2", mask_scp="mask2.scp"),
        "music_mask": dict(backend="music", mask_scp="mask0.scp"),
        "ml_online": dict(chunk_len=8, look_back=12),
        "ml_online_range": dict(chunk_len=10, look_back=5, doa_range="10,170"),
    }
    for run, kw in runs.items():
        args = dict(frame_len=512, frame_hop=256, round_power_of_two=True, window="hann", center=True,
                    backend="ml", srp_pair="", doa_range="0,360", mask_scp="", output="degree",
                    mask_eps=-1.0, chunk_len=-1, look_back=125)
        args.update(kw)
        if args["mask_scp"]:
            args["mask_scp"] = ",".join(os.path.join(tmp, s) for s in args["mask_scp"].split(","))
        args.update(wav_scp=os.path.join(tmp, "wav.scp"), steer_vector=sv_path,
                    doa_scp=os.path.join(tmp, run + ".txt"))
        do_ssl.run(argparse.Namespace(**args))
        with open(args["doa_scp"]) as f:
            text = f.read()
        out[f"cli/{run}/doa_scp"] = np.array(text)
        out[f"cli/{run}/flags"] = np.array(json.dumps(kw, sort_keys=True))
        report[f"cli/{run}"] = text.strip().replace("\t", " ")


def steer_vector_cases(out):
    csv = importlib.import_module("compute_steer_vector")
    tmp = tempfile.mkdtemp()
    for name, kw in (("linear", dict(geometry="linear", linear_topo=(0, 0.05, 0.1), num_doas=13,
                                     normalize=False)),
                     ("circular", dict(geometry="circular", circular_around=6, circular_radius=0.04,
                                       circular_center=True, num_doas=12, normalize=True))):
        args = dict(num_bins=33, sr=16000, speed=343.0, linear_topo=(), circular_around=6,
                    circular_radius=0.05, circular_center=False, geometry="linear", normalize=False)
        args.update(kw)
        args["steer_vector"] = os.path.join(tmp, name + ".npy")
        csv.run(argparse.Namespace(**args))
        out[f"steer/{name}"] = np.load(args["steer_vector"])
        out[f"steer/{name}/flags"] = np.array(json.dumps(kw, sort_keys=True))


def pin(out, report):
    """How the oracle compares with the stored reference results."""
    worst = {"reference": 0.0, "float64": 0.0}
    idx_ok = {"reference": True, "float64": True}
    for name in so.FIXTURE_GEOMETRY:
        g = {k.split("/", 1)[1]: v for k, v in out.items() if k.startswith(name + "/")}
        S, sv = g["stft"], g["sv"]
        pairs = (list(g["pairs"][:, 0]), list(g["pairs"][:, 1]))
        for flow in worst:
            calls = {
                "ml": lambda: so.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, flow=flow),
                "ml_mask": lambda: so.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, mask=g["mask"], flow=flow),
                "ml_norm": lambda: so.ml_ssl(S, sv, norm=True, mask=g["mask"], flow=flow),
                "ml_mask3": lambda: so.ml_ssl(S, sv, compression=-1, eps=so.EPSILON, mask=g["mask3"], flow=flow),
                "ml_pow": lambda: so.ml_ssl(S, sv, compression=0.5, mask=g["mask"], flow=flow),
                "srp": lambda: so.srp_ssl(S, sv, srp_pair=pairs, flow=flow),
                "srp_mask": lambda: so.srp_ssl(S, sv, srp_pair=pairs, mask=g["mask"], flow=flow),
                "music": lambda: so.music_ssl(S, sv, flow=flow),
                "music_mask": lambda: so.music_ssl(S, sv, mask=g["mask_zero_bin"], flow=flow),
            }
            for run, fn in calls.items():
                idx, sc = fn()
                ref_sc = g[run + "/scores"]
                rel = float(np.max(np.abs(sc - ref_sc)) / np.max(np.abs(ref_sc)))
                report[f"{name}/{run}/oracle_{flow}_scores_rel_to_max"] = rel
                worst[flow] = max(worst[flow], rel)
                idx_ok[flow] &= bool(np.array_equal(idx, g[run + "/index"]))
    for flow in worst:
        report[f"oracle_{flow}_worst_scores_rel_to_max"] = worst[flow]
        report[f"oracle_{flow}_indices_equal"] = idx_ok[flow]


def main():
    ref = ref_shim.load_reference()
    sys.path.insert(0, ref_shim.REFERENCE_SPTK)
    ref_ssl = importlib.import_module("libs.ssl")
    rec = _Recorder()
    ref_ssl.np = rec                                   # the reference module's `np` name
    report = {"generated_by": "oracle/make_golden_ssl.py", "numpy": np.__version__,
              "reference": "funcwj/setk @ 50e4da0 under oracle/ref_shim.py"}
    out, full = cases(ref, ref_ssl, rec, report)
    do_ssl_cases(ref, out, report)
    steer_vector_cases(out)
    pin(full, report)
    np.savez_compressed(os.path.join(GOLD, "ref_ssl.npz"), **out)
    with open(os.path.join(GOLD, "PINNING_ssl.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps({k: v for k, v in report.items() if "worst" in k or "equal" in k or "cli" in k},
                     indent=1, sort_keys=True))
    return 0


if __name__ == "__main__":
    sys.exit(main())
