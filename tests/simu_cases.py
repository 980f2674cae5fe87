"""
Shared cases and tolerances of the simulation tests (csrc/simu.cu: setk_convolve, setk_simulate_mix;
setk_b200/simu.py; scripts/sptk/wav_simulate.py).

  TOL_CONV   convolution vs float64 np.convolve, max |error| over each channel's peak: 2e-6, about ten
             times the reference's own float32 spread (2.2e-7 measured on the doc far-field speaker);
             the kernel measures about 3e-7 in the CPU execution model.
  PCM16_LSB  PCM-16 outputs vs the oracle or the reference: 1 LSB (the reference's float32 and float64
             paths already differ by 1 LSB in 0.08 % of samples).
"""
import argparse
import hashlib
import json
import os

import numpy as np
import scipy.io.wavfile as wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import simu_oracle as so  # noqa: E402
from oracle.stft_oracle import pcm16_from_float  # noqa: E402

TOL_CONV = 2e-6
PCM16_LSB = 1

DEFAULTS = dict(mix="out.wav", dump_ref_dir="", src_spk="", src_rir="", src_sdr="", src_begin="", point_noise="",
                point_noise_rir="", point_noise_snr="", point_noise_begin="", point_noise_offset="",
                point_noise_repeat=0, isotropic_noise="", isotropic_noise_snr="", isotropic_noise_offset=0,
                dump_channel=-1, norm_factor=0.9, sr=16000)
PATH_FLAGS = ("src_spk", "src_rir", "point_noise", "point_noise_rir", "isotropic_noise")


def namespace(flags, folder, mix="out.wav"):
    d = dict(DEFAULTS, **flags)
    for k in PATH_FLAGS:
        if d[k]:
            d[k] = ",".join(os.path.join(folder, p) for p in d[k].split(","))
    d["mix"] = os.path.join(folder, mix)
    if d["dump_ref_dir"]:
        d["dump_ref_dir"] = os.path.join(folder, d["dump_ref_dir"])
    return argparse.Namespace(**d)


def command_line(flags, folder, mix):
    """the wav_simulate.py arguments of a flags dict"""
    a = vars(namespace(flags, folder, mix))
    out = []
    for k, v in a.items():
        if k == "mix" or v == DEFAULTS[k]:
            continue
        out += [f"--{k.replace('_', '-')}", str(v)]
    return out + [a["mix"]]


def oracle_read(path, beg, end, sr):
    from setk_b200.libs.utils import read_wav
    return read_wav(path, beg=beg, end=end, sr=sr)


def load_fixture():
    with np.load(os.path.join(GOLD, "ref_simu.npz")) as z:
        return {k: z[k] for k in z.files}


def load_pinning():
    with open(os.path.join(GOLD, "PINNING_simu.json")) as f:
        return json.load(f)


def write_assets(store, folder):
    """the input files the reference read, under folder: the isotropic noise's channel 0 back at its
    offset, in a file of its channel count with zeros elsewhere (oracle/make_golden_simu.py)"""
    pin = load_pinning()
    off, n_ch = pin["iso_offset"], pin["iso_channels"]
    for k, v in store.items():
        if not k.startswith("in/"):
            continue
        if k == "in/iso.wav":
            full = np.zeros((off + v.size, n_ch), np.int16)
            full[off:, 0] = v
            v = full
        wavfile.write(os.path.join(folder, k[3:]), 16000, v)


def cases(store):
    return sorted({k.split("/")[0] for k in store if k.endswith("/args")})


def case_flags(store, name):
    return json.loads(str(store[f"{name}/args"]))


def oracle_outputs(args):
    mix, spk, noise = so.simulate(args, oracle_read)
    out = {"mix": mix, **{f"spk{i + 1}": s for i, s in enumerate(spk)}}
    if noise is not None:
        out["noise"] = noise
    return out


def reference_outputs(store, name, oracle):
    """the reference's PCM-16 outputs of a case, rebuilt from the oracle's and checked by hash"""
    out = {}
    for k in oracle:
        if f"{name}/{k}" not in store:
            continue
        ref = (pcm16_from_float(oracle[k].astype(np.float32)).astype(np.int32) + store[f"{name}/{k}"]).astype(np.int16)
        digest = hashlib.sha256(np.ascontiguousarray(ref).tobytes()).hexdigest()
        assert digest == str(store[f"{name}/{k}.sha256"]), f"{name}/{k}: the oracle no longer rebuilds the reference"
        out[k] = ref
    return out


def synth_assets(folder, seed=0, n_spk=(4000, 3100), rir_len=700, noise_len=3000, iso_len=9000, channels=4):
    """short seeded stand-ins for the doc assets"""
    rng = np.random.default_rng(seed)

    def pcm(a):
        return np.clip(np.round(a * 32768), -32768, 32767).astype(np.int16)

    for i, n in enumerate(n_spk):
        wavfile.write(os.path.join(folder, f"spk{i + 1}.wav"), 16000,
                      pcm(0.3 * np.sin(np.arange(n) * (0.03 + 0.01 * i)) * rng.uniform(0.5, 1, n)))
    decay = np.exp(-np.arange(rir_len) / (rir_len / 5))
    for i in range(3):
        h = rng.standard_normal((rir_len, channels)) * decay[:, None] * 0.2
        wavfile.write(os.path.join(folder, f"4ch-rir{i + 1}.wav"), 16000, pcm(h))
    h = rng.standard_normal(rir_len) * decay * 0.2
    wavfile.write(os.path.join(folder, "1ch-rir.wav"), 16000, pcm(h))
    wavfile.write(os.path.join(folder, "noise.wav"), 16000, pcm(0.1 * rng.standard_normal(noise_len)))
    wavfile.write(os.path.join(folder, "noise2.wav"), 16000, pcm(0.1 * rng.standard_normal(noise_len // 2)))
    wavfile.write(os.path.join(folder, "iso.wav"), 16000, pcm(0.05 * rng.standard_normal((iso_len, channels))))
    wavfile.write(os.path.join(folder, "spk4ch.wav"), 16000, pcm(0.2 * rng.standard_normal((1500, channels))))


# the eight commands of doc/data_simu/README.md on the synthetic assets
DOC_COMMANDS = {
    "reverb_1": dict(src_spk="spk1.wav", src_rir="1ch-rir.wav"),
    "reverb_2": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", dump_channel=1),
    "noisy1": dict(src_spk="spk1.wav", point_noise="noise.wav", point_noise_snr="5"),
    "noisy2": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", point_noise="noise.wav", point_noise_snr="5",
                   point_noise_rir="4ch-rir3.wav"),
    "noisy3": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", point_noise="noise.wav", point_noise_snr="5",
                   point_noise_rir="4ch-rir3.wav", isotropic_noise_snr="8", isotropic_noise="iso.wav",
                   isotropic_noise_offset=1000),
    "mix1": dict(src_spk="spk1.wav,spk2.wav", src_begin="800,0", src_sdr="3"),
    "mix2": dict(src_spk="spk1.wav,spk2.wav", src_begin="800,0", src_sdr="3", point_noise="noise.wav",
                 point_noise_snr="5"),
    "far_field": dict(src_spk="spk1.wav,spk2.wav", src_rir="4ch-rir1.wav,4ch-rir2.wav", src_begin="800,0",
                      src_sdr="3", point_noise="noise.wav", point_noise_snr="5", point_noise_rir="4ch-rir3.wav",
                      isotropic_noise_snr="8", isotropic_noise="iso.wav", isotropic_noise_offset=1000,
                      dump_ref_dir="ref"),
}


def peak_err(got, want):
    got, want = np.atleast_2d(got), np.atleast_2d(want)
    return float(max(np.abs(g - w).max() / max(np.abs(w).max(), 1e-30) for g, w in zip(got, want)))


def compare(results, oracle, tol):
    """a simulate() result (float32) against oracle outputs: worst error over each output's peak"""
    mix, spk, noise = results
    err = peak_err(mix, oracle["mix"])
    for i, s in enumerate(spk):
        err = max(err, peak_err(s, oracle[f"spk{i + 1}"]))
    if "noise" in oracle:
        assert noise is not None
        err = max(err, peak_err(noise, oracle["noise"]))
    return err
