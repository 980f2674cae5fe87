"""
oracle/make_golden_simu.py -- tests/golden/ref_simu.npz and PINNING_simu.json from the reference's own
run_simu (scripts/sptk/wav_simulate.py) on the eight commands of doc/data_simu/README.md, imported
unmodified under oracle/ref_shim.py (plus a distutils.util.strtobool stub: Python 3.12 has no distutils).

The npz holds, per command <case>:
  <case>/args       the command's flags as JSON (paths as asset names)
  <case>/mix, <case>/spk{i}, <case>/noise   the reference's outputs as write_wav stores them (PCM-16),
                    each kept as its difference from the float64 oracle's PCM-16 (int8, almost all 0:
                    the outputs whole would take 8 MB), with <case>/<output>.sha256 of the reference's
                    PCM-16 bytes, so that a reader rebuilds them exactly and checks that it did
                    (tests/simu_cases.py, reference_outputs);
and, under in/<asset>, the PCM-16 input files the reference read, which are the doc assets cut to what
keeps the file small (every command runs unchanged on them):
  spk1.wav, spk2.wav    their first SPK_SAMPLES (4 s);
  noise.wav             its first NOISE_SAMPLES, the longest mixture (the reference never reads past
                        the mixture's length there);
  iso.wav               channel 0 of the window from ISO_OFFSET over NOISE_SAMPLES, 1-D: the file
                        the reference read has iso.wav's channel count (ISO_CHANNELS), that channel 0
                        and zeros elsewhere -- the reference uses only channel 0's samples of it
                        (wav_simulate.py:294);
  4ch-rir{1,2,3}.wav    whole; 4ch-rir1-ch2.wav is channel 2 of 4ch-rir1.wav (the README's sox remix 2).
PINNING_simu.json holds, per case, the float64 oracle's largest distance from the reference's float
outputs over their peak and the oracle's PCM-16 distance in LSB, and the layout of iso.wav.
Run from the repository root where the reference tree exists.
"""
import argparse
import hashlib
import importlib.util
import json
import os
import sys
import types

import numpy as np
import scipy.io.wavfile as wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, simu_oracle  # noqa: E402
from oracle.stft_oracle import pcm16_from_float  # noqa: E402

ASSET = "/root/reference/doc/data_simu/asset"
ISO_OFFSET = 16000
SPK_SAMPLES = 64000
NOISE_SAMPLES = 32000 + SPK_SAMPLES   # the longest mixture: speaker 1 begins at 32000

CASES = {
    "reverb_1": dict(src_spk="spk1.wav", src_rir="4ch-rir1-ch2.wav"),
    "reverb_2": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", dump_channel=1),
    "noisy1": dict(src_spk="spk1.wav", point_noise="noise.wav", point_noise_snr="5"),
    "noisy2": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", point_noise="noise.wav", point_noise_snr="5",
                   point_noise_rir="4ch-rir3.wav"),
    "noisy3": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", point_noise="noise.wav", point_noise_snr="5",
                   point_noise_rir="4ch-rir3.wav", isotropic_noise_snr="8", isotropic_noise="iso.wav",
                   isotropic_noise_offset=ISO_OFFSET),
    "mix1": dict(src_spk="spk1.wav,spk2.wav", src_begin="32000,0", src_sdr="3"),
    "mix2": dict(src_spk="spk1.wav,spk2.wav", src_begin="32000,0", src_sdr="3", point_noise="noise.wav",
                 point_noise_snr="5"),
    "far_field": dict(src_spk="spk1.wav,spk2.wav", src_rir="4ch-rir1.wav,4ch-rir2.wav", src_begin="32000,0",
                      src_sdr="3", point_noise="noise.wav", point_noise_snr="5", point_noise_rir="4ch-rir3.wav",
                      isotropic_noise_snr="8", isotropic_noise="iso.wav", isotropic_noise_offset=ISO_OFFSET,
                      dump_ref_dir="ref"),
}

DEFAULTS = dict(mix="out.wav", dump_ref_dir="", src_spk="", src_rir="", src_sdr="", src_begin="", point_noise="",
                point_noise_rir="", point_noise_snr="", point_noise_begin="", point_noise_offset="",
                point_noise_repeat=0, isotropic_noise="", isotropic_noise_snr="", isotropic_noise_offset=0,
                dump_channel=-1, norm_factor=0.9, sr=16000)


def namespace(flags, prefix=""):
    d = dict(DEFAULTS, **flags)
    for k in ("src_spk", "src_rir", "point_noise", "point_noise_rir", "isotropic_noise"):
        if d[k]:
            d[k] = ",".join(os.path.join(prefix, p) for p in d[k].split(","))
    return argparse.Namespace(**d)


def main():
    ref_shim.load_reference()
    if "distutils.util" not in sys.modules:
        from setk_b200.libs.opts import strtobool
        d, u = types.ModuleType("distutils"), types.ModuleType("distutils.util")
        u.strtobool = strtobool
        d.util = u
        sys.modules["distutils"], sys.modules["distutils.util"] = d, u
    spec = importlib.util.spec_from_file_location("ref_wav_simulate", os.path.join(ref_shim.REFERENCE_SPTK,
                                                                                   "wav_simulate.py"))
    ws = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ws)

    import tempfile
    tmp = tempfile.mkdtemp()
    inputs = {}
    for f in ("4ch-rir1.wav", "4ch-rir2.wav", "4ch-rir3.wav"):
        inputs[f] = wavfile.read(os.path.join(ASSET, f))[1]
    inputs["4ch-rir1-ch2.wav"] = np.ascontiguousarray(inputs["4ch-rir1.wav"][:, 1])
    for f in ("spk1.wav", "spk2.wav"):
        inputs[f] = wavfile.read(os.path.join(ASSET, f))[1][:SPK_SAMPLES]
    inputs["noise.wav"] = wavfile.read(os.path.join(ASSET, "noise.wav"))[1][:NOISE_SAMPLES]
    iso = wavfile.read(os.path.join(ASSET, "iso.wav"))[1]
    iso_channels = iso.shape[1]
    inputs["iso.wav"] = np.ascontiguousarray(iso[ISO_OFFSET:ISO_OFFSET + NOISE_SAMPLES, 0])
    for f, v in inputs.items():
        if f == "iso.wav":   # the file as read: zeros before the offset and on channels 1..
            full = np.zeros((ISO_OFFSET + v.size, iso_channels), np.int16)
            full[ISO_OFFSET:, 0] = v
            v = full
        wavfile.write(os.path.join(tmp, f), 16000, v)

    store, pin = {}, {}

    def read(path, beg, end, sr):
        return ws.read_wav(path, sr=sr, beg=beg, end=end)

    for name, flags in CASES.items():
        args = namespace(flags, tmp)
        mix, spk, noise = ws.run_simu(args)
        mix_o, spk_o, noise_o = simu_oracle.simulate(args, read)
        outs = {"mix": (mix, mix_o), **{f"spk{i + 1}": (s, so) for i, (s, so) in enumerate(zip(spk, spk_o))}}
        if noise is not None and np.ndim(noise) > 0:
            outs["noise"] = (noise, noise_o)
        spread, lsb = 0.0, 0
        for k, (r, o) in outs.items():
            r = np.asarray(r, np.float64)
            spread = max(spread, float(np.abs(r - o).max() / np.abs(r).max()))
            rp = pcm16_from_float(r.astype(np.float32))
            lsb = max(lsb, int(np.abs(rp.astype(np.int32) - pcm16_from_float(o.astype(np.float32))).max()))
            d = rp.astype(np.int32) - pcm16_from_float(o.astype(np.float32))
            store[f"{name}/{k}"] = d.astype(np.int8)
            store[f"{name}/{k}.sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(rp).tobytes()).hexdigest())
        store[f"{name}/args"] = np.array(json.dumps(flags))
        pin[name] = dict(float_spread=spread, pcm16_lsb=lsb)
        assert mix.shape[-1] <= NOISE_SAMPLES
        print(name, pin[name], {k: np.shape(v[0]) for k, v in outs.items()})
    for f, v in inputs.items():
        store[f"in/{f}"] = v
    out = os.path.join(ROOT, "tests", "golden", "ref_simu.npz")
    np.savez_compressed(out, **store)
    with open(os.path.join(ROOT, "tests", "golden", "PINNING_simu.json"), "w") as f:
        json.dump({"iso_offset": ISO_OFFSET, "iso_channels": iso_channels, "oracle_vs_reference": pin}, f, indent=1)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
