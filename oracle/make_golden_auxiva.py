#!/usr/bin/env python
"""
oracle/make_golden_auxiva.py -- generate tests/golden/ref_auxiva.npz from the REFERENCE's own
apply_auxiva.auxiva and apply_auxiva.run (imported under oracle/ref_shim.py), and record in
tests/golden/PINNING_auxiva.json how oracle/auxiva_oracle.py and the port's apply_auxiva.py
compare with them.

Run in the build container only (needs the reference tree and the CPU execution model,
tests/emu/build_emu.sh):
    python -m oracle.make_golden_auxiva

TEST INFRASTRUCTURE.  Three inputs (fixture_inputs below):
  egs     doc/fixed_beamformer/asset/egs.wav, 4 channels, the first 1 s
  spk7    doc/spatial_clustering/asset/2spk.wav, 7 channels (odd, not a power of two), 0.5 s from 1 s
  mix2    spk1 / spk2 of doc/data_simu/asset convolved with channels 0, 1 of 4ch-rir1 / 4ch-rir2, 1 s
For each: the PCM-16 input, the reference's Y = auxiva(X, 20) on every 32nd bin, and the PCM-16
files the reference's run() writes (<key>.src{1..N}.wav).  The STFTs are not stored: the tests
rebuild them from the audio (oracle/stft_oracle.py, checked here to equal the reference's).
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import scipy.io.wavfile as wavfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import auxiva_oracle as ao  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle import stft_oracle  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SR = 16000
EPOCHS = 20
BIN_STEP = 32
N_SAMPLES = 16000
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)


def _read(rel):
    sr, d = wavfile.read(os.path.join(os.path.dirname(ref_shim.REFERENCE_SPTK), "..", rel))
    assert sr == SR
    return d


def fixture_inputs():
    """name -> PCM-16 input, C x S int16."""
    egs = _read("doc/fixed_beamformer/asset/egs.wav")[:N_SAMPLES].T
    spk7 = _read("doc/spatial_clustering/asset/2spk.wav")[16000:24000].T
    s1 = _read("doc/data_simu/asset/spk1.wav")[:N_SAMPLES].astype(np.float64) / 32768
    s2 = _read("doc/data_simu/asset/spk2.wav")[:N_SAMPLES].astype(np.float64) / 32768
    r1 = _read("doc/data_simu/asset/4ch-rir1.wav").astype(np.float64) / 32768
    r2 = _read("doc/data_simu/asset/4ch-rir2.wav").astype(np.float64) / 32768
    mix = np.stack([np.convolve(s1, r1[:, c])[:N_SAMPLES] + np.convolve(s2, r2[:, c])[:N_SAMPLES] for c in (0, 1)])
    mix = (0.5 * mix / np.max(np.abs(mix))).astype(np.float32)
    return {"egs": np.ascontiguousarray(egs), "spk7": np.ascontiguousarray(spk7),
            "mix2": stft_oracle.pcm16_from_float(mix)}


def fixture_stft(pcm):
    """N x T x F complex64 STFT of PCM-16 audio, as the reference's SpectrogramReader computes it."""
    return stft_oracle.multichannel_stft(stft_oracle.float_from_pcm16(pcm), transpose=True, out_dtype=np.complex64,
                                         **STFT_KW)


def run_port_cli(tmp, out_dir):
    """The port's scripts/sptk/apply_auxiva.py on the CPU execution model of the same kernel sources."""
    lib = os.path.join(ROOT, "tests", "emu", "libsetk_b200_emu.so")
    runner = ("import os, sys, runpy; sys.argv = sys.argv[1:];"
              "from setk_b200 import _lib; _lib.use_library(os.environ['SETK_B200_TEST_LIBRARY']);"
              "from setk_b200.libs import utils; utils.set_default_device('cpu');"
              "runpy.run_path(sys.argv[0], run_name='__main__')")
    env = dict(os.environ, PYTHONPATH=ROOT, SETK_B200_TEST_LIBRARY=lib)
    subprocess.run([sys.executable, "-c", runner, os.path.join(ROOT, "scripts", "sptk", "apply_auxiva.py"),
                    os.path.join(tmp, "wav.scp"), out_dir], check=True, env=env, cwd=ROOT)


def main():
    ref = ref_shim.load_reference()
    aux = importlib.import_module("apply_auxiva")
    report = {"generated_by": "oracle/make_golden_auxiva.py", "numpy": np.__version__,
              "reference": "funcwj/setk @ 50e4da0 under oracle/ref_shim.py", "epochs": EPOCHS,
              "stored_bins": f"every {BIN_STEP}nd bin of Y"}
    out = {}
    tmp = tempfile.mkdtemp()
    scp = []
    for name, pcm in fixture_inputs().items():
        x = stft_oracle.float_from_pcm16(pcm)
        X = np.stack([ref.utils.forward_stft(np.ascontiguousarray(c), transpose=True, **STFT_KW) for c in x])
        assert np.array_equal(X, fixture_stft(pcm)), "oracle STFT differs from the reference's"
        Y = aux.auxiva(X, EPOCHS)                                         # N x T x F complex128
        Yo = ao.auxiva(X, EPOCHS)
        report[f"{name}/shape_NTF"] = list(X.shape)
        report[f"{name}/oracle_vs_reference_rel_to_max"] = float(np.max(np.abs(Yo - Y)) / np.max(np.abs(Y)))
        out[name + "/pcm16"] = pcm
        out[name + "/Y_bins"] = Y[:, :, ::BIN_STEP]
        path = os.path.join(tmp, name + ".wav")
        wavfile.write(path, SR, pcm.T)
        scp.append(f"{name} {path}")
    with open(os.path.join(tmp, "wav.scp"), "w") as f:
        f.write("\n".join(scp) + "\n")
    ref_dir, port_dir = os.path.join(tmp, "ref"), os.path.join(tmp, "port")
    aux.run(argparse.Namespace(wav_scp=os.path.join(tmp, "wav.scp"), dst_dir=ref_dir, epochs=EPOCHS, sr=SR,
                               **{k: v for k, v in STFT_KW.items()}))
    run_port_cli(tmp, port_dir)
    for name, pcm in fixture_inputs().items():
        got, want = [], []
        for idx in range(pcm.shape[0]):
            want.append(wavfile.read(os.path.join(ref_dir, f"{name}.src{idx + 1}.wav"))[1])
            got.append(wavfile.read(os.path.join(port_dir, f"{name}.src{idx + 1}.wav"))[1])
        want, got = np.stack(want), np.stack(got)
        out[name + "/cli_pcm16"] = want
        d = np.abs(got.astype(np.int32) - want.astype(np.int32))
        report[f"{name}/port_cli_vs_reference_max_lsb"] = int(d.max())
        report[f"{name}/port_cli_vs_reference_identical_fraction"] = float(np.mean(d == 0))
    report["port_cli_run_on"] = "CPU execution model of the kernel sources (tests/emu)"
    np.savez_compressed(os.path.join(GOLD, "ref_auxiva.npz"), **out)
    with open(os.path.join(GOLD, "PINNING_auxiva.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))
    print("npz bytes", os.path.getsize(os.path.join(GOLD, "ref_auxiva.npz")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
