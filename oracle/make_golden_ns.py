#!/usr/bin/env python
"""
oracle/make_golden_ns.py -- generate tests/golden/ref_ns.npz from the REFERENCE's own
libs.ns.iMCRA (imported under oracle/ref_shim.py), and record in tests/golden/PINNING_ns.json how
oracle/ns_oracle.py and the port's apply_ns.py compare with it.

Run in the build container only (needs the reference tree and the CPU execution model,
tests/emu/build_emu.sh):
    python -m oracle.make_golden_ns

TEST INFRASTRUCTURE.  Stored:
  egs/pcm16       doc/ns/asset/egs.wav (8.2 s, 16 kHz)
  egs/ns_pcm16    the shipped doc/ns/asset/egs_ns.wav (the reference's apply_ns.py output)
  egs/gain_frames the reference's iMCRA().run gains on that clip, every 8th frame (float64)
  a/stft, a/gain  digital silence: an all-zero first frame, a zero run in the middle, an all-zero bin
  b/stft, b/gain  a non-default configuration (CASE_B_CONF: U > V, w_mcra = 2, Hamming, ...)
The clip's STFT is not stored: the tests rebuild it from the PCM (oracle/stft_oracle.py, checked
here to equal the reference's).
"""
import importlib
import json
import os
import subprocess
import sys
import tempfile
import warnings

import numpy as np
import scipy.io.wavfile as wavfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ns_oracle as no  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle import stft_oracle  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SR = 16000
FRAME_STEP = 8
STFT_KW = dict(frame_len=512, frame_hop=256, window="hann", center=True, round_power_of_two=True)
H100_CLI_EXACT = 0.999657
CASE_B_CONF = dict(U=20, V=7, w_mcra=2, h_mcra="hamming", alpha=0.9, beta=1.2, gamma0=5.0, gmin_db=-15)


def case_inputs():
    """(a) T = 200, F = 33 with digital silence; (b) T = 200, F = 65.  T x F complex64."""
    rng = np.random.default_rng(2024)

    def noisy(T, F):
        env = 0.05 + rng.gamma(0.6, 1.0, (T, 1)) * (rng.random((T, 1)) < 0.5)
        return ((rng.standard_normal((T, F)) + 1j * rng.standard_normal((T, F))) * (0.02 + env)).astype(np.complex64)

    a = noisy(200, 33)
    a[0] = 0
    a[90:104] = 0
    a[:, 5] = 0
    return {"a": a, "b": noisy(200, 65)}


def fixture_stft(pcm):
    """T x F complex64 STFT of PCM-16 audio, as the reference's SpectrogramReader computes it."""
    return stft_oracle.forward_stft(stft_oracle.float_from_pcm16(pcm), transpose=True, out_dtype=np.complex64,
                                    **STFT_KW)


def run_port_cli(tmp, out_dir):
    """The port's scripts/sptk/apply_ns.py on the CPU execution model of the same kernel sources."""
    lib = os.path.join(ROOT, "tests", "emu", "libsetk_b200_emu.so")
    runner = ("import os, sys, runpy; sys.argv = sys.argv[1:];"
              "from setk_b200 import _lib; _lib.use_library(os.environ['SETK_B200_TEST_LIBRARY']);"
              "from setk_b200.libs import utils; utils.set_default_device('cpu');"
              "runpy.run_path(sys.argv[0], run_name='__main__')")
    env = dict(os.environ, PYTHONPATH=ROOT, SETK_B200_TEST_LIBRARY=lib)
    subprocess.run([sys.executable, "-c", runner, os.path.join(ROOT, "scripts", "sptk", "apply_ns.py"),
                    os.path.join(tmp, "wav.scp"), out_dir], check=True, env=env, cwd=ROOT)


def main():
    ref = ref_shim.load_reference()
    ns = importlib.import_module("libs.ns")
    asset = os.path.join(os.path.dirname(ref_shim.REFERENCE_SPTK), "..", "doc", "ns", "asset")
    sr, pcm = wavfile.read(os.path.join(asset, "egs.wav"))
    sr2, shipped = wavfile.read(os.path.join(asset, "egs_ns.wav"))
    assert sr == SR and sr2 == SR and pcm.ndim == 1
    report = {"generated_by": "oracle/make_golden_ns.py", "numpy": np.__version__,
              "reference": "funcwj/setk @ 50e4da0 under oracle/ref_shim.py",
              "stored_frames": f"every {FRAME_STEP}th frame of the clip's gain", "case_b_conf": CASE_B_CONF}
    out = {"egs/pcm16": pcm, "egs/ns_pcm16": shipped}

    X = ref.utils.forward_stft(stft_oracle.float_from_pcm16(pcm), transpose=True, **STFT_KW)
    assert np.array_equal(X, fixture_stft(pcm)), "oracle STFT differs from the reference's"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        G = ns.iMCRA().run(X)
    Go = no.iMCRA().run(X)
    report["egs/shape_TF"] = list(X.shape)
    report["egs/oracle_vs_reference_max_abs"] = float(np.max(np.abs(Go - G)))
    out["egs/gain_frames"] = G[::FRAME_STEP]
    y = ref.utils.inverse_stft(G * X, **{k: v for k, v in STFT_KW.items() if k != "round_power_of_two"})
    d = np.abs(stft_oracle.pcm16_from_float(np.asarray(y)).astype(np.int32) - shipped.astype(np.int32))
    report["egs/reference_rerun_vs_shipped_max_lsb"] = int(d.max())
    report["egs/reference_rerun_vs_shipped_differing_samples"] = int(np.count_nonzero(d))

    for name, S in case_inputs().items():
        conf = CASE_B_CONF if name == "b" else {}
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            G = ns.iMCRA(**conf).run(S)
        Go = no.iMCRA(**conf).run(S)
        out[name + "/stft"] = S
        out[name + "/gain"] = G
        report[f"{name}/shape_TF"] = list(S.shape)
        report[f"{name}/oracle_vs_reference_max_rel"] = float(np.max(np.abs(Go - G) / np.maximum(1, np.abs(G))))
        report[f"{name}/max_gain"] = float(np.max(G))

    tmp = tempfile.mkdtemp()
    wavfile.write(os.path.join(tmp, "egs.wav"), SR, pcm)
    with open(os.path.join(tmp, "wav.scp"), "w") as f:
        f.write(f"egs {os.path.join(tmp, 'egs.wav')}\n")
    port_dir = os.path.join(tmp, "port")
    run_port_cli(tmp, port_dir)
    got = wavfile.read(os.path.join(port_dir, "egs.wav"))[1]
    d = np.abs(got.astype(np.int32) - shipped.astype(np.int32))
    report["egs/port_cli_vs_shipped_max_lsb"] = int(d.max())
    report["egs/port_cli_vs_shipped_identical_fraction"] = float(np.mean(d == 0))
    report["port_cli_run_on"] = "CPU execution model of the kernel sources (tests/emu)"
    # tests/test_gpu_ns.py::test_apply_ns_cli on an NVIDIA H100 80GB HBM3 (400 W power limit): the
    # device's float32 iSTFT moves a few more samples across a rounding boundary
    report["egs/port_cli_vs_shipped_identical_fraction_h100"] = H100_CLI_EXACT
    np.savez_compressed(os.path.join(GOLD, "ref_ns.npz"), **out)
    with open(os.path.join(GOLD, "PINNING_ns.json"), "w") as f:
        json.dump(report, f, indent=1, sort_keys=True)
    print(json.dumps(report, indent=1, sort_keys=True))
    print("npz bytes", os.path.getsize(os.path.join(GOLD, "ref_ns.npz")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
