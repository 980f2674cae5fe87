#!/usr/bin/env python
"""
oracle/make_golden_rir.py -- generate tests/golden/ref_rir.npz from the REFERENCE's own image-method
generator (include/rir-generator.cc, compiled by oracle/rir_ref/build.sh into oracle/_ref/rir_ref),
and record in tests/golden/PINNING_rir.json how oracle/rir_oracle.py compares with it.

Run in the build container only (needs the reference tree):
    python oracle/make_golden_rir.py

TEST INFRASTRUCTURE.  Each case <name>/ stores its inputs (room, beta as given to the reference --
one T60 or six coefficients --, source, receivers, n_samples, fs, c, order, mic_type, orientation,
hp_filter) and <name>/ref, the reference's float32 response (M, L).  The cases (CASES below):
  doc1d_*, doc2d_*  doc/rir/asset/{1d,2d}_rir.json: the first two sources of each room, the four
                    receivers, 8000 samples, c = 340 (1d) and 343 (2d) as the scripts' defaults
  pattern_*         the four non-omni patterns, oriented
  order_{0,1,3}     reflection orders
  beta6             six coefficients with zeros among them
  t60_zero          T60 = 0: the direct path only
  no_hp             the high-pass off
"""
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import rir_oracle as ro  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
REF_BIN = os.path.join(HERE, "_ref", "rir_ref")
DOC = "/root/reference/doc/rir/asset"

SMALL = dict(room=[3.2, 2.6, 2.3], source=[0.9, 1.7, 1.4], receivers=[[2.1, 1.0, 1.2], [2.3, 1.1, 1.25]],
             n_samples=2000, fs=16000, c=340, order=-1, mic_type="omnidirectional", orientation=(0.0, 0.0),
             hp_filter=True, beta=[0.35])


def _cases():
    cases = {}
    for tag, c in (("1d", 340), ("2d", 343)):
        with open(os.path.join(DOC, f"{tag}_rir.json")) as f:
            rooms = json.load(f)
        for r, room in enumerate(rooms):
            for s in range(2):
                cases[f"doc{tag}_r{r + 1}s{s + 1}"] = dict(
                    room=room["room_size"], beta=np.atleast_1d(room["beta"]).tolist(),
                    source=room["spk"][s]["pos"], receivers=room["receiver_location"], n_samples=8000,
                    fs=16000, c=c, order=-1, mic_type="omnidirectional", orientation=(0.0, 0.0), hp_filter=True)
    for mic in ro.MIC_TYPES[1:]:
        cases[f"pattern_{mic}"] = dict(SMALL, mic_type=mic, orientation=(0.7, 0.3))
    for order in (0, 1, 3):
        cases[f"order_{order}"] = dict(SMALL, order=order)
    cases["beta6"] = dict(SMALL, beta=[0.9, 0.0, 0.7, 0.8, 0.0, 0.6])
    cases["t60_zero"] = dict(SMALL, beta=[0.0])
    cases["no_hp"] = dict(SMALL, hp_filter=False, fs=8000, n_samples=1200)
    return cases


def run_reference(case):
    f3 = lambda p: ",".join(f"{float(v):.6f}" for v in p)  # noqa: E731
    args = [REF_BIN, f"--sound-velocity={case['c']}", f"--samp-frequency={case['fs']}",
            f"--hp-filter={'true' if case['hp_filter'] else 'false'}", f"--number-samples={case['n_samples']}",
            f"--order={case['order']}", f"--microphone-type={case['mic_type']}",
            f"--receiver-location={';'.join(f3(p) for p in case['receivers'])}",
            f"--source-location={f3(case['source'])}", f"--room-topo={f3(case['room'])}",
            f"--angle={f3(case['orientation'])}", f"--beta={f3(case['beta'])}"]
    out = subprocess.run(args, check=True, capture_output=True).stdout
    rows, cols = np.frombuffer(out[:8], np.int32)
    return np.frombuffer(out[8:], np.float32).reshape(rows, cols).copy()


def oracle_of(case):
    beta = case["beta"]
    beta = ro.t60_to_beta(case["room"], beta[0], case["c"]) if len(beta) == 1 else np.asarray(beta)
    return ro.rir(case["room"], beta, case["source"], case["receivers"], case["n_samples"], fs=case["fs"],
                  c=case["c"], order=case["order"], mic_type=case["mic_type"], orientation=case["orientation"],
                  hp_filter=case["hp_filter"])


def main():
    if not os.path.exists(REF_BIN):
        subprocess.run([os.path.join(HERE, "rir_ref", "build.sh")], check=True)
    store, pin = {}, {}
    for name, case in _cases().items():
        ref = run_reference(case)
        err = ro.peak_err(oracle_of(case), ref)
        pin[name] = float(f"{err:.3e}")
        for k, v in case.items():
            store[f"{name}/{k}"] = np.asarray(v)
        store[f"{name}/ref"] = ref
        print(f"{name}: oracle vs reference {err:.3e}")
    np.savez_compressed(os.path.join(GOLD, "ref_rir.npz"), **store)
    with open(os.path.join(GOLD, "PINNING_rir.json"), "w") as f:
        json.dump({"measure": "max |oracle - reference| over the channel's peak |reference|, worst channel",
                   "oracle_vs_reference": pin}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
