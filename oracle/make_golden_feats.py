"""
oracle/make_golden_feats.py -- tests/golden/ref_feats.npz and PINNING_feats.json: the reference's own
scripts/sptk/compute_spectrogram.py and compute_fbank.py, unmodified, run under oracle/ref_shim.py (plus
a distutils.util.strtobool stub, as in make_golden_cacgmm.py, and a librosa.filters stub served by
oracle/feats_oracle.mel), and the distance of oracle/feats_oracle.py from each run.

TEST INFRASTRUCTURE, BUILD-CONTAINER ONLY (needs the reference tree).

Runs:
  doc_spec      the Spectral Feature doc's spectrogram command on doc/spectral_feature/asset/egs.wav:
                400 -> 512 / 256, center, 257-dim log spectrogram
  doc_fbank     the doc's fbank command: the same geometry, 80-bin log fbank
  fbank_default compute_fbank.py's defaults: 512 / 256, 40 bins, linear, raw int16 samples
  pow_sqrthann  --apply-pow true --window sqrthann --center false on a 1 s cut of the 5-channel
                doc/adaptive_beamformer/asset/egs.wav (channel 0 is written)
  fbank_1024    an n_fft 1024 fbank with --min-freq 20 --max-freq 7600
  fbank_400     --round-power-of-two false --frame-len 400 (n_fft 400)
  exraw         one --format exraw run (the archive's bytes are stored)
The inputs are stored as int16 (in/<key>, C x N).
"""
import io
import json
import os
import runpy
import sys
import tempfile
import types
from contextlib import redirect_stderr

import numpy as np
import scipy.io.wavfile as wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from oracle.make_golden_cacgmm import stub_distutils  # noqa: E402

DOC = "/root/reference/doc"
DOC_FLAGS = ["--frame-len", "400", "--frame-hop", "256", "--round-power-of-two", "true", "--center", "true",
             "--apply-log", "true"]
RUNS = {
    "doc_spec": ("compute_spectrogram.py", ["egs"], DOC_FLAGS),
    "doc_fbank": ("compute_fbank.py", ["egs"], DOC_FLAGS + ["--num-bins", "80"]),
    "fbank_default": ("compute_fbank.py", ["cut_a", "cut_b"], []),
    "pow_sqrthann": ("compute_spectrogram.py", ["bf5"], ["--apply-pow", "true", "--window", "sqrthann",
                                                         "--center", "false"]),
    "fbank_1024": ("compute_fbank.py", ["cut_a"], ["--frame-len", "1024", "--min-freq", "20", "--max-freq", "7600",
                                                   "--apply-log", "true", "--num-bins", "64"]),
    "fbank_400": ("compute_fbank.py", ["cut_b"], ["--round-power-of-two", "false", "--frame-len", "400",
                                                  "--apply-log", "true"]),
    "exraw": ("compute_fbank.py", ["cut_a", "cut_b"], ["--format", "exraw", "--apply-log", "true",
                                                       "--normalize-samples", "true"]),
}


def stub_librosa_filters():
    import librosa  # the shim's stub module
    from oracle import feats_oracle
    filters = types.ModuleType("librosa.filters")
    filters.mel = feats_oracle.mel
    librosa.filters = filters
    sys.modules["librosa.filters"] = filters


def inputs():
    egs = wavfile.read(os.path.join(DOC, "spectral_feature", "asset", "egs.wav"))[1]
    bf = wavfile.read(os.path.join(DOC, "adaptive_beamformer", "asset", "egs.wav"))[1]
    pcm = {"egs": egs[None], "cut_a": egs[None, 16000:36000], "cut_b": egs[None, 50000:61234],
           "bf5": bf[32000:48000].T}
    return {k: np.ascontiguousarray(v, dtype=np.int16) for k, v in pcm.items()}


def run_reference(tmp, name, script, keys, flags, store):
    from setk_b200.libs.data_handler import ArchiveReader
    scp = os.path.join(tmp, name + ".scp")
    with open(scp, "w") as f:
        for k in keys:
            f.write(f"{k} {os.path.join(tmp, k + '.wav')}\n")
    ark = os.path.join(tmp, name + ".ark")
    sys.argv = [script, *flags, scp, ark]
    with redirect_stderr(io.StringIO()):
        runpy.run_path(os.path.join(ref_shim.REFERENCE_SPTK, script), run_name="__main__")
    if "exraw" in flags:
        with open(ark, "rb") as f:
            store[f"{name}/bytes"] = np.frombuffer(f.read(), dtype=np.uint8)
        from setk_b200.libs.exraw import BinaryObjectReader
        items = list(BinaryObjectReader(ark))
    else:
        items = list(ArchiveReader(ark))
    assert [k for k, _ in items] == keys, name
    for k, v in items:
        store[f"{name}/feats/{k}"] = v


def main():
    ref_shim.load_reference()
    stub_distutils()
    stub_librosa_filters()
    from oracle import feats_oracle as fo
    pcm = inputs()
    tmp = tempfile.mkdtemp()
    for k, x in pcm.items():
        wavfile.write(os.path.join(tmp, k + ".wav"), 16000, np.ascontiguousarray(x.T if x.shape[0] > 1 else x[0]))
    store = {f"in/{k}": v for k, v in pcm.items()}
    for name, (script, keys, flags) in RUNS.items():
        run_reference(tmp, name, script, keys, flags, store)
        store[f"{name}/script"] = np.array(script)
        store[f"{name}/keys"] = np.array(json.dumps(keys))
        store[f"{name}/flags"] = np.array(json.dumps(flags))
    out = os.path.join(ROOT, "tests", "golden", "ref_feats.npz")
    np.savez_compressed(out, **store)
    pin = {}
    for name, (script, keys, flags) in RUNS.items():
        err = 0.0
        for k in keys:
            ref = store[f"{name}/feats/{k}"]
            o = fo.run(script, pcm[k], flags)
            assert o.shape == ref.shape, (name, o.shape, ref.shape)
            err = max(err, float(np.max(np.abs(o - ref)) / max(np.max(np.abs(ref)), 1e-30)))
        pin[name] = {"script": script, "flags": flags, "shapes": [list(store[f"{name}/feats/{k}"].shape)
                                                                  for k in keys], "oracle_rel_inf": err}
        print(name, pin[name])
    with open(os.path.join(ROOT, "tests", "golden", "PINNING_feats.json"), "w") as f:
        json.dump(pin, f, indent=1)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
