"""
Spectral features, CPU tier: inputs the fixture does not hold.  Command lines over an scp that mixes
PCM-16, 32-bit PCM and float WAVs (every utterance gives the same bytes whatever shares its batch), an
utterance too short for one frame (the keys before it are written, then the run fails), and a dense mel
table whose weights do not fit in shared memory.
"""
import os

import numpy as np
import pytest
import scipy.io.wavfile as wavfile
import torch

import feats_cases as fc
from oracle import feats_oracle as fo
from script_runner import run_script


def _read(path):
    from setk_b200.libs.data_handler import ArchiveReader
    return list(ArchiveReader(path))


def _mixed_scp(tmp, rng):
    """An scp of the same kind of speech-like int16 signals stored as PCM-16, float32 and 32-bit PCM
    WAVs (each exactly representable in every format); returns (scp path, {key: int16 samples})."""
    pcm, lines = {}, []
    for i, fmt in enumerate(["pcm16", "float", "pcm16", "int32", "float", "pcm16"]):
        x = (rng.standard_normal(6000 + 777 * i) * 3000).clip(-32768, 32767).astype(np.int16)
        key = f"u{i}_{fmt}"
        data = {"pcm16": x, "float": x.astype(np.float32) / np.float32(32768.0),
                "int32": x.astype(np.int32) << 16}[fmt]
        path = os.path.join(tmp, key + ".wav")
        wavfile.write(path, 16000, data)
        pcm[key] = x
        lines.append(f"{key} {path}\n")
    scp = os.path.join(tmp, "mixed.scp")
    with open(scp, "w") as f:
        f.writelines(lines)
    return scp, pcm


@pytest.mark.parametrize("script,flags", [
    ("compute_spectrogram.py", ["--apply-log", "true"]),
    ("compute_fbank.py", ["--apply-log", "true", "--num-bins", "40"]),
    ("compute_fbank.py", ["--normalize-samples", "true", "--frame-len", "400", "--round-power-of-two", "false"]),
])
def test_cli_mixed_wav_formats(emu_library_path, tmp_path, script, flags):
    scp, pcm = _mixed_scp(str(tmp_path), np.random.default_rng(11))
    blobs = []
    for bs in (1, 2, 4):
        out = str(tmp_path / f"out{bs}.ark")
        run_script(script, [*flags, "--batch-size", str(bs), scp, out], library=emu_library_path)
        blobs.append(open(out, "rb").read())
    assert blobs[1] == blobs[0] and blobs[2] == blobs[0]
    o = fo.parse_flags(script, flags)
    items = _read(str(tmp_path / "out1.ark"))
    assert [k for k, _ in items] == list(pcm)
    for k, v in items:
        if script == "compute_spectrogram.py":
            lin = fo.spectrogram(pcm[k], dict(o, apply_log=False))
        else:
            lin = fo.fbank(pcm[k], o, linear=True)
        fc.compare(v, lin, o["apply_log"])


@pytest.mark.parametrize("bs", [1, 2, 3])
def test_cli_short_utterance_writes_the_keys_before_it(emu_library_path, tmp_path, bs):
    rng = np.random.default_rng(5)
    lines = []
    for key, n in (("a", 4000), ("b", 3000), ("short", 200), ("c", 4000)):
        path = str(tmp_path / f"{key}.wav")
        wavfile.write(path, 16000, (rng.standard_normal(n) * 1000).astype(np.int16))
        lines.append(f"{key} {path}\n")
    scp, out = str(tmp_path / "w.scp"), str(tmp_path / "f.ark")
    with open(scp, "w") as f:
        f.writelines(lines)
    with pytest.raises(AssertionError, match="too short"):
        run_script("compute_fbank.py", ["--batch-size", str(bs), scp, out], library=emu_library_path)
    assert [k for k, _ in _read(out)] == ["a", "b"]


@pytest.mark.parametrize("fl", [512, 1024, 400])
def test_dense_mel_table_read_from_global_memory(emu, fl):
    """A non-negative table with every weight non-zero (W = M F > 12 288 floats) is read from global memory."""
    from setk_b200 import plan as P
    rng = np.random.default_rng(fl)
    x = (rng.standard_normal((2, 2, 3000)) * 0.3).astype(np.float32)
    pl = P.StftPlan(2, fl, 256, True, fl != 400, "hann", 2, 3000, emu)
    w = rng.uniform(0.01, 1.0, size=(80, pl.num_bins)).astype(np.float32)
    pl.set_mel(w)
    out = pl.spectral_feats(torch.from_numpy(x), mel=True, apply_log=True).numpy()
    for b in range(2):
        ref = fc.oracle_linear(x[b], fl, 256, True, fl != 400, "hann", weights=w)
        fc.compare(out[b], ref, True)
