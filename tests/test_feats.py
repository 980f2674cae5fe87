"""
Spectral features, CPU tier: the mel filterbank against an independent implementation, the oracle against
the reference's own runs (tests/golden/ref_feats.npz), the kernels of both routes on the CPU execution
model against the oracle, the C-ABI checks, the exraw format and both command lines.
"""
import ctypes
import io
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

import feats_cases as fc
from oracle import feats_oracle as fo
from script_runner import ROOT, run_script

MEL_CONFIGS = [(16000, 512, 40, 0, None), (16000, 512, 80, 0, None), (16000, 1024, 80, 20, 7600),
               (8000, 256, 23, 0, None), (16000, 400, 40, 0, None)]


@pytest.mark.parametrize("sr,n_fft,n_mels,fmin,fmax", MEL_CONFIGS)
def test_mel_matches_oracle_and_torchaudio(sr, n_fft, n_mels, fmin, fmax):
    import torchaudio.functional as AF
    from setk_b200.libs.filters import mel
    w = mel(sr, n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax, htk=True)
    assert w.dtype == np.float32 and w.shape == (n_mels, n_fft // 2 + 1)
    assert np.array_equal(w, fo.mel(sr, n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax, htk=True))
    ta = AF.melscale_fbanks(n_fft // 2 + 1, float(fmin), float(fmax if fmax else sr / 2), n_mels, sr,
                            norm="slaney", mel_scale="htk").T.double().numpy()
    rel = np.abs(w - ta).max(axis=1) / np.maximum(ta.max(axis=1), 1e-30)
    assert rel.max() <= 2e-5, rel.max()


def test_mel_empty_filters_warn_and_are_zero():
    from setk_b200.libs.filters import mel
    with pytest.warns(UserWarning, match="Empty filters"):
        w = mel(16000, 256, n_mels=80, htk=True)
    empty = ~w.any(axis=1)
    assert empty.sum() == 2


def test_mel_rejects_what_the_reference_never_asks_for():
    from setk_b200.libs.filters import mel
    with pytest.raises(ValueError):
        mel(16000, 512, htk=False)
    with pytest.raises(ValueError):
        mel(16000, 512, htk=True, norm=None)


def test_oracle_reproduces_reference_runs():
    g = fc.fixture()
    pin = json.load(open(os.path.join(fc.GOLD, "PINNING_feats.json")))
    for name in fc.fixture_runs(g):
        script, keys, flags = fc.run_info(g, name)
        for k in keys:
            ref = g[f"{name}/feats/{k}"]
            o = fo.run(script, g[f"in/{k}"], flags)
            assert o.shape == ref.shape
            assert np.max(np.abs(o - ref)) <= 1e-6 * np.max(np.abs(ref)), name
        assert pin[name]["oracle_rel_inf"] <= 1e-6


@pytest.mark.parametrize("C,fl,hop,center,window,rp2,lens,n_mels,pw,log", [
    (1, 32, 8, True, "hann", True, (300,), None, False, False),            # generic, n_fft 32
    (1, 32, 7, False, "hamming", True, (301, 200), 8, False, True),       # generic, odd hop, mel + log
    (1, 400, 160, True, "hann", False, (2000,), 40, False, True),         # generic, n_fft 400
    (1, 512, 256, True, "hann", True, (3000, 1700), None, False, True),   # fused 512, log spectrogram
    (5, 400, 128, False, "sqrthann", True, (2400,), None, True, False),   # fused 512, C = 5, power
    (2, 512, 254, True, "hann", True, (2600,), 40, False, False),         # fused 512, even hop, mel
    (1, 1024, 256, True, "hann", True, (4000, 2500), 64, False, True),    # fused 1024, mel + log
    (5, 1024, 512, False, "hann", True, (3000,), None, False, False),     # fused 1024, C = 5
])
def test_kernels_vs_oracle(emu, C, fl, hop, center, window, rp2, lens, n_mels, pw, log):
    rng = np.random.default_rng(fl + hop + C)
    fc.check_plan(emu, rng, C, fl, hop, center, window, rp2, lens, n_mels, pw, log)


@pytest.mark.parametrize("fl,hop,rp2", [(512, 256, True), (1024, 256, True), (400, 160, False)])
def test_ragged_batch_equals_each_alone(emu, fl, hop, rp2):
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    rng = np.random.default_rng(3)
    lens = [2600, 1024, 1900]
    N = max(lens)
    x = np.zeros((3, 2, N), np.float32)
    for b, n in enumerate(lens):
        x[b, :, :n] = rng.standard_normal((2, n))
    pl = P.StftPlan(2, fl, hop, True, rp2, "hann", 3, N, emu)
    pl.set_mel(mel(16000, pl.n_fft, n_mels=24, htk=True))
    out = pl.spectral_feats(torch.from_numpy(x), n_samples=torch.tensor(lens, dtype=torch.int32), mel=True,
                            apply_log=True).numpy()
    for b, n in enumerate(lens):
        alone = pl.spectral_feats(torch.from_numpy(x[b:b + 1, :, :n].copy()), mel=True, apply_log=True).numpy()[0]
        T = alone.shape[1]
        assert np.array_equal(out[b, :, :T], alone)
        assert not out[b, :, T:].any()


@pytest.mark.parametrize("fl,rp2", [(512, True), (1024, True), (400, False)])
def test_sample_scale_equals_scaling_the_samples(emu, fl, rp2):
    from setk_b200 import plan as P
    from setk_b200.libs.filters import mel
    rng = np.random.default_rng(4)
    pcm = rng.integers(-20000, 20000, size=(1, 1, 3000)).astype(np.float32)
    pl = P.StftPlan(1, fl, 256, True, rp2, "hann", 1, 3000, emu)
    pl.set_mel(mel(16000, pl.n_fft, n_mels=40, htk=True))
    for kw in (dict(), dict(apply_pow=True), dict(mel=True, apply_log=True)):
        raw = pl.spectral_feats(torch.from_numpy(pcm), **kw).numpy()
        scaled = pl.spectral_feats(torch.from_numpy(pcm / np.float32(32768.0)), sample_scale=32768.0, **kw).numpy()
        assert np.array_equal(raw, scaled), kw


def test_argument_errors(emu):
    from setk_b200 import _lib
    from setk_b200 import plan as P
    pl = P.StftPlan(1, 512, 256, True, True, "hann", 2, 4000, emu)
    x = torch.zeros((1, 1, 4000))
    with pytest.raises(ValueError):
        pl.spectral_feats(x, mel=True)                          # no table
    with pytest.raises(ValueError):
        pl.spectral_feats(x, sample_scale=0.0)
    with pytest.raises(ValueError):
        pl.spectral_feats(torch.zeros((1, 2, 4000)))            # channel count
    with pytest.raises(ValueError):
        pl.set_mel(np.zeros((4, 100), np.float32))               # F
    with pytest.raises(ValueError):
        pl.set_mel(-np.ones((4, 257), np.float32))
    lib = _lib.library()
    out = np.zeros((1, 1, 17, 257), np.float32)
    xa = np.zeros((1, 1, 4000), np.float32)
    f = lambda *a: lib.setk_spectral_feats(pl._h, _lib.ptr(xa), None, *a, _lib.ptr(out), None)  # noqa: E731
    assert f(1, 4000, _lib.FEAT_MEL, 1.0) == _lib.SETK_EINVAL
    assert f(1, 4000, 8, 1.0) == _lib.SETK_EINVAL
    assert f(1, 4000, 0, float("nan")) == _lib.SETK_EINVAL
    assert f(1, 4000, 0, -1.0) == _lib.SETK_EINVAL
    assert f(3, 4000, 0, 1.0) == _lib.SETK_ESHAPE
    assert f(1, 100, 0, 1.0) == _lib.SETK_ESHAPE
    assert lib.setk_spectral_feats(pl._h, None, None, 1, 4000, 0, 1.0, _lib.ptr(out), None) == _lib.SETK_EINVAL
    bad = np.full((2, 257), np.nan, np.float32)
    assert lib.setk_plan_set_mel(pl._h, 2, bad.ctypes.data_as(ctypes.c_void_p)) == _lib.SETK_EINVAL
    assert lib.setk_plan_set_mel(pl._h, 1025, bad.ctypes.data_as(ctypes.c_void_p)) == _lib.SETK_EINVAL
    assert lib.setk_plan_set_mel(pl._h, 2, None) == _lib.SETK_EINVAL
    assert lib.setk_plan_set_mel(pl._h, 0, None) == 0
    assert f(1, 4000, 0, 1.0) == 0


def test_exraw_round_trip(tmp_path):
    from setk_b200.libs.exraw import BinaryObjectReader, BinaryScriptReader, BinaryWriter
    rng = np.random.default_rng(0)
    items = {"a": rng.standard_normal((7, 3)).astype(np.float32), "b": np.arange(5, dtype=np.int64),
             "c": rng.standard_normal((2, 4)), "d": np.arange(6, dtype=np.int32).reshape(2, 3)}
    ark, scp = str(tmp_path / "x.bin"), str(tmp_path / "x.scp")
    with BinaryWriter(ark, scp) as w:
        for k, v in items.items():
            w.write(k, v)
    for k, v in BinaryObjectReader(ark):
        assert v.dtype == items[k].dtype and np.array_equal(v, items[k])
    rd = BinaryScriptReader(scp)
    assert len(rd) == 4 and "c" in rd
    for k, v in items.items():
        assert np.array_equal(rd[k], v)
    with pytest.raises(TypeError):
        with BinaryWriter(ark) as w:
            w.write("e", np.zeros(3, np.float16))


def _read_output(path, fmt):
    from setk_b200.libs.data_handler import ArchiveReader
    from setk_b200.libs.exraw import BinaryObjectReader
    return list((ArchiveReader if fmt == "kaldi" else BinaryObjectReader)(path))


def cli_against_fixture(g, tmp, library=None, batch_sizes=(64,)):
    """Every fixture run through its script; the outputs must match the fixture within the tolerances and
    be the same bytes at every batch size.  Returns {run: (rel, dlog)}."""
    import scipy.io.wavfile as wavfile
    from setk_b200.libs.filters import mel  # noqa: F401  (import check before the children)
    report = {}
    for k in {f.split("/")[1] for f in g.files if f.startswith("in/")}:
        x = g[f"in/{k}"]
        wavfile.write(os.path.join(tmp, k + ".wav"), 16000, np.ascontiguousarray(x.T if x.shape[0] > 1 else x[0]))
    for name in fc.fixture_runs(g):
        script, keys, flags = fc.run_info(g, name)
        fmt = "exraw" if "exraw" in flags else "kaldi"
        lines = "".join(f"{k} {os.path.join(tmp, k + '.wav')}\n" for k in keys)
        blobs = []
        for bs in batch_sizes:
            out, scp = os.path.join(tmp, f"{name}.{bs}.ark"), os.path.join(tmp, f"{name}.{bs}.scp")
            scp_in = os.path.join(tmp, name + ".wav.scp")
            with open(scp_in, "w") as f:
                f.write(lines)
            run_script(script, [*flags, "--batch-size", str(bs), "--scp", scp, scp_in, out], library=library)
            blobs.append(open(out, "rb").read())
            assert [ln.split()[0] for ln in open(scp)] == keys
        assert all(b == blobs[0] for b in blobs), name
        if fmt == "exraw":
            ref_bytes = g[f"{name}/bytes"].tobytes()
            assert len(blobs[0]) == len(ref_bytes)
        worst = (0.0, 0.0)
        o = fo.parse_flags(script, flags)
        for (k, v), key in zip(_read_output(out, fmt), keys):
            assert k == key
            ref = g[f"{name}/feats/{k}"]
            assert v.shape == ref.shape and v.dtype == np.float32
            pcm = g[f"in/{k}"]
            if script == "compute_spectrogram.py":
                lin = fo.spectrogram(pcm, dict(o, apply_log=False))
            else:
                lin = fo.fbank(pcm, o, linear=True)
            r = fc.compare(v, lin, o["apply_log"], o.get("apply_pow", False))
            worst = tuple(max(a, b) for a, b in zip(worst, r))
        report[name] = worst
    return report


def test_cli_against_fixture_on_emulator(emu_library_path, tmp_path):
    g = fc.fixture()
    cli_against_fixture(g, str(tmp_path), library=emu_library_path, batch_sizes=(1, 64))


def test_cli_stdin_scp_and_doc_command(emu_library_path, tmp_path):
    """The doc's fbank command line with `-` as the scp: a one-entry Kaldi archive, 405 x 80."""
    import scipy.io.wavfile as wavfile
    g = fc.fixture()
    wav = tmp_path / "egs.wav"
    wavfile.write(str(wav), 16000, g["in/egs"][0])
    out = tmp_path / "feats.ark"
    code = ["import runpy, sys", "sys.argv = sys.argv[1:]", "from setk_b200 import _lib",
            f"_lib.use_library({os.fspath(emu_library_path)!r})",
            "from setk_b200.libs import utils; utils.set_default_device('cpu')",
            "runpy.run_path(sys.argv[0], run_name='__main__')"]
    args = ["--frame-len", "400", "--frame-hop", "256", "--round-power-of-two", "true", "--center", "true",
            "--apply-log", "true", "--num-bins", "80", "-", str(out)]
    r = subprocess.run([sys.executable, "-c", "\n".join(code), os.path.join(ROOT, "scripts", "sptk",
                       "compute_fbank.py"), *args], input=f"egs {wav}\n", text=True, capture_output=True,
                       env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-2000:]
    items = _read_output(str(out), "kaldi")
    assert [k for k, _ in items] == ["egs"] and items[0][1].shape == (405, 80)
    o = fo.parse_flags("compute_fbank.py", args[:-2])
    fc.compare(items[0][1], fo.fbank(g["in/egs"], o, linear=True), True)


def test_cli_rejects_max_freq_above_nyquist(emu_library_path, tmp_path):
    with pytest.raises(AssertionError, match="Max frequency"):
        run_script("compute_fbank.py", ["--max-freq", "9000", str(tmp_path / "x.scp"), str(tmp_path / "x.ark")],
                   library=emu_library_path)
