"""
GPU tier of mixture simulation on the H100: the eight doc commands against the reference's outputs
(tests/golden/ref_simu.npz) and the float64 oracle, a 2 s RIR with 10 s of speech, a batch of 256
mixtures of mixed shapes (bit-identical run to run and to each mixture alone) and wav_simulate.py
--batch on the doc commands.
"""
import os

import numpy as np
import pytest
import scipy.io.wavfile as wavfile
import torch

import simu_cases as sc
from script_runner import run_script

pytestmark = pytest.mark.gpu

STORE = sc.load_fixture()


@pytest.fixture(scope="module")
def golden_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("simu_assets")
    sc.write_assets(STORE, str(d))
    return str(d)


@pytest.mark.parametrize("name", sc.cases(STORE))
def test_doc_commands_vs_reference_and_oracle(cuda, golden_dir, name):
    from setk_b200 import simu
    args = sc.namespace(sc.case_flags(STORE, name), golden_dir)
    m = simu.plan_mixture(args)
    oracle = sc.oracle_outputs(args)
    ref = sc.reference_outputs(STORE, name, oracle)
    err = sc.compare(simu.simulate([m], device=cuda)[0], oracle, sc.TOL_CONV)
    mix, spk, noise = simu.simulate([m], device=cuda, pcm16=True)[0]
    got = {"mix": mix, **{f"spk{i + 1}": s for i, s in enumerate(spk)}}
    if noise is not None:
        got["noise"] = noise
    worst = max(int(np.abs(got[k].astype(np.int32) - r).max()) for k, r in ref.items())
    frac = max(float((got[k] != r).mean()) for k, r in ref.items())
    print(f"{name}: float vs oracle {err:.2e}, PCM-16 vs reference {worst} LSB in {frac:.4%} of samples")
    assert err <= sc.TOL_CONV
    assert worst <= sc.PCM16_LSB


def test_two_second_rir_ten_second_speech(cuda):
    from setk_b200 import plan
    rng = np.random.default_rng(5)
    x = (0.3 * np.sin(np.arange(160000) * 0.02) * rng.uniform(0.3, 1, 160000)).astype(np.float32)
    h = (rng.standard_normal((4, 32000)) * np.exp(-np.arange(32000) / 6000) * 0.1).astype(np.float32)
    for n_out in (160000, 160000 + 32000 - 1):
        y = plan.convolve(torch.from_numpy(x).to(cuda), torch.from_numpy(h).to(cuda), n_out=n_out).cpu().numpy()
        import scipy.signal as ss
        want = ss.fftconvolve(x[None].astype(np.float64), h.astype(np.float64), axes=-1)[:, :n_out]
        err = sc.peak_err(y, want)
        print(f"32000 taps, n_out {n_out}: {err:.2e}")
        assert err <= sc.TOL_CONV


def _random_mixtures(rng, n):
    from setk_b200 import _lib
    from setk_b200.simu import Conv, Mixture, Term
    out = []
    for i in range(n):
        M = int(rng.choice([1, 4]))
        S = [int(rng.integers(2000, 40000)) for _ in range(2)]
        L = int(rng.integers(100, 9000))
        beg = [int(rng.integers(0, 5000)), 0]
        T = max(b + s for b, s in zip(beg, S))
        m = Mixture(f"m{i}", T, M, 0.9)
        for k in range(2):
            x = (0.3 * rng.standard_normal(S[k])).astype(np.float32)
            h = (rng.standard_normal((M, L)) * np.exp(-np.arange(L) / (L / 4)) * 0.2).astype(np.float32)
            m.terms.append(Term(_lib.SIMU_SPEAKER, Conv(x, h, S[k]), beg[k], S[k], 0, (0, S[k]), float(k * 2)))
        nz = (0.1 * rng.standard_normal((1, T))).astype(np.float32)
        m.terms.append(Term(_lib.SIMU_POINT_NOISE, nz, 0, T, 0, (0, T), 5.0))
        if M == 4:
            iso = (0.05 * rng.standard_normal((1, T // 2))).astype(np.float32)
            m.terms.append(Term(_lib.SIMU_ISOTROPIC, iso, 0, T // 2, 0, (0, T // 2), 8.0))
        out.append(m)
    return out


def test_batch_of_256_bit_identical(cuda):
    from setk_b200 import simu
    mixtures = _random_mixtures(np.random.default_rng(9), 256)
    a = simu.simulate(mixtures, device=cuda)
    b = simu.simulate(mixtures, device=cuda)
    for i, m in enumerate(mixtures):
        assert np.array_equal(a[i][0], b[i][0]) and np.array_equal(a[i][2], b[i][2])
    for i in range(0, 256, 5):
        alone = simu.simulate([mixtures[i]], device=cuda)[0]
        assert np.array_equal(alone[0], a[i][0]), i
        assert all(np.array_equal(x, y) for x, y in zip(alone[1], a[i][1]))
        assert np.array_equal(alone[2], a[i][2])


def test_command_line_batch_vs_reference(cuda, golden_dir, tmp_path):
    from setk_b200 import _lib
    lines, names = [], sc.cases(STORE)
    for name in names:
        flags = dict(sc.case_flags(STORE, name), dump_ref_dir=f"ref_{name}")
        argv = sc.command_line(flags, golden_dir, f"{name}.wav")
        argv = [a.replace(golden_dir, str(tmp_path)) if a.endswith(".wav") and a == argv[-1] else a for a in argv]
        argv = [a.replace(os.path.join(golden_dir, f"ref_{name}"), str(tmp_path / f"ref_{name}")) for a in argv]
        lines.append(" ".join(argv))
    listing = tmp_path / "list.txt"
    listing.write_text("\n".join(lines) + "\n")
    out = run_script("wav_simulate.py", ["--batch", str(listing)], _lib.library_path(), cwd=tmp_path).stdout
    assert out.count("RTF = ") == len(names)
    for name in names:
        flags = sc.case_flags(STORE, name)
        oracle = sc.oracle_outputs(sc.namespace(flags, golden_dir))
        ref = sc.reference_outputs(STORE, name, oracle)
        ref_dir = tmp_path / f"ref_{name}"
        n_spk = len(flags["src_spk"].split(","))
        files = {"mix": tmp_path / f"{name}.wav"}
        files.update({"spk1": ref_dir / "clean" / f"{name}.wav"} if n_spk == 1 else
                     {f"spk{i + 1}": ref_dir / f"spk{i + 1}" / f"{name}.wav" for i in range(n_spk)})
        if "noise" in ref:
            files["noise"] = ref_dir / "noise" / f"{name}.wav"
        for k, path in files.items():
            sr, data = wavfile.read(str(path))
            got = data.T if data.ndim == 2 else data
            assert got.shape == ref[k].shape
            assert np.abs(got.astype(np.int32) - ref[k]).max() <= sc.PCM16_LSB, (name, k)
