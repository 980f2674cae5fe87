"""
GPU tier of the separation metrics: libsetk_b200.so (sm_90a) at full size against the fp64 oracle,
run-to-run bit identity, and the two command lines.
"""
import numpy as np
import pytest
import torch

import sep_eval_cases as sc
from oracle import sep_eval_oracle as so
from script_runner import run_script

pytestmark = pytest.mark.gpu


def _batch(N, B, S, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(S - 16000, S + 1, size=B)
    lens[0] = S
    refs = np.zeros((B, N, S), np.float32)
    ests = np.zeros((B, N, S), np.float32)
    for b, n in enumerate(lens):
        r = sc.sources(N, 60000, offset=97 * b)
        reps = -(-n // 60000)
        refs[b, :, :n] = np.tile(r, (1, reps))[:, :n] * (1 + 0.01 * rng.standard_normal((N, n)))
        ests[b, :, :n] = sc.estimates(refs[b, :, :n], seed=b, swap=b % 2 == 1)
    return refs, ests, lens


@pytest.mark.parametrize("N", [2, 3, 4])
def test_full_size_against_the_oracle(cuda, N):
    from setk_b200 import plan
    B, S, L = 16, 160000, 512
    refs, ests, lens = _batch(N, B, S, N)
    crit, dropped, status = plan.bss_eval(torch.from_numpy(ests).to(cuda), torch.from_numpy(refs).to(cuda), lens,
                                          flen=L)
    again, _, _ = plan.bss_eval(torch.from_numpy(ests).to(cuda), torch.from_numpy(refs).to(cuda), lens, flen=L)
    assert torch.equal(crit, again)
    assert int(status.abs().sum()) == 0
    crit = crit.cpu().numpy()
    for b in (0, B - 1):
        n = lens[b]
        want = sc.oracle_criteria(refs[b, :, :n], ests[b, :, :n], L)
        sc.assert_criteria_close(crit[b], want, f"N={N} utterance {b}")
    si = plan.si_snr(torch.from_numpy(ests).to(cuda), torch.from_numpy(refs).to(cuda), lens)
    assert torch.equal(si, plan.si_snr(torch.from_numpy(ests).to(cuda), torch.from_numpy(refs).to(cuda), lens))
    si = si.cpu().numpy()
    for b in (0, B - 1):
        n = lens[b]
        mo = np.array([[so.si_snr(ests[b, j, :n], refs[b, i, :n]) for i in range(N)] for j in range(N)])
        assert np.abs(si[b] - mo).max() <= 1e-9


def test_dependent_references(cuda):
    from setk_b200 import plan
    refs = sc.delayed_pair(4000)
    rng = np.random.default_rng(3)
    ests = np.stack([refs[0] + 0.02 * rng.standard_normal(4000),
                     0.5 * refs[1] + 0.3 * sc.sources(2, 4000)[1]]).astype(np.float32)
    crit, dropped, status = plan.bss_eval(torch.from_numpy(ests[None]).to(cuda), torch.from_numpy(refs[None]).to(cuda),
                                          flen=64)
    assert int(status[0]) == 0 and int(dropped[0]) > 0
    sc.assert_criteria_close(crit[0].cpu().numpy(), sc.oracle_criteria(refs, ests, 64, explicit=True))


def test_clis_on_the_device(cuda, tmp_path):
    utts = {}
    for u, S in enumerate([16000, 12000, 14000]):
        refs = sc.sources(2, S, offset=500 * u)
        utts[f"utt{u}"] = (refs, sc.estimates(refs, seed=u, swap=u == 1))
    sep, ref, stored = sc.write_corpus(str(tmp_path), utts, 2, "g")
    r = run_script("compute_sdr.py", [sep, ref, "--per-utt", str(tmp_path / "sdr"), "--utt-ali", str(tmp_path / "ali")])
    with open(tmp_path / "sdr") as f, open(tmp_path / "ali") as g:
        for line, aline in zip(f, g):
            key, val = line.split()
            refs = np.stack([stored[(key, "ref", k)] for k in range(2)])
            ests = np.stack([stored[(key, "sep", k)] for k in range(2)])
            sdr, _, _, perm = so.bss_eval_sources(refs, ests)
            assert abs(float(val) - np.mean(sdr)) <= 0.0051
            assert aline.split("\t")[1].strip() == " ".join(map(str, perm))
    assert r.stdout.splitlines()[0] == "SDR(dB) Report: "
    r = run_script("compute_si_snr.py", [sep, ref, "--per-utt", str(tmp_path / "si")])
    with open(tmp_path / "si") as f:
        for line in f:
            key, val = line.split()
            e = [stored[(key, "sep", k)] for k in range(2)]
            s = [stored[(key, "ref", k)] for k in range(2)]
            best = max((so.si_snr(e[0], s[p[0]]) + so.si_snr(e[1], s[p[1]])) / 2 for p in [(0, 1), (1, 0)])
            assert abs(float(val) - best) <= 0.0051
    assert r.stdout.splitlines()[0] == "Si-SDR(dB) Report: "


def test_fixture_on_the_device(cuda):
    from setk_b200 import plan
    z = sc.golden()
    for name in ("two", "three"):
        for key in sc.golden_keys(z, name):
            r, e = sc.golden_signals(z, name, key)
            crit, _, status = plan.bss_eval(torch.from_numpy(e[None]).to(cuda), torch.from_numpy(r[None]).to(cuda))
            assert int(status[0]) == 0
            sc.assert_criteria_close(crit[0].cpu().numpy(), z[f"bss_explicit/{name}/{key}"], f"{name}/{key}")
            si = plan.si_snr(torch.from_numpy(e[None]).to(cuda), torch.from_numpy(r[None]).to(cuda))[0].cpu().numpy()
            assert np.abs(si - z[f"si_snr_ref/{name}/{key}"]).max() <= 1e-3


@pytest.mark.parametrize("run", ["sdr_two", "sdr_three", "si_two", "si_three", "si_single"])
def test_fixture_runs_on_the_device(cuda, tmp_path, run):
    sc.check_golden_run(sc.golden(), run, run_script, tmp_path)
