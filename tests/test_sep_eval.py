"""
CPU tier of the separation metrics: the oracle's two routes against each other, the kernels
(csrc/sep_eval.cu on the CPU execution model) against the oracle, determinism, the errors, and the
compute_sdr.py / compute_si_snr.py command lines.
"""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import sep_eval_oracle as so
import sep_eval_cases as sc
from script_runner import run_script


@pytest.fixture()
def emu_metric(emu):
    """the CPU execution model, with setk_b200.libs' default device the CPU"""
    from setk_b200.libs import utils
    utils.set_default_device("cpu")
    try:
        yield emu
    finally:
        utils.set_default_device(None)


def _rand(N, S, seed):
    rng = np.random.default_rng(seed)
    refs = rng.standard_normal((N, S)).astype(np.float32)
    return refs, sc.estimates(refs, seed=seed + 1)


@pytest.mark.parametrize("N", [1, 2, 3])
@pytest.mark.parametrize("L", [8, 64])
@pytest.mark.parametrize("kind", ["random", "speech"])
def test_oracle_routes_agree(N, L, kind):
    S = 600 if kind == "random" else 1500
    refs, ests = _rand(N, S, N * 10 + L) if kind == "random" else (sc.sources(N, S), None)
    if ests is None:
        ests = sc.estimates(refs, seed=N)
    for j in range(N):
        p_fft = so._fft_project(refs.astype(np.float64), ests[j].astype(np.float64), L)
        p_exp = so.explicit_projection(refs, ests[j], L)
        assert np.abs(p_fft - p_exp).max() <= 1e-10 * np.abs(p_exp).max()
    a = sc.oracle_criteria(refs, ests, L)
    b = sc.oracle_criteria(refs, ests, L, explicit=True)
    finite = np.isfinite(b)
    assert np.array_equal(np.isfinite(a), finite)
    assert np.abs(a[finite] - b[finite]).max() <= 1e-8


CASES = [(1, 8, 700), (2, 8, 900), (3, 8, 600), (1, 64, 900), (2, 64, 1200), (3, 64, 800), (2, 512, 1100)]


@pytest.mark.parametrize("N,L,S", CASES)
def test_kernels_match_oracle(emu, N, L, S):
    from setk_b200 import plan
    from setk_b200.libs.metric import _select
    refs = sc.sources(N, S, offset=37 * N + L)
    ests = sc.estimates(refs, seed=N + L, swap=N > 1)
    crit, dropped, status = plan.bss_eval(torch.from_numpy(ests[None]), torch.from_numpy(refs[None]), flen=L)
    assert int(status[0]) == 0
    want = sc.oracle_criteria(refs, ests, L, explicit=S * N * L < 4e6)
    sc.assert_criteria_close(crit[0].numpy(), want, f"N={N} L={L}")
    assert np.array_equal(_select(crit[0].numpy(), True)[3], so.best_permutation(want[1]))
    m = plan.si_snr(torch.from_numpy(ests[None]), torch.from_numpy(refs[None]))[0].numpy()
    mo = np.array([[so.si_snr(ests[j], refs[i]) for i in range(N)] for j in range(N)])
    assert np.abs(m - mo).max() <= 1e-9


@pytest.mark.parametrize("L", [64, 512])
def test_dependent_references_give_the_least_squares_projection(emu, L):
    from setk_b200 import plan
    refs = sc.delayed_pair(1000)
    rng = np.random.default_rng(3)
    ests = np.stack([refs[0] + 0.02 * rng.standard_normal(1000),
                     0.5 * refs[1] + 0.3 * sc.sources(2, 1000)[1]]).astype(np.float32)
    crit, dropped, status = plan.bss_eval(torch.from_numpy(ests[None]), torch.from_numpy(refs[None]), flen=L)
    assert int(status[0]) == 0
    assert int(dropped[0]) > 0
    sc.assert_criteria_close(crit[0].numpy(), sc.oracle_criteria(refs, ests, L, explicit=True), "dependent")


def test_ragged_batch_is_bit_identical_to_single_utterances(emu):
    from setk_b200 import plan
    N, L, lens = 2, 16, [700, 512, 903]
    S = max(lens)
    refs = np.zeros((3, N, S), np.float32)
    ests = np.zeros((3, N, S), np.float32)
    for b, n in enumerate(lens):
        refs[b, :, :n] = sc.sources(N, n, offset=100 * b)
        ests[b, :, :n] = sc.estimates(refs[b, :, :n], seed=b)
    crit, dropped, _ = plan.bss_eval(torch.from_numpy(ests), torch.from_numpy(refs), lens, flen=L)
    again, _, _ = plan.bss_eval(torch.from_numpy(ests), torch.from_numpy(refs), lens, flen=L)
    assert torch.equal(crit, again)
    si = plan.si_snr(torch.from_numpy(ests), torch.from_numpy(refs), lens)
    for b, n in enumerate(lens):
        one, d1, _ = plan.bss_eval(torch.from_numpy(ests[b:b + 1, :, :n].copy()),
                                   torch.from_numpy(refs[b:b + 1, :, :n].copy()), flen=L)
        assert torch.equal(one[0], crit[b]) and int(d1[0]) == int(dropped[b])
        s1 = plan.si_snr(torch.from_numpy(ests[b:b + 1, :, :n].copy()), torch.from_numpy(refs[b:b + 1, :, :n].copy()))
        assert torch.equal(s1[0], si[b])


def test_silent_source_and_shape_errors(emu_metric):
    from setk_b200.libs import metric
    refs = sc.sources(2, 800)
    ests = sc.estimates(refs)
    with pytest.raises(ValueError, match="reference sources is all 0s"):
        metric.bss_eval_sources(np.stack([refs[0], np.zeros(800, np.float32)]), ests)
    with pytest.raises(ValueError, match="estimated sources is all 0s"):
        metric.bss_eval_sources(refs, np.stack([ests[0], np.zeros(800, np.float32)]))
    with pytest.raises(ValueError, match="should match"):
        metric.bss_eval_sources(refs, ests[:, :700])
    sdr, sir, sar, perm = metric.bss_eval_sources(refs, ests[::-1])
    assert list(perm) == [1, 0] and sdr.shape == (2,)
    sdr2, _, _, perm2 = metric.bss_eval_sources(refs, ests[::-1], compute_permutation=False)
    assert list(perm2) == [0, 1] and sdr2[0] < sdr[0]


def test_silent_status_from_the_kernels(emu):
    from setk_b200 import _lib, plan
    refs = sc.sources(2, 600)
    refs[1] = 0
    _, _, status = plan.bss_eval(torch.from_numpy(sc.sources(2, 600)[None]), torch.from_numpy(refs[None]), flen=8)
    assert int(status[0]) & _lib.ST_SILENT


def test_metric_module_matches_the_reference_formulas(emu_metric):
    from setk_b200.libs import metric
    refs = sc.sources(3, 900)
    ests = sc.estimates(refs, seed=5)[[2, 0, 1]]
    assert abs(metric.si_snr(ests[1], refs[0]) - so.si_snr(ests[1], refs[0])) <= 1e-9
    best, ali = metric.permute_si_snr(list(ests), list(refs), align=True)
    scores = {p: sum(so.si_snr(ests[k], refs[p[k]]) for k in range(3)) / 3 for p in itertools.permutations(range(3))}
    want = max(scores, key=lambda p: scores[p])
    assert ali == want and abs(best - scores[want]) <= 1e-9
    assert metric.permute_si_snr(list(ests), list(refs)) == best
    with pytest.raises(RuntimeError):
        metric.permute_si_snr(list(ests), list(refs[:2]))


def test_cabi_argument_checks(emu):
    from setk_b200 import _lib
    lib = _lib.library()
    x = np.zeros((2, 2, 64), np.float32)
    out = np.zeros((2, 3, 2, 2))
    st = np.zeros(2, np.uint32)
    p = _lib.ptr
    assert lib.setk_bss_eval(None, p(x), None, 2, 2, 64, 8, p(out), None, p(st), None) == _lib.SETK_EINVAL
    assert lib.setk_bss_eval(p(x), p(x), None, 2, 0, 64, 8, p(out), None, p(st), None) == _lib.SETK_EINVAL
    assert lib.setk_bss_eval(p(x), p(x), None, 2, 2, 64, 0, p(out), None, p(st), None) == _lib.SETK_EINVAL
    assert lib.setk_bss_eval(p(x), p(x), None, 2, 9, 64, 8, p(out), None, p(st), None) == _lib.SETK_EUNSUPPORTED
    assert lib.setk_bss_eval(p(x), p(x), None, 2, 2, 64, 513, p(out), None, p(st), None) == _lib.SETK_EUNSUPPORTED
    assert lib.setk_bss_eval(p(x), p(x), None, 1, 8, 64, 513, p(out), None, p(st), None) == _lib.SETK_EUNSUPPORTED
    bad = np.array([64, 65], np.int32)
    assert lib.setk_bss_eval(p(x), p(x), _lib.ctypes.c_void_p(bad.ctypes.data), 2, 2, 64, 8, p(out), None, p(st),
                             None) == _lib.SETK_EINVAL
    assert lib.setk_si_snr(p(x), p(x), None, 2, 2, 64, 1, -1.0, p(out), None) == _lib.SETK_EINVAL
    assert lib.setk_si_snr(p(x), p(x), None, 2, 9, 64, 1, 1e-8, p(out), None) == _lib.SETK_EUNSUPPORTED
    assert lib.setk_si_snr(p(x), None, None, 2, 2, 64, 1, 1e-8, p(out), None) == _lib.SETK_EINVAL


def _cli_corpus(tmp):
    """two-speaker utterances: ragged, one swapped, one with estimates longer than its references"""
    utts = {}
    for u, S in enumerate([1500, 1100, 1300]):
        refs = sc.sources(2, S, offset=500 * u)
        ests = sc.estimates(refs, seed=u, swap=u == 1)
        if u == 2:
            ests = np.concatenate([ests, 0.01 * np.ones((2, 40), np.float32)], axis=1)
        utts[f"utt{u}"] = (refs, ests)
    sep, ref, stored = sc.write_corpus(str(tmp), utts, 2, "m")
    return utts, sep, ref, stored


def _read_lines(path):
    with open(path) as f:
        return [line.rstrip("\n").split("\t") for line in f]


@pytest.mark.parametrize("batch", ["0", "2"])
def test_compute_sdr_cli(emu_library_path, tmp_path, batch):
    utts, sep, ref, stored = _cli_corpus(tmp_path)
    r = run_script("compute_sdr.py", [sep, ref, "--per-utt", str(tmp_path / "sdr"), "--utt-ali",
                                      str(tmp_path / "ali"), "--batch-size", batch], library=emu_library_path)
    per = _read_lines(tmp_path / "sdr")
    ali = _read_lines(tmp_path / "ali")
    means = []
    for (key, val), (key2, a) in zip(per, ali):
        refs = np.stack([stored[(key, "ref", k)] for k in range(2)])
        ests = np.stack([stored[(key, "sep", k)] for k in range(2)])
        n = min(refs.shape[-1], ests.shape[-1])
        sdr, _, _, perm = so.bss_eval_sources(refs[:, :n], ests[:, :n], project=so._fft_project)
        assert key == key2 and a == " ".join(map(str, perm))
        assert abs(float(val) - np.mean(sdr)) <= 0.0051
        means.append(np.mean(sdr))
    assert [k for k, _ in per] == list(utts)
    lines = r.stdout.splitlines()
    assert lines[0] == "SDR(dB) Report: " and lines[1].startswith("Total: 3/")
    assert abs(float(lines[1].split("/")[1]) - np.mean(means)) <= 1e-3 and lines[2].startswith("\tNG: 3/")


@pytest.mark.parametrize("batch", ["0", "2"])
def test_compute_si_snr_cli(emu_library_path, tmp_path, batch):
    utts, sep, ref, stored = _cli_corpus(tmp_path)
    run_script("compute_si_snr.py", [sep, ref, "--per-utt", str(tmp_path / "m"), "--utt-ali", str(tmp_path / "a"),
                                     "--batch-size", batch], library=emu_library_path)
    for (key, val), (_, a) in zip(_read_lines(tmp_path / "m"), _read_lines(tmp_path / "a")):
        refs = [stored[(key, "ref", k)] for k in range(2)]
        ests = [stored[(key, "sep", k)] for k in range(2)]
        n = min(refs[0].size, ests[0].size)
        scores = {p: sum(so.si_snr(ests[k][:n], refs[p[k]][:n]) for k in range(2)) / 2
                  for p in itertools.permutations(range(2))}
        best = max(scores, key=lambda p: scores[p])
        assert a == " ".join(map(str, best)) and abs(float(val) - scores[best]) <= 0.0051
    s_sep, s_ref = sep.split(",")[0], ref.split(",")[0]
    r = run_script("compute_si_snr.py", [s_sep, s_ref, "--per-utt", str(tmp_path / "s"), "--batch-size", batch],
                   library=emu_library_path)
    for key, val in _read_lines(tmp_path / "s"):
        x, s = stored[(key, "sep", 0)], stored[(key, "ref", 0)]
        n = min(x.size, s.size)
        assert abs(float(val) - so.si_snr(x[:n], s[:n])) <= 0.0051
    assert r.stdout.splitlines()[0] == "Si-SDR(dB) Report: "


def test_clis_do_not_import_mir_eval():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for name in ("compute_sdr.py", "compute_si_snr.py"):
        with open(os.path.join(root, "scripts", "sptk", name)) as f:
            src = f.read()
        assert "import mir_eval" not in src and "from mir_eval" not in src


def test_three_cycle_permutation(emu_metric):
    # estimate j is built from reference (j + 1) % 3, so reference k is matched by estimate (k - 1) % 3:
    # bss_eval_sources' perm (estimate per reference) is [2, 0, 1], permute_si_snr's alignment
    # (reference per estimate) is (1, 2, 0) -- two different permutations, each the other's inverse
    from setk_b200.libs import metric
    refs = sc.sources(3, 1000, offset=211)
    ests = sc.estimates(refs, seed=9)[[1, 2, 0]]
    _, _, _, perm = metric.bss_eval_sources(refs, ests)
    assert list(perm) == [2, 0, 1]
    _, ali = metric.permute_si_snr(list(ests), list(refs), align=True)
    assert ali == (1, 2, 0)


def test_a_bench_sized_batch_runs_in_one_call(emu):
    from setk_b200 import _lib, plan
    for N in (2, 3, 4):
        assert plan.bss_eval_batch_step(64, N, 160000, 512) == 64
        assert _lib.library().setk_bss_eval_scratch_bytes(64, N, 160000, 512) <= plan.SEP_SCRATCH_BYTES
    assert _lib.library().setk_bss_eval_scratch_bytes(1, 9, 1000, 512) == -1
    # 8 sources at L = 512 (128 MB of system per utterance) are split to stay under the cap
    step = plan.bss_eval_batch_step(64, 8, 160000, 512)
    assert 1 <= step < 64
    assert _lib.library().setk_bss_eval_scratch_bytes(step, 8, 160000, 512) <= plan.SEP_SCRATCH_BYTES
    assert _lib.library().setk_bss_eval_scratch_bytes(step + 1, 8, 160000, 512) > plan.SEP_SCRATCH_BYTES
