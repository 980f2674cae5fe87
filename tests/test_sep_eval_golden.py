"""
CPU tier: the separation metrics against tests/golden/ref_sep_eval.npz, the reference's own
compute_si_snr.py and compute_sdr.py runs (oracle/make_golden_sep_eval.py): the oracle against the
reference's float32 SI-SNR and the explicit-route criteria, the kernels on the CPU execution model on one
fixture utterance, and both command lines on the CPU execution model against the stored outputs.
"""
import numpy as np
import pytest
import torch

import sep_eval_cases as sc
from oracle import sep_eval_oracle as so
from oracle.make_golden_sep_eval import RUNS
from script_runner import run_script
from setk_b200.libs.metric import best_mean_permutation

Z = sc.golden()


@pytest.mark.parametrize("name", ["two", "three"])
def test_oracle_reproduces_the_fixture(name):
    for key in sc.golden_keys(Z, name):
        r, e = sc.golden_signals(Z, name, key)
        N = r.shape[0]
        m = np.array([[so.si_snr(e[j], r[i]) for i in range(N)] for j in range(N)])
        want = Z[f"si_snr_ref/{name}/{key}"]
        assert np.abs(m - want).max() <= 1e-3
        assert best_mean_permutation(m)[1] == best_mean_permutation(want)[1]
        fft = so.criteria(r, e, so.FLEN)
        assert np.abs(fft - Z[f"bss_explicit/{name}/{key}"]).max() <= 1e-8


def test_kernels_on_a_fixture_utterance(emu):
    from setk_b200 import plan
    r, e = sc.golden_signals(Z, "two", "u2")
    crit, _, status = plan.bss_eval(torch.from_numpy(e[None]), torch.from_numpy(r[None]), flen=512)
    assert int(status[0]) == 0
    sc.assert_criteria_close(crit[0].numpy(), Z["bss_explicit/two/u2"], "u2")
    si = plan.si_snr(torch.from_numpy(e[None]), torch.from_numpy(r[None]))[0].numpy()
    assert np.abs(si - Z["si_snr_ref/two/u2"]).max() <= 1e-3


@pytest.mark.parametrize("run", sorted(RUNS))
def test_cli_reproduces_the_reference_run(emu_library_path, tmp_path, run):
    sc.check_golden_run(Z, run, run_script, tmp_path, library=emu_library_path, batch_size=2)
