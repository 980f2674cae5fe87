"""
GPU tier of image-method RIR simulation (setk_rir_image on the H100): the reference's responses on
the doc geometries and the option cases (tests/golden/ref_rir.npz), the float64 oracle, a
multi-segment case, run-to-run bit identity and both command lines.
"""
import numpy as np
import pytest
import torch

import rir_cases as rc
from oracle import rir_oracle as ro

pytestmark = pytest.mark.gpu

G = rc.load_fixture()


@pytest.mark.parametrize("name", sorted(G))
def test_golden_cases_vs_reference_and_oracle(cuda, name):
    case = G[name]
    got = rc.kernel_case(cuda, case)
    err_ref = ro.peak_err(got, case["ref"])
    m = 0 if name.startswith("doc") else slice(None)     # the oracle on one channel of the 8000-sample cases
    rcv = np.asarray(case["receivers"])[[0]] if m == 0 else None
    err_or = ro.peak_err(got[[0]] if m == 0 else got, rc.oracle_case(case, receivers=rcv))
    print(f"{name}: vs reference {err_ref:.2e}, vs oracle {err_or:.2e}")
    assert err_ref <= rc.ref_tol(name)
    assert err_or <= rc.TOL_ORACLE


def test_multi_segment_two_seconds(cuda):
    """2 s at 16 kHz (4 segments of 8192) with order 10, filter on; and the same without the filter"""
    from setk_b200 import plan
    room, src, rcv = [5.0, 4.0, 3.0], [1.2, 2.9, 1.5], [[3.1, 1.2, 1.4], [3.3, 1.2, 1.4]]
    beta = plan.rir_beta(room, 0.4, 340)
    for hp in (True, False):
        got = rc.kernel(cuda, room, beta, src, rcv, 32000, order=10, hp_filter=hp)[0]
        want = ro.rir(room, beta, src, rcv[:1], 32000, order=10, hp_filter=hp)
        assert ro.peak_err(got[:1], want) <= rc.TOL_ORACLE


def test_batch_bit_identical(cuda):
    from setk_b200 import plan
    rng = np.random.default_rng(11)
    room = rng.uniform([4, 4, 2], [7, 7, 3], (16, 3))
    src = room * rng.uniform(0.2, 0.8, (16, 3))
    rcv = room[:, None, :] * rng.uniform(0.2, 0.8, (16, 4, 3))
    beta = np.stack([plan.rir_beta(r, 0.35, 340) for r in room])
    a = plan.rir_image(room, beta, src, rcv, 8000, device=cuda)
    b = plan.rir_image(room, beta, src, rcv, 8000, device=cuda)
    assert torch.equal(a, b)
    one = plan.rir_image(room[5:6], beta[5:6], src[5:6], rcv[5:6], 8000, device=cuda)
    assert torch.equal(one[0], a[5])


@pytest.mark.parametrize("which", ["1d", "2d"])
def test_command_lines(cuda, tmp_path, which):
    extra = ["--num-rirs", "25", "--rir-dur", "0.5", "--room-dim", "4,7;4,7;2,3", "--rt60", "0.2,0.5"]
    if which == "1d":
        extra += ["--array-topo", "0,0.05,0.1,0.15"]
    cfg, worst = rc.run_cli(tmp_path, which, extra, check_sources=2)   # the oracle on 2 of 25 per room
    assert sum(len(room["spk"]) for room in cfg) == 50
    assert all(len(room["receiver_location"]) == 4 for room in cfg)
    assert worst <= 1
