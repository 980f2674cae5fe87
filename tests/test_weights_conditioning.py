"""
CPU tier: the per-bin weight solves on the CPU execution model (tests/emu) against the 40-digit
reference of solve_cases.py, at a few shapes.  test_gpu_weights_conditioning.py runs the full
sweep on the device.  Run with -rP to see the worst err / bound per route.
"""
import numpy as np
import pytest

import solve_cases as sc

FAMILIES = [("cond", 1e8), ("gap", 1e-7), ("pgap", 1e-4), ("rank1", None), ("scale", -40)]


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    """Collect this module's worst err / bound per route; -rP shows them after its last test."""
    sc.WORST.clear()
    yield
    print("\nweights vs the 40-digit reference (emulator):\n" + sc.report())


@pytest.mark.parametrize("C,dtype,pmwf", [
    (3, np.complex128, True),        # one thread per bin, every kind
    (4, np.complex128, False),       # both C = 4 routes
    (4, np.complex64, False),
    (6, np.complex128, False),       # the 8-thread groups
])
def test_sweep(emu, C, dtype, pmwf):
    sc.check_sweep(emu, C, 2, FAMILIES, dtype, pmwf=pmwf)


def test_ban_rank1(emu):
    sc.check_post(emu, 3, 2, FAMILIES, np.complex128)
    sc.check_post(emu, 5, 2, FAMILIES[:2], np.complex64)


@pytest.mark.parametrize("C", [3, 6])
def test_status_contract(emu, C):
    sc.check_dead_channel(emu, C)
    sc.check_ladder_depth(emu, C)
    sc.check_rank_deficient(emu, C)
    sc.check_silent(emu, C)


@pytest.mark.parametrize("C,B,F", [(4, 2, 11), (6, 2, 7)])
def test_batch_invariance(emu, C, B, F):
    kinds = [("mvdr", False), ("mvdr", True), ("pevd", False)]
    if C > 4:
        kinds += [("gevd", False), ("gevd", True)]
    sc.check_invariance(emu, C, B, F, kinds)


@pytest.mark.parametrize("C", [4, 6])
def test_exact_scaling(emu, C):
    sc.check_scaling(emu, C, F=2)
    sc.check_eps_floor(emu, C, F=2)
