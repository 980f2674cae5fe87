"""
The random draws of scripts/sptk/rir_generate_{1d,2d}.py (setk_b200/rir_cli.py), pinned: each
configuration's rir.json with random.seed(7) against tests/golden/rir_cli_draws.json, which was recorded
with the two scripts' earlier, separate implementations.  rir.json holds only host-side draws and
rounding (rooms, receivers, sources, beta), so it is the same on any device.  The configurations reach
both geometries, the vertical linear array, the absorption-coefficient path (--rt60 "") and T60 = 0;
every run's files are also checked for name, format and shape.
"""
import json
import os

import pytest

import rir_cases as rc

SHORT = ["--num-rirs", "3", "--rir-dur", "0.02"]
CONFIGS = {
    "1d": ("1d", SHORT),
    "1d_vertical": ("1d", SHORT + ["--vertical-oriented", "true"]),
    "1d_absorption": ("1d", SHORT + ["--rt60", ""]),
    "1d_rt60_zero": ("1d", SHORT + ["--rt60", "0,0"]),
    "2d": ("2d", SHORT),
    "2d_topo": ("2d", SHORT + ["--array-topo", "0,0;0.08,0;0.04,0.07"]),
}

with open(os.path.join(rc.GOLD, "rir_cli_draws.json")) as f:
    DRAWS = json.load(f)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_draws_match_fixture(emu, tmp_path, name):
    which, extra = CONFIGS[name]
    cfg, _ = rc.run_cli(tmp_path, which, extra, check_sources=0)
    assert cfg == DRAWS[name]
