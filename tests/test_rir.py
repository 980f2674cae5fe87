"""
CPU tier of image-method RIR simulation (csrc/rir.cu, setk_rir_image): the float64 oracle against
the reference's generator (tests/golden/ref_rir.npz), the kernel's own source on the CPU execution
model (tests/emu) against the oracle, bit identity, the C-ABI's argument checks, rir_beta and both
command lines.  The multi-segment path runs twice: with the shipped 8192-sample segments in a large
room (few images, L > 8192), and in a second build of the model with SETK_RIR_SEG=256, where the
small rooms' short responses span several segments.
"""
import ctypes

import numpy as np
import pytest
import torch

import rir_cases as rc
from oracle import rir_oracle as ro

G = rc.load_fixture()
PIN = rc.load_pinning()


@pytest.fixture(scope="session")
def emu_seg256_path(tmp_path_factory):
    return rc.build_emu_variant(str(tmp_path_factory.mktemp("emu_seg256")),
                                ["SETK_TABLE_CHUNK=8", "SETK_RIR_SEG=256"])


@pytest.fixture()
def emu_seg256(emu_seg256_path):
    """the CPU execution model with 256-sample RIR segments"""
    from setk_b200 import _lib
    _lib.use_library(emu_seg256_path)
    yield torch.device("cpu")


@pytest.mark.parametrize("name", sorted(G))
def test_oracle_vs_reference_within_pinned_spread(name):
    case = G[name]
    err = ro.peak_err(rc.oracle_case(case), case["ref"])
    assert err <= PIN[name] * 1.01 + 1e-9, (err, PIN[name])


@pytest.mark.parametrize("L", [1, 63, 64, 129, 700])
@pytest.mark.parametrize("fs", [8000, 16000])
def test_emu_lengths_and_rates(emu, L, fs):
    from setk_b200 import plan
    beta = plan.rir_beta(rc.SMALL_ROOM["room"], 0.3, 340)
    got = rc.kernel(emu, rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], L, fs=fs)
    want = ro.rir(rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], L, fs=fs)
    assert got.shape == (1, 2, L) and got.dtype == np.float32
    if np.abs(want).max() == 0:
        assert not got.any()
    else:
        assert ro.peak_err(got[0], want) <= rc.TOL_ORACLE_DENSE


OPTIONS = {
    "subcardioid": dict(mic_type="subcardioid", orientation=(0.4, 0.1)),
    "cardioid": dict(mic_type="cardioid", orientation=(1.0, -0.3)),
    "hypercardioid": dict(mic_type="hypercardioid", orientation=(2.5, 0.6)),
    "bidirectional": dict(mic_type="bidirectional", orientation=(0.0, 0.0)),
    "order0": dict(order=0),
    "order1": dict(order=1),
    "order3": dict(order=3),
    "no_hp": dict(hp_filter=False),
}


@pytest.mark.parametrize("name", list(OPTIONS))
def test_emu_options(emu, name):
    from setk_b200 import plan
    kw = dict(OPTIONS[name])
    L = kw.pop("L", 200)
    beta = plan.rir_beta(rc.SMALL_ROOM["room"], 0.25, 340)
    args = (rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], L)
    got = rc.kernel(emu, *args, **kw)
    want = ro.rir(*args, **kw)
    assert ro.peak_err(got[0], want) <= rc.TOL_ORACLE_DENSE


@pytest.mark.parametrize("L", [257, 512, 700])
@pytest.mark.parametrize("fs", [8000, 16000])
@pytest.mark.parametrize("hp", [True, False], ids=["hp", "no_hp"])
def test_emu_multi_segment_short_segments(emu_seg256, L, fs, hp):
    """256-sample segments: 2 to 3 segments, taps straddling every boundary, with and without the filter"""
    from setk_b200 import plan
    beta = plan.rir_beta(rc.SMALL_ROOM["room"], 0.3, 340)
    args = (rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], L)
    got = rc.kernel(emu_seg256, *args, fs=fs, hp_filter=hp)
    assert ro.peak_err(got[0], ro.rir(*args, fs=fs, hp_filter=hp)) <= rc.TOL_ORACLE_DENSE


@pytest.mark.parametrize("name", ["cardioid", "order2"])
def test_emu_multi_segment_options(emu_seg256, name):
    from setk_b200 import plan
    kw = dict(mic_type="cardioid", orientation=(1.0, -0.3)) if name == "cardioid" else dict(order=2)
    beta = plan.rir_beta(rc.SMALL_ROOM["room"], 0.25, 340)
    args = (rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], 900)
    got = rc.kernel(emu_seg256, *args, **kw)
    assert ro.peak_err(got[0], ro.rir(*args, **kw)) <= rc.TOL_ORACLE_DENSE


def test_emu_short_segments_give_the_same_response(emu_seg256, emu_library_path):
    """the split into segments changes no bit of the response (fixed-point sums)"""
    from setk_b200 import _lib, plan
    beta = plan.rir_beta(rc.SMALL_ROOM["room"], 0.3, 340)
    args = (rc.SMALL_ROOM["room"], beta, rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], 700)
    seg = rc.kernel(emu_seg256, *args, fs=8000, hp_filter=False)
    _lib.use_library(emu_library_path)
    one = rc.kernel(torch.device("cpu"), *args, fs=8000, hp_filter=False)
    assert np.array_equal(seg, one)


@pytest.mark.parametrize("L", [8193, 9000])
@pytest.mark.parametrize("hp", [True, False], ids=["hp", "no_hp"])
def test_emu_multi_segment_shipped_length(emu, L, hp):
    """the shipped 8192-sample segments: a 20 m room at 8 kHz keeps the lattice small past L = 8192"""
    room, src, rcv = [20.0, 18.0, 16.0], [5.0, 7.0, 3.0], [[12.0, 9.0, 8.0]]
    beta = np.full(6, 0.9)
    got = rc.kernel(emu, room, beta, src, rcv, L, fs=8000, hp_filter=hp)
    assert ro.peak_err(got[0], ro.rir(room, beta, src, rcv, L, fs=8000, hp_filter=hp)) <= rc.TOL_ORACLE


@pytest.mark.parametrize("beta", [[0.9, 0.0, 0.7, 0.8, 0.0, 0.6], [0.0] * 6, [1.0, 1.0, 0.5, 0.5, 0.9, 0.9]])
def test_emu_six_coefficients(emu, beta):
    args = (rc.SMALL_ROOM["room"], np.asarray(beta), rc.SMALL_ROOM["source"], rc.SMALL_ROOM["receivers"], 300)
    got = rc.kernel(emu, *args)
    assert ro.peak_err(got[0], ro.rir(*args)) <= rc.TOL_ORACLE_DENSE


def test_emu_batch_matches_each_problem_alone_and_is_bit_identical(emu):
    from setk_b200 import plan
    rng = np.random.default_rng(4)
    room = np.array([[2.0, 1.5, 1.2], [1.6, 1.9, 1.1], [2.2, 1.4, 1.3]])
    src = room * rng.uniform(0.2, 0.8, (3, 3))
    rcv = room[:, None, :] * rng.uniform(0.2, 0.8, (3, 2, 3))
    beta = np.stack([plan.rir_beta(r, t, 340) for r, t in zip(room, [0.2, 0.3, 0.0])])
    a = plan.rir_image(room, beta, src, rcv, 400, sr=8000, device=emu)
    b = plan.rir_image(room, beta, src, rcv, 400, sr=8000, device=emu)
    assert torch.equal(a, b)
    for i in range(3):
        one = plan.rir_image(room[i], beta[i], src[i], rcv[i], 400, sr=8000, device=emu)
        assert torch.equal(one[0], a[i])
        assert ro.peak_err(a[i].numpy(), ro.rir(room[i], beta[i], src[i], rcv[i], 400, fs=8000)) <= \
            rc.TOL_ORACLE_DENSE


def _call(cfg_kw=None, B=1, M=1, room=(2.0, 1.5, 1.2), null=None):
    from setk_b200 import _lib
    cfg = dict(sound_velocity=340.0, samp_frequency=16000.0, azimuth=0.0, elevation=0.0, n_samples=100, order=-1,
               mic_type=0, hp_filter=1)
    cfg.update(cfg_kw or {})
    bufs = dict(room=np.tile(np.asarray(room, np.float64), (max(B, 1), 1)), beta=np.full((max(B, 1), 6), 0.5),
                source=np.full((max(B, 1), 3), 0.5), receivers=np.full((max(B, 1), max(M, 1), 3), 0.4),
                rir=np.zeros((max(B, 1), max(M, 1), max(cfg["n_samples"], 1)), np.float32))
    ptrs = {k: (None if k == null else ctypes.c_void_p(v.ctypes.data)) for k, v in bufs.items()}
    c = _lib.RirConfig(**cfg)
    return _lib.library().setk_rir_image(ctypes.byref(c), ptrs["room"], ptrs["beta"], ptrs["source"],
                                         ptrs["receivers"], B, M, ptrs["rir"], None, None)


EINVAL = {
    "B0": dict(B=0), "M0": dict(M=0), "L0": dict(cfg_kw=dict(n_samples=0)),
    "c<1": dict(cfg_kw=dict(sound_velocity=0.5)), "fs<1": dict(cfg_kw=dict(samp_frequency=0.0)),
    "fs_nan": dict(cfg_kw=dict(samp_frequency=float("nan"))), "order-2": dict(cfg_kw=dict(order=-2)),
    "mic5": dict(cfg_kw=dict(mic_type=5)), "mic-1": dict(cfg_kw=dict(mic_type=-1)),
    "room0": dict(room=(2.0, 0.0, 1.0)), "room_neg": dict(room=(-1.0, 2.0, 1.0)),
    "null_room": dict(null="room"), "null_beta": dict(null="beta"), "null_source": dict(null="source"),
    "null_receivers": dict(null="receivers"), "null_rir": dict(null="rir"),
}


@pytest.mark.parametrize("name", list(EINVAL))
def test_cabi_einval(emu, name):
    assert _call(**EINVAL[name]) == -1


@pytest.mark.parametrize("kw", [dict(cfg_kw=dict(n_samples=64000), room=(1.0, 1.0, 1.0)),   # 2.2e10 images
                                dict(cfg_kw=dict(n_samples=200000), room=(0.5, 20.0, 20.0)),  # half-width 4255
                                dict(cfg_kw=dict(samp_frequency=96000.0))],                   # Tw = 768
                         ids=["candidates", "half_width", "window"])
def test_cabi_unsupported(emu, kw):
    assert _call(**kw) == -4


def test_cabi_accepts_the_smallest_call(emu):
    assert _call(cfg_kw=dict(n_samples=1)) == 0


def test_nonfinite_status_raises(emu):
    from setk_b200 import plan
    room = [2.0, 1.5, 1.2]
    with pytest.raises(ValueError, match="problem 0"):
        plan.rir_image(room, np.full(6, 0.5), [0.5, 0.5, 0.5], [[0.5, 0.5, 0.5]], 64, device=emu)


def test_rir_beta():
    from setk_b200 import plan
    room = [5.0, 4.0, 3.0]
    b = plan.rir_beta(room, 0.3, 340)
    assert b.shape == (6,) and np.allclose(b, ro.t60_to_beta(room, 0.3, 340), rtol=0, atol=0)
    assert not plan.rir_beta(room, 0, 340).any()
    assert np.array_equal(plan.rir_beta(room, [0.1, 0.2, 0.3, 0.4, 0.5, 0.6], 340), [0.1, 0.2, 0.3, 0.4, 0.5, 0.6])
    with pytest.raises(ValueError, match="cannot be calculated"):
        plan.rir_beta(room, 0.05, 340)
    with pytest.raises(ValueError):
        plan.rir_beta(room, [0.1, 0.2], 340)


@pytest.mark.parametrize("which,extra", [
    ("1d", ["--num-rirs", "2", "--rir-dur", "0.02", "--array-topo", "0,0.05,0.1", "--room-dim", "4,5;4,5;2.5,3",
            "--rt60", "0.2,0.3"]),
    ("2d", ["--num-rirs", "2", "--rir-dur", "0.02", "--room-dim", "4,5;4,5;2.5,3", "--rt60", "0.2,0.3"]),
])
def test_command_lines(emu, tmp_path, which, extra):
    cfg, worst = rc.run_cli(tmp_path, which, extra)
    assert all(len(room["spk"]) == 2 for room in cfg)
    assert worst <= 1
