"""
CPU tier of mixture simulation (csrc/simu.cu: setk_convolve, setk_simulate_mix; setk_b200/simu.py;
scripts/sptk/wav_simulate.py): the float64 oracle against the reference's outputs on the eight doc
commands (tests/golden/ref_simu.npz), the kernels' own source on the CPU execution model (tests/emu)
against float64 convolutions and the oracle, bit identity, every kept quirk and error of the reference,
the C-ABI's argument checks and the command line in single and --batch mode.  The convolution runs in
the shipped build (1024-sample blocks) and in a build with SETK_CONV_BLOCK=64, where short filters span
many partitions.
"""
import argparse
import ctypes
import os

import numpy as np
import pytest
import scipy.io.wavfile as wavfile
import torch

import rir_cases
import simu_cases as sc
from script_runner import run_script

STORE = sc.load_fixture()
PIN = sc.load_pinning()["oracle_vs_reference"]


@pytest.fixture(scope="session")
def emu_block64_path(tmp_path_factory):
    return rir_cases.build_emu_variant(str(tmp_path_factory.mktemp("emu_block64")),
                                       ["SETK_TABLE_CHUNK=8", "SETK_CONV_BLOCK=64"])


@pytest.fixture(params=["block1024", "block64"])
def conv_emu(request, emu_library_path, emu_block64_path):
    """(device, P): the CPU execution model with the shipped or the 64-sample block"""
    from setk_b200 import _lib
    _lib.use_library(emu_library_path if request.param == "block1024" else emu_block64_path)
    yield torch.device("cpu"), 1024 if request.param == "block1024" else 64


@pytest.fixture(scope="module")
def golden_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("simu_assets")
    sc.write_assets(STORE, str(d))
    return str(d)


@pytest.fixture(scope="module")
def synth_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("simu_synth")
    sc.synth_assets(str(d))
    return str(d)


@pytest.mark.parametrize("name", sc.cases(STORE))
def test_oracle_vs_reference_within_pinned_spread(golden_dir, name):
    oracle = sc.oracle_outputs(sc.namespace(sc.case_flags(STORE, name), golden_dir))
    ref = sc.reference_outputs(STORE, name, oracle)
    assert set(ref) == set(oracle)
    for k, r in ref.items():
        o = sc.pcm16_from_float(oracle[k].astype(np.float32)).astype(np.int32)
        assert np.abs(o - r).max() <= PIN[name]["pcm16_lsb"] * 1.01
    assert PIN[name]["float_spread"] <= 1e-6


def _conv_case(rng, S, L, M):
    x = (rng.standard_normal(S)).astype(np.float32)
    h = (rng.standard_normal((M, L)) * np.exp(-np.arange(L) / max(L / 4, 1))).astype(np.float32)
    return x, h


def _conv_err(y, x, h, n_out):
    err = 0.0
    for m in range(h.shape[0]):
        want = np.convolve(x.astype(np.float64), h[m].astype(np.float64))
        want = np.concatenate([want, np.zeros(max(0, n_out - want.size))])[:n_out]
        assert y[m].shape == (n_out,)
        peak = np.abs(want).max()
        err = max(err, float(np.abs(y[m] - want).max() / peak) if peak > 0 else float(np.abs(y[m]).max()))
    return err


@pytest.mark.parametrize("L_kind", ["1", "P-1", "P", "P+1", "3P+5"])
@pytest.mark.parametrize("S_kind", ["1", "L-1", "P", "5P+3"])
def test_convolve_vs_float64(conv_emu, L_kind, S_kind):
    from setk_b200 import plan
    dev, P = conv_emu
    L = {"1": 1, "P-1": P - 1, "P": P, "P+1": P + 1, "3P+5": 3 * P + 5}[L_kind]
    S = {"1": 1, "L-1": max(L - 1, 1), "P": P, "5P+3": 5 * P + 3}[S_kind]
    rng = np.random.default_rng(S * 7 + L)
    for M, n_out in zip((1, 4, 7), (max(S // 2, 1), S, S + L - 1)):
        x, h = _conv_case(rng, S, L, M)
        y = plan.convolve(torch.from_numpy(x), torch.from_numpy(h), n_out=n_out).numpy()
        assert _conv_err(y, x, h, n_out) <= sc.TOL_CONV, (M, n_out)


def test_convolve_ragged_batch_bit_identity(conv_emu):
    """a ragged batch: each problem within tolerance, the same bits twice, and alone as inside the batch"""
    from setk_b200 import plan
    dev, P = conv_emu
    rng = np.random.default_rng(3)
    shapes = [(5 * P + 3, 3 * P + 5), (P, 1), (17, P + 1), (2 * P + 9, P - 1)]
    Sx, Lh, M = max(s for s, _ in shapes), max(l for _, l in shapes), 4
    x = np.zeros((len(shapes), Sx), np.float32)
    h = np.zeros((len(shapes), M, Lh), np.float32)
    probs = []
    for i, (S, L) in enumerate(shapes):
        xi, hi = _conv_case(rng, S, L, M)
        x[i, :S], h[i, :, :L] = xi, hi
        probs.append((xi, hi))
    n_out = [S + L - 1 for S, L in shapes]
    kw = dict(n_out=n_out, s_len=[s for s, _ in shapes], h_len=[l for _, l in shapes])
    a = plan.convolve(torch.from_numpy(x), torch.from_numpy(h), **kw)
    b = plan.convolve(torch.from_numpy(x), torch.from_numpy(h), **kw)
    assert torch.equal(a, b)
    for i, ((xi, hi), n) in enumerate(zip(probs, n_out)):
        assert not a[i, :, n:].any()
        assert _conv_err(a[i, :, :n].numpy(), xi, hi, n) <= sc.TOL_CONV
        one = plan.convolve(torch.from_numpy(xi), torch.from_numpy(hi), n_out=n)
        assert torch.equal(one, a[i, :, :n])


def _simulate(flags, folder, mix="out.wav"):
    from setk_b200 import simu
    args = sc.namespace(flags, folder, mix)
    return simu.simulate([simu.plan_mixture(args)], device="cpu")[0], args


@pytest.mark.parametrize("name", list(sc.DOC_COMMANDS))
def test_doc_commands_vs_oracle(emu, synth_dir, name):
    got, args = _simulate(sc.DOC_COMMANDS[name], synth_dir)
    assert sc.compare(got, sc.oracle_outputs(args), sc.TOL_CONV) <= sc.TOL_CONV


QUIRKS = {
    # the mixing loop's stale dur: both noises 3000 / 1500 samples, the last one's dur is used for both;
    # noise2 last and shorter: noise 1's image is cut to it -> a result
    "stale_dur_result": dict(src_spk="spk1.wav", point_noise="noise.wav,noise2.wav", point_noise_snr="5,3",
                             point_noise_begin="0,100", point_noise_offset=""),
    "isotropic_channel0": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", isotropic_noise="iso.wav",
                               isotropic_noise_snr="4", point_noise="noise.wav", point_noise_snr="6",
                               point_noise_rir="4ch-rir2.wav"),
    "multichannel_source_no_rir": dict(src_spk="spk4ch.wav,spk2.wav", src_sdr="2", src_begin="0,50",
                                       isotropic_noise="iso.wav", isotropic_noise_snr="10"),
    "dump_channel": dict(src_spk="spk1.wav,spk2.wav", src_rir="4ch-rir1.wav,4ch-rir2.wav", src_sdr="-2",
                         dump_channel=2, point_noise="noise.wav", point_noise_snr="0", point_noise_rir="4ch-rir3.wav",
                         isotropic_noise="iso.wav", isotropic_noise_snr="5"),
    "single_offset": dict(src_spk="spk1.wav", point_noise="noise.wav,noise2.wav", point_noise_snr="5",
                          point_noise_offset="700"),
    "repeat": dict(src_spk="spk1.wav,spk2.wav", src_begin="0,3000", src_sdr="1", point_noise="noise2.wav",
                   point_noise_snr="3", point_noise_repeat=1, point_noise_begin="200"),
    "repeat_with_rir": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", point_noise="noise2.wav",
                            point_noise_snr="3", point_noise_repeat=1, point_noise_rir="4ch-rir2.wav"),
    "norm_factor": dict(src_spk="spk2.wav", point_noise="noise.wav", point_noise_snr="-5", norm_factor=0.3),
}


@pytest.mark.parametrize("name", list(QUIRKS))
def test_quirks_vs_oracle(emu, synth_dir, name):
    got, args = _simulate(QUIRKS[name], synth_dir)
    oracle = sc.oracle_outputs(args)
    assert sc.compare(got, oracle, sc.TOL_CONV) <= sc.TOL_CONV
    if name == "multichannel_source_no_rir":   # mix_nsamps counts the 4 channels of spk4ch.wav
        assert got[0].shape == (4, 4 * 1500)
    if name == "single_offset":                # one offset: zip() reads one noise file
        from setk_b200 import simu
        assert sum(t.kind == 1 for t in simu.plan_mixture(args).terms) == 1


def test_stale_dur_broadcast_error_names_the_mixture(emu, synth_dir):
    """the last noise is longer than the first: numpy's broadcast fails, ValueError names the mixture"""
    flags = dict(src_spk="spk1.wav", point_noise="noise2.wav,noise.wav", point_noise_snr="5,3")
    args = sc.namespace(flags, synth_dir, "bad_mix.wav")
    with pytest.raises(ValueError):
        sc.oracle_outputs(args)
    from setk_b200 import simu
    with pytest.raises(ValueError, match="bad_mix.wav"):
        simu.plan_mixture(args)


RUNTIME_ERRORS = {
    "rir_count": dict(src_spk="spk1.wav,spk2.wav", src_sdr="1", src_rir="4ch-rir1.wav"),
    "no_sdr": dict(src_spk="spk1.wav,spk2.wav"),
    "sdr_count": dict(src_spk="spk1.wav,spk2.wav", src_sdr="1,2"),
    "noise_rir_count": dict(src_spk="spk1.wav", point_noise="noise.wav", point_noise_snr="1",
                            point_noise_rir="4ch-rir1.wav,4ch-rir2.wav"),
    "no_snr": dict(src_spk="spk1.wav", point_noise="noise.wav"),
    "snr_count": dict(src_spk="spk1.wav", point_noise="noise.wav", point_noise_snr="1,2"),
    "no_iso_snr": dict(src_spk="spk1.wav", isotropic_noise="iso.wav"),
    "noise_channels": dict(src_spk="spk1.wav", point_noise="noise.wav", point_noise_snr="1",
                           point_noise_rir="4ch-rir1.wav"),
    "iso_single_channel": dict(src_spk="spk1.wav", isotropic_noise="iso.wav", isotropic_noise_snr="1"),
    "iso_channels": dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", isotropic_noise="noise.wav",
                         isotropic_noise_snr="1"),
    "multichannel_convolve": dict(src_spk="spk4ch.wav", src_rir="4ch-rir1.wav"),
    "sample_rate": dict(src_spk="spk1.wav", sr=8000),
}


@pytest.mark.parametrize("name", list(RUNTIME_ERRORS))
def test_reference_runtime_errors(emu, synth_dir, name):
    from setk_b200 import simu
    args = sc.namespace(RUNTIME_ERRORS[name], synth_dir)
    with pytest.raises(RuntimeError):
        sc.oracle_outputs(args)
    with pytest.raises(RuntimeError):
        simu.plan_mixture(args)


def test_dump_channel_on_single_channel_iso(emu, synth_dir):
    """a one-channel mixture with --dump-channel takes that channel of a multichannel isotropic file"""
    got, args = _simulate(dict(src_spk="spk1.wav", src_rir="4ch-rir1.wav", dump_channel=3, isotropic_noise="iso.wav",
                               isotropic_noise_snr="2"), synth_dir)
    assert sc.compare(got, sc.oracle_outputs(args), sc.TOL_CONV) <= sc.TOL_CONV


def test_batch_bit_identical_to_alone(emu, synth_dir):
    from setk_b200 import simu
    plans = [simu.plan_mixture(sc.namespace(f, synth_dir, f"{n}.wav")) for n, f in sc.DOC_COMMANDS.items()]
    batch = simu.simulate(plans, device="cpu", pcm16=True)
    again = simu.simulate(plans, device="cpu", pcm16=True)
    for i, p in enumerate(plans):
        alone = simu.simulate([p], device="cpu", pcm16=True)[0]
        for got in (again[i], alone):
            assert np.array_equal(got[0], batch[i][0])
            assert all(np.array_equal(a, b) for a, b in zip(got[1], batch[i][1]))
            assert (got[2] is None) == (batch[i][2] is None)
            assert got[2] is None or np.array_equal(got[2], batch[i][2])


def _call_conv(B=1, M=1, Sx=8, Lh=4, Ny=8, null=None, s_len=None, h_len=None, n_out=None):
    from setk_b200 import _lib
    x = np.zeros((max(B, 1), max(Sx, 1)), np.float32)
    h = np.zeros((max(B, 1), max(M, 1), max(Lh, 1)), np.float32)
    y = np.zeros((max(B, 1), max(M, 1), max(Ny, 1)), np.float32)
    p = {k: (None if k == null else ctypes.c_void_p(v.ctypes.data)) for k, v in dict(x=x, h=h, y=y).items()}

    def lens(v):
        return None if v is None else (ctypes.c_int32 * len(v))(*v)

    return _lib.library().setk_convolve(p["x"], Sx, p["h"], Lh, B, M, lens(s_len), lens(h_len), lens(n_out),
                                        p["y"], Ny, None)


CONV_EINVAL = {
    "B0": dict(B=0), "M0": dict(M=0), "Sx0": dict(Sx=0), "Lh0": dict(Lh=0), "Ny0": dict(Ny=0),
    "B_big": dict(B=65536), "null_x": dict(null="x"), "null_h": dict(null="h"), "null_y": dict(null="y"),
    "S_over": dict(s_len=[9]), "S0": dict(s_len=[0]), "L_over": dict(h_len=[5]), "n_out_over": dict(n_out=[9]),
    "n_out0": dict(n_out=[0]),
}


@pytest.mark.parametrize("name", list(CONV_EINVAL))
def test_convolve_einval(emu, name):
    assert _call_conv(**CONV_EINVAL[name]) == -1


def test_convolve_unsupported_and_smallest(emu):
    assert _call_conv(Lh=(1 << 24) + 1) == -4
    assert _call_conv(B=1, M=1, Sx=1, Lh=1, Ny=1) == 0


def _call_mix(mix_kw=None, term_kw=None, B=1, M=1, K=1, n_pitch=16, pool_len=64, null=None, extra_terms=()):
    from setk_b200 import _lib
    pool = np.zeros(max(pool_len, 1), np.float32)
    out = np.zeros((max(B, 1), max(M, 1), max(n_pitch, 1)), np.float32)
    terms = [dict(src=0, kind=0, n_channels=1, pitch=16, begin=0, length=16, repeat=0, power_begin=0,
                  power_end=16, reserved=0, level_db=0.0, **{})]
    terms[0].update(term_kw or {})
    terms += [dict(terms[0], **t) for t in extra_terms]
    mixes = [dict(first_term=0, n_terms=len(terms), n_samples=16, n_channels=1, norm_factor=0.9)] * max(B, 1)
    mixes = [dict(m, **(mix_kw or {})) for m in mixes]
    mx = (_lib.SimuMix * len(mixes))(*[_lib.SimuMix(**m) for m in mixes])
    tm = (_lib.SimuTerm * len(terms))(*[_lib.SimuTerm(**t) for t in terms])
    ptr = {"pool": ctypes.c_void_p(pool.ctypes.data), "mixes": ctypes.cast(mx, ctypes.c_void_p),
           "terms": ctypes.cast(tm, ctypes.c_void_p), "mix": ctypes.c_void_p(out.ctypes.data)}
    ptr[null] = None
    return _lib.library().setk_simulate_mix(ptr["pool"], pool_len, ptr["mixes"], B, ptr["terms"], len(terms), M, K,
                                            n_pitch, 0, ptr["mix"], None, None, None, None)


MIX_EINVAL = {
    "null_pool": dict(null="pool"), "null_mixes": dict(null="mixes"), "null_terms": dict(null="terms"),
    "null_mix": dict(null="mix"), "B0": dict(B=0), "M0": dict(M=0), "K0": dict(K=0), "pitch0": dict(n_pitch=0),
    "pool0": dict(pool_len=0), "n_samples_over": dict(mix_kw=dict(n_samples=17)),
    "n_samples0": dict(mix_kw=dict(n_samples=0)), "channels_over": dict(mix_kw=dict(n_channels=2)),
    "term_range": dict(mix_kw=dict(first_term=1)), "no_terms": dict(mix_kw=dict(n_terms=0)),
    "no_speaker": dict(term_kw=dict(kind=1)), "bad_kind": dict(term_kw=dict(kind=3)),
    "out_of_order": dict(extra_terms=[dict(kind=1), dict(kind=0)]),
    "two_isotropic": dict(extra_terms=[dict(kind=2), dict(kind=2)]),
    "too_many_speakers": dict(extra_terms=[dict(kind=0)]),
    "term_channels": dict(term_kw=dict(n_channels=3)), "negative_begin": dict(term_kw=dict(begin=-1)),
    "past_mixture": dict(term_kw=dict(begin=4)), "outside_pool": dict(term_kw=dict(src=60)),
    "empty_power": dict(term_kw=dict(power_end=0)), "power_outside_pool": dict(term_kw=dict(power_end=65)),
}


@pytest.mark.parametrize("name", list(MIX_EINVAL))
def test_simulate_mix_einval(emu, name):
    assert _call_mix(**MIX_EINVAL[name]) == -1


def test_simulate_mix_unsupported_and_smallest(emu):
    assert _call_mix(K=70, extra_terms=[dict()] * 64) == -4
    assert _call_mix() == 0


def _run_cli(argv, cwd):
    from setk_b200 import _lib
    return run_script("wav_simulate.py", argv, _lib.library_path(), cwd=cwd).stdout


def _outputs(folder, name, flags):
    files = {"mix": os.path.join(folder, name)}
    if flags.get("dump_ref_dir"):
        ref = os.path.join(folder, flags["dump_ref_dir"])
        n_spk = len(flags["src_spk"].split(","))
        if n_spk == 1:
            files["spk1"] = os.path.join(ref, "clean", name)
        else:
            files.update({f"spk{i + 1}": os.path.join(ref, f"spk{i + 1}", name) for i in range(n_spk)})
        if flags.get("point_noise") or flags.get("isotropic_noise"):
            files["noise"] = os.path.join(ref, "noise", name)
    return files


def test_command_line_single_and_batch(emu, synth_dir, tmp_path):
    out_single, out_batch = tmp_path / "single", tmp_path / "batch"
    lines = []
    for name, flags in sc.DOC_COMMANDS.items():
        flags = dict(flags, dump_ref_dir=flags.get("dump_ref_dir") or "ref")
        for out in (out_single, out_batch):
            os.makedirs(out, exist_ok=True)
        argv = sc.command_line(flags, synth_dir, f"{name}.wav")
        argv = [a.replace(os.path.join(synth_dir, "ref"), str(out_single / "ref")) for a in argv]
        argv[-1] = str(out_single / f"{name}.wav")
        stdout = _run_cli(argv, str(tmp_path))
        assert stdout.startswith("Time cost: ") and "RTF = " in stdout
        files = _outputs(str(out_single), f"{name}.wav", flags)
        oracle = sc.oracle_outputs(sc.namespace(flags, synth_dir, f"{name}.wav"))
        for k, path in files.items():
            sr, data = wavfile.read(path)
            assert sr == 16000 and data.dtype == np.int16
            want = sc.pcm16_from_float(oracle[k].astype(np.float32))
            got = data.T if data.ndim == 2 else data
            assert got.shape == want.shape, (k, got.shape, want.shape)
            assert np.abs(got.astype(np.int32) - want).max() <= sc.PCM16_LSB, (name, k)
        lines.append(" ".join(a.replace(str(out_single), str(out_batch)) for a in argv))
    listing = tmp_path / "list.txt"
    listing.write_text("\n\n".join(lines) + "\n")
    stdout = _run_cli(["--batch", str(listing)], str(tmp_path))
    assert stdout.count("RTF = ") == len(lines)
    for name, flags in sc.DOC_COMMANDS.items():
        flags = dict(flags, dump_ref_dir=flags.get("dump_ref_dir") or "ref")
        for k, path in _outputs(str(out_single), f"{name}.wav", flags).items():
            with open(path, "rb") as a, open(path.replace(str(out_single), str(out_batch)), "rb") as b:
                assert a.read() == b.read(), (name, k)
