"""
The CGMM and CACGMM mask estimators share one host path; what they compute and what they refuse stays
as it was.  Against tests/golden/cgmm_family_emu_sha256.json on the CPU execution model:
  * sha256 of the CACGMM masks through StftPlan.cacgmm_masks and cacgmm_from_stft (C = 2, 3, 5, 9;
    K = 2, 3, 4; a given start and cgmm_init; alignment on and off; a ragged batch; num_iters = 0) and
    the library's launch count of every call, CGMM calls included (their masks are pinned by
    cgmm_emu_sha256.json);
  * (return code, message) of refused calls on the four C entry points and setk_permu_align, and the
    Python exception of the same bad arguments through plan.py and the trainers;
  * the output bytes, log lines (timestamps and source locations stripped) and --help text of
    estimate_cgmm_masks.py and estimate_cacgmm_masks.py over the tile and the generic STFT routes.
family_digests(device) computes the mask table on any device.
"""
import ctypes
import hashlib
import json
import os
import re

import numpy as np
import pytest
import torch

import parity_cases as pc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cgmm_family_emu_sha256.json")

# CACGMM: (C, n_fft, K, start "given" / "cgmm", aligned, ragged, num_iters)
CACGMM_CASES = [
    (2, 512, 2, "cgmm", True, False, 2),
    (3, 512, 3, "given", False, True, 2),
    (5, 1024, 4, "given", True, True, 1),
    (9, 512, 2, "cgmm", False, False, 1),
    (9, 512, 3, "given", True, False, 1),
    (2, 512, 4, "given", False, False, 0),
    (3, 512, 2, "cgmm", True, True, 0),
]
# CGMM: (C, n_fft, K, given start, update_alpha, ragged, num_iters)
CGMM_CASES = [
    (4, 512, 2, False, False, False, 2),
    (3, 1024, 3, True, True, True, 2),
    (9, 512, 2, False, False, False, 1),
    (2, 512, 4, True, False, False, 0),
]


def _sha(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def _counted(fn):
    """(fn(), the library launches it made)"""
    from setk_b200 import _lib
    before = _lib.launch_count()
    out = fn()
    return out, _lib.launch_count() - before


def _case_input(device, C, n_fft, K, ragged, seed, dtype):
    from setk_b200 import plan as P
    rng = np.random.default_rng(seed)
    B, N = 2, 3000 if n_fft == 512 else 4200
    pl = P.StftPlan(C, n_fft, 256, True, True, "hann", B, N, device)
    x = torch.from_numpy(pc.structured_audio(rng, B, C, N)).to(device)
    ns = torch.tensor([N, N // 2], dtype=torch.int32).to(device) if ragged else None
    T, F = pl.num_frames(N), pl.num_bins
    g = rng.uniform(0.05, 1.0, size=(B, K, T, F))
    return pl, x, ns, torch.from_numpy((g / g.sum(1, keepdims=True)).astype(dtype)).to(device)


def family_digests(device):
    """{case/call: [sha256 of the masks, launches]} for every CACGMM and CGMM case."""
    from setk_b200 import plan as P
    out = {}
    for C, n_fft, K, start, aligned, ragged, iters in CACGMM_CASES:
        key = f"cacgmm/C{C}/{n_fft}/K{K}/{start}/{'aligned' if aligned else 'raw'}/" + \
              ("ragged/" if ragged else "") + f"it{iters}"
        pl, x, ns, g = _case_input(device, C, n_fft, K, ragged, 100 * C + K, np.float64)
        kw = dict(init_gamma=g if start == "given" else None, cgmm_init=start == "cgmm",
                  permu_plan=P.PERMU_PLANS[pl.num_bins] if aligned else None)
        (m, st), n = _counted(lambda: pl.cacgmm_masks(x, K, iters, n_samples=ns, **kw))
        assert int(st.abs().sum()) == 0
        out[f"{key}/masks"] = [_sha(m), n]
        X = pl.stft(x)
        (m, st), n = _counted(lambda: P.cacgmm_from_stft(X, K, iters, update_alpha=False, **kw))
        assert int(st.abs().sum()) == 0
        out[f"{key}/stft"] = [_sha(m), n]
        pl.close()
    for C, n_fft, K, given, alpha, ragged, iters in CGMM_CASES:
        key = f"cgmm/C{C}/{n_fft}/K{K}/{'given' if given else 'uniform'}/" + ("ragged/" if ragged else "") + \
              f"it{iters}"
        pl, x, ns, g = _case_input(device, C, n_fft, K, ragged, 200 * C + K, np.float32)
        g = g if given else None
        (m, _), n = _counted(lambda: pl.cgmm_masks(x, K, iters, init_gamma=g, update_alpha=alpha, n_samples=ns))
        out[f"{key}/masks"] = [_sha(m), n]
        X = pl.stft(x)
        (m, _), n = _counted(lambda: P.cgmm_from_stft(X, K, iters, init_gamma=g, update_alpha=alpha))
        out[f"{key}/stft"] = [_sha(m), n]
        pl.close()
    return out


def cabi_refusals(device):
    """{call: [return code, message]} of refused calls; none of them launches anything."""
    from setk_b200 import _lib
    from setk_b200 import plan as P
    lib = _lib.library()
    buf = torch.zeros(1 << 16, dtype=torch.float64)
    p = ctypes.c_void_p(buf.data_ptr())
    rows = (ctypes.c_int32 * 3)(2, 0, 8)
    bad = (ctypes.c_int32 * 3)(2, 4, 4)
    plans = {"p2": P.StftPlan(2, 512, 256, True, True, "hann", 2, 3000, device),
             "p1": P.StftPlan(1, 512, 256, True, True, "hann", 2, 3000, device),
             "p256": P.StftPlan(2, 256, 64, True, True, "hann", 2, 3000, device)}
    h = {k: v._h for k, v in plans.items()}
    # setk_cgmm_masks(plan, audio, n_samples, B, N, K, iters, init_gamma, update_alpha, masks, status)
    cgmm = {
        "null_plan": (None, p, None, 1, 3000, 2, 2, None, 0, p, p),
        "null_audio": (h["p2"], None, None, 1, 3000, 2, 2, None, 0, p, p),
        "null_masks": (h["p2"], p, None, 1, 3000, 2, 2, None, 0, None, p),
        "batch": (h["p2"], p, None, 3, 3000, 2, 2, None, 0, p, p),
        "samples": (h["p2"], p, None, 1, 3001, 2, 2, None, 0, p, p),
        "short": (h["p2"], p, None, 1, 100, 2, 2, None, 0, p, p),
        "K1": (h["p2"], p, None, 1, 3000, 1, 2, None, 0, p, p),
        "K5": (h["p2"], p, None, 1, 3000, 5, 2, p, 0, p, p),
        "K3_no_start": (h["p2"], p, None, 1, 3000, 3, 2, None, 0, p, p),
        "iters": (h["p2"], p, None, 1, 3000, 2, -1, None, 0, p, p),
        "K3_no_start_iters": (h["p2"], p, None, 1, 3000, 3, -1, None, 0, p, p),
        "n_fft256": (h["p256"], p, None, 1, 3000, 2, 2, None, 0, p, p),
        "n_fft256_iters": (h["p256"], p, None, 1, 3000, 2, -1, None, 0, p, p),
    }
    # setk_cgmm_stft(stft, B, C, F, T, K, iters, init_gamma, update_alpha, masks, status)
    cgmm_stft = {
        "null_stft": (None, 1, 2, 8, 4, 2, 2, None, 0, p, p),
        "null_masks": (p, 1, 2, 8, 4, 2, 2, None, 0, None, p),
        "B0": (p, 0, 2, 8, 4, 2, 2, None, 0, p, p),
        "B65536": (p, 65536, 2, 8, 4, 2, 2, None, 0, p, p),
        "C0": (p, 1, 0, 8, 4, 2, 2, None, 0, p, p),
        "C17": (p, 1, 17, 8, 4, 2, 2, None, 0, p, p),
        "F0": (p, 1, 2, 0, 4, 2, 2, None, 0, p, p),
        "T0": (p, 1, 2, 8, 0, 2, 2, None, 0, p, p),
        "K5": (p, 1, 2, 8, 4, 5, 2, p, 0, p, p),
        "K3_no_start": (p, 1, 2, 8, 4, 3, 2, None, 0, p, p),
        "iters": (p, 1, 2, 8, 4, 2, -1, None, 0, p, p),
        "K3_no_start_iters": (p, 1, 2, 8, 4, 3, -1, None, 0, p, p),
    }
    # setk_cacgmm_masks(plan, audio, n_samples, B, N, K, iters, init_gamma, cgmm_init, update_alpha, plan rows,
    #                   R, masks, status)
    cacgmm = {
        "null_plan": (None, p, None, 1, 3000, 2, 2, None, 1, 1, None, 0, p, p),
        "null_audio": (h["p2"], None, None, 1, 3000, 2, 2, None, 1, 1, None, 0, p, p),
        "batch": (h["p2"], p, None, 0, 3000, 2, 2, None, 1, 1, None, 0, p, p),
        "K5": (h["p2"], p, None, 1, 3000, 5, 2, p, 0, 1, None, 0, p, p),
        "C1": (h["p1"], p, None, 1, 3000, 2, 2, None, 1, 1, None, 0, p, p),
        "iters": (h["p2"], p, None, 1, 3000, 2, -1, None, 1, 1, None, 0, p, p),
        "no_start": (h["p2"], p, None, 1, 3000, 2, 2, None, 0, 1, None, 0, p, p),
        "K3_cgmm_init": (h["p2"], p, None, 1, 3000, 3, 2, None, 1, 1, None, 0, p, p),
        "no_start_iters": (h["p2"], p, None, 1, 3000, 3, -1, None, 0, 1, None, 0, p, p),
        "row": (h["p2"], p, None, 1, 3000, 2, 2, None, 1, 1, bad, 1, p, p),
        "rows_negative": (h["p2"], p, None, 1, 3000, 2, 2, None, 1, 1, rows, -1, p, p),
        "rows_65": (h["p2"], p, None, 1, 3000, 2, 2, None, 1, 1, rows, 65, p, p),
        "n_fft256": (h["p256"], p, None, 1, 3000, 2, 2, None, 1, 1, None, 0, p, p),
        "n_fft256_row": (h["p256"], p, None, 1, 3000, 2, 2, None, 1, 1, bad, 1, p, p),
    }
    # setk_cacgmm_stft(stft, B, C, F, T, K, iters, init_gamma, cgmm_init, update_alpha, plan rows, R, masks,
    #                  status)
    cacgmm_stft = {
        "null_stft": (None, 1, 2, 8, 4, 2, 2, None, 1, 1, None, 0, p, p),
        "null_masks": (p, 1, 2, 8, 4, 2, 2, None, 1, 1, None, 0, None, p),
        "B0": (p, 0, 2, 8, 4, 2, 2, None, 1, 1, None, 0, p, p),
        "C17": (p, 1, 17, 8, 4, 2, 2, None, 1, 1, None, 0, p, p),
        "T0": (p, 1, 2, 8, 0, 2, 2, None, 1, 1, None, 0, p, p),
        "K1": (p, 1, 2, 8, 4, 1, 2, p, 0, 1, None, 0, p, p),
        "C1": (p, 1, 1, 8, 4, 2, 2, None, 1, 1, None, 0, p, p),
        "C1_K5": (p, 1, 1, 8, 4, 5, 2, None, 1, 1, None, 0, p, p),
        "iters": (p, 1, 2, 8, 4, 2, -1, None, 1, 1, None, 0, p, p),
        "no_start": (p, 1, 2, 8, 4, 2, 2, None, 0, 1, None, 0, p, p),
        "no_start_iters": (p, 1, 2, 8, 4, 3, -1, None, 0, 1, None, 0, p, p),
        "row": (p, 1, 2, 8, 4, 2, 2, None, 1, 1, bad, 1, p, p),
        "row_hi": (p, 1, 2, 4, 4, 2, 2, None, 1, 1, rows, 1, p, p),
        "rows_65": (p, 1, 2, 8, 4, 2, 2, None, 1, 1, rows, 65, p, p),
        "aligner_smem": (p, 1, 2, 8193, 4, 4, 2, p, 0, 1, rows, 1, p, p),
    }
    # setk_permu_align(masks, n_frames, B, K, T, F, plan rows, R, out, mapping)
    permu = {
        "null_masks": (None, None, 1, 2, 4, 8, rows, 1, p, None),
        "K5": (p, None, 1, 5, 4, 8, rows, 1, p, None),
        "shape": (p, None, 1, 2, 0, 8, rows, 1, p, None),
        "no_plan": (p, None, 1, 2, 4, 8, None, 0, p, None),
        "row": (p, None, 1, 2, 4, 8, bad, 1, p, None),
        "smem": (p, None, 1, 4, 4, 8193, rows, 1, p, None),
    }
    out = {}
    for name, table in (("setk_cgmm_masks", cgmm), ("setk_cgmm_stft", cgmm_stft), ("setk_cacgmm_masks", cacgmm),
                        ("setk_cacgmm_stft", cacgmm_stft), ("setk_permu_align", permu)):
        fn = getattr(lib, name)
        for case, args in table.items():
            rc, n = _counted(lambda: fn(*args, None))
            assert n == 0 and rc != 0, (name, case)
            out[f"{name}/{case}"] = [rc, lib.setk_last_error_string().decode()]
    for pl in plans.values():
        pl.close()
    return out


def python_refusals(device):
    """{call: [exception type, message]} through plan.py and the trainers; none of them launches anything."""
    from setk_b200 import plan as P
    from setk_b200.libs import utils
    from setk_b200.libs.cluster import CacgmmTrainer, CgmmTrainer
    utils.set_default_device(device)
    pl = P.StftPlan(2, 512, 256, True, True, "hann", 1, 3000, device)
    pl256 = P.StftPlan(2, 256, 64, True, True, "hann", 1, 3000, device)
    x = torch.zeros((1, 2, 3000), device=device)
    T, F = pl.num_frames(3000), 257
    X = torch.zeros((1, 2, F, 4), dtype=torch.complex64, device=device)
    X1 = torch.zeros((1, 1, F, 4), dtype=torch.complex64, device=device)
    g64 = torch.zeros((1, 2, T, F), dtype=torch.float64, device=device)
    obs = np.zeros((2, F, 4), np.complex64)
    calls = {
        "cgmm_masks/K3_no_start": lambda: pl.cgmm_masks(x, 3, 2),
        "cgmm_masks/K5": lambda: pl.cgmm_masks(x, 5, 2),
        "cgmm_masks/iters": lambda: pl.cgmm_masks(x, 2, -1),
        "cgmm_masks/gamma_shape": lambda: pl.cgmm_masks(x, 2, 2, init_gamma=torch.zeros((1, 2, T + 1, F))),
        "cgmm_masks/n_fft256": lambda: pl256.cgmm_masks(x, 2, 2),
        "cgmm_masks/short": lambda: pl.cgmm_masks(x[..., :100], 2, 2),
        "cgmm_from_stft/K3_no_start": lambda: P.cgmm_from_stft(X, 3, 2),
        "cgmm_from_stft/iters": lambda: P.cgmm_from_stft(X, 2, -1),
        "cgmm_from_stft/K1": lambda: P.cgmm_from_stft(X, 1, 2),
        "cacgmm_masks/K3_no_start": lambda: pl.cacgmm_masks(x, 3, 2),
        "cacgmm_masks/no_start": lambda: pl.cacgmm_masks(x, 2, 2),
        "cacgmm_masks/K5": lambda: pl.cacgmm_masks(x, 5, 2, init_gamma=torch.zeros((1, 5, T, F), dtype=torch.float64)),
        "cacgmm_masks/iters": lambda: pl.cacgmm_masks(x, 2, -1, cgmm_init=True),
        "cacgmm_masks/gamma_shape": lambda: pl.cacgmm_masks(x, 2, 2, init_gamma=g64[:, :, 1:]),
        "cacgmm_masks/row_hi": lambda: pl.cacgmm_masks(x, 2, 2, cgmm_init=True, permu_plan=[(2, 10, 300)]),
        "cacgmm_masks/row_empty": lambda: pl.cacgmm_masks(x, 2, 2, cgmm_init=True, permu_plan=[(2, 50, 50)]),
        "cacgmm_masks/no_rows": lambda: pl.cacgmm_masks(x, 2, 2, cgmm_init=True, permu_plan=[]),
        "cacgmm_masks/n_fft256": lambda: pl256.cacgmm_masks(x, 2, 2, cgmm_init=True),
        "cacgmm_from_stft/C1": lambda: P.cacgmm_from_stft(X1, 2, 2, cgmm_init=True),
        "cacgmm_from_stft/iters": lambda: P.cacgmm_from_stft(X, 2, -1, cgmm_init=True),
        "cacgmm_from_stft/K5": lambda: P.cacgmm_from_stft(X, 5, 2, cgmm_init=True),
        "cacgmm_from_stft/gamma_shape": lambda: P.cacgmm_from_stft(X, 2, 2, init_gamma=g64),
        "CgmmTrainer/K3_no_start": lambda: CgmmTrainer(obs, 3),
        "CgmmTrainer/gamma_shape": lambda: CgmmTrainer(obs, 3, gamma=np.zeros((3, F, 5))),
        "CgmmTrainer/real": lambda: CgmmTrainer(obs.real, 2),
        "CgmmTrainer/pickle": lambda: CgmmTrainer(obs, 2, cgmm="model.pkl"),
        "CgmmTrainer/K5": lambda: CgmmTrainer(obs, 5, gamma=np.full((5, F, 4), 0.2)).train(2),
        "CgmmTrainer/iters": lambda: CgmmTrainer(obs, 2).train(-1),
        "CacgmmTrainer/gamma_shape": lambda: CacgmmTrainer(obs, 3, gamma=np.zeros((3, F, 5))),
        "CacgmmTrainer/pickle": lambda: CacgmmTrainer(obs, 2, cacgmm="model.pkl"),
        "CacgmmTrainer/C1": lambda: CacgmmTrainer(obs[:1], 2, cgmm_init=True).train(2),
        "CacgmmTrainer/K5": lambda: CacgmmTrainer(obs, 5, gamma=np.full((5, F, 4), 0.2)).train(2),
        "CacgmmTrainer/iters": lambda: CacgmmTrainer(obs, 2, cgmm_init=True).train(-1),
    }
    out = {}
    for name, call in calls.items():
        def refused():
            with pytest.raises(Exception) as e:
                call()
            return e
        e, n = _counted(refused)
        assert n == 0, name
        out[name] = [type(e.value).__name__, str(e.value)]
    pl.close()
    pl256.close()
    return out


# (script, case, extra argv, first key's output present, init mask "T x F" / "K x T x F" / None)
SCRIPT_CASES = [
    ("estimate_cgmm_masks.py", "tile_skip", ["--num-iters", "2"], True, None),
    ("estimate_cgmm_masks.py", "tile_K3_permu", ["--num-iters", "2", "--num-classes", "3", "--seed", "11",
                                                 "--solve-permu", "true", "--update-alpha", "true"], False, None),
    ("estimate_cgmm_masks.py", "tile_init", ["--num-iters", "2", "--solve-permu", "true"], False, "TF"),
    ("estimate_cgmm_masks.py", "generic_256_K3", ["--num-iters", "2", "--num-classes", "3", "--frame-len", "256",
                                                  "--frame-hop", "128"], True, None),
    ("estimate_cgmm_masks.py", "generic_400_init", ["--num-iters", "2", "--frame-len", "400", "--frame-hop", "160",
                                                    "--round-power-of-two", "false"], False, "TF"),
    ("estimate_cgmm_masks.py", "generic_hop130", ["--num-iters", "1", "--frame-hop", "130"], False, None),
    ("estimate_cacgmm_masks.py", "tile_skip", ["--num-iters", "2"], True, None),
    ("estimate_cacgmm_masks.py", "tile_K3_init", ["--num-iters", "2", "--num-classes", "3"], False, "KTF"),
    ("estimate_cacgmm_masks.py", "tile_cgmm_init_raw", ["--num-iters", "2", "--cgmm-init", "true",
                                                        "--solve-permu", "false", "--update-alpha", "false"],
     False, None),
    ("estimate_cacgmm_masks.py", "tile_1024_K3", ["--num-iters", "1", "--num-classes", "3", "--seed", "5",
                                                  "--frame-len", "1024"], False, None),
    ("estimate_cacgmm_masks.py", "generic_256_K3", ["--num-iters", "2", "--num-classes", "3", "--frame-len", "256",
                                                    "--frame-hop", "128", "--solve-permu", "false"], True, None),
    ("estimate_cacgmm_masks.py", "generic_400_init", ["--num-iters", "2", "--frame-len", "400", "--frame-hop",
                                                      "160", "--round-power-of-two", "false", "--solve-permu",
                                                      "false"], False, "KTF"),
    ("estimate_cacgmm_masks.py", "generic_hop130", ["--num-iters", "1", "--frame-hop", "130"], False, None),
]
KEYS = ["utt_a", "utt_b", "utt_c"]


def _log_lines(stderr):
    """the log lines with their timestamp and source location stripped: "LEVEL message" """
    return [re.sub(r"^\S+ \S+ \[.* - (\w+) \] ", r"\1 ", ln) for ln in stderr.splitlines()]


def _frames(argv, N):
    o = dict(zip(argv[::2], argv[1::2]))
    n_fft = int(o.get("--frame-len", 512))
    if o.get("--round-power-of-two", "true") == "true":
        n_fft = 1 << (n_fft - 1).bit_length()
    return N // int(o.get("--frame-hop", 256)) + 1, n_fft // 2 + 1


def script_outputs(library, tmp):
    """{script/case: {"files": {key: sha256 of the .npy}, "log": [...]}} and {script/help: text}."""
    import scipy.io.wavfile as wavfile
    from script_runner import run_script
    rng = np.random.default_rng(2024)
    lengths = [2600, 3400, 2200]
    scp = os.path.join(tmp, "wav.scp")
    with open(scp, "w") as f:
        for key, N in zip(KEYS, lengths):
            x = pc.structured_audio(rng, 1, 3, N)[0]
            pcm = np.clip(np.round(x / np.abs(x).max() * 20000), -32768, 32767).astype(np.int16)
            wavfile.write(os.path.join(tmp, key + ".wav"), 16000, np.ascontiguousarray(pcm.T))
            f.write(f"{key} {os.path.join(tmp, key + '.wav')}\n")
    out = {}
    for script, case, argv, skip_first, init in SCRIPT_CASES:
        dst = os.path.join(tmp, script[:-3], case)
        os.makedirs(dst)
        if skip_first:
            np.save(os.path.join(dst, KEYS[0] + ".npy"), np.zeros(1, np.float32))
        argv = list(argv)
        if init:
            K = int(dict(zip(argv[::2], argv[1::2])).get("--num-classes", 2))
            with open(os.path.join(dst + "_init.scp"), "w") as f:
                for key, N in list(zip(KEYS, lengths))[:2]:          # the last key has no init mask
                    T, F = _frames(argv, N)
                    m = rng.uniform(0.05, 1.0, size=(K, T, F))
                    m = (m / m.sum(0, keepdims=True)).astype(np.float32)
                    path = os.path.join(dst + "_init", key + ".npy")
                    os.makedirs(os.path.dirname(path), exist_ok=True)
                    np.save(path, m[0] if init == "TF" else m)
                    f.write(f"{key} {path}\n")
            argv += ["--init-mask", dst + "_init.scp"]
        r = run_script(script, [*argv, scp, dst], library=library)
        files = {}
        for key in KEYS:
            with open(os.path.join(dst, key + ".npy"), "rb") as f:
                files[key] = hashlib.sha256(f.read()).hexdigest()
        out[f"{script}/{case}"] = {"files": files, "log": _log_lines(r.stderr)}
    for script in ("estimate_cgmm_masks.py", "estimate_cacgmm_masks.py"):
        out[f"{script}/help"] = run_script(script, ["--help"]).stdout
    return out


def _golden():
    with open(GOLD) as f:
        return json.load(f)


def test_cacgmm_masks_and_launches_unchanged(emu):
    want = _golden()["masks"]
    got = family_digests(emu)
    assert sorted(got) == sorted(want)
    assert [k for k in want if got[k] != want[k]] == []


def test_refusals_unchanged(emu):
    want = _golden()
    assert cabi_refusals(emu) == want["cabi"]
    assert python_refusals(emu) == want["python"]


def test_scripts_unchanged(emu_library_path, tmp_path, monkeypatch):
    monkeypatch.setenv("COLUMNS", "100")          # argparse wraps --help to the terminal's width
    want = _golden()["scripts"]
    got = script_outputs(emu_library_path, str(tmp_path))
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], k
