"""
Shared cases and tolerances of the RIR tests (csrc/rir.cu, setk_rir_image): small rooms for the CPU
execution model, the golden cases of tests/golden/ref_rir.npz, and the command lines' check.

Error measure: max |got - want| over the channel's peak |want|, the worst channel (rir_oracle.peak_err).
  TOL_ORACLE      kernel vs the float64 oracle: float32 taps, fp64 geometry.  The error of float32
                  taps grows with the sum of |taps| over a sample relative to the peak, so the dense
                  small rooms of the CPU tier (up to 6.6e-6 measured) get TOL_ORACLE_DENSE.
  ref_tol(name)   kernel vs the reference: twice the case's pinned oracle-vs-reference spread
                  (PINNING_rir.json: 5.4e-6 .. 5.0e-5, the reference's float32 geometry) plus
                  TOL_ORACLE.
"""
import json
import os
import subprocess

import numpy as np
import torch

from script_runner import run_script

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import rir_oracle as ro  # noqa: E402

TOL_ORACLE = 5e-6
TOL_ORACLE_DENSE = 1e-5

SMALL_ROOM = dict(room=[2.0, 1.5, 1.2], source=[0.5, 0.7, 0.6], receivers=[[1.2, 0.9, 0.5], [1.5, 0.4, 0.8]])


def build_emu_variant(out_dir, defines):
    """
    The CPU execution model of every csrc/*.cu (tests/emu) built into out_dir with extra -D
    definitions, e.g. SETK_RIR_SEG=256 so that short responses take the multi-segment path.
    Returns the library's path.
    """
    emu_dir, csrc = os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "setk_b200", "csrc")
    flags = ["g++", "-O2", "-std=c++17", "-DSETK_EMU", "-fPIC", "-pthread", "-I" + emu_dir,
             "-I" + os.path.join(ROOT, "include")] + ["-D" + d for d in defines]
    jobs, objs = [], []
    for src in sorted(f for f in os.listdir(csrc) if f.endswith(".cu")):
        o = os.path.join(out_dir, src[:-3] + ".o")
        objs.append(o)
        jobs.append(subprocess.Popen(flags + ["-x", "c++", "-c", os.path.join(csrc, src), "-o", o]))
    o = os.path.join(out_dir, "cuda_emu.o")
    objs.append(o)
    jobs.append(subprocess.Popen(flags + ["-c", os.path.join(emu_dir, "cuda_emu.cc"), "-o", o]))
    assert all(j.wait() == 0 for j in jobs), "building the CPU execution model failed"
    lib = os.path.join(out_dir, "libsetk_b200_emu.so")
    subprocess.run(["g++", "-shared", "-pthread", "-o", lib] + objs, check=True)
    return lib


def load_fixture():
    with np.load(os.path.join(GOLD, "ref_rir.npz")) as z:
        store = {k: z[k] for k in z.files}
    names = sorted({k.split("/")[0] for k in store})
    return {n: {k.split("/")[1]: v for k, v in store.items() if k.startswith(n + "/")} for n in names}


def load_pinning():
    with open(os.path.join(GOLD, "PINNING_rir.json")) as f:
        return json.load(f)["oracle_vs_reference"]


def ref_tol(name):
    return 2 * load_pinning()[name] + TOL_ORACLE


def case_kwargs(case):
    return dict(fs=int(case["fs"]), c=float(case["c"]), order=int(case["order"]), mic_type=str(case["mic_type"]),
                orientation=tuple(float(v) for v in case["orientation"]), hp_filter=bool(case["hp_filter"]))


def case_beta(case):
    from setk_b200 import plan
    beta = np.atleast_1d(np.asarray(case["beta"], np.float64))
    return plan.rir_beta(case["room"], beta[0] if beta.size == 1 else beta, float(case["c"]))


def kernel(device, room, beta, source, receivers, L, fs=16000, c=340, **kw):
    from setk_b200 import plan
    return plan.rir_image(torch.as_tensor(np.asarray(room, np.float64), device=device), beta, source, receivers,
                          L, sr=fs, c=c, **kw).cpu().numpy()


def kernel_case(device, case):
    kw = case_kwargs(case)
    fs, c = kw.pop("fs"), kw.pop("c")
    return kernel(device, case["room"], case_beta(case), case["source"], case["receivers"], int(case["n_samples"]),
                  fs=fs, c=c, **kw)[0]


def oracle_case(case, receivers=None):
    return ro.rir(case["room"], case_beta(case), case["source"],
                  case["receivers"] if receivers is None else receivers, int(case["n_samples"]),
                  **case_kwargs(case))


def run_cli(tmp_path, which, extra=(), check_sources=None):
    """
    runs scripts/sptk/rir_generate_{which}.py for 2 rooms (seeded, in tmp_path, --dump-dir rir) and
    checks every file's name, format and shape, and those of the first `check_sources` sources of
    each room (all when None) against the oracle run on rir.json.  Returns (rir.json, worst
    |PCM-16 difference| in LSB).
    """
    from setk_b200 import _lib
    import scipy.io.wavfile as wavfile
    run_script(f"rir_generate_{which}.py", ["--dump-dir", "rir", *extra, "2"], library=_lib.library_path(),
               cwd=tmp_path, seed=7)
    with open(tmp_path / "rir" / "rir.json") as f:
        cfg = json.load(f)
    assert len(cfg) == 2
    worst = 0
    for r, room in enumerate(cfg):
        assert set(room) == {"beta", "receiver_location", "room_size", "receiver_geometric", "spk"}
        for i, spk in enumerate(room["spk"]):
            assert set(spk) == {"pos", "doa", "dst", "loc"}
            assert spk["loc"] == f"rir/Room{r + 1}-{i + 1}.wav"
            sr, data = wavfile.read(tmp_path / spk["loc"])
            assert sr == 16000 and data.dtype == np.int16 and data.shape[1] == len(room["receiver_location"])
            pcm = data.T
            if check_sources is not None and i >= check_sources:
                continue
            want = ro.rir(room["room_size"], case_beta(dict(room=room["room_size"], beta=room["beta"], c=cfg_c(which))),
                          spk["pos"], room["receiver_location"], pcm.shape[-1], fs=16000, c=cfg_c(which))
            ref = np.clip(np.floor(want * 32768.0), -32768, 32767)
            worst = max(worst, int(np.max(np.abs(pcm.astype(np.int64) - ref))))
    return cfg, worst


def cfg_c(which):
    return 340.0 if which == "1d" else 343.0
