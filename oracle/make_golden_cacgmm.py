"""
oracle/make_golden_cacgmm.py -- tests/golden/ref_cacgmm.npz and PINNING_cacgmm.json: the reference's
own scripts/sptk/estimate_cacgmm_masks.py, unmodified, run under oracle/ref_shim.py (plus a
distutils.util.strtobool stub: Python 3.12 has no distutils) on cuts of the spatial-clustering doc
assets, and the distance of oracle/cacgmm_oracle.py from its masks in each dtype mode.

TEST INFRASTRUCTURE, BUILD-CONTAINER ONLY (needs the reference tree).

Runs (every one --frame-len 512, the doc's):
  2spk         the blind-separation doc command: 7 ch, --num-classes 3 --num-iters 20
  noisy        the enhancement doc command: 5 ch, --num-classes 2 --num-iters 20 --solve-permu false
               --cgmm-init true --update-alpha false
  nopermu      2spk cut, 2 classes, --solve-permu false
  fixed_alpha  noisy cut, random start, --update-alpha false
  init_mask    noisy cut, --init-mask = the noisy run's masks
  two_utts     two 2spk cuts in one scp: the second utterance's start is the seed stream's second draw
  skip         the same scp with the first key's .npy already present: it is skipped and draws nothing
The audio is cut to 8000 samples per utterance so that the fixture stays under 1 MB.
"""
import io
import json
import os
import runpy
import sys
import tempfile
import types
from contextlib import redirect_stderr

import numpy as np
import scipy.io.wavfile as wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

ASSET = "/root/reference/doc/spatial_clustering/asset"
CUT = 8000
INPUTS = {"2spk_a": ("2spk.wav", 32000), "2spk_b": ("2spk.wav", 64000), "noisy": ("noisy.wav", 32000)}
RUNS = {
    "2spk": (["2spk_a"], ["--num-classes", "3", "--num-iters", "20"]),
    "noisy": (["noisy"], ["--num-classes", "2", "--num-iters", "20", "--solve-permu", "false", "--cgmm-init",
                          "true", "--update-alpha", "false"]),
    "nopermu": (["2spk_a"], ["--num-classes", "2", "--num-iters", "10", "--solve-permu", "false"]),
    "fixed_alpha": (["noisy"], ["--num-classes", "2", "--num-iters", "10", "--update-alpha", "false"]),
    "init_mask": (["noisy"], ["--num-classes", "2", "--num-iters", "10", "--init-mask", "@noisy"]),
    "two_utts": (["2spk_a", "2spk_b"], ["--num-classes", "2", "--num-iters", "10"]),
    "skip": (["2spk_a", "2spk_b"], ["--num-classes", "2", "--num-iters", "10"]),
}
COMMON = ["--frame-len", "512"]


def stub_distutils():
    if "distutils.util" not in sys.modules:
        from setk_b200.libs.opts import strtobool
        d, u = types.ModuleType("distutils"), types.ModuleType("distutils.util")
        u.strtobool = strtobool
        d.util = u
        sys.modules["distutils"], sys.modules["distutils.util"] = d, u


def write_inputs(tmp, pcm):
    for key, x in pcm.items():
        wavfile.write(os.path.join(tmp, key + ".wav"), 16000, np.ascontiguousarray(x.T))


def scp(tmp, name, keys):
    path = os.path.join(tmp, name + ".scp")
    with open(path, "w") as f:
        for k in keys:
            f.write(f"{k} {os.path.join(tmp, k + '.wav')}\n")
    return path


def run_reference(tmp, name, keys, flags, store):
    dst = os.path.join(tmp, "out_" + name)
    os.makedirs(dst, exist_ok=True)
    if name == "skip":
        np.save(os.path.join(dst, keys[0] + ".npy"), np.zeros(1, np.float32))
    flags = list(flags)
    if "@noisy" in flags:
        with open(os.path.join(tmp, "init.scp"), "w") as f:
            f.write(f"noisy {os.path.join(tmp, 'out_noisy', 'noisy.npy')}\n")
        flags[flags.index("@noisy")] = os.path.join(tmp, "init.scp")
    sys.argv = ["estimate_cacgmm_masks.py", *COMMON, *flags, scp(tmp, name, keys), dst]
    with redirect_stderr(io.StringIO()):
        runpy.run_path(os.path.join(ref_shim.REFERENCE_SPTK, "estimate_cacgmm_masks.py"), run_name="__main__")
    for k in keys[1:] if name == "skip" else keys:
        store[f"{name}/masks/{k}"] = np.load(os.path.join(dst, k + ".npy"))


def main():
    ref_shim.load_reference()
    stub_distutils()
    from oracle import cacgmm_oracle as ao
    from oracle import stft_oracle as so
    pcm = {}
    for key, (f, beg) in INPUTS.items():
        pcm[key] = np.ascontiguousarray(wavfile.read(os.path.join(ASSET, f))[1][beg:beg + CUT].T)   # C x N int16
    tmp = tempfile.mkdtemp()
    write_inputs(tmp, pcm)
    store = {f"in/{k}": v for k, v in pcm.items()}
    for name, (keys, flags) in RUNS.items():
        run_reference(tmp, name, keys, flags, store)
        store[f"{name}/keys"] = np.array(json.dumps(keys))
        store[f"{name}/flags"] = np.array(json.dumps(COMMON + flags))
    out = os.path.join(ROOT, "tests", "golden", "ref_cacgmm.npz")
    np.savez_compressed(out, **store)
    pin = {}
    g = np.load(out)
    for name in RUNS:
        pin[name] = {}
        for mode, kw in (("complex64", dict(obs_dtype=np.complex64, start_dtype=np.complex64)), ("float64", {})):
            d = [np.abs(m - r) for m, r in oracle_runs(g, name, ao, so, **kw)]
            pin[name][mode] = dict(max=float(max(x.max() for x in d)), mean=float(np.mean([x.mean() for x in d])))
        print(name, pin[name])
    with open(os.path.join(ROOT, "tests", "golden", "PINNING_cacgmm.json"), "w") as f:
        json.dump({"cut_samples": CUT, "oracle_vs_reference": pin}, f, indent=1)
    print(out, os.path.getsize(out), "bytes")


def parse_flags(flags):
    """The fixture run's options the oracle needs, with the reference script's defaults."""
    o = dict(num_classes=2, num_iters=50, seed=777, cgmm_init=False, solve_permu=True, update_alpha=True,
             init_mask=False)
    i = 0
    while i < len(flags):
        k, v = flags[i][2:].replace("-", "_"), flags[i + 1]
        if k in ("num_classes", "num_iters", "seed"):
            o[k] = int(v)
        elif k in ("cgmm_init", "solve_permu", "update_alpha"):
            o[k] = v.lower() in ("true", "1", "yes")
        elif k == "init_mask":
            o[k] = True
        i += 2
    return o


def oracle_runs(g, name, ao, so, **dtypes):
    """
    (oracle masks, reference masks) of every utterance the fixture run `name` trained, the oracle fed
    the reference's complex64 STFT and its seed stream.  `dtypes` go to cacgmm_posteriors.
    """
    keys = json.loads(str(g[f"{name}/keys"]))
    o = parse_flags(json.loads(str(g[f"{name}/flags"])))
    np.random.seed(o["seed"])
    K = o["num_classes"]
    out = []
    for i, key in enumerate(keys):
        if name == "skip" and i == 0:
            continue
        x = so.float_from_pcm16(g[f"in/{key}"])
        obs = so.multichannel_stft(x, frame_len=512, frame_hop=256, round_power_of_two=True, center=True,
                                   window="hann", transpose=False, out_dtype=np.complex64)
        _, F, T = obs.shape
        gamma = None
        if o["init_mask"]:   # the reference takes the float32 file as it is; the kernels take it in fp64
            gamma = np.transpose(g["noisy/masks/noisy"], (0, 2, 1))
            gamma = gamma if dtypes.get("obs_dtype") == np.complex64 else gamma.astype(np.float64)
        elif not (o["cgmm_init"] and K == 2):
            gamma = np.random.uniform(size=[K, F, T])
            gamma = gamma / np.sum(gamma, 0, keepdims=True)
        post = ao.cacgmm_posteriors(obs, K, o["num_iters"], gamma=gamma, cgmm_init=o["cgmm_init"],
                                    update_alpha=o["update_alpha"], **dtypes)
        masks = np.transpose(post, (0, 2, 1))
        if o["solve_permu"]:
            masks = ao.permu_align(masks)[0]
        out.append((masks.astype(np.float32), g[f"{name}/masks/{key}"]))
    return out


if __name__ == "__main__":
    main()
