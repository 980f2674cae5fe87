#!/usr/bin/env python
"""
tools/bench_ssl.py -- throughput of mask-informed sound source localisation (setk_ssl).

Workload: B = 64 utterances of 10 s at 16 kHz, STFT 512 / 256 (T = 626 frames, F = 257 bins),
seeded synthetic audio and TF-masks, one offline window per utterance.  Cases: ML at A = 181 and
360 directions with M = 4 and 8 microphones, SRP (7 adjacent pairs) and MUSIC at A = 360, M = 8.
Each case is timed with CUDA events over --iters calls after --warmup calls.

The fp64 rate of ML is computed from the operation count of the kernel's inner loop: per
(direction, frame, bin) cell 4 M DFMA for s^H x, 2 for |.|^2, 1 for the (1 + eps) scaling,
1 subtraction and 1 masked accumulate = 4 M + 5 fp64 FMA-pipe operations, plus one fp64 log
(not counted).  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from setk_b200 import _lib, plan  # noqa: E402

B, N_SAMPLES, SR = 64, 160000, 16000


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def steering(A, M, F, circular):
    """Geometry steering vectors A x M x F: a 4-mic linear array (4 cm) or a 7-mic circular one."""
    omega = np.pi * np.arange(F) * SR / (F - 1)
    doas = np.linspace(0, 180, A) if not circular else np.arange(A) * 360 / A
    if not circular:
        dist = np.cos(doas[:, None] * np.pi / 180) * (np.arange(M) * 0.04)[None]
    else:
        ang = np.arange(M - 1) * 2 * np.pi / (M - 1)
        dist = -np.concatenate([np.zeros((A, 1)), np.cos(ang[None] - doas[:, None] * np.pi / 180) * 0.05], 1)
    return np.exp(-1j * omega[None, None, :] * dist[:, :, None] / 343.0)


def time_call(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[1])
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--iters", type=int, default=50)
    args = p.parse_args()
    if args.iters < 50:
        raise SystemExit("--iters must be at least 50")
    dev = torch.device("cuda:0")
    _lib.use_library(_lib.DEFAULT_LIBRARY)
    gen = torch.Generator(device=dev).manual_seed(1234)
    result = {"workload": f"B={B} x 10 s @ 16 kHz, STFT 512/256 (T=626, F=257), one TF-mask per utterance",
              "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
              "iters": args.iters, "warmup": args.warmup, "cases": {}}
    stft = {}
    for M in (4, 8):
        sp = plan.StftPlan(M, 512, 256, max_batch=B, max_samples=N_SAMPLES, device=dev)
        audio = torch.randn((B, M, N_SAMPLES), generator=gen, device=dev) * 0.1
        stft[M] = sp.stft(audio)
    T, F = stft[4].shape[-1], stft[4].shape[-2]
    mask = torch.rand((B, 1, T, F), generator=gen, device=dev)
    cases = [("ml", 181, 4), ("ml", 360, 4), ("ml", 181, 8), ("ml", 360, 8), ("srp", 360, 8), ("music", 360, 8)]
    for backend, A, M in cases:
        sv = torch.from_numpy(steering(A, M, F, circular=M == 8)).to(dev)
        kw = dict(compression=-1, eps=float(np.finfo(np.float32).eps)) if backend == "ml" else {}
        if backend == "srp":
            kw["pairs"] = [(i, i + 1) for i in range(M - 1)]
        ms = time_call(lambda: plan.ssl(stft[M], sv, backend=backend, mask=mask, **kw), args.warmup, args.iters)
        entry = {"ms_per_batch": round(ms, 3), "utt_per_s": round(B / ms * 1e3, 1)}
        if backend == "ml":
            ops = (4 * M + 5) * A * T * F * B
            entry["fp64_fma_pipe_tflops"] = round(2 * ops / (ms * 1e-3) / 1e12, 2)
        result["cases"][f"{backend}_A{A}_M{M}"] = entry
    result["h100_sxm_fp64_peak_tflops"] = 67.0 / 2     # data sheet: 67 TF fp64 tensor core, 34 TF fp64 FMA pipe
    result["reference_on_host"] = "not measured"
    print(json.dumps(result))


if __name__ == "__main__":
    main()
