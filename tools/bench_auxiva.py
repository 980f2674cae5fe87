#!/usr/bin/env python
"""
tools/bench_auxiva.py -- throughput of AuxIVA blind source separation (setk_auxiva_stft).

Workload: B = 64 utterances of 10 s at 16 kHz, STFT 512 / 256 (T = 626 frames, F = 257 bins),
seeded synthetic audio, 20 epochs (apply_auxiva.py's default), N = 2, 4 and 8 channels (= sources).
Each case is timed with CUDA events over --iters calls after --warmup calls.

Algorithmic traffic and work, from the shapes (auxiva.cuh):
  bytes  every epoch reads X twice (power pass, update pass), the final demix reads X once and
         writes Y (complex128); W and Gr are small beside X and not counted
  fp64   update pass: per (utterance, bin, frame, i <= j) 6 flops for x_i conj(x_j) and 4 N for the
         N weighted sums; power pass: per (utterance, bin, frame) 8 N^2 for y = W^H x and 3 N for
         |y|^2; the final demix 8 N^2; the per-bin solves are O(F N^4) and not counted
The larger of bytes / 3.35 TB/s (HBM3) and flops / 33.5 TFLOP/s (fp64 FMA pipe) is the bound; its
share is that least time over the measured time.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from setk_b200 import _lib, plan  # noqa: E402

B, N_SAMPLES, EPOCHS = 64, 160000, 20
HBM_BPS, FP64_FLOPS = 3.35e12, 33.5e12     # H100 SXM data sheet (700 W)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def cost(N, F, T, epochs):
    x_bytes = 8 * B * N * F * T
    nbytes = (2 * epochs + 1) * x_bytes + 2 * x_bytes
    P = N * (N + 1) // 2
    update = B * F * T * P * (6 + 4 * N)
    demix = B * F * T * (8 * N * N + 3 * N)
    flops = epochs * (update + demix) + B * F * T * 8 * N * N
    return nbytes, flops


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
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--iters", type=int, default=50)
    args = p.parse_args()
    if args.iters < 50:
        raise SystemExit("--iters must be at least 50")
    dev = torch.device("cuda:0")
    _lib.use_library(_lib.DEFAULT_LIBRARY)
    gen = torch.Generator(device=dev).manual_seed(1234)
    result = {"workload": f"B={B} x 10 s @ 16 kHz, STFT 512/256 (T=626, F=257), {EPOCHS} epochs",
              "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
              "iters": args.iters, "warmup": args.warmup, "cases": {}}
    for N in (2, 4, 8):
        sp = plan.StftPlan(N, 512, 256, max_batch=B, max_samples=N_SAMPLES, device=dev)
        audio = torch.randn((B, N, N_SAMPLES), generator=gen, device=dev) * 0.1
        stft = sp.stft(audio)
        F, T = stft.shape[-2], stft.shape[-1]
        ms = time_call(lambda: plan.auxiva_from_stft(stft, num_epochs=EPOCHS), args.warmup, args.iters)
        nbytes, flops = cost(N, F, T, EPOCHS)
        t_mem, t_fp64 = nbytes / HBM_BPS, flops / FP64_FLOPS
        result["cases"][f"N{N}"] = {
            "ms_per_batch": round(ms, 3), "utt_per_s": round(B / ms * 1e3, 1),
            "algorithmic_gbytes": round(nbytes / 1e9, 2), "fp64_gflop": round(flops / 1e9, 2),
            "bound": "hbm" if t_mem >= t_fp64 else "fp64",
            "share_of_bound": round(max(t_mem, t_fp64) / (ms * 1e-3), 3)}
        sp.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
