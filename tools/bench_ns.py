#!/usr/bin/env python
"""
tools/bench_ns.py -- throughput of iMCRA / OM-LSA noise suppression (setk_ns_imcra).

Workload: B = 64 and 256 utterances of 10 s at 16 kHz, STFT 512 / 256 (T = 626, F = 257), and B = 64
at 1024 / 256 (F = 513); seeded synthetic noisy speech (a harmonic tone stack under a syllable-rate
envelope plus white noise).  Each case times setk_ns_imcra alone and the chain setk_stft ->
setk_ns_imcra -> setk_istft with CUDA events over --iters calls after --warmup calls.

Bounds, from the shapes:
  bytes  8 B of STFT in, 8 B of enh and 8 B of gain out per (utterance, bin, frame), over 3.35 TB/s
  fp64   FP64_PER_CELL flops per cell, counted from the kernel with E1 on its series branch (26 FMAs,
         a log); cells on the continued-fraction branch cost more and are not counted, so the fp64
         bound is a lower bound.  Over 33.5 TFLOP/s (fp64 FMA pipe, H100 SXM data sheet, 700 W)
The larger of the two is the bound; its share is that least time over the measured time.  The
frame-to-frame chain (one CTA per utterance, T dependent steps) rather than either bound is what
limits the kernel at these sizes: ms_per_frame_step is the kernel time over T.  Prints one JSON line.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from setk_b200 import _lib, plan  # noqa: E402

N_SAMPLES, SR = 160000, 16000
HBM_BPS, FP64_FLOPS = 3.35e12, 33.5e12     # H100 SXM data sheet (700 W)
# per cell: |x|^2 (3), gamma / xi / v / gh1 (~16 + E1 series 2 x 26 + log + exp ~ 40), the three
# 3-tap convolutions (18), minima and indicator (~12), p_hat / lambda / gain (~20 + log + exp ~ 40)
FP64_PER_CELL = 180


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def noisy_speech(B, gen, dev):
    t = torch.arange(N_SAMPLES, device=dev, dtype=torch.float32) / SR
    f0 = 100 + 150 * torch.rand((B, 1), generator=gen, device=dev)
    voiced = sum(torch.sin(2 * math.pi * k * f0 * t) / k for k in range(1, 8))
    env = torch.clamp(torch.sin(2 * math.pi * 4 * t + 6.28 * torch.rand((B, 1), generator=gen, device=dev)), min=0)
    noise = torch.randn((B, N_SAMPLES), generator=gen, device=dev)
    return (0.1 * env * voiced + 0.03 * noise)[:, None, :].contiguous()


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
    p.add_argument("--iters", type=int, default=20)
    args = p.parse_args()
    dev = torch.device("cuda:0")
    _lib.use_library(_lib.DEFAULT_LIBRARY)
    gen = torch.Generator(device=dev).manual_seed(1234)
    result = {"workload": "10 s utterances @ 16 kHz, synthetic noisy speech, default iMCRA",
              "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
              "iters": args.iters, "warmup": args.warmup, "cases": {}}
    for B, frame_len in ((64, 512), (256, 512), (64, 1024)):
        sp = plan.StftPlan(1, frame_len, 256, max_batch=B, max_samples=N_SAMPLES, device=dev)
        audio = noisy_speech(B, gen, dev)
        stft = sp.stft(audio)[:, 0].contiguous()
        F, T = stft.shape[-2], stft.shape[-1]
        ms_ns = time_call(lambda: plan.ns_from_stft(stft), args.warmup, args.iters)

        def chain():
            _, enh = plan.ns_from_stft(sp.stft(audio)[:, 0], gain=False)
            return sp.istft(enh)
        ms_chain = time_call(chain, args.warmup, args.iters)
        cells = B * F * T
        t_mem, t_fp64 = 24 * cells / HBM_BPS, FP64_PER_CELL * cells / FP64_FLOPS
        result["cases"][f"B{B}_nfft{frame_len}"] = {
            "F": F, "T": T, "ns_ms": round(ms_ns, 3), "ns_utt_per_s": round(B / ms_ns * 1e3, 1),
            "ms_per_frame_step": round(ms_ns / T, 5), "chain_ms": round(ms_chain, 3),
            "chain_utt_per_s": round(B / ms_chain * 1e3, 1),
            "bound": "hbm" if t_mem >= t_fp64 else "fp64 (lower bound)",
            "share_of_bound": round(max(t_mem, t_fp64) / (ms_ns * 1e-3), 4)}
        sp.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
