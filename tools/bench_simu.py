"""
tools/bench_simu.py -- throughput of mixture simulation (setk_convolve + setk_simulate_mix) on the
README's far-field workload, one JSON line.

Workload: 256 seeded mixtures, each 2 speakers of 4-13 s of seeded synthetic signal at 16 kHz through
4-microphone 0.5 s RIRs made by plan.rir_image in seeded rooms, one point noise through its own RIR and
a 4-channel isotropic noise (channel 0 added), speaker 1 starting at 2 s.  The inputs live on the device
(the in-memory path a data loader takes); the timed region is simu.simulate's device work for all 256
mixtures, from CUDA events after a warm-up, outputs float32.

Reported: mixtures/s and seconds of mixture audio/s; the convolution kernels' time (CUDA events around
the setk_convolve calls alone), their FLOP/s from shapes (real products of an overlap-save with 2P-point
complex FFTs) against the FP32 data-sheet rate, and the bytes of images written and read by the mixing
against the HBM3 bandwidth; the card and its power limit, read in the same run; and a CPU line: the
float64 oracle's float32 scipy path on one host core for 4 of the mixtures.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from setk_b200 import _lib, plan, simu  # noqa: E402
from setk_b200.simu import Conv, Mixture, Term  # noqa: E402

FP32_TFLOPS, HBM_TBS = 67.0, 3.35   # H100 SXM data sheet (700 W)


def workload(n, device, seed=0):
    rng = np.random.default_rng(seed)
    rooms = rng.uniform([4, 4, 2.5], [8, 7, 3.2], (n, 3))
    beta = np.stack([plan.rir_beta(r, rng.uniform(0.3, 0.6), 343) for r in rooms])
    src = rooms[:, None, :] * rng.uniform(0.2, 0.8, (n, 3, 3))
    mic_c = rooms * rng.uniform(0.3, 0.7, (n, 3))
    rcv = mic_c[:, None, :] + np.array([[0, 0, 0], [0.05, 0, 0], [0.1, 0, 0], [0.15, 0, 0]])[None]
    rirs = []
    for s in range(3):
        rirs.append(plan.rir_image(rooms, beta, src[:, s], rcv, 8000, sr=16000, c=343, device=device))
    out = []
    for i in range(n):
        S = [int(rng.integers(4 * 16000, 13 * 16000)) for _ in range(2)]
        beg = [32000, 0]
        T = max(b + s for b, s in zip(beg, S))
        m = Mixture(f"m{i}", T, 4, 0.9)
        for k in range(2):
            x = torch.from_numpy((0.3 * np.sin(np.arange(S[k]) * (0.02 + 0.01 * k)) *
                                  rng.uniform(0.3, 1, S[k])).astype(np.float32)).to(device)
            m.terms.append(Term(_lib.SIMU_SPEAKER, Conv(x, rirs[k][i], S[k]), beg[k], S[k], 0, (0, S[k]),
                                3.0 * k))
        nz = torch.from_numpy((0.1 * rng.standard_normal(T)).astype(np.float32)).to(device)
        m.terms.append(Term(_lib.SIMU_POINT_NOISE, Conv(nz, rirs[2][i], T), 0, T, 0, (0, T), 5.0))
        iso = torch.from_numpy((0.05 * rng.standard_normal((1, T))).astype(np.float32)).to(device)
        m.terms.append(Term(_lib.SIMU_ISOTROPIC, iso, 0, T, 0, (0, T), 8.0))
        out.append(m)
    return out


def conv_flops(mixtures, P=1024):
    """real flops of the overlap-save: forward FFTs of source blocks and filter partitions, the
    spectral products, the inverse FFTs (5 N log2 N per complex FFT of N = 2P)"""
    N = 2 * P
    fft = 5 * N * np.log2(N)
    total = 0.0
    for m in mixtures:
        for t in m.terms:
            if isinstance(t.image, Conv):
                M, L = t.image.h.shape
                blocks, parts = -(-t.image.n_out // P), -(-L // P)
                total += blocks * fft + M * parts * fft + M * blocks * (fft + 8 * (P + 1) * min(parts, blocks))
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mixtures", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_simu.py needs a CUDA device"
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    mixtures = workload(args.mixtures, dev)
    simu.simulate(mixtures[:8], device=dev)   # warm-up
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(args.reps):
        ev0.record()
        simu.simulate(mixtures, device=dev)
        ev1.record()
        torch.cuda.synchronize()
        times.append(ev0.elapsed_time(ev1) / 1e3)
    t = min(times)
    audio_s = sum(m.n_samples for m in mixtures) / 16000.0
    # the convolutions alone: one call per problem kind, as simulate groups them (all M = 4)
    convs = [t_.image for m in mixtures for t_ in m.terms if isinstance(t_.image, Conv)]
    Sx, Lh, Ny = max(c.x.shape[-1] for c in convs), 8000, max(c.n_out for c in convs)
    x = torch.zeros((len(convs), Sx), device=dev)
    h = torch.zeros((len(convs), 4, Lh), device=dev)
    for i, c in enumerate(convs):
        x[i, :c.x.shape[-1]] = c.x
        h[i] = c.h
    kw = dict(n_out=[c.n_out for c in convs], s_len=[c.x.shape[-1] for c in convs])
    y = torch.empty((len(convs), 4, Ny), device=dev)
    plan.convolve(x, h, out=y, **kw)
    ev0.record()
    for _ in range(args.reps):
        plan.convolve(x, h, out=y, **kw)
    ev1.record()
    torch.cuda.synchronize()
    t_conv = ev0.elapsed_time(ev1) / 1e3 / args.reps
    flops = conv_flops(mixtures)
    img_bytes = 4 * sum(c.n_out * 4 for c in convs) * 2 + 4 * sum(m.n_samples * 2 for m in mixtures)
    out_bytes = 4 * sum(m.n_samples * (4 + 2 + 1) for m in mixtures)
    # CPU line: the oracle's float32 scipy path, one core, 4 mixtures
    import scipy.signal as ss
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    t0 = time.perf_counter()
    for m in mixtures[:4]:
        for t_ in m.terms:
            if isinstance(t_.image, Conv):
                ss.convolve(t_.image.x.cpu().numpy()[None], t_.image.h.cpu().numpy())
    cpu_s = (time.perf_counter() - t0) / 4
    print(json.dumps({
        "bench": "simu", "card": q, "mixtures": len(mixtures), "audio_seconds": round(audio_s, 1),
        "gpu_seconds": round(t, 4), "mixtures_per_s": round(len(mixtures) / t, 1),
        "audio_seconds_per_s": round(audio_s / t, 1),
        "conv_seconds": round(t_conv, 4), "conv_tflops": round(flops / t_conv / 1e12, 2),
        "conv_share_of_fp32_peak": round(flops / t_conv / 1e12 / FP32_TFLOPS, 3),
        "mix_image_bytes": img_bytes + out_bytes,
        "mix_bound_by_hbm_s": round((img_bytes + out_bytes) / (HBM_TBS * 1e12), 5),
        "cpu_label": "CPU: scipy float32 convolutions only, one host core, per mixture",
        "cpu_seconds_per_mixture": round(cpu_s, 4),
    }))


if __name__ == "__main__":
    main()
