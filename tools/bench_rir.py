#!/usr/bin/env python
"""
tools/bench_rir.py -- throughput of setk_rir_image (csrc/rir.cu) on the reference's documented
workload (doc/rir/README.md: rir_generate_1d.py, rooms 4-7 x 4-7 x 2-3 m, T60 0.2-0.5 s, a
4-microphone linear array 0.05 m apart, 0.5 s at 16 kHz, 25 sources per room), seeded.  Prints one
JSON line.

  channels/s, rooms/s  over the timed calls (CUDA events, after warm-up)
  taps/s               taps = images with floor(dist) < L, times Tw, counted on the host from the
                       geometry (every such image writes Tw taps, some dropped past L)
  alu_share            taps/s over an ALU bound: 4 x 32 lanes x SMs x max SM clock instructions per
                       second over INSTR_PER_TAP instructions per tap (stated below: an estimate from
                       the source of the tap loop, not a SASS count)
  cpu_reference_s      when oracle/_ref/rir_ref exists: the reference's C++ generator on one host core
                       for one (room, source) pair, 4 microphones -- a CPU number
"""
import argparse
import json
import math
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from setk_b200 import plan  # noqa: E402

# Instructions per (tap, lane) in the spread loop of rir_image_kernel<4>, estimated from the source:
# window (FFMA x2, FMUL), den (FADD), divide (MUFU.RCP + FFMA refinement), select, range test,
# F2I.S64, shared atomic add with its overflow test (LOP3 x3, ISETP), index (IADD, ISETP x2).
INSTR_PER_TAP = 20
TW = 128
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "rir_ref")


def draw(rooms, sources, seed):
    rnd = random.Random(seed)
    topo = [0, 0.05, 0.1, 0.15]
    out = []
    while len(out) < rooms * sources:
        l, w, h = rnd.uniform(4, 7), rnd.uniform(4, 7), rnd.uniform(2, 3)
        t60 = rnd.uniform(0.2, 0.5)
        room = [round(v, 3) for v in (l, w, h)]
        try:
            beta = plan.rir_beta(room, round(t60, 3), 340)
        except ValueError:
            continue
        mx, my, mz = rnd.uniform(0.4 * l, 0.6 * l), rnd.uniform(0.1 * w, 0.2 * w), rnd.uniform(1.2, 1.8)
        rcv = [[round(mx - 0.075 + x, 3), round(my, 3), round(mz, 3)] for x in topo]
        n = 0
        while n < sources:
            d, doa, sz = rnd.uniform(1.5, 3), rnd.uniform(0, math.pi), rnd.uniform(1, 2)
            sx, sy = mx + math.cos(doa) * d, my + math.sin(doa) * d
            if 0 < sx < l and 0 < sy < w and sz < h:
                out.append((room, beta, [round(sx, 3), round(sy, 3), round(sz, 3)], rcv))
                n += 1
    return out[:rooms * sources]


def images_in_range(room, src, rcv, L, fs=16000, c=340):
    cts = c / fs
    T, S, R = np.asarray(room) / cts, np.asarray(src) / cts, np.asarray(rcv) / cts
    n = [int(math.ceil(L / (2 * t))) for t in T]
    axes = []
    for d in range(3):
        x = np.arange(-n[d], n[d] + 1)
        axes.append(np.concatenate([(S[d] - R[d] + 2 * x * T[d]) ** 2, (-S[d] - R[d] + 2 * x * T[d]) ** 2]))
    d2 = axes[0][:, None, None] + axes[1][None, :, None] + axes[2][None, None, :]
    return int(np.count_nonzero(np.floor(np.sqrt(d2)) < L))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rooms", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    L, sources = 8000, 25
    probs = draw(a.rooms, sources, a.seed)
    dev = torch.device("cuda")
    room, beta, src, rcv = (torch.tensor(np.array([p[k] for p in probs], np.float64), device=dev) for k in range(4))
    B, M = room.shape[0], rcv.shape[1]
    for _ in range(2):
        out = plan.rir_image(room, beta, src, rcv, L, device=dev)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        out = plan.rir_image(room, beta, src, rcv, L, device=dev)
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / a.iters
    taps = TW * sum(images_in_range(p[0], p[2], r, L) for p in probs[:50] for r in p[3]) * (B * M) / (50 * M)
    props = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (s.strip() for s in q[0].split(",")) if q else (props.name, "not measured", "")
    mhz = float(clock.split()[0]) if clock else 1980.0
    alu_taps = 4 * 32 * props.multi_processor_count * mhz * 1e6 / INSTR_PER_TAP
    res = dict(workload=f"{a.rooms} rooms x {sources} sources x {M} mics, {L} samples at 16 kHz",
               problems=B, ms_per_call=round(sec * 1e3, 3), channels_per_s=round(B * M / sec, 1),
               rooms_per_s=round(a.rooms / sec, 2), taps_per_s=float(f"{taps / sec:.4g}"),
               taps_per_channel=float(f"{taps / (B * M):.4g}"), instr_per_tap=INSTR_PER_TAP,
               alu_share=round(taps / sec / alu_taps, 3), gpu=name, power_limit=power, max_sm_clock=clock,
               finite=bool(torch.isfinite(out).all()))
    if os.path.exists(REF_BIN):
        p = probs[0]
        f3 = lambda v: ",".join(f"{x:.6f}" for x in v)  # noqa: E731
        t = time.perf_counter()
        subprocess.run([REF_BIN, "--number-samples=8000", f"--room-topo={f3(p[0])}", f"--beta={f3(p[1])}",
                        f"--source-location={f3(p[2])}",
                        f"--receiver-location={';'.join(f3(r) for r in p[3])}"], check=True, capture_output=True)
        res["cpu_reference_s_per_pair"] = round(time.perf_counter() - t, 2)
        res["cpu_reference_note"] = "reference C++ generator, one host CPU core, 4 mics"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
