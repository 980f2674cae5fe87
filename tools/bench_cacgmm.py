#!/usr/bin/env python
"""
tools/bench_cacgmm.py -- CACGMM mask estimation on the GPU: 64 utterances of 10 s at 16 kHz per batch,
C = 4 and 7 channels, K = 2, 3 and 4 classes, 20 and 50 EM iterations, n_fft 512 / hop 256, random
start, the reference's permutation alignment.  Prints one JSON line per configuration and a summary
line with the card's name and power limit, read in the same run.

Every time comes from CUDA events around whole setk_cacgmm_masks calls (median of --reps after
--warmup):
  utt_per_s       utterances per second, alignment included
  em_iter_ms      one EM iteration over the batch (covariance + factor + E-step): the difference of
                  the 50- and 20-iteration calls over 30
  fixed_ms        the rest of a call without alignment: tile STFT, start, export
  align_ms        the aligner: the call with alignment minus the call without
  align_share     align_ms over the whole call with alignment
The sizes are a user's batch: 10 s utterances are the reference's doc-command scale, and 64 of them
fill the 132 SMs in every pass.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from setk_b200 import _lib  # noqa: E402
from setk_b200 import plan as P  # noqa: E402


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cacgmm.py measures the GPU: no CUDA device")
    _lib.use_library(_lib.DEFAULT_LIBRARY)
    import parity_cases as pc
    dev = torch.device("cuda:0")
    B, N = args.utts, int(16000 * args.seconds)
    rng = np.random.default_rng(0)
    for C in (4, 7):
        x = torch.from_numpy(pc.structured_audio(rng, B, C, N)).to(dev)
        pl = P.StftPlan(C, 512, 256, True, True, "hann", B, N, dev)
        T, F = pl.num_frames(N), pl.num_bins
        for K in (2, 3, 4):
            g = torch.rand((B, K, T, F), dtype=torch.float64, device=dev, generator=torch.Generator(dev).manual_seed(K))
            g /= g.sum(1, keepdim=True)

            def call(iters, permu):
                return lambda: pl.cacgmm_masks(x, K, iters, init_gamma=g, permu_plan=P.PERMU_PLANS[F] if permu else None)

            t = {(it, pm): timed(call(it, pm), args.warmup, args.reps) for it in (20, 50) for pm in (False, True)}
            it_ms = (t[(50, False)] - t[(20, False)]) / 30
            for it in (20, 50):
                align = t[(it, True)] - t[(it, False)]
                print(json.dumps(dict(C=C, K=K, iters=it, B=B, seconds=args.seconds, T=T, F=F,
                                      call_ms=round(t[(it, True)], 3), utt_per_s=round(B / t[(it, True)] * 1e3, 1),
                                      em_iter_ms=round(it_ms, 4), fixed_ms=round(t[(it, False)] - it * it_ms, 3),
                                      align_ms=round(align, 3), align_share=round(align / t[(it, True)], 4))),
                      flush=True)
        pl.close()
        del x
    print(json.dumps({"card": card()}))


if __name__ == "__main__":
    main()
