#!/usr/bin/env python
"""
tools/bench_feats.py -- spectral features on the GPU: B utterances of 10 s mono at 16 kHz per batch.
Prints one JSON line per workload, then a summary line with the card's name, power limit and maximum SM
clock, read in the same run.

Workloads (both sides of setk_spectral_feats' route selection):
  spec_512     257-dim log spectrogram, 512 / 256            fused route (n_fft 512)
  fbank_doc    80-bin log fbank, 400 -> 512 / 256            fused route (the doc command)
  fbank_1024   80-bin log fbank, 1024 / 256                  fused route (n_fft 1024)
  fbank_400    80-bin log fbank, 400 / 256, n_fft 400        generic route (STFT in HBM, then the tail)
Per workload:
  kernel_ms    one setk_spectral_feats call on the batch: median of CUDA-event times over --steps warmed calls
  utt_per_s    B / kernel_ms
  gb_per_s     algorithmic bytes (4 N read + 4 T D written per utterance) / kernel_ms, and hbm_share of the
               3.35 TB/s data sheet; fp32_share is the FFT's 5 n log2 n / 2 flops per frame over 67 TFLOP/s
  today_ms     the same features through what a user had before: StftPlan.stft, then torch abs / matmul /
               log; timed alternating with the fused call, outputs compared (today_rel)
  e2e_ms       pinned PCM-16 host buffer -> H2D -> setk_pcm16_to_float -> features -> pinned host features
  cpu_ms_utt   the oracle (numpy, one host core) per utterance, labelled CPU
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

from setk_b200 import _lib  # noqa: E402
from setk_b200 import plan as P  # noqa: E402
from setk_b200.libs.filters import mel  # noqa: E402

WORKLOADS = {
    "spec_512": dict(fl=512, rp2=True, n_mels=None),
    "fbank_doc": dict(fl=400, rp2=True, n_mels=80),
    "fbank_1024": dict(fl=1024, rp2=True, n_mels=80),
    "fbank_400": dict(fl=400, rp2=False, n_mels=80),
}
HBM = 3.35e12
FP32 = 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--hop", type=int, default=256)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_feats.py measures the GPU and needs a CUDA device")
    _lib.use_library(_lib.DEFAULT_LIBRARY)
    dev = torch.device("cuda:0")
    B, N, hop = args.utts, int(args.seconds * 16000), args.hop
    rng = np.random.default_rng(0)
    pcm = torch.from_numpy(rng.integers(-8000, 8000, size=(B, N), dtype=np.int16)).pin_memory()
    x = P.pcm16_to_float(pcm.to(dev)).view(B, 1, N)
    for name in args.workloads.split(","):
        w = WORKLOADS[name]
        pl = P.StftPlan(1, w["fl"], hop, True, w["rp2"], "hann", B, N, dev)
        F, T = pl.num_bins, pl.num_frames(N)
        weights = None
        if w["n_mels"]:
            weights = mel(16000, pl.n_fft, n_mels=w["n_mels"], htk=True)
            pl.set_mel(weights)
        D = w["n_mels"] or F
        kw = dict(mel=bool(w["n_mels"]), apply_log=True)
        fused = lambda: pl.spectral_feats(x, **kw)  # noqa: E731
        wt = torch.from_numpy(weights).to(dev) if weights is not None else None

        def today():
            m = pl.stft(x).abs()[:, 0]                    # B x F x T
            if wt is not None:
                m = torch.matmul(wt, m)
            return torch.log(torch.clamp(m, min=float(P.EPSILON))).transpose(-1, -2)

        for _ in range(args.warmup):
            fused()
            today()
        torch.cuda.synchronize()
        tf, tt = [], []
        for _ in range(args.steps):                       # alternate the two
            tf.append(event_ms(fused))
            tt.append(event_ms(today))
        a, b = fused()[:, 0], today()
        lin_a, lin_b = torch.exp(a), torch.exp(b)
        today_rel = float((lin_a - lin_b).abs().max() / lin_b.abs().max())
        out_h = torch.empty((B, T, D), dtype=torch.float32).pin_memory()

        def e2e():
            xd = P.pcm16_to_float(pcm.to(dev, non_blocking=True)).view(B, 1, N)
            out_h.copy_(pl.spectral_feats(xd, **kw)[:, 0], non_blocking=True)

        for _ in range(args.warmup):
            e2e()
        te = [event_ms(e2e) for _ in range(max(5, args.steps // 5))]
        # oracle on one host core (numpy), a few utterances
        from oracle import feats_oracle as fo
        o = dict(frame_len=w["fl"], frame_hop=hop, round_power_of_two=w["rp2"], window="hann", center=True,
                 apply_log=True, apply_pow=False, normalize=True, sr=16000, num_bins=w["n_mels"] or 0,
                 min_freq=0, max_freq=8000)
        pcm_np = pcm[:4].numpy()
        t0 = time.perf_counter()
        for i in range(4):
            (fo.fbank(pcm_np[i], o) if w["n_mels"] else fo.spectrogram(pcm_np[i], o))
        cpu_ms = (time.perf_counter() - t0) / 4 * 1e3
        k_ms = float(np.median(tf))
        nbytes = B * (4 * N + 4 * T * D)
        flops = B * T * 2.5 * pl.n_fft * np.log2(pl.n_fft)
        route = "fused" if pl.n_fft in (512, 1024) else "generic"
        print(json.dumps(dict(
            workload=name, route=route, B=B, seconds=args.seconds, n_fft=pl.n_fft, hop=hop, D=D,
            kernel_ms=round(k_ms, 3), utt_per_s=round(B / k_ms * 1e3, 1),
            gb_per_s=round(nbytes / k_ms / 1e6, 1), hbm_share=round(nbytes / HBM / (k_ms * 1e-3), 3),
            fp32_share=round(flops / FP32 / (k_ms * 1e-3), 3),
            today_ms=round(float(np.median(tt)), 3), speedup_vs_today=round(float(np.median(tt)) / k_ms, 2),
            today_rel=today_rel, e2e_ms=round(float(np.median(te)), 3),
            e2e_utt_per_s=round(B / float(np.median(te)) * 1e3, 1), cpu_ms_utt_oracle_CPU=round(cpu_ms, 2))),
            flush=True)
        pl.close()
    print(json.dumps(dict(card=card(), torch=torch.__version__)), flush=True)


if __name__ == "__main__":
    main()
