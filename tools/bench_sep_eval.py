"""
tools/bench_sep_eval.py -- throughput of the separation metrics (setk_bss_eval, setk_si_snr), one JSON line.

Workload: for N = 2, 3, 4 sources, B = 64 seeded utterances of 4-10 s at 16 kHz (references of seeded
lowpass noise over a white floor 20 dB down, so that no column of the least-squares system is dependent
as on speech; estimates short FIR filters of them with cross-talk and noise), L = 512, the utterances
on the device; plan.bss_eval runs the 64 in one call.  Timed with CUDA events after a warm-up: the
whole plan.bss_eval call (utt/s), and plan.si_snr.  A torch.profiler pass of its own gives each kernel's time.  The fp64 FMAs of each kernel
come from the shapes: the correlations (N(N+1)/2 (2L-1) + N^2 L) S, the Cholesky (NL)^3/6 + N L^3/6,
the substitutions 2 N ((NL)^2 + N L^2), the FIRs 2 N^2 L (S + L); FLOP/s count an FMA as 2 and are set
against the H100 SXM data sheet's 34 TFLOP/s of non-tensor FP64.  The CPU line is the float64 oracle
(mir_eval's FFT route) on one host core for utterance 0 of each N, scaled to 10 s.  The card's name and power
limit are read in the same run.  Reported with each N: the dropped columns (sum and max over the
batch) and the largest distance of utterance 0's criteria from the oracle's, in dB.
"""
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
os.environ.setdefault("MKL_NUM_THREADS", "1")

import numpy as np  # noqa: E402
import scipy.signal  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import sep_eval_oracle as so  # noqa: E402
from setk_b200 import plan  # noqa: E402

FP64_TFLOPS = 34.0   # H100 SXM data sheet, FP64 without tensor cores (700 W)
SR, B, L = 16000, 64, 512


def workload(N, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(4 * SR, 10 * SR + 1, size=B).astype(np.int32)
    S = int(lens.max())
    bl, al = scipy.signal.butter(4, 0.25)
    refs = np.zeros((B, N, S), np.float32)
    ests = np.zeros((B, N, S), np.float32)
    for b, n in enumerate(lens):
        r = scipy.signal.lfilter(bl, al, rng.standard_normal((N, n)), axis=1) + 0.1 * rng.standard_normal((N, n))
        e = scipy.signal.lfilter([1.0, 0.3, -0.1], [1.0], r, axis=1) + 0.2 * np.roll(r, 1, axis=0)
        refs[b, :, :n] = r
        ests[b, :, :n] = e + 0.05 * rng.standard_normal((N, n))
    return refs, ests, lens


def fmas(N, lens):
    n = N * L
    S = lens.astype(np.float64)
    return {
        "sep_corr_kernel": float(((N * (N + 1) // 2) * (2 * L - 1) + N * N * L) * S.sum()),
        "sep_factor_kernel": float(len(lens) * (n ** 3 / 6 + N * L ** 3 / 6 + 2 * N * (n * n + N * L * L))),
        "sep_score_kernel": float(2 * N * N * L * (S + L).sum()),
    }


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / reps


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.key.startswith("_ZN4setk") or "sep_" in ev.key:
            name = next((k for k in ("sep_corr_kernel", "sep_factor_kernel", "sep_score_kernel", "sep_crit_kernel",
                                     "sep_si_snr_kernel") if k in ev.key), ev.key)
            dev_us = getattr(ev, "device_time_total", None)
            if dev_us is None:
                dev_us = ev.cuda_time_total
            out[name] = out.get(name, 0.0) + dev_us / 1e6
    return out


def main():
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    result = {"metric": "sep_eval", "card": card, "B": B, "L": L, "fp64_tflops_datasheet": FP64_TFLOPS}
    for N in (2, 3, 4):
        refs, ests, lens = workload(N, N)
        r, e = torch.from_numpy(refs).to(dev), torch.from_numpy(ests).to(dev)
        t = timed(lambda: plan.bss_eval(e, r, lens, flen=L), 3)
        ts = timed(lambda: plan.si_snr(e, r, lens), 10)
        kt = kernel_times(lambda: plan.bss_eval(e, r, lens, flen=L))
        crit, dropped, status = plan.bss_eval(e, r, lens, flen=L)
        dropped, crit0 = dropped.cpu().numpy(), crit[0].cpu().numpy()
        work = fmas(N, lens)
        per = {k: {"s": round(v, 6)} for k, v in kt.items()}
        for k, f in work.items():
            if k in per and per[k]["s"] > 0:
                per[k]["tflops"] = round(2 * f / per[k]["s"] / 1e12, 3)
                per[k]["share_of_fp64_peak"] = round(2 * f / per[k]["s"] / 1e12 / FP64_TFLOPS, 4)
        n0 = int(lens[0])
        c0 = time.process_time()
        want = so.criteria(refs[0, :, :n0], ests[0, :, :n0], L)
        cpu = (time.process_time() - c0) * (10 * SR) / n0   # scaled to a 10 s utterance
        result[f"N{N}"] = {"bss_eval_s": round(t, 5), "bss_eval_utt_per_s": round(B / t, 1),
                           "audio_s_per_s": round(float(lens.sum()) / SR / t, 1),
                           "si_snr_utt_per_s": round(B / ts, 1), "kernels": per,
                           "oracle_cpu_s_per_10s_utt": round(cpu, 3),
                           "dropped_columns_sum": int(dropped.sum()), "dropped_columns_max": int(dropped.max()),
                           "status_nonzero": int((status.cpu().numpy() != 0).sum()),
                           "utt0_max_abs_db_vs_oracle": float(np.abs(crit0 - want).max())}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
