#!/usr/bin/env python
# coding=utf-8
"""
Command to eval speech separation (SDR), BSS-Eval v3 as mir_eval.separation.bss_eval_sources defines it

Drop-in for the reference's scripts/sptk/compute_sdr.py: the same positional arguments (comma-separated
scps of the separated and the reference speakers), flags (--spk2class, --per-utt, --utt-ali), defaults,
printed report ("SDR(dB) Report:", "Total: n/mean", one line per class) and file formats
(--per-utt "key\\t{:.2f}" of the mean SDR of the chosen permutation, --utt-ali the permutation).
Kept: channel 0 of a multichannel file; both sides truncated to the shorter one; mir_eval's permutation
(the best mean SIR, first in itertools order) and its ValueErrors (silent sources, shape mismatch),
raised after the lines of the utterances before the failing one are written, as in the reference.
Added: --batch-size, the utterances per device batch (grouped by length); 0 runs one utterance at a
time, as the reference does.  A thread pool reads the files.  mir_eval is not needed.
Deviations: the scores are computed in fp64 on libsetk_b200's kernels (setk_bss_eval), with direct
correlations in place of mir_eval's FFTs; where references are linearly dependent (one a delayed copy
of another), numpy.linalg.solve is ill-posed in mir_eval and here the least-squares projection is used.
"""
import argparse
import os
import sys
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from setk_b200.libs.data_handler import ScpReader, WaveReader  # noqa: E402
from setk_b200.libs.metric import bss_eval_sources_batch, first_failure, validate  # noqa: E402

WINDOW = 1024   # utterances read and scored together before their lines are written


class AudioReader(object):

    def __init__(self, spks_scp):
        self.wav_reader = [WaveReader(scp) for scp in spks_scp.split(",")]

    def __len__(self):
        return len(self.wav_reader[0])

    def __getitem__(self, key):
        data = []
        for reader in self.wav_reader:
            wave = reader[key]
            data.append(wave if wave.ndim == 1 else wave[0])
        return np.stack(data, axis=0)

    def keys(self):
        return list(self.wav_reader[0].index_keys)


class Report(object):

    def __init__(self, spk2class=None):
        self.s2c = ScpReader(spk2class) if spk2class else None
        self.snr = defaultdict(float)
        self.cnt = defaultdict(int)

    def add(self, key, val):
        cls_str = "NG"
        if self.s2c:
            cls_str = self.s2c[key]
        self.snr[cls_str] += val
        self.cnt[cls_str] += 1

    def report(self):
        print("SDR(dB) Report: ")
        tot_utt = sum([self.cnt[cls_str] for cls_str in self.cnt])
        tot_snr = sum([self.snr[cls_str] for cls_str in self.snr])
        print("Total: {:d}/{:.3f}".format(tot_utt, tot_snr / tot_utt))
        for cls_str in self.snr:
            cls_snr = self.snr[cls_str]
            num_utt = self.cnt[cls_str]
            print("\t{}: {:d}/{:.3f}".format(cls_str, num_utt, cls_snr / num_utt))


def _caught(load):
    def run(key):
        try:
            return load(key)
        except Exception as err:  # noqa: BLE001 -- raised in input order by run()
            return err
    return run


def _check(pair):
    if isinstance(pair, Exception):
        raise pair
    validate(*pair)


def run(args):
    sep_reader = AudioReader(args.sep_scp)
    ref_reader = AudioReader(args.ref_scp)
    utt_snr = open(args.per_utt, "w") if args.per_utt else None
    utt_ali = open(args.utt_ali, "w") if args.utt_ali else None
    reporter = Report(args.spk2class)

    def load(key):
        sep, ref = sep_reader[key], ref_reader[key]
        nsamps = min(sep.shape[-1], ref.shape[-1])
        return ref[:, :nsamps], sep[:, :nsamps]

    keys = sep_reader.keys()
    with ThreadPoolExecutor(max_workers=8) as pool:
        for w0 in range(0, len(keys), WINDOW):
            window = keys[w0:w0 + WINDOW]
            pairs = list(pool.map(_caught(load), window))
            # the utterances before the first failing one are scored and written, then it raises
            n_ok, err = first_failure(pairs, _check)
            pairs = pairs[:n_ok]
            scores = bss_eval_sources_batch([p[0] for p in pairs], [p[1] for p in pairs],
                                            batch_size=args.batch_size)
            for key, (sdr, _, _, ali) in zip(window, scores):
                sdr = np.mean(sdr)
                reporter.add(key, sdr)
                if utt_snr:
                    utt_snr.write("{}\t{:.2f}\n".format(key, sdr))
                if utt_ali:
                    ali_str = " ".join(map(str, ali))
                    utt_ali.write(f"{key}\t{ali_str}\n")
            if err is not None:
                for f in (utt_snr, utt_ali):
                    if f:
                        f.close()
                raise err
    reporter.report()
    if utt_snr:
        utt_snr.close()
    if utt_ali:
        utt_ali.close()


if __name__ == "__main__":
    parser = argparse.ArgumentParser(
        description="Command to eval speech separation (SDR) using "
        "mir_eval (https://github.com/craffel/mir_eval)",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("sep_scp", type=str,
                        help="Separated speech scripts, waiting for measure"
                        "(support multi-speaker, egs: spk1.scp,spk2.scp)")
    parser.add_argument("ref_scp", type=str,
                        help="Reference speech scripts, as ground truth for "
                        "separation evaluation")
    parser.add_argument("--spk2class", type=str, default="",
                        help="If assigned, report results"
                        " per class (gender or degree)")
    parser.add_argument("--per-utt", type=str, default="",
                        help="If assigned, report snr "
                        "improvement for each utterance")
    parser.add_argument("--utt-ali", type=str, default="",
                        help="If assigned, output audio alignments")
    parser.add_argument("--batch-size", type=int, default=32,
                        help="Utterances per device batch (grouped by length); 0 scores one at a time")
    args = parser.parse_args()
    run(args)
