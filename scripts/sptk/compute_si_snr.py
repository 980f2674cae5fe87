#!/usr/bin/env python
# coding=utf-8
"""
Compute Si-SDR as the evaluation metric

Drop-in for the reference's scripts/sptk/compute_si_snr.py: the same positional arguments, flags
(--spk2class, --per-utt, --utt-ali), defaults, printed report ("Si-SDR(dB) Report:") and file formats.
Kept: one scp runs the single-speaker mode (si_snr of each pair), several the multi-speaker mode
(permute_si_snr with the alignment, first best permutation in itertools order); a length mismatch is
truncated to the first speaker's shorter side; channel 0 of multichannel files in multi-speaker mode;
SpeakersReader's RuntimeError for one scp and permute_si_snr's for a speaker count mismatch; an
utterance's error is raised after the lines of the utterances before it are written.
Added: --batch-size, the utterances per device batch (grouped by length); 0 runs one utterance at a
time, as the reference does.  A thread pool reads the files.
Deviations: fp64 throughout on libsetk_b200's kernels (setk_si_snr), where the reference computes in
float32; a multichannel file in single-speaker mode raises ValueError (the reference's numpy fails on it).
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
from setk_b200.libs.metric import best_mean_permutation, first_failure, si_snr_matrix_batch  # noqa: E402

WINDOW = 1024   # utterances read and scored together before their lines are written


class SpeakersReader(object):

    def __init__(self, scps):
        split_scps = scps.split(",")
        if len(split_scps) == 1:
            raise RuntimeError("Construct SpeakersReader need more "
                               "than one script, got {}".format(scps))
        self.readers = [WaveReader(scp) for scp in split_scps]

    def __len__(self):
        first_reader = self.readers[0]
        return len(first_reader)

    def __getitem__(self, key):
        data = []
        for reader in self.readers:
            wave = reader[key]
            # if multi-channel, choose ch0 as reference
            # we always use ch0 as training targets
            data.append(wave if wave.ndim == 1 else wave[0])
        return data

    def keys(self):
        return list(self.readers[0].index_keys)


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
        print("Si-SDR(dB) Report: ")
        tot_utt = sum([self.cnt[cls_str] for cls_str in self.cnt])
        tot_snr = sum([self.snr[cls_str] for cls_str in self.snr])
        print("Total: {:d}/{:.3f}".format(tot_utt, tot_snr / tot_utt))
        for cls_str in self.snr:
            cls_snr = self.snr[cls_str]
            num_utt = self.cnt[cls_str]
            print("\t{}: {:d}/{:.3f}".format(cls_str, num_utt, cls_snr / num_utt))


def _single(sep_reader, ref_reader):
    def load(key):
        sep, ref = sep_reader[key], ref_reader[key]
        if sep.ndim != 1 or ref.ndim != 1:
            raise ValueError(f"{key}: single-speaker Si-SDR needs single-channel audio, got "
                             f"{sep.shape} and {ref.shape}")
        if sep.size != ref.size:
            end = min(sep.size, ref.size)
            sep, ref = sep[:end], ref[:end]
        return sep[None], ref[None]
    return load


def _multi(sep_reader, ref_reader):
    def load(key):
        sep_list, ref_list = sep_reader[key], ref_reader[key]
        if len(sep_list) != len(ref_list):
            raise RuntimeError("size do not match between xlist " +
                               f"and slist: {len(sep_list)} vs {len(ref_list)}")
        if sep_list[0].size != ref_list[0].size:
            end = min(sep_list[0].size, ref_list[0].size)
            sep_list = [s[:end] for s in sep_list]
            ref_list = [s[:end] for s in ref_list]
        if len({s.shape for s in sep_list + ref_list}) != 1:
            raise ValueError(f"{key}: speakers differ in length after truncation to the first speaker's")
        return np.stack(sep_list), np.stack(ref_list)
    return load


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


def run(args):
    single_speaker = len(args.sep_scp.split(",")) == 1
    reporter = Report(args.spk2class)
    utt_snr = open(args.per_utt, "w") if args.per_utt else None
    utt_ali = open(args.utt_ali, "w") if args.utt_ali else None

    if single_speaker:
        sep_reader = WaveReader(args.sep_scp)
        ref_reader = WaveReader(args.ref_scp)
        keys = list(sep_reader.index_keys)
        load = _single(sep_reader, ref_reader)
    else:
        sep_reader = SpeakersReader(args.sep_scp)
        ref_reader = SpeakersReader(args.ref_scp)
        keys = sep_reader.keys()
        load = _multi(sep_reader, ref_reader)
    with ThreadPoolExecutor(max_workers=8) as pool:
        for w0 in range(0, len(keys), WINDOW):
            window = keys[w0:w0 + WINDOW]
            pairs = list(pool.map(_caught(load), window))
            # the utterances before the first failing one are scored and written, then it raises
            n_ok, err = first_failure(pairs, _check)
            pairs = pairs[:n_ok]
            mats = si_snr_matrix_batch([p[0] for p in pairs], [p[1] for p in pairs], batch_size=args.batch_size)
            for key, m in zip(window, mats):
                if single_speaker:
                    snr = float(m[0, 0])
                    reporter.add(key, snr)
                    if utt_snr:
                        utt_snr.write("{}\t{:.2f}\n".format(key, snr))
                    continue
                snr, ali = best_mean_permutation(m)
                reporter.add(key, snr)
                if utt_snr:
                    utt_snr.write(f"{key}\t{snr:.2f}\n")
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
        description="Command to compute SI-SDR, as metric of the separation quality",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("sep_scp", type=str,
                        help="Separated speech scripts, waiting for measure"
                        "(support multi-speaker, egs: spk1.scp,spk2.scp)")
    parser.add_argument("ref_scp", type=str,
                        help="Reference speech scripts, as ground truth for"
                        " Si-SDR computation")
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
