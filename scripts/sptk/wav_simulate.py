#!/usr/bin/env python
"""
Command to do audio data simulation: speakers through RIRs, point-source and isotropic noises, mixed
and normalised.

Drop-in for the reference's scripts/sptk/wav_simulate.py: the same positional mix, flags, defaults,
output paths (mix, and <dump-ref-dir>/{noise,clean,spk{i}}/<basename of mix>, PCM-16), the
"Time cost ... RTF = ..." line and the reference's RuntimeErrors.  The long convolutions run through
setk_convolve and the mixing and normalisation through setk_simulate_mix (csrc/simu.cu); the host
restatement of run_simu's bookkeeping is setk_b200.simu.plan_mixture.

One added flag, --batch LIST: every non-empty line of LIST holds the arguments of one invocation (the
flags and the output path, split with shlex and parsed by this parser).  A thread pool reads the files
and all lines go through the device in batches; each RTF line then reports the batch's time shared
evenly among its mixtures.  A mixture gives the same files alone and inside a batch.

Kept quirks of the reference (see setk_b200/simu.py):
  * mix_nsamps = max(begin + source.size): a multichannel source's size counts all its channels;
  * the point-noise mixing loop uses the last noise's duration for every noise; where numpy's
    broadcast fails there, ValueError names the mixture;
  * only channel 0 of the isotropic noise is added, to every channel, though the file must have the
    mixture's channel count;
  * --point-noise-offset is split on whitespace, so it takes one offset, and it limits how many noise
    files are read;
  * --point-noise-repeat pads with numpy's wrap mode;
  * every power is taken on channel 0.
Deviations: the mixture is computed in fp64 from float32 images (the reference mixes float32 images
in float64 too, but takes its powers and speaker coefficients in float32), and with an isotropic noise
but no point noise the noise reference is written as the isotropic noise's channel-0 track, where the
reference fails writing a scalar.  --sr other than the files' rate raises as read_wav does.
"""
import argparse
import os
import shlex
import sys
import time
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from setk_b200 import simu  # noqa: E402
from setk_b200.libs.opts import strtobool  # noqa: E402
from setk_b200.libs.utils import write_wav  # noqa: E402


def make_parser():
    parser = argparse.ArgumentParser(description="Command to do audio data simulation",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("mix", type=str, help="Audio to output")
    parser.add_argument("--dump-ref-dir", type=str, default="", help="Directory of the reference audio to output")
    parser.add_argument("--src-spk", type=str, required=True, help="Source speakers, e.g., spk1.wav,spk2.wav")
    parser.add_argument("--src-rir", type=str, default="", help="RIRs for each source speakers")
    parser.add_argument("--src-sdr", type=str, default="", help="SDR for each speakers (if needed)")
    parser.add_argument("--src-begin", type=str, default="", help="Begining samples on the mixture utterances")
    parser.add_argument("--point-noise", type=str, default="", help="Add pointsource noises")
    parser.add_argument("--point-noise-rir", type=str, default="", help="RIRs of the pointsource noises (if needed)")
    parser.add_argument("--point-noise-snr", type=str, default="", help="SNR of the pointsource noises")
    parser.add_argument("--point-noise-begin", type=str, default="",
                        help="Begining samples of the pointsource noises on the mixture utterances (if needed)")
    parser.add_argument("--point-noise-offset", type=str, default="",
                        help="Add from the offset position of the pointsource noise")
    parser.add_argument("--point-noise-repeat", type=strtobool, default="false",
                        help="Repeat the pointsource noise or not")
    parser.add_argument("--isotropic-noise", type=str, default="", help="Add isotropic noises")
    parser.add_argument("--isotropic-noise-snr", type=str, default="", help="SNR of the isotropic noises")
    parser.add_argument("--isotropic-noise-offset", type=int, default=0,
                        help="Add noise from the offset position of the isotropic noise")
    parser.add_argument("--dump-channel", type=int, default=-1, help="Index of the channel to dump out (-1 means all)")
    parser.add_argument("--norm-factor", type=float, default=0.9, help="Normalization factor of the final output")
    parser.add_argument("--sr", type=int, default=16000, help="Value of the sample rate")
    return parser


def run_many(arg_list, workers=8):
    """plans every invocation (files read by a thread pool), simulates them in device batches, writes
    the files and prints one RTF line per mixture"""
    with ThreadPoolExecutor(max_workers=workers) as pool:
        plans = list(pool.map(simu.plan_mixture, arg_list))
    done = 0
    for group in simu.batches(plans):
        start = time.time()
        results = simu.simulate(group, pcm16=True, budget=float("inf"))
        share = (time.time() - start) / len(group)
        for m, r in zip(group, results):
            args = arg_list[done]
            done += 1
            utt_dur = m.n_samples / float(args.sr)
            print(f"Time cost: {share:.4f}s, Utterance duration: {utt_dur:.2f}s, RTF = {share / utt_dur:.4f}",
                  flush=True)
            simu.write_outputs(m, r, args.dump_ref_dir, args.sr, write_wav)


def run(args):
    start = time.time()
    m = simu.plan_mixture(args)
    result = simu.simulate([m], pcm16=True)[0]
    utt_dur = m.n_samples / float(args.sr)
    time_cost = float(time.time() - start)
    print(f"Time cost: {time_cost:.4f}s, Utterance duration: {utt_dur:.2f}s, RTF = {time_cost / utt_dur:.4f}",
          flush=True)
    simu.write_outputs(m, result, args.dump_ref_dir, args.sr, write_wav)


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--batch", type=str, default="")
    known, rest = pre.parse_known_args(argv)
    parser = make_parser()
    parser.add_argument("--batch", type=str, default="",
                        help="File of invocations, one per line (flags and output path), run in device batches")
    if not known.batch:
        run(parser.parse_args(argv))
        return
    if rest:
        parser.error(f"--batch takes no other arguments (got {' '.join(rest)})")
    with open(known.batch) as f:
        lines = [ln for ln in f.read().splitlines() if ln.strip()]
    run_many([make_parser().parse_args(shlex.split(ln)) for ln in lines])


if __name__ == "__main__":
    main()
