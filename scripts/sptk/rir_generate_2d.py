#!/usr/bin/env python
"""
Simulate multi-channel RIRs of 2D (e.g. circular) microphone arrays in random rooms (image method)

Drop-in for the reference's scripts/sptk/rir_generate_2d.py: the same positional num_rooms, flags,
defaults, random draws (RoomGenerator, _place_mic, _place_spk and the retry loop over
random.uniform, through libs.sampler.UniformSampler) and outputs:
  <dump-dir>/Room{r}-{i}.wav  the M receivers' responses, PCM-16 through write_wav, as the
                              reference's pyrirgen branch writes them
  <dump-dir>/rir.json         the rooms, receivers and sources, same schema and rounding
Every response is computed on the GPU by setk_rir_image (csrc/rir.cu) from the geometry and T60
rounded as the reference's rir-simulate branch rounds them ({:.3f}, round(beta, 3)), so rir.json
alone reproduces every file.  All rooms are drawn first; then every (room, source) pair goes to the
device in batches bounded by a memory budget, and the files are written.

--gpu is accepted and has no effect: every path runs on the GPU.  gpuRIR's different algorithm
(Sabine-estimated beta, lookup tables, image-count truncation) is not reproduced.

Implemented in setk_b200/rir_cli.py (main("2d")), which lists the deviations from the reference.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from setk_b200.rir_cli import main  # noqa: E402

if __name__ == "__main__":
    main("2d")
