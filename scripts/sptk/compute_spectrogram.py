#!/usr/bin/env python
# coding=utf-8
"""
scripts/sptk/compute_spectrogram.py of funcwj/setk on libsetk_b200's CUDA kernels: the same positional
arguments, flags and defaults, plus --batch-size (utterances per device batch); implemented in
setk_b200/cli_tools.py (spectrogram_main).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from setk_b200.cli_tools import spectrogram_main  # noqa: E402

if __name__ == "__main__":
    spectrogram_main()
