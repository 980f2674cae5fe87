#!/usr/bin/env python
# coding=utf-8
"""
scripts/sptk/do_ssl.py of funcwj/setk on libsetk_b200's CUDA kernels (csrc/ssl.cuh): the same positional
arguments, flags and defaults; implemented in setk_b200/cli_tools.py (ssl_main).

Repaired reference bug: in online mode (--chunk-len > 0, --look-back > 0) with --mask-scp, the reference
slices the T x F mask along its FREQUENCY axis (do_ssl.py:106) and fails with a broadcast error; here each
chunk uses the mask's frames of that chunk.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from setk_b200.cli_tools import ssl_main  # noqa: E402

if __name__ == "__main__":
    ssl_main()
