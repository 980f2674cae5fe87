#!/usr/bin/env python
# coding=utf-8
"""
scripts/sptk/compute_steer_vector.py of funcwj/setk (host numpy: geometry constants, no kernel): the same positional
arguments, flags and defaults; implemented in setk_b200/cli_tools.py (steer_vector_main).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from setk_b200.cli_tools import steer_vector_main  # noqa: E402

if __name__ == "__main__":
    steer_vector_main()
