"""
`libs` as seen from scripts/sptk/, like in the reference tree: the modules are
the CUDA-backed mirrors in setk_b200.libs, so `from libs.beamformer import
MvdrBeamformer` or `from libs.utils import forward_stft` keep working for code
written against the reference's scripts/sptk layout.
"""
import importlib
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

for _name in ("utils", "stft", "beamformer", "cluster", "wpe", "spatial", "data_handler", "opts", "sampler", "metric",
              "filters", "exraw"):
    _mod = importlib.import_module("setk_b200.libs." + _name)
    sys.modules[__name__ + "." + _name] = _mod
    globals()[_name] = _mod
