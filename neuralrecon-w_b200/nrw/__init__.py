"""nrw - H100-native per-ray training core for NeuralRecon-W.

Drop-in replacements for the reference's hot-path classes:

    from nrw import NeuconW, NeRF, NeuconWRenderer

keep the constructor signatures, attributes, result dictionary and checkpoint layout of
models/neuconw.py, models/nerf.py and rendering/renderer.py while running the arithmetic in
hand-written sm_90a CUDA (libnrw.so, C ABI in include/nrw.h).  There is no CPU or eager fallback.
"""
from ._lib import NrwError, LIB_PATH  # noqa: F401
from .models import NeRF, NeuconW, RenderingNetwork, SDFNetwork, SingleVarianceNetwork  # noqa: F401
from .renderer import NeuconWRenderer  # noqa: F401
from .engine import Engine  # noqa: F401

__all__ = ["NeuconW", "NeRF", "NeuconWRenderer", "SDFNetwork", "RenderingNetwork", "SingleVarianceNetwork",
           "Engine", "NrwError"]
