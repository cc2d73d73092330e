"""lightglue_b200 -- an H100-native (sm_90a) implementation of the LightGlue matcher forward path.

``LightGlue`` is a drop-in for ``lightglue.LightGlue`` (cvg/LightGlue): same constructor, same
``forward({"image0": ..., "image1": ...})`` -> output dict; the math runs in hand-written CUDA
kernels behind the C ABI declared in ``include/lightglue_b200.h``.
"""
from .disk import DISK  # noqa: F401
from .dog_hardnet import DoGHardNet  # noqa: F401
from .matcher import LightGlue  # noqa: F401
from .nn_matcher import NearestNeighborMatcher  # noqa: F401
from .sift import SIFT  # noqa: F401

__all__ = ["DISK", "DoGHardNet", "LightGlue", "NearestNeighborMatcher", "SIFT"]
