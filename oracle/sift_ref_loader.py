"""Loader of the UNMODIFIED reference SIFT file (test / measurement infrastructure only).

``make -C oracle -f sift_ref.mk`` (run by ``__graft_entry__.build()``) copies the reference's ``lightglue/sift.py`` to
``oracle/_ref/sift_ref.py`` (git-ignored).  The file imports ``kornia.color.rgb_to_grayscale`` (kornia is not a
dependency here) and ``.utils.Extractor`` (which imports kornia).  This loader provides stand-ins for exactly those:
  * ``kornia.color.rgb_to_grayscale`` with kornia's formula, ``0.299 r + 0.587 g + 0.114 b`` in fp32, in that order;
  * a minimal ``Extractor`` base that only builds ``self.conf`` the way the reference's utils.py does
    (``default_conf`` overridden by the keyword arguments).
``cv2`` and ``packaging`` are the real ones.  Used by oracle/make_golden_sift.py, tests/test_sift_oracle_golden.py and
tools/sift_bench.py; nothing under ``lightglue_b200/`` imports it."""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import warnings
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_FILE = os.path.join(HERE, "_ref", "sift_ref.py")
_mod = None


def available() -> bool:
    if not os.path.exists(REF_FILE):
        return False
    return all(importlib.util.find_spec(m) is not None for m in ("cv2", "packaging"))


def rgb_to_grayscale(image: torch.Tensor) -> torch.Tensor:
    """kornia.color.rgb_to_grayscale with its default weights."""
    w = torch.tensor([0.299, 0.587, 0.114], dtype=image.dtype, device=image.device)
    r, g, b = image[..., 0:1, :, :], image[..., 1:2, :, :], image[..., 2:3, :, :]
    return w[0] * r + w[1] * g + w[2] * b


def load():
    """The reference module, or None when the copy (or cv2) is missing."""
    global _mod
    if _mod is not None or not available():
        return _mod
    kornia = sys.modules.get("kornia") or types.ModuleType("kornia")
    color = sys.modules.get("kornia.color") or types.ModuleType("kornia.color")
    color.rgb_to_grayscale = rgb_to_grayscale
    kornia.color = color
    sys.modules["kornia"] = kornia
    sys.modules["kornia.color"] = color

    class Extractor(torch.nn.Module):  # conf = default_conf overridden by kwargs, nothing else
        def __init__(self, **conf):
            super().__init__()
            self.conf = SimpleNamespace(**{**self.default_conf, **conf})

    pkg = types.ModuleType("lg_ref_sift_pkg")
    pkg.__path__ = []
    utils = types.ModuleType("lg_ref_sift_pkg.utils")
    utils.Extractor = Extractor
    sys.modules["lg_ref_sift_pkg"] = pkg
    sys.modules["lg_ref_sift_pkg.utils"] = utils
    spec = importlib.util.spec_from_file_location("lg_ref_sift_pkg.sift", REF_FILE)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["lg_ref_sift_pkg.sift"] = mod
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        spec.loader.exec_module(mod)
    _mod = mod
    return mod


def build_model(**conf):
    """The reference ``SIFT(**conf)`` (backend opencv)."""
    mod = load()
    if mod is None:
        raise RuntimeError("oracle/_ref/sift_ref.py or cv2 is missing (run `make -C oracle -f sift_ref.mk`)")
    return mod.SIFT(**conf).eval()
