"""Loader of the UNMODIFIED reference DoG-HardNet file (test infrastructure only).

``make -C oracle -f doghardnet_ref.mk`` (run by ``__graft_entry__.build()``) copies the reference's
``lightglue/dog_hardnet.py`` to ``oracle/_ref/dog_hardnet_ref.py`` (git-ignored).  It is loaded as the ``dog_hardnet``
module of the package ``sift_ref_loader`` builds around the reference ``sift.py`` (so its ``from .sift import SIFT`` is
the reference SIFT with real cv2), with stand-ins for the kornia names it imports: ``kornia.color.rgb_to_grayscale``
(sift_ref_loader's) and ``kornia.feature.HardNet`` / ``LAFDescriptor`` / ``laf_from_center_scale_ori`` (those of
oracle/doghardnet_oracle.py)."""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import warnings

from . import doghardnet_oracle as dho
from . import sift_ref_loader

HERE = os.path.dirname(os.path.abspath(__file__))
REF_FILE = os.path.join(HERE, "_ref", "dog_hardnet_ref.py")
_mod = None


def available() -> bool:
    return os.path.exists(REF_FILE) and sift_ref_loader.available()


def load():
    """The reference module, or None when a copy (or cv2) is missing."""
    global _mod
    if _mod is not None or not available():
        return _mod
    sift_ref_loader.load()
    feature = sys.modules.get("kornia.feature") or types.ModuleType("kornia.feature")
    feature.HardNet = dho.HardNet
    feature.LAFDescriptor = dho.LAFDescriptor
    feature.laf_from_center_scale_ori = dho.laf_from_center_scale_ori
    sys.modules["kornia"].feature = feature
    sys.modules["kornia.feature"] = feature
    spec = importlib.util.spec_from_file_location("lg_ref_sift_pkg.dog_hardnet", REF_FILE)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["lg_ref_sift_pkg.dog_hardnet"] = mod
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        spec.loader.exec_module(mod)
    _mod = mod
    return mod


def build_model(sd: dict, **conf):
    """The reference ``DoGHardNet(**conf)`` whose ``HardNet(True)`` holds the state_dict ``sd``."""
    mod = load()
    if mod is None:
        raise RuntimeError("oracle/_ref/dog_hardnet_ref.py, oracle/_ref/sift_ref.py or cv2 is missing")
    dho.HardNet.state_dict_source = sd
    return mod.DoGHardNet(**conf).eval()
