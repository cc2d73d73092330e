"""Loader of the UNMODIFIED reference ALIKED file (test / measurement infrastructure only).

``make -C oracle -f aliked_ref.mk`` (run by ``__graft_entry__.build()``) copies the reference's ``lightglue/aliked.py``
to ``oracle/_ref/aliked_ref.py`` (git-ignored).
The file imports ``kornia.color.grayscale_to_rgb`` (kornia is not a dependency here), ``.utils.Extractor`` (which
imports kornia and cv2) and downloads its checkpoint in the constructor.  None of that is on the path the fixtures
pin (3-channel images, ``forward``), so this loader provides stand-ins for exactly those three things:
  * a ``kornia.color`` stub whose ``grayscale_to_rgb`` raises (the fixtures feed RGB images);
  * a minimal ``Extractor`` base that only builds ``self.conf`` the way the reference's utils.py does
    (``default_conf`` overridden by the keyword arguments);
  * ``torch.hub.load_state_dict_from_url`` returning the given state_dict, patched only while the model is built.
Everything else that runs is the reference's own code (it needs torch and torchvision).  Used by
oracle/make_golden_aliked.py and tools/aliked_bench.py; nothing under ``lightglue_b200/`` imports it."""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import warnings
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_FILE = os.path.join(HERE, "_ref", "aliked_ref.py")
_mod = None


def available() -> bool:
    if not os.path.exists(REF_FILE):
        return False
    return importlib.util.find_spec("torchvision") is not None


def load():
    """The reference module, or None when the copy (or torchvision) is missing."""
    global _mod
    if _mod is not None or not available():
        return _mod

    def never(*a, **k):
        raise RuntimeError("grayscale_to_rgb is outside the pinned path (RGB inputs only)")

    if "kornia" not in sys.modules:
        kornia = types.ModuleType("kornia")
        color = types.ModuleType("kornia.color")
        color.grayscale_to_rgb = never
        kornia.color = color
        sys.modules["kornia"] = kornia
        sys.modules["kornia.color"] = color

    class Extractor(torch.nn.Module):  # conf = default_conf overridden by kwargs, nothing else
        def __init__(self, **conf):
            super().__init__()
            self.conf = SimpleNamespace(**{**self.default_conf, **conf})

    pkg = types.ModuleType("lg_ref_aliked_pkg")
    pkg.__path__ = []
    utils = types.ModuleType("lg_ref_aliked_pkg.utils")
    utils.Extractor = Extractor
    sys.modules["lg_ref_aliked_pkg"] = pkg
    sys.modules["lg_ref_aliked_pkg.utils"] = utils
    spec = importlib.util.spec_from_file_location("lg_ref_aliked_pkg.aliked", REF_FILE)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["lg_ref_aliked_pkg.aliked"] = mod
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        spec.loader.exec_module(mod)
    _mod = mod
    return mod


def build_model(state_dict, **conf):
    """The reference ``ALIKED(**conf)`` with ``state_dict`` loaded by its own constructor (strict), in eval mode."""
    mod = load()
    if mod is None:
        raise RuntimeError("oracle/_ref/aliked_ref.py or torchvision is missing (run `make -C oracle -f aliked_ref.mk`)")
    orig = torch.hub.load_state_dict_from_url
    torch.hub.load_state_dict_from_url = lambda *a, **k: state_dict
    try:
        return mod.ALIKED(**conf).eval()
    finally:
        torch.hub.load_state_dict_from_url = orig
