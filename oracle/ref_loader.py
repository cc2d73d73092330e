"""Loader of the UNMODIFIED reference matcher (test / bench infrastructure only).

``oracle/Makefile`` copies ``/root/reference/lightglue/lightglue.py`` to ``oracle/_ref/lightglue_ref.py`` in the build
container (git-ignored, travels to the GPU box with the repo snapshot).  The package ``lightglue`` itself cannot be
imported (``__init__`` pulls in kornia, absent here) but this one file only needs torch + numpy (SURVEY.md 8c), so it is
loaded by path.  Used by ``bench.py --impl reference`` (the reference's own CPU path), by the ``reference_gpu`` leg of
the bench (the same file on the same GPU) and by ``oracle/make_golden.py``.  Nothing under ``lightglue_b200/`` imports
this."""
from __future__ import annotations

import importlib.util
import os
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
REF_FILE = os.path.join(HERE, "_ref", "lightglue_ref.py")
_mod = None


def available() -> bool:
    return os.path.exists(REF_FILE)


def load():
    """The reference module (``lightglue/lightglue.py``), or None when the copy is absent."""
    global _mod
    if _mod is None and available():
        spec = importlib.util.spec_from_file_location("lightglue_ref", REF_FILE)
        mod = importlib.util.module_from_spec(spec)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            spec.loader.exec_module(mod)
        _mod = mod
    return _mod


def build_matcher(state_dict, device="cpu", **conf):
    """``LightGlue(features=None, **conf)`` of the reference with ``state_dict`` loaded (reference key names)."""
    mod = load()
    if mod is None:
        raise RuntimeError("oracle/_ref/lightglue_ref.py is missing (run `make -C oracle ref` where /root/reference exists)")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = mod.LightGlue(features=None, **conf)
    missing, unexpected = m.load_state_dict(state_dict, strict=False)
    assert not unexpected, unexpected
    assert all(k == "confidence_thresholds" for k in missing), missing
    return m.eval().to(device)
