"""Host-side contract of the ALIKED extractor (include/aliked_b200.h, lightglue_b200/aliked.py); no GPU needed."""
import ctypes as C
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.aliked import ALIKED
from oracle import aliked_synth as als

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "aliked")


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "aliked_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(al_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.AL_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.AL_EXPORTS:
        assert hasattr(lib, s), s


@pytest.mark.parametrize("model_name", sorted(ALIKED.cfgs))
def test_blob_size_is_parameters_plus_bn_statistics(model_name):
    m = ALIKED(model_name=model_name, weights=None)
    n_param = sum(p.numel() for p in m.parameters())
    n_stats = sum(b.numel() for k, b in m.named_buffers() if k.endswith(("running_mean", "running_var")))
    cfg = m._config()
    assert _cabi.load().al_weight_blob_floats(C.byref(cfg)) == n_param + n_stats == m._blob().numel()


@pytest.mark.parametrize("model_name", sorted(ALIKED.cfgs))
def test_state_dict_keys_equal_the_reference(model_name):
    fixtures = {"aliked-t16": "al_t16", "aliked-n32": "al_n32"}
    fix = torch.load(os.path.join(GOLDEN, fixtures.get(model_name, "al_240x320") + ".pt"), weights_only=False)
    ref = [(k, tuple(s)) for k, s in fix["state_dict_layout"]]
    if model_name in fixtures:
        ours = [(k, tuple(v.shape)) for k, v in ALIKED(model_name=model_name, weights=None).state_dict().items()]
        assert ours == ref
    else:  # aliked-n16 / n16rot share the fixture's (n16) layout
        assert [k for k, _ in ALIKED(model_name=model_name, weights=None).state_dict().items()] == [k for k, _ in ref]
    # the synthetic weights load strictly
    ALIKED(model_name=model_name, weights=None).load_state_dict(als.make_aliked_state_dict(model_name), strict=True)


def test_cpu_tensor_raises():
    m = ALIKED(weights=None)
    with pytest.raises(RuntimeError):
        m({"image": torch.rand(1, 3, 32, 32)})


def test_missing_weights_raise(tmp_path, monkeypatch):
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError):
        ALIKED(model_name="aliked-n16")


def test_weights_found_in_weights_dir(tmp_path, monkeypatch):
    torch.save(als.make_aliked_state_dict("aliked-t16"), tmp_path / "aliked-t16.pth")
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    m = ALIKED(model_name="aliked-t16")
    assert torch.equal(m.desc_head.agg_weights, als.make_aliked_state_dict("aliked-t16")["desc_head.agg_weights"])


def test_unknown_model_name_raises():
    with pytest.raises(ValueError):
        ALIKED(model_name="aliked-x99", weights=None)
