"""The nearest-neighbour matcher without a GPU: the header's exports, constants and struct layouts, the argument checks
of the C ABI and of ``NearestNeighborMatcher``, and the workspace size (include/nn_b200.h, lightglue_b200/nn_matcher.py)."""
import ctypes
import os
import re

import pytest
import torch

from lightglue_b200 import NearestNeighborMatcher, _cabi
from lightglue_b200.ragged import split_outputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "nn_b200.h")) as f:
        return f.read()


def _struct_fields(name):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), _header(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [n for decl in body.split(";") for n in re.findall(r"\**(\w+)\s*(?:,|$)", decl.strip())]


def test_header_entry_points_are_the_binding_table_and_exported():
    declared = re.findall(r"LG_API \w+\*? (nn_\w+)\(", _header())
    assert declared == list(_cabi.NN_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.NN_EXPORTS:
        assert getattr(lib, s).argtypes is not None, s


def test_header_constants_match_the_bindings():
    h = _header()
    for name, value in (("NN_ABI_VERSION", _cabi.NN_ABI_VERSION), ("NN_MIN_DIM", _cabi.NN_MIN_DIM),
                        ("NN_MAX_DIM", _cabi.NN_MAX_DIM), ("NN_GROUP_ROWS", _cabi.NN_GROUP_ROWS)):
        m = re.search(rf"#define {name} (\d+)", h)
        assert m and int(m.group(1)) == value, name


def test_struct_layouts_match_the_header():
    for cls in (_cabi.NnConfig, _cabi.NnInputs, _cabi.NnOutputs):
        assert [f for f, _ in cls._fields_] == _struct_fields(cls.__name__), cls.__name__
    assert ctypes.sizeof(_cabi.NnConfig) == 20 and _cabi.NnConfig.ratio_thresh.offset == 12
    assert _cabi.NnInputs.desc0.offset == 16 and ctypes.sizeof(_cabi.NnInputs) == 48
    assert ctypes.sizeof(_cabi.NnOutputs) == 56


def test_output_names_mirror_lightglue():
    lg = [f for f, _ in _cabi.LgOutputs._fields_]
    for f, _ in _cabi.NnOutputs._fields_:
        assert f in lg, f


def test_workspace_is_far_below_the_similarity_matrix_and_grows_with_the_sizes():
    lib = _cabi.load()
    big = lib.nn_workspace_bytes(32, 8192, 8192, 256)
    assert 0 < big < 32 * 8192 * 8192 * 4 // 32
    sizes = [lib.nn_workspace_bytes(32, n, n, 256) for n in (512, 1024, 2048, 4096, 8192)]
    assert sizes == sorted(sizes) and len(set(sizes)) == len(sizes)
    assert lib.nn_workspace_bytes(32, 2048, 2048, 128) < lib.nn_workspace_bytes(32, 2048, 2048, 256)
    assert lib.nn_workspace_bytes(8, 300, 5000, 128) > lib.nn_workspace_bytes(8, 300, 300, 128)


@pytest.mark.parametrize("d", [0, 32, 96, 100, 576, 1024])
def test_workspace_rejects_a_bad_dim(d):
    assert _cabi.load().nn_workspace_bytes(4, 100, 100, d) == 0


def test_nn_match_rejects_bad_arguments_before_any_launch():
    lib = _cabi.load()
    cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 0.8, 0.0)
    ins = _cabi.NnInputs(1, 10, 10, None, None, None, None)
    outs = _cabi.NnOutputs()
    assert lib.nn_match(None, ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None) != 0
    assert b"null" in lib.lg_last_error()
    fake = ctypes.c_void_p(1)  # never dereferenced: every check below fails first
    for bad, what in ((_cabi.NnConfig(_cabi.NN_ABI_VERSION + 1, 128, 1, 0.8, 0.0), b"ABI"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 96, 1, 0.8, 0.0), b"dim"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 1024, 1, 0.8, 0.0), b"dim"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 1.5, 0.0), b"ratio"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 0.8, float("inf")), b"distance")):
        assert lib.nn_match(fake, ctypes.byref(bad), ctypes.byref(ins), ctypes.byref(outs), None, 0, None) != 0
        assert what in lib.lg_last_error(), what
    assert lib.nn_match(fake, ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None) != 0
    assert b"null" in lib.lg_last_error()


def test_default_conf():
    assert NearestNeighborMatcher.default_conf == {"ratio_thresh": None, "distance_thresh": None, "mutual_check": True}
    assert NearestNeighborMatcher().conf == NearestNeighborMatcher.default_conf
    assert NearestNeighborMatcher(ratio_thresh=0.8).conf["ratio_thresh"] == 0.8
    NearestNeighborMatcher(ratio_thresh=1.0, distance_thresh=0.7, mutual_check=False)


@pytest.mark.parametrize("conf", [{"ratio_thresh": 0.0}, {"ratio_thresh": -0.5}, {"ratio_thresh": 1.01},
                                  {"distance_thresh": 0.0}, {"distance_thresh": -1.0},
                                  {"distance_thresh": float("inf")}, {"k": 2}])
def test_bad_conf_is_a_value_error(conf):
    with pytest.raises(ValueError):
        NearestNeighborMatcher(**conf)


def _data(b0, m, d0, b1, n, d1):
    return {"image0": {"descriptors": torch.zeros(b0, m, d0)}, "image1": {"descriptors": torch.zeros(b1, n, d1)}}


@pytest.mark.parametrize("shapes", [(1, 10, 96, 1, 10, 96), (1, 10, 32, 1, 10, 32), (1, 10, 576, 1, 10, 576),
                                    (1, 10, 128, 1, 10, 256), (2, 10, 128, 1, 10, 128)])
def test_bad_descriptors_are_a_value_error(shapes):
    with pytest.raises(ValueError):
        NearestNeighborMatcher()(_data(*shapes))


def test_cpu_tensors_are_a_runtime_error():
    with pytest.raises(RuntimeError, match="CUDA"):
        NearestNeighborMatcher()(_data(1, 10, 128, 1, 12, 128))


def test_split_outputs_without_lightglues_adaptive_keys():
    out = {"matches0": torch.tensor([[1, -1], [0, 0]]), "matches1": torch.tensor([[-1, 0, -1], [0, -1, -1]]),
           "matching_scores0": torch.ones(2, 2), "matching_scores1": torch.ones(2, 3),
           "matches": [torch.tensor([[0, 1]]), torch.tensor([[0, 0]])], "scores": [torch.ones(1), torch.ones(1)]}
    res = split_outputs(out, [2, 1], [3, 1])
    assert set(res[0]) == {"matches0", "matches1", "matching_scores0", "matching_scores1", "matches", "scores"}
    assert res[1]["matches0"].shape == (1, 1) and res[1]["matches1"].shape == (1, 1)
