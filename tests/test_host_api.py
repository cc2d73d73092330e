"""CPU-side checks: the C-ABI library loads and exports every symbol include/lightglue_b200.h
declares, and the host-side mirror of the reference interface behaves like the reference's
(constructor / conf / state_dict names / error behaviour).  No compute calls (no GPU here)."""
import os
import re

import pytest
import torch

from lightglue_b200 import LightGlue, _cabi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = _cabi.load()
    header = open(os.path.join(ROOT, "include", "lightglue_b200.h")).read()
    declared = re.findall(r"LG_API\s+[\w\s\*]+?\b(lg_\w+)\s*\(", header)
    assert sorted(declared) == sorted(_cabi.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.lg_build_info()


def test_blob_size_matches_parameter_count():
    lib = _cabi.load()
    for d, so in ((256, False), (128, False), (128, True)):
        m = LightGlue(features=None, input_dim=d, add_scale_ori=so)
        assert lib.lg_weight_blob_floats(d, 4 if so else 2, 9) == sum(t.numel() for t in m._blob_tensors())
    assert sum(p.numel() for p in LightGlue(features=None).parameters()) == 11_851_601  # SURVEY.md §8a


def test_state_dict_uses_reference_key_names():
    m = LightGlue(features=None, input_dim=128)
    sd = synth.make_state_dict(input_dim=128)
    keys = set(m.state_dict().keys())
    assert set(sd.keys()) | {"confidence_thresholds"} == keys
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert missing == ["confidence_thresholds"] and not unexpected


def test_legacy_checkpoint_names_are_renamed():
    sd = {"self_attn.3.Wqkv.weight": torch.zeros(1), "cross_attn.0.to_qk.bias": torch.zeros(1), "posenc.Wr.weight": 0}
    out = LightGlue._rename_legacy(sd, 9)
    assert "transformers.3.self_attn.Wqkv.weight" in out and "transformers.0.cross_attn.to_qk.bias" in out


def test_constructor_contract():
    with pytest.raises(ValueError):
        LightGlue(features="orb")
    m = LightGlue(features=None, depth_confidence=-1, filter_threshold=0.2)
    assert m.conf.depth_confidence == -1 and m.conf.width_confidence == 0.99 and m.conf.filter_threshold == 0.2
    assert m.conf.n_layers == 9 and m.conf.num_heads == 4 and m.conf.descriptor_dim == 256
    assert LightGlue.pruning_keypoint_thresholds == {"cpu": -1, "mps": -1, "cuda": 1024, "flash": 1536}
    assert LightGlue.required_data_keys == ["image0", "image1"]
    assert torch.allclose(
        m.confidence_thresholds,
        torch.tensor([0.9000, 0.8641, 0.8411, 0.8264, 0.8169, 0.8108, 0.8069, 0.8045, 0.8029]), atol=5e-5,
    )
    m.compile()
    assert m.static_lengths == [256, 512, 768, 1024, 1280, 1536]


def test_forward_rejects_missing_keys_and_cpu_tensors():
    m = LightGlue(features=None)
    data, _ = synth.make_pair(16)
    with pytest.raises(AssertionError):
        m({"image0": data["image0"]})
    with pytest.raises(RuntimeError):  # no CPU path: fail loudly
        m(data)


def test_ctypes_structs_match_the_header_layout(tmp_path):
    """sizeof / offsetof of the C-ABI structs as gcc lays them out == the ctypes mirrors in _cabi.py."""
    import ctypes as C
    import subprocess

    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "lightglue_b200.h"\n#include "superpoint_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %d ", sizeof(SpConfig), offsetof(SpConfig, detection_threshold), SP_ABI_VERSION);\n'
        '  printf("%zu %zu %zu %zu %zu %zu %zu %d\\n", sizeof(LgConfig), sizeof(LgInputs), sizeof(LgOutputs),\n'
        "         offsetof(LgInputs, pruning_threshold), offsetof(LgInputs, lens0), offsetof(LgInputs, lens1),\n"
        "         offsetof(LgOutputs, log_assignment), LG_ABI_VERSION);\n"
        "  return 0;\n}\n"
    )
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [
        C.sizeof(_cabi.SpConfig), _cabi.SpConfig.detection_threshold.offset, _cabi.SP_ABI_VERSION,
        C.sizeof(_cabi.LgConfig), C.sizeof(_cabi.LgInputs), C.sizeof(_cabi.LgOutputs),
        _cabi.LgInputs.pruning_threshold.offset, _cabi.LgInputs.lens0.offset, _cabi.LgInputs.lens1.offset,
        _cabi.LgOutputs.log_assignment.offset, _cabi.ABI_VERSION,
    ]
    assert got == want


def test_ragged_padding_and_splitting_host_logic():
    from lightglue_b200.ragged import pad_pairs, split_outputs

    pairs = []
    for m, n in ((5, 3), (2, 7), (0, 4)):
        data, _ = synth.make_pair(max(m, n, 1), b=1, seed=m + n, m=max(m, 1))
        f0 = {k: (v[:, :m] if v.dim() == 3 else v) for k, v in data["image0"].items()}
        f1 = {k: (v[0, :n] if v.dim() == 3 else v) for k, v in data["image1"].items()}  # unbatched form
        pairs.append({"image0": f0, "image1": f1})
    data = pad_pairs(pairs)
    assert data["image0"]["keypoints"].shape == (3, 5, 2) and data["image1"]["descriptors"].shape == (3, 7, 256)
    assert data["image0"]["num_keypoints"].tolist() == [5, 2, 0] and data["image1"]["num_keypoints"].tolist() == [3, 7, 4]
    assert data["image0"]["image_size"].shape == (3, 2)
    assert torch.equal(data["image1"]["keypoints"][0, :3], pairs[0]["image1"]["keypoints"])
    assert float(data["image0"]["descriptors"][1, 2:].abs().sum()) == 0.0  # zero padding
    out = {
        "matches0": torch.full((3, 5), -1), "matches1": torch.full((3, 7), -1),
        "matching_scores0": torch.zeros(3, 5), "matching_scores1": torch.zeros(3, 7),
        "matches": [torch.zeros(0, 2, dtype=torch.int64)] * 3, "scores": [torch.zeros(0)] * 3,
        "prune0": torch.ones(3, 5), "prune1": torch.ones(3, 7), "stop": 9, "stops": [9, 4, 1],
    }
    parts = split_outputs(out, data["image0"]["num_keypoints"], data["image1"]["num_keypoints"])
    assert [p["matches0"].shape[1] for p in parts] == [5, 2, 0] and [p["matches1"].shape[1] for p in parts] == [3, 7, 4]
    assert [p["stop"] for p in parts] == [9, 4, 1] and isinstance(parts[0]["matches"], list)
    with pytest.raises(ValueError):
        pairs[1]["image0"].pop("image_size")
        pad_pairs(pairs)


def test_caller_glue_rbd_batch_to_device_match_pair():
    """utils.rbd / batch_to_device / match_pair behave like the reference's (utils.py:41-69, 150-165)."""
    import numpy as np

    from lightglue_b200 import utils

    d = {"a": torch.arange(6).reshape(1, 3, 2), "b": [torch.ones(2)], "stop": 7, "n": np.zeros((1, 4)), "s": "name"}
    r = utils.rbd(d)
    assert r["a"].shape == (3, 2) and torch.equal(r["b"], torch.ones(2)) and r["stop"] == 7 and r["n"].shape == (4,)
    assert r["s"] == "name"
    moved = utils.batch_to_device({"x": torch.ones(2, requires_grad=True), "l": [torch.zeros(1)], "k": "v", "i": 3}, "cpu")
    assert not moved["x"].requires_grad and isinstance(moved["l"], list) and moved["k"] == "v" and moved["i"] == 3

    class Extractor:
        def extract(self, img, **conf):
            n = int(img.shape[-1])
            return {"keypoints": torch.zeros(1, n, 2), "descriptors": torch.zeros(1, n, 256),
                    "image_size": torch.tensor([[float(n), 1.0]]), "resize": conf.get("resize")}

    def matcher(data):
        m, n = data["image0"]["keypoints"].shape[1], data["image1"]["keypoints"].shape[1]
        return {"matches0": torch.full((1, m), -1), "matches1": torch.full((1, n), -1),
                "matches": [torch.zeros(0, 2, dtype=torch.int64)], "scores": [torch.zeros(0)], "stop": 3}

    f0, f1, m01 = utils.match_pair(Extractor(), matcher, torch.zeros(1, 8, 5), torch.zeros(1, 8, 9), resize=512)
    assert f0["keypoints"].shape == (5, 2) and f1["descriptors"].shape == (9, 256) and f0["resize"] == 512
    assert m01["matches0"].shape == (5,) and m01["matches"].shape == (0, 2) and m01["stop"] == 3


def test_numa_binding_helpers_never_raise():
    """sharding.bind_to_gpu_numa_node: cpulist parsing, and a graceful no-op where there is no GPU / sysfs topology."""
    from lightglue_b200 import sharding

    assert sharding._parse_cpulist("0-3,8,10-11\n") == [0, 1, 2, 3, 8, 10, 11]
    assert sharding._parse_cpulist("") == []
    info = sharding.bind_to_gpu_numa_node(0)
    assert info["device"] == 0 and isinstance(info["bound"], bool)
