"""DISK without a GPU: the oracle's detection rules on hand-built heatmaps, the module's parameter layout, checkpoint
loading, conf validation and the header's export table (include/disk_b200.h, lightglue_b200/disk.py)."""
import os
import re

import pytest
import torch

from lightglue_b200 import DISK, _cabi
from oracle import disk_oracle as do
from oracle import disk_synth as ds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- oracle detection rules
def test_plateau_keeps_only_its_first_pixel():
    heat = torch.zeros(8, 8)
    heat[3:5, 3:5] = 1.0
    xy, logp = do.detect(heat, 5, 0.0, None)
    assert xy.tolist() == [[3, 3]] and logp.tolist() == [1.0]


def test_nms_keeps_separated_maxima_in_row_major_order():
    heat = torch.zeros(9, 12)
    heat[7, 1], heat[1, 10], heat[1, 2] = 3.0, 2.0, 1.0
    xy, logp = do.detect(heat, 3, 0.0, None)
    assert xy.tolist() == [[2, 1], [10, 1], [1, 7]] and logp.tolist() == [1.0, 2.0, 3.0]


def test_topk_with_count_at_most_n_drops_the_minimum():
    heat = torch.zeros(9, 12)
    heat[1, 1], heat[1, 6], heat[6, 1], heat[6, 6] = 4.0, 1.0, 3.0, 1.0
    xy, logp = do.detect(heat, 3, 0.0, 10)  # 4 candidates <= 10: both values equal to the minimum go
    assert xy.tolist() == [[1, 1], [1, 6]] and logp.tolist() == [4.0, 3.0]


def test_topk_drops_every_candidate_tied_at_the_cut():
    heat = torch.zeros(9, 16)
    for x, v in ((1, 5.0), (5, 2.0), (9, 2.0), (13, 7.0)):
        heat[4, x] = v
    xy, logp = do.detect(heat, 3, 0.0, 2)  # the 3rd largest (2.0) is tied with the 2nd: only values > 2 stay
    assert xy.tolist() == [[1, 4], [13, 4]] and logp.tolist() == [5.0, 7.0]
    xy, _ = do.detect(heat, 3, 0.0, 3)  # cut at the 4th largest (2.0 again): room for 3, yet both 2.0s go
    assert xy.tolist() == [[1, 4], [13, 4]]
    heat[4, 9] = 3.0
    xy, _ = do.detect(heat, 3, 0.0, 2)  # cut at 3.0: keep 5 and 7, in row-major order
    assert xy.tolist() == [[1, 4], [13, 4]]
    xy, _ = do.detect(heat, 3, 0.0, 3)  # cut at 2.0: keep 5, 3, 7
    assert xy.tolist() == [[1, 4], [9, 4], [13, 4]]


def test_threshold_is_strict():
    heat = torch.zeros(6, 6)
    heat[1, 1], heat[4, 4] = 0.5, 0.25
    xy, _ = do.detect(heat, 3, 0.25, None)
    assert xy.tolist() == [[1, 1]]


def test_even_window_raises():
    with pytest.raises(ValueError):
        do.detect(torch.zeros(8, 8), 4, 0.0, None)


def test_one_pixel_at_sixteenth_resolution_raises():
    sd = ds.make_disk_state_dict(0)
    with pytest.raises(ValueError):
        do.heads(sd, torch.rand(1, 3, 16, 16))
    heat, desc = do.heads(sd, torch.rand(1, 3, 16, 17))  # padded to 16 x 32: two pixels at 1/16
    assert heat.shape == (1, 16, 17) and desc.shape == (1, 128, 16, 17)


def test_synthetic_case_is_not_vacuous():
    """The synthetic weights and image give hundreds of keypoints at 240 x 320 with the default conf."""
    out = do.forward(ds.make_disk_state_dict(0), ds.make_image(240, 320, 1, 1))
    assert 100 <= out["keypoints"].shape[1] <= 2000
    assert torch.allclose(out["descriptors"].norm(dim=-1), torch.ones(1))


# ---------------------------------------------------------------------------------------------- module
def test_state_dict_names_and_shapes_are_kornias():
    m = DISK(weights=None)
    ours = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert ours == [(f"model.{k}", s) for k, s in ds.layout()]
    assert sum(p.numel() for p in m.parameters()) == 1092372
    assert m._blob().numel() == 1092372 == _cabi.load().disk_weight_blob_floats()


def test_checkpoint_loads_strictly_from_weights_dir(tmp_path, monkeypatch):
    sd = ds.make_disk_state_dict(3)
    torch.save({"extractor": sd}, tmp_path / "epipolar-save.pth")
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    m = DISK(weights="epipolar")
    assert torch.equal(m.model.unet.path_up[3].conv[3].weight, sd["unet.path_up.3.conv.3.weight"])
    bad = dict(sd)
    bad["unet.extra"] = torch.zeros(1)
    torch.save({"extractor": bad}, tmp_path / "depth-save.pth")
    with pytest.raises(RuntimeError):
        DISK(weights="depth")


def test_missing_checkpoint_raises(tmp_path, monkeypatch):
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError):
        DISK()


@pytest.mark.parametrize("conf", [dict(desc_dim=64), dict(weights="outdoor"), dict(nms_window_size=4),
                                  dict(nms_window_size=0), dict(max_num_keypoints=-1), dict(max_num_keypoints=2.5)])
def test_bad_conf_raises(conf):
    with pytest.raises(ValueError):
        DISK(**{"weights": None, **conf})


def test_conf_struct():
    c = DISK(weights=None, max_num_keypoints=None, nms_window_size=7, detection_threshold=0.5,
             pad_if_not_divisible=False)._config()
    assert (c.abi_version, c.max_num_keypoints, c.nms_window_size, c.pad_if_not_divisible) == (1, -1, 7, 0)
    assert c.detection_threshold == 0.5
    assert DISK(weights=None, max_num_keypoints=2048)._config().max_num_keypoints == 2048


def test_reference_confs():
    assert DISK.default_conf == {"weights": "depth", "max_num_keypoints": None, "desc_dim": 128, "nms_window_size": 5,
                                 "detection_threshold": 0.0, "pad_if_not_divisible": True}
    assert DISK.preprocess_conf == {"resize": 1024, "grayscale": False}
    assert DISK.required_data_keys == ["image"]


def test_cpu_tensor_raises():
    with pytest.raises(RuntimeError):
        DISK(weights=None)({"image": torch.rand(1, 3, 32, 32)})


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "disk_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(disk_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.DISK_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.DISK_EXPORTS:
        assert hasattr(lib, s), s
        assert getattr(lib, s).argtypes is not None, s
