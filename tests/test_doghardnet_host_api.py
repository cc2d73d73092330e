"""DoG-HardNet without a GPU: the oracle's pyramid and patch rules on hand-built LAFs, the unmodified reference file
against the oracle, the module's parameter layout, checkpoint loading, conf validation and the header's export table
(include/doghardnet_b200.h, lightglue_b200/dog_hardnet.py)."""
import os
import re

import pytest
import torch

from lightglue_b200 import SIFT, DoGHardNet, _cabi
from oracle import doghardnet_oracle as dho
from oracle import doghardnet_ref_loader, sift_ref_loader, sift_synth
from oracle import doghardnet_synth as dhs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = torch.float64


def _laf(x, y, s, deg=0.0):
    """One LAF [1, 2, 3] with A = s R(deg) at (x, y)."""
    t = torch.tensor
    return dho.laf_from_center_scale_ori(t([[[x, y]]], dtype=D), t([[[[s]]]], dtype=D), t([[[deg]]], dtype=D))[0]


# ---------------------------------------------------------------------------------------------- oracle rules
def test_laf_is_scaled_rotation_at_the_centre():
    laf = _laf(10.0, 20.0, 3.0, 90.0)
    want = torch.tensor([[0.0, 3.0, 10.0], [-3.0, 0.0, 20.0]], dtype=D)
    assert torch.allclose(laf[0], want, atol=1e-12)


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_level_selection_at_and_around_powers_of_two(k):
    s = 16.0 * 2**k  # 2 s / 32 = 2^k
    for f, want in ((1.0, k), (1 - 1e-9, k - 1), (1 + 1e-9, k), (1.999, k)):
        assert int(dho.pyramid_levels(_laf(500.0, 400.0, s * f), 768, 1024)) == want, (f, want)
    assert int(dho.pyramid_levels(_laf(500.0, 400.0, 1.0), 768, 1024)) == 0  # log2 < 0 clamps to 0


def test_level_clamp():
    assert int(dho.pyramid_levels(_laf(50.0, 50.0, 1e6), 100, 130)) == 2  # min side 100: 100 // 32 - 1
    assert int(dho.pyramid_levels(_laf(10.0, 10.0, 1e6), 31, 40)) == 0   # max(0, 0 - 1)
    assert int(dho.pyramid_levels(_laf(500.0, 400.0, 1e9), 768, 1024)) == 23


def test_zero_patch_beyond_the_last_sampled_level():
    img = sift_synth.make_image(768, 1024, 1, 3).to(D)
    assert dho.level_count(768, 1024) == 6  # 768 384 192 96 48 24
    lafs = torch.cat([_laf(500.0, 400.0, 16.0 * 2**5 * 1.5), _laf(500.0, 400.0, 16.0 * 2**6 * 1.5)])
    assert dho.pyramid_levels(lafs, 768, 1024).tolist() == [5, 6]
    p = dho.extract_patches(img, lafs)
    assert p[0].abs().sum() > 0 and torch.equal(p[1], torch.zeros_like(p[1]))


def test_pyramid_shapes_for_odd_sides():
    img = torch.rand(1, 1, 203, 317, dtype=D)
    shapes = [tuple(l.shape[-2:]) for l in dho.pyramid(img)]
    assert shapes == [(203, 317), (101, 158), (50, 79), (25, 39)]
    assert dho.level_count(203, 317) == 4
    assert tuple(dho.pyrdown(torch.rand(1, 1, 33, 47, dtype=D)).shape[-2:]) == (16, 23)


def test_pyrdown_of_a_constant_is_the_constant():
    assert torch.allclose(dho.pyrdown(torch.full((1, 1, 40, 57), 0.25, dtype=D)), torch.tensor(0.25, dtype=D))


def test_identity_laf_on_a_ramp_gives_the_analytic_bilinear_values():
    h, w, s, cx, cy = 120, 160, 10.0, 70.3, 50.8
    yy, xx = torch.meshgrid(torch.arange(h, dtype=D), torch.arange(w, dtype=D), indexing="ij")
    img = (0.002 * xx + 0.003 * yy + 0.1)[None, None]
    p = dho.extract_patches(img, _laf(cx, cy, s))[0, 0]
    base = (2 * torch.arange(32, dtype=D) + 1) / 32 - 1  # affine_grid, align_corners=False
    px = (s * base + cx) * w / (w - 1) - 0.5  # 2 g / (w - 1) - 1, then grid_sample's unnormalise
    py = (s * base + cy) * h / (h - 1) - 0.5
    want = 0.002 * px[None, :] + 0.003 * py[:, None] + 0.1
    assert torch.allclose(p, want, atol=1e-12)


def test_border_clamp():
    img = torch.rand(1, 1, 64, 64, dtype=D)
    p = dho.extract_patches(img, _laf(0.0, 0.0, 20.0))[0, 0]
    assert torch.all(p[:8, :8] == img[0, 0, 0, 0])  # the top-left quarter samples left of / above pixel 0


def test_hardnet_output_is_unit_and_scale_invariant():
    sd = dhs.make_state_dict(1)
    x = torch.rand(5, 1, 32, 32, dtype=D)
    d = dho.hardnet(sd, x)
    assert d.shape == (5, 128) and torch.allclose(d.norm(dim=1), torch.ones(5, dtype=D))
    assert torch.allclose(dho.hardnet(sd, 3.0 * x + 1.0), d, atol=1e-4)  # up to the std's 1e-6


@pytest.mark.skipif(not doghardnet_ref_loader.available(), reason="oracle/_ref/ reference files or cv2 missing")
def test_reference_file_equals_oracle_forward():
    """The unmodified reference dog_hardnet.py + sift.py (real cv2; kornia stand-ins from the oracle) equals
    doghardnet_oracle.forward on the reference SIFT's own keypoints: crop, 6 x scale, rad2deg, no RootSIFT, per image."""
    sd = dhs.make_state_dict(2)
    conf = dict(max_num_keypoints=48, nms_radius=None)  # equal counts: the reference stacks them
    img = sift_synth.make_image(240, 320, 2, 21, channels=3)
    size = torch.tensor([[320, 240], [301, 223]])
    ref = doghardnet_ref_loader.build_model(sd, **conf)({"image": img, "image_size": size})
    sift = sift_ref_loader.build_model(**conf)
    g = dho.gray(img)
    feats = [sift.extract_single_image(g[k][:, :int(size[k, 1]), :int(size[k, 0])]) for k in range(2)]
    got = dho.forward(sd, img, feats, size)
    assert ref["keypoints"].shape == (2, 48, 2)
    for k in ("keypoints", "scales", "oris", "keypoint_scores"):
        assert torch.equal(ref[k], got[k]), k
    assert torch.allclose(ref["descriptors"], got["descriptors"], atol=1e-6)
    assert not torch.allclose(ref["descriptors"][:, :, :128], ref["descriptors"].new_zeros(()))  # not vacuous


# ---------------------------------------------------------------------------------------------- module
def test_state_dict_names_and_shapes_are_kornias():
    m = DoGHardNet(weights=None)
    ours = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert ours == [(f"laf_desc.descriptor.{k}", s) for k, s in dhs.layout()]
    assert sum(p.numel() for p in m.parameters()) == 1334560
    assert m._blob().numel() == 1334560 + 1152 == _cabi.load().dhn_weight_blob_floats()


def test_blob_order():
    m = DoGHardNet(weights=None)
    m.laf_desc.descriptor.load_state_dict(dhs.make_state_dict(4), strict=True)
    f = m.laf_desc.descriptor.features
    blob = m._blob()
    assert torch.equal(blob[:288], f[0].weight.reshape(-1))
    assert torch.equal(blob[288:320], f[1].running_mean) and torch.equal(blob[320:352], f[1].running_var)
    assert torch.equal(blob[-128:], f[20].running_var)


def test_checkpoint_loads_strictly_from_weights_dir(tmp_path, monkeypatch):
    sd = dhs.make_state_dict(3)
    torch.save({"state_dict": sd}, tmp_path / "checkpoint_liberty_with_aug.pth")
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    m = DoGHardNet()
    assert torch.equal(m.laf_desc.descriptor.features[19].weight, sd["features.19.weight"])
    assert torch.equal(m.laf_desc.descriptor.features[7].running_var, sd["features.7.running_var"])
    bad = dict(sd)
    bad["features.99.weight"] = torch.zeros(1)
    torch.save({"state_dict": bad}, tmp_path / "bad.pth")
    with pytest.raises(RuntimeError):
        DoGHardNet(weights="bad.pth")


def test_missing_checkpoint_raises(tmp_path, monkeypatch):
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError):
        DoGHardNet()


@pytest.mark.parametrize("conf", [dict(backend="pycolmap"), dict(max_num_keypoints=0), dict(max_num_keypoints=2.5),
                                  dict(max_num_keypoints=None), dict(nms_radius=-1), dict(num_octaves=0),
                                  dict(num_octaves=9), dict(weights=3)])
def test_bad_conf_raises(conf):
    with pytest.raises(ValueError):
        DoGHardNet(**{"weights": None, **conf})


def test_confs_are_sifts():
    assert DoGHardNet.default_conf == {**SIFT.default_conf, "weights": "checkpoint_liberty_with_aug.pth"}
    assert DoGHardNet.preprocess_conf == SIFT.preprocess_conf
    assert DoGHardNet.required_data_keys == ["image"]


def test_conf_struct():
    c = DoGHardNet(weights=None, nms_radius=None, max_num_keypoints=2048, num_octaves=3, detection_threshold=0.01,
                   edge_threshold=12, rootsift=False)._config()
    assert (c.abi_version, c.num_octave_layers, c.nms_radius, c.max_num_keypoints) == (1, 3, -1, 2048)
    assert (c.detection_threshold, c.edge_threshold) == (0.01, 12.0)
    assert bytes(c) == bytes(DoGHardNet(weights=None, nms_radius=None, max_num_keypoints=2048, num_octaves=3,
                                        detection_threshold=0.01, edge_threshold=12)._config())  # rootsift is ignored


def test_conf_struct_layout():
    import ctypes as C
    assert C.sizeof(_cabi.DhnConfig) == 32 and _cabi.DhnConfig.detection_threshold.offset == 16


def test_cpu_tensor_raises():
    with pytest.raises(RuntimeError):
        DoGHardNet(weights=None)({"image": torch.rand(1, 1, 64, 64)})


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "doghardnet_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(dhn_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.DHN_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.DHN_EXPORTS:
        assert hasattr(lib, s), s
        assert getattr(lib, s).argtypes is not None, s
