"""GPU parity of the SIFT extractor (include/sift_b200.h) against the fixtures made by the unmodified reference with
OpenCV, against the host emulation of the same functors, and its own invariances."""
import os

import pytest
import torch

from lightglue_b200 import synth
from lightglue_b200.sift import SIFT
from oracle import make_golden_sift as mg
from oracle import sift_compare, sift_emul, sift_synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sift")
CASES = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.startswith("sift_") and f.endswith(".pt"))
KEYS = ("keypoints", "scales", "oris", "keypoint_scores", "descriptors")


def _run(conf, image, image_size=None):
    data = {"image": image.cuda()}
    if image_size is not None:
        data["image_size"] = torch.as_tensor(image_size).cuda()
    return {k: v.cpu() for k, v in SIFT(**conf)(data).items()}


@pytest.mark.parametrize("name", CASES)
def test_sift_cuda_matches_reference_fixture(name):
    fix = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    rc, conf = fix["recipe"], fix["conf"]
    image = mg.make_image(rc)
    assert synth.checksum(image) == fix["image_checksum"]
    out = _run(conf, image, rc.get("image_size"))
    ordered = conf["max_num_keypoints"] == 4096  # far above these images' raw counts: OpenCV's order
    for b, ref in enumerate(fix["out"]):
        got = {k: out[k][b] for k in KEYS}
        st = sift_compare.compare(got, ref, ordered=ordered, is_rootsift=conf["rootsift"])
        sift_compare.check(st, ordered=ordered)


@pytest.mark.skipif(not sift_emul.available(), reason="oracle/_build/libsift_emul.so is not built")
@pytest.mark.parametrize("hw", [(240, 320), (480, 640)])
def test_sift_cuda_counts_match_host_emulation(hw):
    conf = dict(SIFT.default_conf)
    image = sift_synth.make_image(*hw, 1, 11)
    out = _run(conf, image)
    emu = sift_emul.forward(conf, image)[0]
    n, ne = out["keypoints"].shape[1], len(emu["keypoints"])
    assert abs(n - ne) <= 0.005 * ne, (n, ne)
    st = sift_compare.compare({k: out[k][0] for k in KEYS}, emu, ordered=True)
    assert st["frac_ref"] >= 0.99 and st["frac_test"] >= 0.99, st


def test_rgb_equals_gray_of_the_same_image():
    rgb = sift_synth.make_image(240, 320, 1, 12, channels=3)
    gray = 0.299 * rgb[:, 0:1] + 0.587 * rgb[:, 1:2] + 0.114 * rgb[:, 2:3]  # kornia's rgb_to_grayscale in fp32
    a, b = _run({}, rgb), _run({}, gray)
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k


def test_batch_equals_single_and_crop_equals_cropped_image():
    conf = dict(max_num_keypoints=64, nms_radius=None)
    img = sift_synth.make_image(240, 320, 2, 13)
    both = _run(conf, img)
    for i in range(2):
        one = _run(conf, img[i:i + 1])
        for k in KEYS:
            assert torch.equal(both[k][i], one[k][0]), k
    sizes = [[320, 240], [301, 211]]
    crop = _run(conf, img, sizes)
    alone = _run(conf, img[1:2, :, :211, :301].contiguous())
    for k in KEYS:
        assert torch.equal(crop[k][1], alone[k][0]), k
        assert torch.equal(crop[k][0], both[k][0]), k


def test_unequal_counts_in_a_batch_raise_value_error():
    img = torch.cat([sift_synth.make_image(240, 320, 1, 14), sift_synth.make_image(240, 320, 1, 15)])
    with pytest.raises(ValueError):
        SIFT()({"image": img.cuda()})


def test_integer_translation_shifts_interior_keypoints():
    """Cropping the same image at an offset that is a multiple of 2^(octaves - 1) shifts the first-octave keypoints away
    from the borders by exactly that offset, with equal descriptors.  filter_dog_point is off: it lets keypoints of the
    coarse octaves, which see the crop borders, remove first-octave ones at the same pixel."""
    conf = dict(max_num_keypoints=100000, nms_radius=None)
    h, w, d = 480, 640, 256  # 9 octaves at 480x640
    big = sift_synth.make_image(h + d, w + d, 1, 16)
    a = _run(conf, big[:, :, d:, d:].contiguous())  # a's pixel p is b's pixel p + d
    b = _run(conf, big[:, :, :h, :w].contiguous())
    kb = b["keypoints"][0]
    margin, found = 64, 0

    def interior(x, y):
        return margin <= x < w - margin and margin <= y < h - margin

    for j, ((x, y), s) in enumerate(zip(a["keypoints"][0].tolist(), a["scales"][0].tolist())):
        if s > 3.6 or not (interior(x, y) and interior(x + d, y + d)):  # first octave, away from both crops' borders
            continue
        # the same octave-pixel computation; only the final fp32 sum `pixel + offset` rounds at a different magnitude
        dist = (kb - torch.tensor([x + d, y + d])).abs().max(dim=1).values
        cands = torch.nonzero(dist <= 1e-3).flatten().tolist()
        assert cands, (x, y, s)
        assert any(float(a["scales"][0][j]) == float(b["scales"][0][k]) and float(a["oris"][0][j]) == float(b["oris"][0][k])
                   and torch.equal(a["descriptors"][0][j], b["descriptors"][0][k]) for k in cands), (x, y, s)
        found += 1
    assert found >= 20, found


def test_sift_feeds_the_matcher():
    from lightglue_b200 import LightGlue

    sift = SIFT(max_num_keypoints=256, nms_radius=None)
    lg = LightGlue(features=None, input_dim=128, add_scale_ori=True, depth_confidence=-1, width_confidence=-1)
    lg.load_state_dict(synth.make_state_dict(input_dim=128, add_scale_ori=True), strict=False)
    lg = lg.eval().cuda()
    im0 = sift_synth.make_image(240, 320, 1, 17).cuda()
    im1 = torch.roll(im0, shifts=(8, 16), dims=(2, 3))
    f0, f1 = sift({"image": im0}), sift({"image": im1})
    n0, n1 = f0["keypoints"].shape[1], f1["keypoints"].shape[1]
    size = torch.tensor([[320.0, 240.0]], device="cuda")
    out = lg({"image0": {**f0, "image_size": size}, "image1": {**f1, "image_size": size}})
    assert out["matches0"].shape == (1, n0) and out["matches1"].shape == (1, n1)
    assert out["matching_scores0"].shape == (1, n0)


def test_conf_change_after_the_first_call_takes_effect():
    """Setting ``conf.max_num_keypoints`` on a module that has run rebuilds its C handle, as a fresh module would.  (The
    ``nfeatures`` cut comes before filter_dog_point, so the count may end below the cap.)"""
    image = sift_synth.make_image(240, 320, 1, 13).cuda()
    s = SIFT()
    assert s({"image": image})["keypoints"].shape[1] > 100
    s.conf.max_num_keypoints = 100
    out = s({"image": image})
    want = SIFT(max_num_keypoints=100)({"image": image})
    assert 0 < out["keypoints"].shape[1] <= 100
    for k in KEYS:
        assert torch.equal(out[k], want[k]), k
