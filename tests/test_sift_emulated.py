"""Host emulation of the SIFT CUDA path (oracle/sift_emul.cpp runs the functors of csrc/sift_pipeline.h with g++)
against the fixtures made by the unmodified reference with OpenCV; no GPU needed."""
import os

import pytest
import torch

from lightglue_b200 import synth
from oracle import make_golden_sift as mg
from oracle import sift_compare, sift_emul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sift")
CASES = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.startswith("sift_") and f.endswith(".pt"))


def uncapped(fix) -> bool:
    """OpenCV's order survives when neither the nfeatures cut nor the top-k applied: the fixtures with the default
    max_num_keypoints have far fewer raw keypoints than that."""
    return fix["conf"]["max_num_keypoints"] == 4096


@pytest.mark.skipif(not sift_emul.available(), reason="oracle/_build/libsift_emul.so is not built")
@pytest.mark.parametrize("name", CASES)
def test_sift_emulation_matches_reference_fixture(name):
    fix = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    rc, conf = fix["recipe"], fix["conf"]
    image = mg.make_image(rc)
    assert synth.checksum(image) == fix["image_checksum"]
    out = sift_emul.forward(conf, image, rc.get("image_size"))
    for b, (got, ref) in enumerate(zip(out, fix["out"])):
        st = sift_compare.compare(got, ref, ordered=uncapped(fix), is_rootsift=conf["rootsift"])
        sift_compare.check(st, ordered=uncapped(fix))


def test_truncating_quantisation_is_exercised():
    """The k/255 fixture is an RGB image with equal channels on exact k/255 levels: its gray value, times 255 in fp32,
    truncates to k - 1 at some pixels."""
    img = mg.make_image(mg.CASES["sift_exact_levels"][0])
    assert bool((img[:, 0] == img[:, 1]).all() and (img[:, 0] == img[:, 2]).all())
    k = torch.round(img[:, :1] * 255.0)
    gray = 0.299 * img[:, 0:1] + 0.587 * img[:, 1:2] + 0.114 * img[:, 2:3]
    q = (gray * 255.0).to(torch.uint8).float()
    assert bool((q == k - 1).any()) and bool((q == k).any())
