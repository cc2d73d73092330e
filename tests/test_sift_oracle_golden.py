"""The SIFT fixtures are reproducible: the unmodified reference (oracle/_ref/sift_ref.py with the real cv2) rerun on a
fixture's recipe gives the stored output.  Skipped where the reference copy or cv2 is missing."""
import os

import pytest
import torch

from oracle import make_golden_sift as mg
from oracle import sift_ref_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sift")


@pytest.mark.skipif(not sift_ref_loader.available(), reason="oracle/_ref/sift_ref.py or cv2 is missing")
@pytest.mark.parametrize("name", ["sift_240x320", "sift_rgb_layers3", "sift_b2_image_size"])
def test_reference_reproduces_fixture(name):
    import cv2

    fix = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    if cv2.__version__ != fix["cv2_version"]:
        pytest.skip(f"fixture made with cv2 {fix['cv2_version']}, this is {cv2.__version__}")
    out = mg.run_reference(fix["recipe"], fix["conf"])
    for got, ref in zip(out, fix["out"]):
        for k in ref:
            torch.testing.assert_close(got[k], ref[k], rtol=0, atol=0)
