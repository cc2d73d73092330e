"""The ALIKED oracle (oracle/aliked_oracle.py: pure torch, no torchvision) against fixtures produced by the reference's
own aliked.py (oracle/make_golden_aliked.py): identical integer NMS positions in the same order, refined keypoints
within 1e-4 px, scores within 1e-6, descriptors within 1e-5.  CPU only."""
import os

import pytest
import torch

from lightglue_b200 import synth
from oracle import aliked_oracle as alo
from oracle import aliked_synth as als
from oracle.make_golden_aliked import FIXTURE_THREADS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aliked")
CASES = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.startswith("al_") and f.endswith(".pt"))


def test_fixtures_exist():
    assert len(CASES) >= 7


@pytest.mark.parametrize("name", CASES)
def test_aliked_oracle_matches_reference_fixture(name):
    fix = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    rc, conf, gold = fix["recipe"], fix["conf"], fix["out"]
    w = als.make_aliked_state_dict(rc["model"], 0)
    for k, v in fix["weights_checksum"].items():
        assert synth.checksum(w[k]) == v, k
    image = als.make_image(rc["h"], rc["w"], rc["b"], rc["seed"])
    assert synth.checksum(image) == fix["image_checksum"]
    image_size = torch.tensor(rc["image_size"]) if "image_size" in rc else None
    threads = torch.get_num_threads()
    torch.set_num_threads(FIXTURE_THREADS)  # the fixtures' summation order (see make_golden_aliked.py)
    try:
        with torch.no_grad():
            out = alo.forward(w, image, image_size=image_size, **conf)
    finally:
        torch.set_num_threads(threads)
    for b in range(rc["b"]):
        assert torch.equal(out["nms_positions"][b], gold["nms_positions"][b]), "NMS positions / order differ"
        assert float((out["keypoints"][b] - gold["keypoints"][b]).abs().max()) <= 1e-4
        assert float((out["keypoint_scores"][b] - gold["keypoint_scores"][b]).abs().max()) <= 1e-6
        d = out["descriptors"][b][:: gold["desc_stride"][b]]
        assert d.shape == gold["descriptors"][b].shape
        assert float((d - gold["descriptors"][b]).abs().max()) <= 1e-5
