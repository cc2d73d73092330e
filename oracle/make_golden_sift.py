"""Generate tests/golden/sift/*.pt by running the UNMODIFIED reference SIFT (lightglue/sift.py, backend "opencv",
through oracle/sift_ref_loader.py) with the real cv2 on seeded synthetic images (oracle/sift_synth.py).

Each fixture holds the image recipe and its checksum, the conf, cv2.__version__ and the reference's outputs per image.
They live in tests/golden/sift/ because the matcher suites load every tests/golden/*.pt.

    make -C oracle -f sift_ref.mk && python oracle/make_golden_sift.py
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from lightglue_b200 import synth  # noqa: E402
from oracle import sift_ref_loader, sift_synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sift")

# name: (recipe, conf overrides); recipe = image arguments of sift_synth.make_image (+ image_size)
CASES = {
    "sift_240x320": (dict(h=240, w=320, b=1, seed=0), {}),
    "sift_480x640_top256": (dict(h=480, w=640, b=1, seed=1), dict(max_num_keypoints=256)),
    "sift_odd_203x317": (dict(h=203, w=317, b=1, seed=2), {}),
    "sift_nms3_norootsift": (dict(h=240, w=320, b=1, seed=3), dict(nms_radius=3, rootsift=False)),
    "sift_nms_none": (dict(h=240, w=320, b=1, seed=4), dict(nms_radius=None)),
    "sift_rgb_layers3": (dict(h=240, w=320, b=1, seed=5, channels=3),
                         dict(num_octaves=3, detection_threshold=0.02, edge_threshold=5)),
    "sift_b2_image_size": (dict(h=240, w=320, b=2, seed=6, image_size=[[320, 240], [288, 197]]),
                           dict(max_num_keypoints=64, nms_radius=None)),
    "sift_exact_levels": (dict(h=240, w=320, b=1, seed=7, channels=3, exact_levels=True), {}),
}


def make_image(rc: dict) -> torch.Tensor:
    return sift_synth.make_image(rc["h"], rc["w"], rc["b"], rc["seed"], rc.get("channels", 1), rc.get("exact_levels", False))


def run_reference(rc: dict, conf: dict) -> list:
    import cv2  # noqa: F401  (the reference's backend)

    model = sift_ref_loader.build_model(**conf)
    image = make_image(rc)
    data = {"image": image}
    if "image_size" in rc:
        data["image_size"] = torch.tensor(rc["image_size"])
    with torch.no_grad():
        out = model(data)
    keys = ("keypoints", "scales", "oris", "keypoint_scores", "descriptors")
    return [{k: out[k][b].clone() for k in keys} for b in range(rc["b"])]


def main():
    import cv2

    os.makedirs(OUT, exist_ok=True)
    for name, (rc, over) in CASES.items():
        conf = {**sift_ref_loader.load().SIFT.default_conf, **over}
        image = make_image(rc)
        out = run_reference(rc, conf)
        torch.save({"recipe": rc, "conf": conf, "image_checksum": synth.checksum(image), "cv2_version": cv2.__version__,
                    "out": out}, os.path.join(OUT, name + ".pt"))
        print(name, [len(o["keypoints"]) for o in out])


if __name__ == "__main__":
    main()
