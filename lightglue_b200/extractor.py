"""Host glue shared by the extractors (``SuperPoint``, ``ALIKED``): checkpoint lookup and ``Extractor.extract``."""
from __future__ import annotations

import os
from pathlib import Path

import torch


def find_checkpoint(fname: str, url: str, cls_name: str):
    """The reference downloads the checkpoint; offline we look in $LIGHTGLUE_WEIGHTS_DIR, torch hub's checkpoints and
    the package's ``weights/``, in that order."""
    cands = [
        Path(os.environ["LIGHTGLUE_WEIGHTS_DIR"]) / fname if os.environ.get("LIGHTGLUE_WEIGHTS_DIR") else None,
        Path(torch.hub.get_dir()) / "checkpoints" / fname,
        Path(__file__).parent / "weights" / fname,
    ]
    for c in cands:
        if c is not None and c.exists():
            return torch.load(str(c), map_location="cpu")
    raise FileNotFoundError(
        f"{fname} not found (no network access: put it under $LIGHTGLUE_WEIGHTS_DIR or torch hub's checkpoints, "
        f"or construct {cls_name}(weights=None)); upstream URL: {url}"
    )


@torch.no_grad()
def extract(model, img: torch.Tensor, **conf) -> dict:
    """``Extractor.extract`` (utils.py:136-147): add the batch dimension, resize the longer side to ``resize``
    (``ImagePreprocessor``, utils.py:26-38: ``kornia.geometry.transform.resize(side="long", antialias=True)``: the long
    side becomes ``resize`` and the other ``int(resize / aspect)`` -- truncated, kornia's ``_side_to_image_size``; kornia
    itself is not a dependency here), run ``forward``, map keypoints back to the original pixels."""
    if img.dim() == 3:
        img = img[None]
    assert img.dim() == 4 and img.shape[0] == 1
    h, w = img.shape[-2:]
    resize = {**model.preprocess_conf, **conf}.get("resize")
    nh, nw = h, w
    if resize is not None:
        aspect = w / h
        nh, nw = (int(resize / aspect), int(resize)) if aspect >= 1.0 else (int(resize), int(resize * aspect))
    if (nh, nw) != (h, w):
        img = torch.nn.functional.interpolate(img, size=(nh, nw), mode="bilinear", antialias=True, align_corners=False)
    scales = torch.tensor([nw / w, nh / h], device=img.device, dtype=torch.float32)
    feats = model.forward({"image": img})
    feats["image_size"] = torch.tensor([[w, h]], device=img.device, dtype=torch.float32)
    feats["keypoints"] = (feats["keypoints"] + 0.5) / scales[None] - 0.5
    return feats
