"""Drop-in host mirror of ``lightglue.ALIKED`` (reference lightglue/aliked.py) over the C ABI in ``include/aliked_b200.h``.

The forward runs in CUDA (``csrc/al_api.cu``, fp32 on CUDA cores): padding, encoder with the deformable blocks, score
head, DKD and SDDH.  This module holds the parameters under the reference's names (an official ``{model_name}.pth``
loads with ``strict=True``), passes them to the library as one blob, and does the host glue outside ``forward``'s
math: gray -> RGB (``kornia.color.grayscale_to_rgb``: the channel repeated, on the device) and ``extract``'s resize
(lightglue_b200/extractor.py, shared with the other extractors).  CUDA tensors only, no CPU path.

Deviations from the reference, both in cases where its result is not well defined:
  * top-k mode (``detection_threshold <= 0``, ``max_num_keypoints = k > 0``) on an image with fewer than k NMS maxima:
    the reference fills up with zero-score pixels in whatever order ``torch.topk`` returns them; here the filler pixels
    are the first zero-score pixels in row-major order (mostly the border).  The maxima themselves come first, by
    descending score, ties by lower pixel index.
  * ``image_size`` with a batch: the reference's DKD loop rebinds its ``w, h`` to the last image's ``image_size`` and
    then decodes and scales every image's keypoints with them; here each image's keypoints are its own score-map pixel
    positions (the two agree when the last image's ``image_size`` is the image's full size).
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
from torch import nn

from . import _cabi
from . import extractor as _extractor


class _Module(nn.Module):
    """A bare parameter container (the reference's submodule names; the math runs in CUDA)."""


def _dcn(ci, co):
    m = _Module()
    m.offset_conv = nn.Conv2d(ci, 18, 3, padding=1, bias=True)
    m.regular_conv = nn.Conv2d(ci, co, 3, padding=1, bias=False)
    return m


def _block(ci, co, dcn, res):
    m = _Module()
    m.conv1 = _dcn(ci, co) if dcn else nn.Conv2d(ci, co, 3, padding=1, bias=False)
    m.bn1 = nn.BatchNorm2d(co)
    m.conv2 = _dcn(co, co) if dcn else nn.Conv2d(co, co, 3, padding=1, bias=False)
    m.bn2 = nn.BatchNorm2d(co)
    if res:
        m.downsample = nn.Conv2d(ci, co, 1)
    return m


class ALIKED(_extractor.CudaExtractor):
    _abi = "al"
    default_conf = {
        "model_name": "aliked-n16",
        "max_num_keypoints": -1,
        "detection_threshold": 0.2,
        "nms_radius": 2,
        # extension: None = keep the (random) initial parameters instead of looking for {model_name}.pth
        "weights": "default",
    }
    checkpoint_url = "https://github.com/Shiaoming/ALIKED/raw/main/models/{}.pth"
    n_limit_max = 20000
    # c1, c2, c3, c4, dim, K, M
    cfgs = {
        "aliked-t16": [8, 16, 32, 64, 64, 3, 16],
        "aliked-n16": [16, 32, 64, 128, 128, 3, 16],
        "aliked-n16rot": [16, 32, 64, 128, 128, 3, 16],
        "aliked-n32": [16, 32, 64, 128, 128, 3, 32],
    }
    preprocess_conf = {"resize": 1024}
    required_data_keys = ["image"]

    def __init__(self, **conf):
        super().__init__()
        self.conf = SimpleNamespace(**{**self.default_conf, **conf})
        if self.conf.model_name not in self.cfgs:
            raise ValueError(f"unknown model_name {self.conf.model_name!r}; one of {sorted(self.cfgs)}")
        c1, c2, c3, c4, dim, K, M = self.cfgs[self.conf.model_name]
        self.block1 = _block(3, c1, False, False)
        self.block2 = _block(c1, c2, False, True)
        self.block3 = _block(c2, c3, True, True)
        self.block4 = _block(c3, c4, True, True)
        self.conv1 = nn.Conv2d(c1, dim // 4, 1, bias=False)
        self.conv2 = nn.Conv2d(c2, dim // 4, 1, bias=False)
        self.conv3 = nn.Conv2d(c3, dim // 4, 1, bias=False)
        self.conv4 = nn.Conv2d(dim, dim // 4, 1, bias=False)
        self.score_head = nn.Sequential(
            nn.Conv2d(dim, 8, 1, bias=False), nn.SELU(), nn.Conv2d(8, 4, 3, padding=1, bias=False), nn.SELU(),
            nn.Conv2d(4, 4, 3, padding=1, bias=False), nn.SELU(), nn.Conv2d(4, 1, 3, padding=1, bias=False),
        )
        self.desc_head = _Module()
        self.desc_head.agg_weights = nn.Parameter(torch.rand(M, dim, dim))
        self.desc_head.offset_conv = nn.Sequential(nn.Conv2d(dim, 2 * M, K, bias=True), nn.SELU(),
                                                   nn.Conv2d(2 * M, 2 * M, 1, bias=True))
        self.desc_head.sf_conv = nn.Conv2d(dim, dim, 1, bias=False)
        if self.conf.weights is not None:
            name = self.conf.model_name if self.conf.weights == "default" else self.conf.weights
            self.load_state_dict(
                _extractor.find_checkpoint(f"{name}.pth", self.checkpoint_url.format(name), "ALIKED"), strict=True)
        self.requires_grad_(False)
        self.eval()

    # ------------------------------------------------------------------ C handle
    def _config(self) -> _cabi.AlConfig:
        c1, c2, c3, c4, dim, K, M = self.cfgs[self.conf.model_name]
        return _cabi.AlConfig(_cabi.AL_ABI_VERSION, c1, c2, c3, c4, dim, K, M, int(self.conf.nms_radius),
                              int(self.conf.max_num_keypoints), float(self.conf.detection_threshold))

    def _blob(self) -> torch.Tensor:
        """The state_dict without the BatchNorm counters, in state_dict order (include/aliked_b200.h)."""
        parts = [t.detach().reshape(-1).to(torch.float32) for k, t in self.state_dict().items()
                 if not k.endswith("num_batches_tracked")]
        return torch.cat(parts).contiguous()

    def _create(self, lib, cfg, blob, stream, out):
        assert blob.numel() == lib.al_weight_blob_floats(cfg)
        _cabi.check(lib.al_create(cfg, blob.data_ptr(), blob.numel(), stream, out), "al_create")

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, data: dict) -> dict:
        """Keypoints (pixels), descriptors and keypoint_scores of an image batch [B, 1 or 3, H, W], H, W >= 8."""
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        image = self._cuda_image(data["image"])
        if image.shape[1] == 1:  # kornia.color.grayscale_to_rgb
            image = image.expand(-1, 3, -1, -1)
        b, c, hh, ww = image.shape
        assert c == 3
        if hh < 8 or ww < 8:
            raise ValueError(f"image size {ww}x{hh}: height and width must be at least 8")
        image = image.detach().to(torch.float32).contiguous()
        size = data.get("image_size")
        if size is not None:
            size = torch.as_tensor(size).to(device=image.device, dtype=torch.float32).reshape(b, 2).contiguous()

        def call(lib, handle, cap, p, tail):
            return lib.al_forward(handle, image.data_ptr(), size.data_ptr() if size is not None else None, b, hh, ww, cap,
                                  p["keypoints"], p["keypoint_scores"], p["descriptors"], *tail)

        dim = self.cfgs[self.conf.model_name][4]
        return self._run(image, {"keypoints": (2,), "descriptors": (dim,), "keypoint_scores": ()}, call)
