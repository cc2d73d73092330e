"""Drop-in host mirror of ``lightglue.DISK`` (reference lightglue/disk.py, which wraps ``kornia.feature.DISK``) over the
C ABI in ``include/disk_b200.h``.

The forward runs in CUDA (``csrc/disk_api.cu``): the padding to multiples of 16, the U-Net (instance norm, PReLU and 5x5
convolutions; the convolutions of down1 .. up2 on tensor cores with split-bf16 operands), NMS, the threshold, the
kthvalue top-k and the descriptors.  The 128 descriptor channels of the last convolution are computed at the selected
keypoints only.  This module holds the parameters under kornia's names (``model.unet.path_down.{i}.1.{1,3}.*``,
``model.unet.path_up.{i}.conv.{1,3}.*``; a DISK checkpoint's ``["extractor"]`` loads into ``model`` with
``strict=True``) and passes them to the library as one blob.  CUDA tensors only, no CPU path.

Deviations from the reference:
  * ``desc_dim`` other than 128 raises ``ValueError`` (the reference ignores it: the network always has 128 channels);
  * with ``max_num_keypoints`` set, an image without NMS candidates gives zero rows (the reference's ``kthvalue``
    raises);
  * sizes that are not multiples of 16 with ``pad_if_not_divisible=False`` raise ``ValueError`` up front (the reference
    fails inside the U-Net), as does a padded image with a single pixel at 1/16 resolution (``F.instance_norm`` raises);
  * a batch whose images end with different keypoint counts raises ``ValueError`` (the reference's ``torch.stack``
    fails).
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
from torch import nn

from . import _cabi
from . import extractor as _extractor

DOWN = [16, 32, 64, 64, 64]
UP = [64, 64, 64, 129]


class _Module(nn.Module):
    """A bare parameter container (kornia's submodule names; the math runs in CUDA)."""


def _conv(ci: int, co: int) -> nn.Sequential:
    """kornia's ``Conv`` block: InstanceNorm2d (no parameters), PReLU, a parameter-free slot, Conv2d(5x5)."""
    return nn.Sequential(nn.InstanceNorm2d(ci), nn.PReLU(ci), nn.Identity(), nn.Conv2d(ci, co, 5, padding=2))


def _unet() -> _Module:
    unet = _Module()
    cins = [3] + DOWN[:-1]
    unet.path_down = nn.ModuleList(
        nn.Sequential(nn.AvgPool2d(2) if i else nn.Identity(), _conv(ci, co)) for i, (ci, co) in enumerate(zip(cins, DOWN)))
    unet.path_up = nn.ModuleList()
    for cb, ch, co in zip([DOWN[-1]] + UP[:-1], DOWN[-2::-1], UP):
        blk = _Module()
        blk.conv = _conv(cb + ch, co)
        unet.path_up.append(blk)
    return unet


class DISK(_extractor.CudaExtractor):
    _abi = "disk"
    default_conf = {
        "weights": "depth",
        "max_num_keypoints": None,
        "desc_dim": 128,
        "nms_window_size": 5,
        "detection_threshold": 0.0,
        "pad_if_not_divisible": True,
    }
    preprocess_conf = {
        "resize": 1024,
        "grayscale": False,
    }
    required_data_keys = ["image"]
    checkpoint_url = "https://raw.githubusercontent.com/cvlab-epfl/disk/master/{}-save.pth"

    def __init__(self, **conf):
        super().__init__()
        self.conf = c = SimpleNamespace(**{**self.default_conf, **conf})
        if c.desc_dim != 128:
            raise ValueError(f"desc_dim={c.desc_dim}: DISK's network has 128 descriptor channels")
        if c.weights not in ("depth", "epipolar", None):
            raise ValueError(f"weights={c.weights!r}: one of 'depth', 'epipolar' or None")
        w = c.nms_window_size
        if not isinstance(w, int) or isinstance(w, bool) or w < 1 or w % 2 == 0:
            raise ValueError(f"nms_window_size={w!r}: a positive odd int")
        n = c.max_num_keypoints
        if n is not None and (not isinstance(n, int) or isinstance(n, bool) or n < 0 or n >= 2**31):
            raise ValueError(f"max_num_keypoints={n!r}: None or an int >= 0")
        self.model = _Module()
        self.model.unet = _unet()
        if c.weights is not None:
            ckpt = _extractor.find_checkpoint(f"{c.weights}-save.pth", self.checkpoint_url.format(c.weights), "DISK")
            self.model.load_state_dict(ckpt["extractor"], strict=True)
        self.requires_grad_(False)
        self.eval()

    # ------------------------------------------------------------------ C handle
    def _config(self) -> _cabi.DiskConfig:
        c = self.conf
        n = -1 if c.max_num_keypoints is None else int(c.max_num_keypoints)
        return _cabi.DiskConfig(_cabi.DISK_ABI_VERSION, n, int(c.nms_window_size), int(bool(c.pad_if_not_divisible)),
                                float(c.detection_threshold))

    def _blob(self) -> torch.Tensor:
        """kornia's DISK state_dict in state_dict order (include/disk_b200.h)."""
        return torch.cat([t.detach().reshape(-1).to(torch.float32) for t in self.model.state_dict().values()]).contiguous()

    def _create(self, lib, cfg, blob, stream, out):
        assert blob.numel() == lib.disk_weight_blob_floats()
        _cabi.check(lib.disk_create(cfg, blob.data_ptr(), blob.numel(), stream, out), "disk_create")

    # ------------------------------------------------------------------ forward
    def _image(self, image: torch.Tensor) -> torch.Tensor:
        image = self._cuda_image(image)
        if image.dim() != 4 or image.shape[1] not in (1, 3):
            raise ValueError(f"image of shape {tuple(image.shape)}: expected [B, 1 or 3, H, W]")
        hh, ww = image.shape[-2:]
        if not self.conf.pad_if_not_divisible and (hh % 16 or ww % 16):
            raise ValueError(f"image size {ww}x{hh} is not a multiple of 16 and pad_if_not_divisible is off")
        if -(-hh // 16) * -(-ww // 16) < 2:
            raise ValueError(f"image size {ww}x{hh}: the padded image needs at least two pixels at 1/16 resolution")
        return image.detach().to(torch.float32).contiguous()

    @torch.no_grad()
    def forward(self, data: dict) -> dict:
        """keypoints [B, n, 2] (x, y pixels), keypoint_scores [B, n] and descriptors [B, n, 128] of an image batch
        [B, 1 or 3, H, W]; rows in row-major pixel order."""
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        image = self._image(data["image"])
        b, c, hh, ww = image.shape

        def call(lib, handle, cap, p, tail):
            return lib.disk_forward(handle, image.data_ptr(), c, b, hh, ww, cap, p["keypoints"], p["keypoint_scores"],
                                    p["descriptors"], *tail)

        return self._run(image, {"keypoints": (2,), "keypoint_scores": (), "descriptors": (128,)}, call)

    @torch.no_grad()
    def heads(self, image: torch.Tensor, pos: torch.Tensor):
        """The network alone (``disk_heads``): the heatmap [B, H, W] cropped to the image, and the raw (un-normalised)
        128 descriptor channels [B, P, 128] at the pixels ``pos`` [B, P] (flat index y W + x)."""
        image = self._image(image)
        b, c, hh, ww = image.shape
        pos = pos.to(device=image.device, dtype=torch.int32).reshape(b, -1).contiguous()
        if pos.numel() and (int(pos.min()) < 0 or int(pos.max()) >= hh * ww):
            raise ValueError("pos: pixel indices outside the image")
        device = image.device
        with torch.cuda.device(device):
            lib = _cabi.load()
            handle = self._get_handle(device)
            ws = self._workspace(lib, handle, device, b, hh, ww)
            heat = torch.empty(b, hh, ww, dtype=torch.float32, device=device)
            desc = torch.empty(b, pos.shape[1], 128, dtype=torch.float32, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(lib.disk_heads(handle, image.data_ptr(), c, b, hh, ww, pos.data_ptr(), pos.shape[1], heat.data_ptr(),
                                       desc.data_ptr(), ws.data_ptr(), ws.numel(), stream), "disk_heads")
        return heat, desc
