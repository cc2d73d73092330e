"""Drop-in host mirror of ``lightglue.DoGHardNet`` (reference lightglue/dog_hardnet.py: the SIFT extractor's keypoints,
then kornia's ``LAFDescriptor(HardNet(pretrained=True))``) over the C ABI in ``include/doghardnet_b200.h``.

The forward runs in CUDA (``csrc/dhn_api.cu``): SIFT's detection exactly as ``lightglue_b200.SIFT`` runs it (without
its descriptor histograms, which the reference discards), then per keypoint the LAF ``laf_from_center_scale_ori(kpts,
6 scales, rad2deg(oris))``, a 32x32 patch sampled from the pyrdown pyramid of the float gray crop, and HardNet (its
first convolution on CUDA cores, the other six on tensor cores with split-bf16 operands).  This module holds HardNet's
parameters under kornia's names (``laf_desc.descriptor.features.*``; the checkpoint's ``["state_dict"]`` loads into
``laf_desc.descriptor`` with ``strict=True``) and passes them to the library as one blob.  CUDA tensors only, no CPU
path.

The conf keys are SIFT's, plus ``weights``: the HardNet checkpoint's file name, looked up offline through
``find_checkpoint`` (default ``checkpoint_liberty_with_aug.pth``), or ``None`` for randomly initialised weights.
``rootsift`` is accepted and ignored, as in the reference.

Deviations from the reference: those of ``lightglue_b200.SIFT`` (row order when a cut applies, ``backend`` and
``max_num_keypoints`` validation, a batch with unequal keypoint counts raises ``ValueError``).
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
from torch import nn

from . import _cabi
from . import extractor as _extractor
from .sift import SIFT

# (cin, cout, kernel, stride) of HardNet's seven convolutions (kornia.feature.HardNet.features)
LAYERS = [(1, 32, 3, 1), (32, 32, 3, 1), (32, 64, 3, 2), (64, 64, 3, 1), (64, 128, 3, 2), (128, 128, 3, 1), (128, 128, 8, 1)]
CHECKPOINT = "checkpoint_liberty_with_aug.pth"
CHECKPOINT_URL = ("https://github.com/DagnyT/hardnet/raw/master/pretrained/train_liberty_with_aug/"
                  "checkpoint_liberty_with_aug.pth")


class _Module(nn.Module):
    """A bare parameter container (kornia's submodule names; the math runs in CUDA)."""


def hardnet_features() -> nn.Sequential:
    """kornia's ``HardNet.features``: Conv / BatchNorm2d(affine=False) / ReLU triples, Dropout(0.1) before the last
    convolution, no ReLU after the last BatchNorm.  Indices of the convolutions: 0, 3, 6, 9, 12, 15, 19."""
    mods = []
    for i, (ci, co, k, s) in enumerate(LAYERS):
        if i == len(LAYERS) - 1:
            mods.append(nn.Dropout(0.1))
        mods += [nn.Conv2d(ci, co, k, stride=s, padding=1 if k == 3 else 0, bias=False), nn.BatchNorm2d(co, affine=False)]
        if i < len(LAYERS) - 1:
            mods.append(nn.ReLU())
    return nn.Sequential(*mods)


class DoGHardNet(_extractor.CudaExtractor):
    _abi = "dhn"
    default_conf = {**SIFT.default_conf, "weights": CHECKPOINT}
    preprocess_conf = dict(SIFT.preprocess_conf)
    required_data_keys = ["image"]

    def __init__(self, **conf):
        super().__init__()
        self.conf = c = SimpleNamespace(**{**self.default_conf, **conf})
        if c.backend != "opencv":
            raise ValueError(f"backend {c.backend!r}: lightglue_b200.DoGHardNet implements backend='opencv' only")
        k = c.max_num_keypoints
        if not isinstance(k, int) or isinstance(k, bool) or k <= 0 or k >= 2**31:
            raise ValueError(f"max_num_keypoints={k!r}: must be a positive int")
        if c.nms_radius is not None and int(c.nms_radius) < 0:
            raise ValueError(f"nms_radius={c.nms_radius!r}: must be >= 0 or None")
        if not 1 <= int(c.num_octaves) <= 8:
            raise ValueError(f"num_octaves={c.num_octaves!r}: must be in [1, 8]")
        if c.weights is not None and not isinstance(c.weights, str):
            raise ValueError(f"weights={c.weights!r}: a checkpoint file name or None")
        self.laf_desc = _Module()
        self.laf_desc.descriptor = _Module()
        self.laf_desc.descriptor.features = hardnet_features()
        if c.weights is not None:
            ckpt = _extractor.find_checkpoint(c.weights, CHECKPOINT_URL, "DoGHardNet")
            self.laf_desc.descriptor.load_state_dict(ckpt["state_dict"], strict=True)
        self.requires_grad_(False)
        self.eval()

    # ------------------------------------------------------------------ C handle
    def _config(self) -> _cabi.DhnConfig:
        c = self.conf
        return _cabi.DhnConfig(
            abi_version=_cabi.DHN_ABI_VERSION, num_octave_layers=int(c.num_octaves),
            nms_radius=-1 if c.nms_radius is None else int(c.nms_radius), max_num_keypoints=int(c.max_num_keypoints),
            detection_threshold=float(c.detection_threshold), edge_threshold=float(c.edge_threshold),
        )

    def _blob(self) -> torch.Tensor:
        """Per convolution: its weight, then its BatchNorm's running mean and variance (include/doghardnet_b200.h)."""
        f = self.laf_desc.descriptor.features
        parts = []
        for m, bn in zip(f, f[1:]):
            if isinstance(m, nn.Conv2d):
                parts += [m.weight, bn.running_mean, bn.running_var]
        return torch.cat([t.detach().reshape(-1).to(torch.float32) for t in parts]).contiguous()

    def _create(self, lib, cfg, blob, stream, out):
        assert blob.numel() == lib.dhn_weight_blob_floats()
        _cabi.check(lib.dhn_create(cfg, blob.data_ptr(), blob.numel(), stream, out), "dhn_create")

    # ------------------------------------------------------------------ forward
    def _image(self, image: torch.Tensor) -> torch.Tensor:
        image = self._cuda_image(image)
        if image.dim() != 4 or image.shape[1] not in (1, 3):
            raise ValueError(f"image of shape {tuple(image.shape)}: expected [B, 1 or 3, H, W]")
        return image.detach().to(torch.float32).contiguous()

    @staticmethod
    def _size(size, b: int):
        if size is None:
            return None
        return torch.as_tensor(size).reshape(b, 2).cpu().to(torch.int32).contiguous()  # host copy: shapes depend on it

    @torch.no_grad()
    def forward(self, data: dict) -> dict:
        """keypoints [B, n, 2], scales [B, n], oris [B, n] (radians), keypoint_scores [B, n] as ``SIFT`` gives them,
        and HardNet descriptors [B, n, 128] (unit norm)."""
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        image = self._image(data["image"])
        b, c, hh, ww = image.shape
        size = self._size(data.get("image_size"), b)

        def call(lib, handle, cap, p, tail):
            return lib.dhn_forward(handle, image.data_ptr(), c, size.data_ptr() if size is not None else None, b, hh, ww,
                                   cap, p["keypoints"], p["scales"], p["oris"], p["keypoint_scores"], p["descriptors"],
                                   *tail)

        return self._run(image, {"keypoints": (2,), "scales": (), "oris": (), "keypoint_scores": (), "descriptors": (128,)},
                         call)

    @torch.no_grad()
    def describe(self, image: torch.Tensor, keypoints: torch.Tensor, scales: torch.Tensor, oris: torch.Tensor,
                 counts=None, image_size=None) -> torch.Tensor:
        """kornia's ``LAFDescriptor(HardNet)`` for the reference's LAFs of given keypoints [B, n, 2], scales [B, n]
        (cv2 sizes) and oris [B, n] (radians) on the gray crop of each image: descriptors [B, n, 128].  ``counts`` [B]:
        only the first counts[b] rows of image b are described, the others are zero (default: all n)."""
        image = self._image(image)
        b, c, hh, ww = image.shape
        dev = image.device
        n = keypoints.shape[1]
        if n > self.conf.max_num_keypoints:
            raise ValueError(f"{n} keypoints per image: at most max_num_keypoints={self.conf.max_num_keypoints}")
        kp = keypoints.to(device=dev, dtype=torch.float32).reshape(b, n, 2).contiguous()
        sc = scales.to(device=dev, dtype=torch.float32).reshape(b, n).contiguous()
        ori = oris.to(device=dev, dtype=torch.float32).reshape(b, n).contiguous()
        cnt = torch.full((b,), n, dtype=torch.int32) if counts is None else torch.as_tensor(counts).reshape(b)
        cnt = cnt.to(device=dev, dtype=torch.int32).contiguous()
        size = self._size(image_size, b)
        desc = torch.zeros(b, n, 128, dtype=torch.float32, device=dev)
        if n == 0:
            return desc
        with torch.cuda.device(dev):
            lib = _cabi.load()
            handle = self._get_handle(dev)
            ws = self._workspace(lib, handle, dev, b, hh, ww)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _cabi.check(lib.dhn_describe(handle, image.data_ptr(), c, size.data_ptr() if size is not None else None, b, hh,
                                         ww, n, kp.data_ptr(), sc.data_ptr(), ori.data_ptr(), cnt.data_ptr(),
                                         desc.data_ptr(), ws.data_ptr(), ws.numel(), stream), "dhn_describe")
        return desc
