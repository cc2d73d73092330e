"""Drop-in host mirror of ``lightglue.SuperPoint`` (reference lightglue/superpoint.py:99-227) over the C ABI in
``include/superpoint_b200.h`` -- the caller-side row next to the matcher (SURVEY.md 8f1).

First CUDA path: fp32 on CUDA cores (``csrc/sp_pipeline.h``), no tensor cores yet.  Same parameter names, conf keys
and output dict as the reference; CUDA tensors only, no CPU path.  What is host glue here and not kernels: the
RGB -> gray weighting the reference takes from kornia (``rgb_to_grayscale``: 0.299 R + 0.587 G + 0.114 B) and the
optional resize of ``extract`` (the reference uses kornia's antialiased resize, utils.py:17-38; here
``F.interpolate(..., mode="bilinear", antialias=True)``).
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace

import torch
from torch import nn

from . import _cabi
from . import extractor as _extractor

LAYERS = (  # name, out channels, in channels, kernel   (superpoint.py:137-153)
    ("conv1a", 64, 1, 3), ("conv1b", 64, 64, 3), ("conv2a", 64, 64, 3), ("conv2b", 64, 64, 3),
    ("conv3a", 128, 64, 3), ("conv3b", 128, 128, 3), ("conv4a", 128, 128, 3), ("conv4b", 128, 128, 3),
    ("convPa", 256, 128, 3), ("convPb", 65, 256, 1), ("convDa", 256, 128, 3), ("convDb", 256, 256, 1),
)


class SuperPoint(nn.Module):
    default_conf = {  # superpoint.py:112-118
        "descriptor_dim": 256,
        "nms_radius": 4,
        "max_num_keypoints": None,
        "detection_threshold": 0.0005,
        "remove_borders": 4,
        # extension: None = keep the (random) initial parameters instead of looking for superpoint_v1.pth
        "weights": "superpoint_v1",
        # extension: arithmetic of the twelve convolutions -- "bf16x3" (wgmma tensor cores, split-bf16 operands,
        # fp32 accumulate) or "fp32" (CUDA cores: the checker the tensor-core path is validated against)
        "precision": "bf16x3",
    }
    preprocess_conf = {"resize": 1024}  # superpoint.py:120-122
    required_data_keys = ["image"]
    url = "https://github.com/cvg/LightGlue/releases/download/v0.1_arxiv/superpoint_v1.pth"

    def __init__(self, **conf):
        super().__init__()
        self.conf = SimpleNamespace(**{**self.default_conf, **conf})
        if self.conf.descriptor_dim != 256:
            raise ValueError("descriptor_dim is fixed to 256 by the SuperPoint weights")
        if self.conf.precision not in ("fp32", "bf16x3"):
            raise ValueError("precision must be 'fp32' or 'bf16x3'")
        if self.conf.max_num_keypoints is not None and self.conf.max_num_keypoints <= 0:
            raise ValueError("max_num_keypoints must be positive or None")  # superpoint.py:158-159
        for name, co, ci, k in LAYERS:  # parameter containers with the reference's names; the math runs in CUDA
            setattr(self, name, nn.Conv2d(ci, co, kernel_size=k, stride=1, padding=k // 2))
        if self.conf.weights is not None:
            self.load_state_dict(self._find_checkpoint(f"{self.conf.weights}.pth"))
        self.requires_grad_(False)
        self._handle = None  # (C handle, device index, weight signature)
        self._ws = {}

    def _find_checkpoint(self, fname: str):
        """The reference downloads the checkpoint (155-156); offline we look in the usual caches."""
        return _extractor.find_checkpoint(fname, self.url, "SuperPoint")

    # ------------------------------------------------------------------ C handle
    def _blob(self) -> torch.Tensor:
        parts = []
        for name, *_ in LAYERS:
            m = getattr(self, name)
            parts += [m.weight.detach().reshape(-1), m.bias.detach().reshape(-1)]
        return torch.cat(parts).to(torch.float32).contiguous()

    def _get_handle(self, device: torch.device):
        lib = _cabi.load()
        sig = (device.index, tuple(int(getattr(self, n).weight._version) for n, *_ in LAYERS),
               self.conf.nms_radius, self.conf.max_num_keypoints, self.conf.remove_borders, self.conf.detection_threshold,
               self.conf.precision)
        if self._handle is not None and self._handle[1] == sig:
            return self._handle[0]
        self._release()
        blob = self._blob().to(device)
        assert blob.numel() == lib.sp_weight_blob_floats()
        cfg = _cabi.SpConfig(_cabi.SP_ABI_VERSION, int(self.conf.nms_radius), int(self.conf.max_num_keypoints or 0),
                             int(self.conf.remove_borders), float(self.conf.detection_threshold),
                             1 if self.conf.precision == "bf16x3" else 0)
        h = C.c_void_p()
        stream = torch.cuda.current_stream(device).cuda_stream
        _cabi.check(lib.sp_create(C.byref(cfg), blob.data_ptr(), blob.numel(), stream, C.byref(h)), "sp_create")
        torch.cuda.current_stream(device).synchronize()  # the blob may be freed once the copy has run
        self._handle = (h, sig)
        return h

    def _release(self):
        try:
            if getattr(self, "_handle", None) is not None:  # (the constructor may have raised before the attribute exists)
                _cabi.load().sp_destroy(self._handle[0])
                object.__setattr__(self, "_handle", None)
        except Exception:  # noqa: BLE001  (interpreter shutdown: modules may already be torn down)
            pass

    def __del__(self):
        self._release()

    # ------------------------------------------------------------------ forward
    @staticmethod
    def _gray(image: torch.Tensor) -> torch.Tensor:
        """[B, 1 or 3, H, W] CUDA image -> contiguous fp32 [B, 1, H, W]."""
        if image.device.type != "cuda":
            raise RuntimeError("lightglue_b200.SuperPoint runs on CUDA (sm_90a) tensors only; there is no CPU path")
        if image.shape[1] == 3:  # kornia.color.rgb_to_grayscale's weights (superpoint.py:168-169)
            wts = torch.tensor([0.299, 0.587, 0.114], device=image.device, dtype=image.dtype).view(1, 3, 1, 1)
            image = (image * wts).sum(1, keepdim=True)
        _, c, hh, ww = image.shape
        assert c == 1
        if hh < 8 or ww < 8:
            raise ValueError(f"image size {ww}x{hh}: height and width must be at least 8 (one detector cell)")
        return image.detach().to(torch.float32).contiguous()

    def _workspace(self, lib, handle, device: torch.device, b: int, hh: int, ww: int) -> torch.Tensor:
        key = (device.index, b, hh, ww)
        ws = self._ws.get(key)
        if ws is None:
            self._ws.clear()
            ws = self._ws[key] = torch.empty(int(lib.sp_workspace_bytes(handle, b, hh, ww)), dtype=torch.uint8, device=device)
        return ws

    @torch.no_grad()
    def forward(self, data: dict) -> dict:
        """Keypoints, scores and descriptors of an image batch (superpoint.py:163-227)."""
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        image = self._gray(data["image"])
        b, _, hh, ww = image.shape
        device = image.device
        with torch.cuda.device(device):
            lib = _cabi.load()
            handle = self._get_handle(device)
            cap = int(lib.sp_max_keypoints(handle, hh, ww))
            ws = self._workspace(lib, handle, device, b, hh, ww)
            kpts = torch.empty(b, cap, 2, dtype=torch.float32, device=device)
            scores = torch.empty(b, cap, dtype=torch.float32, device=device)
            desc = torch.empty(b, cap, 256, dtype=torch.float32, device=device)
            counts = torch.empty(b, dtype=torch.int32, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(
                lib.sp_forward(handle, image.data_ptr(), b, hh, ww, cap, kpts.data_ptr(), scores.data_ptr(), desc.data_ptr(),
                               counts.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                "sp_forward",
            )
            n = counts.cpu().tolist()  # the one host read-back: keypoint counts
        if len(set(n)) != 1:  # the reference stacks the per-image results (223-227), which needs equal counts
            raise ValueError(f"images of the batch have different keypoint counts {n}; set max_num_keypoints or batch 1")
        k = n[0]
        return {
            "keypoints": kpts[:, :k].contiguous(),
            "keypoint_scores": scores[:, :k].contiguous(),
            "descriptors": desc[:, :k].contiguous(),
        }

    @torch.no_grad()
    def backbone_heads(self, image: torch.Tensor):
        """Block-level parity (``sp_backbone``): the convolution stack alone, as ``forward`` runs it in this precision --
        the detector logits ``[B, 65, H/8, W/8]`` (superpoint.py:185) and the un-normalised descriptor map
        ``[B, 256, H/8, W/8]`` (221), fp32."""
        image = self._gray(image)
        b, _, hh, ww = image.shape
        device = image.device
        with torch.cuda.device(device):
            lib = _cabi.load()
            handle = self._get_handle(device)
            ws = self._workspace(lib, handle, device, b, hh, ww)
            logits = torch.empty(b, 65, hh // 8, ww // 8, dtype=torch.float32, device=device)
            dense = torch.empty(b, 256, hh // 8, ww // 8, dtype=torch.float32, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(lib.sp_backbone(handle, image.data_ptr(), b, hh, ww, logits.data_ptr(), dense.data_ptr(), ws.data_ptr(),
                                        ws.numel(), stream), "sp_backbone")
        return logits, dense

    @torch.no_grad()
    def extract(self, img: torch.Tensor, **conf) -> dict:
        """``Extractor.extract`` (utils.py:136-147): resize, ``forward``, keypoints back in the original pixels
        (lightglue_b200/extractor.py)."""
        return _extractor.extract(self, img, **conf)
