"""Host shell shared by the extractors (``SuperPoint``, ``ALIKED``, ``SIFT``, ``DISK``, ``DoGHardNet``): checkpoint
lookup, the C handle and workspace caches, the forward call with its output allocation and count read-back, and
``Extractor.extract``."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch
from torch import nn

from . import _cabi


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


class CudaExtractor(nn.Module):
    """One C handle per module, rebuilt whenever the device, the config struct or any parameter or buffer (identity or
    in-place version) changes, plus the workspace cache and the forward call.  A subclass names its C prefix
    (``_abi``: ``{_abi}_max_keypoints`` / ``_workspace_bytes`` / ``_destroy``) and supplies ``_config()``, ``_blob()``
    (``None`` when the handle takes no weights) and ``_create()``."""

    _abi: str

    def __init__(self):
        super().__init__()
        self._handle = None  # (C handle, signature)
        self._ws = {}

    def _blob(self):
        return None

    def _signature(self, device: torch.device) -> tuple:
        tensors = list(self.parameters()) + list(self.buffers())
        return device.index, bytes(self._config()), tuple((t.data_ptr(), t._version) for t in tensors)

    def _get_handle(self, device: torch.device):
        sig = self._signature(device)
        if self._handle is not None and self._handle[1] == sig:
            return self._handle[0]
        self._release()
        self._ws.clear()  # the workspace size depends on the config
        lib = _cabi.load()
        blob = self._blob()
        if blob is not None:
            blob = blob.to(device)
        h = C.c_void_p()
        stream = torch.cuda.current_stream(device)
        self._create(lib, C.byref(self._config()), blob, stream.cuda_stream, C.byref(h))
        if blob is not None:
            stream.synchronize()  # the blob may be freed once the copy has run
        self._handle = (h, sig)
        return h

    def _release(self):
        try:
            handle = self.__dict__.get("_handle")  # (the constructor may have raised before the attribute exists)
            if handle is not None and _cabi._lib is not None:  # never load (or build) the library from here
                getattr(_cabi._lib, f"{self._abi}_destroy")(handle[0])
            self.__dict__["_handle"] = None
        except Exception:  # noqa: BLE001  (interpreter shutdown: modules may already be torn down)
            pass

    def __del__(self):
        self._release()

    def _cuda_image(self, image: torch.Tensor) -> torch.Tensor:
        if image.device.type != "cuda":
            raise RuntimeError(
                f"lightglue_b200.{type(self).__name__} runs on CUDA (sm_90a) tensors only; there is no CPU path")
        return image

    def _workspace(self, lib, handle, device: torch.device, b: int, hh: int, ww: int) -> torch.Tensor:
        key = (device.index, b, hh, ww)
        ws = self._ws.get(key)
        if ws is None:
            self._ws.clear()
            nbytes = int(getattr(lib, f"{self._abi}_workspace_bytes")(handle, b, hh, ww))
            ws = self._ws[key] = torch.empty(nbytes, dtype=torch.uint8, device=device)
        return ws

    def _run(self, image: torch.Tensor, outputs: dict, call) -> dict:
        """Allocate the fp32 outputs ``{name: trailing shape}`` at the keypoint cap, run the C forward through
        ``call(lib, handle, cap, ptrs, tail)`` -- ``ptrs`` maps each name to its pointer, ``tail`` is (counts,
        workspace, workspace bytes, stream) -- read the counts back once and return the rows of every image, in the
        order of ``outputs``."""
        b, _, hh, ww = image.shape
        device = image.device
        with torch.cuda.device(device):
            lib = _cabi.load()
            handle = self._get_handle(device)
            cap = int(getattr(lib, f"{self._abi}_max_keypoints")(handle, hh, ww))
            ws = self._workspace(lib, handle, device, b, hh, ww)
            out = {k: torch.empty(b, cap, *s, dtype=torch.float32, device=device) for k, s in outputs.items()}
            counts = torch.empty(b, dtype=torch.int32, device=device)
            tail = (counts.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream)
            _cabi.check(call(lib, handle, cap, {k: t.data_ptr() for k, t in out.items()}, tail), f"{self._abi}_forward")
            n = counts.cpu().tolist()  # the one host read-back: keypoint counts
        if min(n) < 0:
            raise RuntimeError(f"{self._abi}_forward: an image has more raw keypoints than the internal list holds "
                               f"(counts {n})")
        if len(set(n)) != 1:  # the reference stacks the per-image results, which needs equal counts
            raise ValueError(f"images of the batch have different keypoint counts {n}; set max_num_keypoints or batch 1")
        k = n[0]
        return {name: t[:, :k].contiguous() for name, t in out.items()}

    @torch.no_grad()
    def extract(self, img: torch.Tensor, **conf) -> dict:
        """``Extractor.extract`` (utils.py:136-147): add the batch dimension, resize the longer side to ``resize``
        (``ImagePreprocessor``, utils.py:26-38: ``kornia.geometry.transform.resize(side="long", antialias=True)``: the
        long side becomes ``resize`` and the other ``int(resize / aspect)`` -- truncated, kornia's
        ``_side_to_image_size``; kornia itself is not a dependency here), run ``forward``, map keypoints back to the
        original pixels.  Other outputs (SIFT's ``scales``) are returned as ``forward`` gives them, as in the
        reference."""
        if img.dim() == 3:
            img = img[None]
        assert img.dim() == 4 and img.shape[0] == 1
        h, w = img.shape[-2:]
        resize = {**self.preprocess_conf, **conf}.get("resize")
        nh, nw = h, w
        if resize is not None:
            aspect = w / h
            nh, nw = (int(resize / aspect), int(resize)) if aspect >= 1.0 else (int(resize), int(resize * aspect))
        if (nh, nw) != (h, w):
            img = torch.nn.functional.interpolate(img, size=(nh, nw), mode="bilinear", antialias=True, align_corners=False)
        scales = torch.tensor([nw / w, nh / h], device=img.device, dtype=torch.float32)
        feats = self.forward({"image": img})
        feats["image_size"] = torch.tensor([[w, h]], device=img.device, dtype=torch.float32)
        feats["keypoints"] = (feats["keypoints"] + 0.5) / scales[None] - 0.5
        return feats
