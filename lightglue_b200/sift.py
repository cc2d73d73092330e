"""Drop-in host mirror of ``lightglue.SIFT`` (reference lightglue/sift.py, ``backend="opencv"``) over the C ABI in
``include/sift_b200.h``.

The forward runs in CUDA (``csrc/sift_api.cu`` over the functors of ``csrc/sift_pipeline.h``, fp32 on CUDA cores):
gray conversion, the ``image_size`` crop, the reference's 8-bit quantisation, OpenCV's SIFT (2x upsampled first octave,
scale space, extrema, refinement, orientations, descriptors, duplicate removal and the ``nfeatures`` cut),
``filter_dog_point``, the top-k and RootSIFT.  The reference copies every image to the host and runs OpenCV there.
CUDA tensors only, no CPU path.

The conf keys are the reference's.  As there, ``num_octaves`` is passed to OpenCV as the number of layers per octave
(nOctaveLayers); ``first_octave`` only concerns the pycolmap backends and is ignored.

Deviations from the reference:
  * when the ``nfeatures`` cut or the top-k applies, the rows are in descending score, ties in OpenCV's order (the
    reference's order is then whatever ``nth_element`` / ``torch.topk`` leave); otherwise they are in OpenCV's
    (x, y, size desc, angle, response desc) order, as the reference's are;
  * ``backend`` values other than ``"opencv"`` raise ``ValueError``, and ``max_num_keypoints`` must be a positive int;
  * a batch whose images end with different keypoint counts raises ``ValueError`` (the reference's ``torch.stack``
    fails);
  * with ``image_size``, the sizes are read back to the host (the pyramid's shapes depend on them); the keypoint counts
    are read back once per call, as in the other extractors.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from . import _cabi
from . import extractor as _extractor


class SIFT(_extractor.CudaExtractor):
    _abi = "sift"
    default_conf = {
        "rootsift": True,
        "nms_radius": 0,  # None to disable filtering entirely.
        "max_num_keypoints": 4096,
        "backend": "opencv",  # in {opencv, pycolmap, pycolmap_cpu, pycolmap_cuda}
        "detection_threshold": 0.0066667,  # from COLMAP
        "edge_threshold": 10,
        "first_octave": -1,  # only used by pycolmap, the default of COLMAP
        "num_octaves": 4,
    }

    preprocess_conf = {
        "resize": 1024,
    }

    required_data_keys = ["image"]

    def __init__(self, **conf):
        super().__init__()
        self.conf = SimpleNamespace(**{**self.default_conf, **conf})
        if self.conf.backend != "opencv":
            raise ValueError(f"backend {self.conf.backend!r}: lightglue_b200.SIFT implements backend='opencv' only")
        k = self.conf.max_num_keypoints
        if not isinstance(k, int) or k <= 0:
            raise ValueError(f"max_num_keypoints={k!r}: must be a positive int")
        if self.conf.nms_radius is not None and int(self.conf.nms_radius) < 0:
            raise ValueError(f"nms_radius={self.conf.nms_radius!r}: must be >= 0 or None")
        if not 1 <= int(self.conf.num_octaves) <= 8:
            raise ValueError(f"num_octaves={self.conf.num_octaves!r}: must be in [1, 8]")

    def _config(self) -> _cabi.SiftConfig:
        c = self.conf
        return _cabi.SiftConfig(
            abi_version=_cabi.SIFT_ABI_VERSION, num_octave_layers=int(c.num_octaves),
            nms_radius=-1 if c.nms_radius is None else int(c.nms_radius), max_num_keypoints=int(c.max_num_keypoints),
            rootsift=int(bool(c.rootsift)), reserved=0, detection_threshold=float(c.detection_threshold),
            edge_threshold=float(c.edge_threshold),
        )

    def _create(self, lib, cfg, blob, stream, out):
        _cabi.check(lib.sift_create(cfg, None, out), "sift_create")

    @torch.no_grad()
    def forward(self, data: dict) -> dict:
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        image = self._cuda_image(data["image"])
        b, c, hh, ww = image.shape
        if c not in (1, 3):
            raise ValueError(f"image has {c} channels: expected 1 (gray) or 3 (RGB)")
        image = image.detach().to(torch.float32).contiguous()
        size = data.get("image_size")
        if size is not None:  # host copy: the pyramid's shapes depend on it
            size = torch.as_tensor(size).reshape(b, 2).cpu().to(torch.int32).contiguous()

        def call(lib, handle, cap, p, tail):
            return lib.sift_forward(handle, image.data_ptr(), c, size.data_ptr() if size is not None else None, b, hh, ww,
                                    cap, p["keypoints"], p["scales"], p["oris"], p["keypoint_scores"], p["descriptors"],
                                    *tail)

        return self._run(image, {"keypoints": (2,), "scales": (), "oris": (), "keypoint_scores": (), "descriptors": (128,)},
                         call)
