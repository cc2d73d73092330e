"""The classic baseline matcher: mutual nearest neighbours with Lowe's ratio test and a distance threshold on
unit-norm descriptors (C ABI ``include/nn_b200.h``, CUDA ``csrc/nn_api.cu``).

It needs no checkpoint, so any extractor of this package can be matched with it directly, and its output dict has
LightGlue's match keys, so ``matches0`` feeds ``lightglue_b200.geometry`` and ``match_ragged`` / ``match_pairs`` take it
in place of ``LightGlue``.  The similarities run on the tensor cores in split-bf16; the B x M x N similarity matrix is
never written to memory.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
from torch import nn

from . import _cabi


class NearestNeighborMatcher(nn.Module):
    """Nearest-neighbour matching of ``data = {"image0": {"descriptors" [B, M, D], optional "num_keypoints" [B]},
    "image1": {...}}``.  For unit descriptors d0_i, d1_j the squared distance is 2 (1 - d0_i . d1_j).  A row of image 0
    keeps its nearest neighbour j when ``ratio_thresh`` is None or its distance ratio to the second nearest is at most
    ``ratio_thresh`` (compared on squared distances), and ``distance_thresh`` is None or its distance is at most
    ``distance_thresh``; image 1 likewise.  ``mutual_check`` keeps a match only when both directions keep it.  The
    exact rules are stated in ``include/nn_b200.h``.

    Returns ``matches0`` [B, M] / ``matches1`` [B, N] int64 (-1 unmatched), ``matching_scores0`` / ``matching_scores1``
    float32 ((1 + d0_i . d1_j) / 2 for a match, else 0), and per pair ``matches`` [K_b, 2] (i, j) in ascending i with
    ``scores`` [K_b].  D is a multiple of 64 in [64, 512].

    Guided matching: ``forward(data, F=...)`` or ``forward(data, H=...)`` matches each pair again under its estimated
    fundamental matrix (x1^T F x0 = 0) or homography (image 0 -> image 1), [B, 3, 3] of any float dtype, as
    ``lightglue_b200.geometry`` returns them.  A candidate (i, j) counts only when its error under the model (the
    estimators' inlier error: the transfer error for H, the larger point-to-epipolar-line distance for F, squared) is
    below ``max_error``^2 pixels^2; the ratio, distance and mutual tests then run among those candidates only.  It needs
    ``data["image0"]["keypoints"]`` [B, M, 2] and ``data["image1"]["keypoints"]`` [B, N, 2].  A pair whose ``valid``
    [B] entry is zero (e.g. an estimator's ``success``) is matched ungated, exactly as without a model."""

    default_conf = {"ratio_thresh": None, "distance_thresh": None, "mutual_check": True}

    _handles: dict = {}  # device index -> NnHandle (the handle holds only a tensor-map cache)

    def __init__(self, **conf) -> None:
        super().__init__()
        unknown = set(conf) - set(self.default_conf)
        if unknown:
            raise ValueError(f"unknown NearestNeighborMatcher options: {sorted(unknown)}")
        self.conf = {**self.default_conf, **conf}
        r, t = self.conf["ratio_thresh"], self.conf["distance_thresh"]
        if r is not None and not (0.0 < float(r) <= 1.0):
            raise ValueError(f"ratio_thresh={r!r}: None or in (0, 1]")
        if t is not None and not (0.0 < float(t) < math.inf):
            raise ValueError(f"distance_thresh={t!r}: None or a positive number")

    @staticmethod
    def _guide(d0: dict, d1: dict, b: int, m: int, n: int, F, H, valid, max_error):
        """Checks the guided keywords; returns (kind, model, kpts0, kpts1, valid or None) as given."""
        if F is not None and H is not None:
            raise ValueError("give at most one of F and H")
        kind, model = (_cabi.NN_GUIDE_F, F) if F is not None else (_cabi.NN_GUIDE_H, H)
        if not isinstance(model, torch.Tensor) or not model.is_floating_point() or tuple(model.shape) != (b, 3, 3):
            shape = tuple(model.shape) if isinstance(model, torch.Tensor) else type(model).__name__
            raise ValueError(f"model {shape}: expected a float tensor [{b}, 3, 3]")
        try:
            err = float(max_error)
        except (TypeError, ValueError):
            raise ValueError(f"max_error={max_error!r}: a positive number of pixels") from None
        if not 0.0 < err < math.inf:
            raise ValueError(f"max_error={max_error!r}: a positive number of pixels")
        kps = []
        for name, img, rows in (("image0", d0, m), ("image1", d1, n)):
            k = img.get("keypoints")
            if k is None:
                raise ValueError(f"guided matching needs data[{name!r}]['keypoints']")
            if not isinstance(k, torch.Tensor) or tuple(k.shape) != (b, rows, 2):
                shape = tuple(k.shape) if isinstance(k, torch.Tensor) else type(k).__name__
                raise ValueError(f"{name} keypoints {shape}: expected [{b}, {rows}, 2]")
            kps.append(k.detach())
        if valid is not None:
            valid = torch.as_tensor(valid)
            if valid.reshape(-1).numel() != b or valid.dim() > 1:
                raise ValueError(f"valid {tuple(valid.shape)}: expected [{b}]")
            valid = valid.reshape(b)
        return kind, model.detach(), kps[0], kps[1], valid

    @classmethod
    def _handle(cls, device: torch.device):
        h = cls._handles.get(device.index)
        if h is None:
            h = C.c_void_p()
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(_cabi.load().nn_create(stream, C.byref(h)), "nn_create")
            cls._handles[device.index] = h
        return h

    def forward(self, data: dict, *, F=None, H=None, valid=None, max_error: float = 4.0) -> dict:
        d0, d1 = data["image0"], data["image1"]
        x0, x1 = d0["descriptors"], d1["descriptors"]
        if not isinstance(x0, torch.Tensor) or not isinstance(x1, torch.Tensor):
            raise ValueError("descriptors must be torch tensors")
        if x0.dim() != 3 or x1.dim() != 3:
            raise ValueError(f"descriptors {tuple(x0.shape)} and {tuple(x1.shape)}: expected [B, M, D] and [B, N, D]")
        b, m, dim = x0.shape
        n = x1.shape[1]
        if x1.shape[0] != b or x1.shape[2] != dim:
            raise ValueError(f"descriptors {tuple(x0.shape)} and {tuple(x1.shape)}: batch and D must agree")
        if dim % 64 or not _cabi.NN_MIN_DIM <= dim <= _cabi.NN_MAX_DIM:
            raise ValueError(f"descriptor size {dim}: a multiple of 64 in [{_cabi.NN_MIN_DIM}, {_cabi.NN_MAX_DIM}]")
        guide = None if F is None and H is None else self._guide(d0, d1, b, m, n, F, H, valid, max_error)
        if x0.device.type != "cuda" or x1.device.type != "cuda":
            raise RuntimeError("lightglue_b200.NearestNeighborMatcher runs on CUDA (sm_90a) tensors only; there is no "
                               "CPU path")
        if x1.device != x0.device:
            raise ValueError("descriptors must be on one device")
        device = x0.device
        x0 = x0.detach().to(torch.float32).contiguous()
        x1 = x1.detach().to(torch.float32).contiguous()
        if guide is not None:
            kind, model, kp0, kp1, ok = guide
            model = model.to(device=device, dtype=torch.float64).reshape(b, 9).contiguous()
            kp0 = kp0.to(device=device, dtype=torch.float32).contiguous()
            kp1 = kp1.to(device=device, dtype=torch.float32).contiguous()
            ok = None if ok is None else (ok.to(device) != 0).to(torch.uint8).contiguous()

        def lens(img, cap):
            t = img.get("num_keypoints")
            if t is None:
                return None
            t = torch.as_tensor(t, device=device).to(torch.int32).reshape(-1).contiguous()
            if t.numel() != b:
                raise ValueError("num_keypoints must hold one count per pair")
            return t.clamp(0, cap)

        l0, l1 = lens(d0, m), lens(d1, n)
        out = {
            "matches0": torch.empty(b, m, dtype=torch.int64, device=device),
            "matches1": torch.empty(b, n, dtype=torch.int64, device=device),
            "matching_scores0": torch.empty(b, m, dtype=torch.float32, device=device),
            "matching_scores1": torch.empty(b, n, dtype=torch.float32, device=device),
        }
        n_matches = torch.zeros(b, dtype=torch.int32, device=device)
        pairs = torch.empty(b, m, 2, dtype=torch.int64, device=device)
        pscores = torch.empty(b, m, dtype=torch.float32, device=device)
        if b > 0:
            r, t = self.conf["ratio_thresh"], self.conf["distance_thresh"]
            cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, dim, int(bool(self.conf["mutual_check"])),
                                 0.0 if r is None else float(r), 0.0 if t is None else float(t))
            ptr = lambda v: None if v is None else v.data_ptr()  # noqa: E731
            ins = _cabi.NnInputs(b, m, n, ptr(x0), ptr(x1), ptr(l0), ptr(l1))
            outs = _cabi.NnOutputs(*(ptr(out[k]) for k in ("matches0", "matches1", "matching_scores0",
                                                            "matching_scores1")),
                                   ptr(n_matches), ptr(pairs), ptr(pscores))
            with torch.cuda.device(device):
                lib = _cabi.load()
                handle = self._handle(device)
                stream = torch.cuda.current_stream(device).cuda_stream
                if guide is None:
                    ws = torch.empty(max(lib.nn_workspace_bytes(b, m, n, dim), 256), dtype=torch.uint8, device=device)
                    _cabi.check(lib.nn_match(handle, C.byref(cfg), C.byref(ins), C.byref(outs), ws.data_ptr(),
                                             ws.numel(), stream), "nn_match")
                else:
                    g = _cabi.NnGuide(kind, ptr(model), ptr(ok), ptr(kp0), ptr(kp1), float(max_error))
                    ws = torch.empty(max(lib.nn_guided_workspace_bytes(b, m, n, dim), 256), dtype=torch.uint8,
                                     device=device)
                    _cabi.check(lib.nn_match_guided(handle, C.byref(cfg), C.byref(ins), C.byref(g), C.byref(outs),
                                                    ws.data_ptr(), ws.numel(), stream), "nn_match_guided")
        counts = n_matches.tolist()  # the one read-back: the lengths of the per-pair lists
        out["matches"] = [pairs[i, : counts[i]] for i in range(b)]
        out["scores"] = [pscores[i, : counts[i]] for i in range(b)]
        return out
