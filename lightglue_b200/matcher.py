"""Drop-in ``LightGlue`` matcher whose forward runs entirely in liblightglue_b200.so (sm_90a CUDA).

Host-side mirror of the reference interface (reference: lightglue/lightglue.py:321-662):

* same constructor ``LightGlue(features="superpoint", **conf)``, same ``default_conf`` keys, same
  class attributes (``pruning_keypoint_thresholds``, ``features``, ``required_data_keys``,
  ``version``, ``url``), ``compile()`` accepted;
* an ``nn.Module`` whose parameters carry the reference's state_dict key names, so official
  ``*_lightglue.pth`` checkpoints (and legacy-named ones, 427-434) load unchanged;
* ``forward({"image0": ..., "image1": ...})`` returns the reference's output dict (keys, shapes and
  dtypes, 619-629), including the empty-input special case (568-588).

There is no PyTorch implementation of the math in this file and no CPU path: tensors must live on a
CUDA device and the C library must load, otherwise the call raises.  PyTorch only provides device
memory, the current stream and the module/state_dict plumbing.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from pathlib import Path
from types import SimpleNamespace
from typing import Dict, List, Optional

import numpy as np
import torch
from torch import nn

from . import _cabi

DIM = 256


def _block(kind: str) -> nn.Module:
    """Parameter container for one SelfBlock / CrossBlock (reference 140-157 / 175-192)."""
    m = nn.Module()
    if kind == "self":
        m.Wqkv = nn.Linear(DIM, 3 * DIM)
        m.out_proj = nn.Linear(DIM, DIM)
    else:
        m.to_qk = nn.Linear(DIM, DIM)
        m.to_v = nn.Linear(DIM, DIM)
        m.to_out = nn.Linear(DIM, DIM)
    m.ffn = nn.Sequential(nn.Linear(2 * DIM, 2 * DIM), nn.LayerNorm(2 * DIM), nn.GELU(), nn.Linear(2 * DIM, DIM))
    return m


def _holder(**children: nn.Module) -> nn.Module:
    m = nn.Module()
    for k, v in children.items():
        m.add_module(k, v)
    return m


class LightGlue(nn.Module):
    default_conf = {
        "name": "lightglue",
        "input_dim": 256,
        "descriptor_dim": 256,
        "add_scale_ori": False,
        "n_layers": 9,
        "num_heads": 4,
        "flash": True,  # kept for interface compatibility; selects the "flash" pruning threshold
        "mp": False,  # kept for interface compatibility (the kernels choose their own arithmetic)
        "depth_confidence": 0.95,
        "width_confidence": 0.99,
        "filter_threshold": 0.1,
        "weights": None,
        # extension: arithmetic of the linear layers -- "fp32" | "bf16" | "bf16x3" (see LG_PREC_*)
        "precision": "bf16x3",
        # extension: replay the ~100 kernel launches of a forward as one CUDA graph per input shape (the
        # kernels take ragged / pruned lengths from device memory, so the launch sequence is static)
        "cuda_graph": False,
    }

    # reference lightglue.py:339-344; callers mutate it (benchmark.py:178-181)
    pruning_keypoint_thresholds = {"cpu": -1, "mps": -1, "cuda": 1024, "flash": 1536}
    required_data_keys = ["image0", "image1"]
    version = "v0.1_arxiv"
    url = "https://github.com/cvg/LightGlue/releases/download/{}/{}_lightglue.pth"
    features = {
        "superpoint": {"weights": "superpoint_lightglue", "input_dim": 256},
        "disk": {"weights": "disk_lightglue", "input_dim": 128},
        "aliked": {"weights": "aliked_lightglue", "input_dim": 128},
        "sift": {"weights": "sift_lightglue", "input_dim": 128, "add_scale_ori": True},
        "doghardnet": {"weights": "doghardnet_lightglue", "input_dim": 128, "add_scale_ori": True},
    }

    def __init__(self, features: Optional[str] = "superpoint", **conf) -> None:
        super().__init__()
        self.conf = conf = SimpleNamespace(**{**self.default_conf, **conf})
        if features is not None:
            if features not in self.features:
                raise ValueError(f"Unsupported features: {features} not in {{{','.join(self.features)}}}")
            for k, v in self.features[features].items():
                setattr(conf, k, v)
        if conf.descriptor_dim != DIM or conf.num_heads != 4:
            raise ValueError("the sm_90a kernels are specialised for descriptor_dim=256, num_heads=4")
        if conf.precision not in _cabi.PREC:
            raise ValueError(f"precision must be one of {sorted(_cabi.PREC)}")
        n = conf.n_layers
        self.input_proj = nn.Linear(conf.input_dim, DIM) if conf.input_dim != DIM else nn.Identity()
        wr = nn.Linear(2 + 2 * conf.add_scale_ori, 32, bias=False)
        nn.init.normal_(wr.weight.data, mean=0.0, std=1.0)
        self.posenc = _holder(Wr=wr)
        self.transformers = nn.ModuleList(
            [_holder(self_attn=_block("self"), cross_attn=_block("cross")) for _ in range(n)]
        )
        self.log_assignment = nn.ModuleList(
            [_holder(matchability=nn.Linear(DIM, 1), final_proj=nn.Linear(DIM, DIM)) for _ in range(n)]
        )
        self.token_confidence = nn.ModuleList(
            [_holder(token=nn.Sequential(nn.Linear(DIM, 1), nn.Sigmoid())) for _ in range(n - 1)]
        )
        thr = np.clip(0.8 + 0.1 * np.exp(-4.0 * np.arange(n) / n), 0, 1)  # reference 631-634
        self.register_buffer("confidence_thresholds", torch.tensor(thr, dtype=torch.float32))

        state_dict = None
        if features is not None:
            state_dict = self._find_checkpoint(f"{conf.weights}_{self.version.replace('.', '-')}.pth", features)
        elif conf.weights is not None:
            path = Path(__file__).parent / "weights" / f"{conf.weights}.pth"
            state_dict = torch.load(str(path), map_location="cpu")
        if state_dict:
            self.load_state_dict(self._rename_legacy(state_dict, n), strict=False)

        self.static_lengths = None
        self.requires_grad_(False)
        self._handle = None  # (C handle, signature: device index + precision / thresholds + identity of the packed weights)
        self._ws: Dict[tuple, torch.Tensor] = {}
        self._graphs: Dict[tuple, tuple] = {}
        self._meta_pool: Dict[int, list] = {}  # batch size -> free pinned [2, B] int32 read-back buffers
        self.timing = False

    # ------------------------------------------------------------------ weights
    def _find_checkpoint(self, fname: str, features: str):
        """Reference 416-421 downloads the checkpoint; offline we look in the usual caches first."""
        cands = [
            Path(os.environ.get("LIGHTGLUE_WEIGHTS_DIR", "")) / fname if os.environ.get("LIGHTGLUE_WEIGHTS_DIR") else None,
            Path(torch.hub.get_dir()) / "checkpoints" / fname,
            Path(__file__).parent / "weights" / fname,
        ]
        for c in cands:
            if c is not None and c.exists():
                return torch.load(str(c), map_location="cpu")
        return torch.hub.load_state_dict_from_url(self.url.format(self.version, features), file_name=fname)

    @staticmethod
    def _rename_legacy(sd: dict, n_layers: int) -> dict:
        for i in range(n_layers):  # reference 427-433
            sd = {k.replace(f"self_attn.{i}", f"transformers.{i}.self_attn"): v for k, v in sd.items()}
            sd = {k.replace(f"cross_attn.{i}", f"transformers.{i}.cross_attn"): v for k, v in sd.items()}
        return sd

    def _blob_tensors(self) -> List[torch.Tensor]:
        """Parameters in the canonical order of the C-ABI weight blob (include/lightglue_b200.h)."""
        ts: List[torch.Tensor] = [self.posenc.Wr.weight]
        if isinstance(self.input_proj, nn.Linear):
            ts += [self.input_proj.weight, self.input_proj.bias]
        for t in self.transformers:
            s, c = t.self_attn, t.cross_attn
            ts += [s.Wqkv.weight, s.Wqkv.bias, s.out_proj.weight, s.out_proj.bias]
            ts += [s.ffn[0].weight, s.ffn[0].bias, s.ffn[1].weight, s.ffn[1].bias, s.ffn[3].weight, s.ffn[3].bias]
            ts += [c.to_qk.weight, c.to_qk.bias, c.to_v.weight, c.to_v.bias, c.to_out.weight, c.to_out.bias]
            ts += [c.ffn[0].weight, c.ffn[0].bias, c.ffn[1].weight, c.ffn[1].bias, c.ffn[3].weight, c.ffn[3].bias]
        for a in self.log_assignment:
            ts += [a.matchability.weight, a.matchability.bias, a.final_proj.weight, a.final_proj.bias]
        for t in self.token_confidence:
            ts += [t.token[0].weight, t.token[0].bias]
        return ts

    def _signature(self, device: torch.device):
        c = self.conf
        return (
            device.index, c.precision, float(c.depth_confidence), float(c.width_confidence), float(c.filter_threshold),
            tuple((p.data_ptr(), p._version) for p in self._blob_tensors()),
        )

    def _release(self) -> None:
        if self._handle is not None:
            _cabi.load().lg_destroy(self._handle[0])
            self._handle = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _get_handle(self, device: torch.device):
        sig = self._signature(device)
        if self._handle is not None and self._handle[1] == sig:
            return self._handle[0]
        self._release()
        lib = _cabi.load()
        c = self.conf
        pos_dim = 2 + 2 * int(bool(c.add_scale_ori))
        blob = torch.cat([p.detach().to(device=device, dtype=torch.float32).reshape(-1) for p in self._blob_tensors()])
        want = lib.lg_weight_blob_floats(c.input_dim, pos_dim, c.n_layers)
        assert blob.numel() == want, (blob.numel(), want)
        cfg = _cabi.LgConfig(
            _cabi.ABI_VERSION, c.input_dim, pos_dim, c.n_layers, _cabi.PREC[c.precision],
            float(c.depth_confidence), float(c.width_confidence), float(c.filter_threshold),
        )
        handle = C.c_void_p()
        stream = torch.cuda.current_stream(device).cuda_stream
        _cabi.check(lib.lg_create(C.byref(cfg), blob.data_ptr(), blob.numel(), stream, C.byref(handle)), "lg_create")
        torch.cuda.current_stream(device).synchronize()  # the blob may be freed now
        self._handle = (handle, sig)
        self._ws.clear()
        self._graphs.clear()
        return handle

    def _workspace(self, handle, device: torch.device, b: int, m: int, n: int) -> torch.Tensor:
        key = (device.index, b, m, n)
        ws = self._ws.get(key)
        if ws is None:
            nbytes = _cabi.load().lg_workspace_bytes(handle, b, m, n)
            if len(self._ws) > 8:
                self._ws.clear()
            ws = torch.zeros(max(nbytes, 256), dtype=torch.uint8, device=device)  # zero-filled once (header contract)
            self._ws[key] = ws
        return ws

    # ------------------------------------------------------------------ reference API
    def compile(self, mode="reduce-overhead", static_lengths=[256, 512, 768, 1024, 1280, 1536]):
        """Reference 439-454 pads to static lengths for torch.compile.  The CUDA kernels take ragged
        lengths directly, so this only records the lengths for interface compatibility."""
        self.static_lengths = static_lengths

    def pruning_min_kpts(self, device: torch.device) -> int:
        """Reference 658-662."""
        if self.conf.flash and device.type == "cuda":
            return self.pruning_keypoint_thresholds["flash"]
        return self.pruning_keypoint_thresholds[device.type]

    def confidence_threshold(self, layer_index: int) -> float:
        return float(np.clip(0.8 + 0.1 * np.exp(-4.0 * layer_index / self.conf.n_layers), 0, 1))

    def forward(self, data: dict) -> dict:
        """Match keypoints and descriptors between two images (reference 456-481): ``forward_async(data).result()``."""
        return self.forward_async(data).result()

    def forward_async(self, data: dict) -> "PendingMatch":
        """Enqueue one forward on the current stream and return without waiting for the GPU.

        The reference synchronises several times per layer; this path has a single host dependency -- the python
        int ``stop`` and the lengths of the per-pair ``matches`` lists -- which ``PendingMatch.result()`` resolves
        from a pinned read-back buffer.  Callers that keep one forward in flight while they post-process the
        previous one (``lightglue_b200.pipeline.match_stream``, ``bench.py``) never leave the GPU idle.

        data = {"image0": {"keypoints" [B,M,2], "descriptors" [B,M,D], optional "image_size" [B,2],
        optional "scales"/"oris" [B,M]}, "image1": {...}}  ->  dict with matches0/1, matching_scores0/1,
        matches, scores, stop, prune0/1.

        Extension (SURVEY 8f2, ragged batches): an optional "num_keypoints" [B] integer tensor per image
        says how many leading rows of that pair are real keypoints; the rest is padding that no kernel
        reads (the reference pads + masks instead, 46-55, 256-262, 512-520).  Padding rows come back as
        matches -1 / scores 0 / prune 0; every pair's result equals its own B=1 call.

        Deviation from the reference for B > 1 with adaptive depth / width ON: early exit and point pruning are
        decided PER PAIR on the device, ``stop`` is the maximum over the batch and ``stops`` (extra key for B > 1) lists
        every pair's exit layer.  The reference takes one
        batch-global decision (the low-confidence count is summed over the batch and divided by one pair's m + n,
        645-656; ``torch.where(mask)[1]`` concatenates the columns of all rows, 554/562), which is only well defined
        for B == 1 -- there the results are identical (fixtures ``adaptive_*``); in a batch of two COPIES of one pair the
        reference runs all nine layers where the pair alone stops after six (tests/test_reference_batch_semantics.py
        runs the unmodified reference file to show it).  With pruning / early exit off
        (``depth_confidence = width_confidence = -1``) batched and single calls agree bit for bit.
        """
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        d0, d1 = data["image0"], data["image1"]
        k0, k1 = d0["keypoints"], d1["keypoints"]
        b, m, _ = k0.shape
        b, n, _ = k1.shape
        device = k0.device
        if device.type != "cuda":
            raise RuntimeError("lightglue_b200.LightGlue runs on CUDA (sm_90a) tensors only; there is no CPU path")
        x0 = d0["descriptors"].detach()
        x1 = d1["descriptors"].detach()
        assert x0.shape[-1] == self.conf.input_dim
        assert x1.shape[-1] == self.conf.input_dim

        def f32(t):
            return None if t is None else t.detach().to(device=device, dtype=torch.float32).contiguous()

        k0, k1, x0, x1 = f32(k0), f32(k1), f32(x0), f32(x1)
        s0, s1 = d0.get("image_size"), d1.get("image_size")

        def size_tensor(s):
            if s is None:
                return None
            s = torch.as_tensor(s, device=device, dtype=torch.float32)
            return s.expand(b, 2).contiguous() if s.dim() == 1 else s.contiguous()

        s0, s1 = size_tensor(s0), size_tensor(s1)

        def len_tensor(t, cap):
            if t is None:
                return None
            t = torch.as_tensor(t, device=device).to(torch.int32).reshape(-1).contiguous()
            assert t.numel() == b, "num_keypoints must hold one count per pair"
            return t.clamp(0, cap)

        l0, l1 = len_tensor(d0.get("num_keypoints"), m), len_tensor(d1.get("num_keypoints"), n)
        sc0 = or0 = sc1 = or1 = None
        if self.conf.add_scale_ori:
            sc0, or0, sc1, or1 = f32(d0["scales"]), f32(d0["oris"]), f32(d1["scales"]), f32(d1["oris"])

        # reference 514, 529: the padded ("compiled") path disables point pruning for inputs that fit a
        # static length; the kernels need no padding, so only the pruning switch is mirrored.
        do_compile = bool(self.static_lengths) and max(m, n) <= max(self.static_lengths)
        prune = self.conf.width_confidence > 0 and not do_compile
        pruning_th = int(self.pruning_min_kpts(device)) if not do_compile else (1 << 30)

        with torch.cuda.device(device):
            handle = self._get_handle(device)
            lib = _cabi.load()
            use_graph = bool(self.conf.cuda_graph) and m > 0 and n > 0 and not self.timing
            key = (device.index, b, m, n, prune, pruning_th, s0 is None, s1 is None, l0 is None, l1 is None)
            slot = self._graphs.get(key) if use_graph else None
            if slot is None:
                ws = self._workspace(handle, device, b, m, n)
                cap = min(m, n)
                io = {
                    "m0": torch.empty(b, m, dtype=torch.int64, device=device),
                    "m1": torch.empty(b, n, dtype=torch.int64, device=device),
                    "ms0": torch.empty(b, m, dtype=torch.float32, device=device),
                    "ms1": torch.empty(b, n, dtype=torch.float32, device=device),
                    "meta": torch.empty(2, b, dtype=torch.int32, device=device),  # [stop | n_matches]
                    "pr0": torch.empty(b, m, dtype=torch.int32, device=device) if prune else None,
                    "pr1": torch.empty(b, n, dtype=torch.int32, device=device) if prune else None,
                    "pairs": torch.empty(b, cap, 2, dtype=torch.int64, device=device),
                    "pscores": torch.empty(b, cap, dtype=torch.float32, device=device),
                }
                ins = [k0, k1, x0, x1, s0, s1, sc0, or0, sc1, or1, l0, l1]
                if use_graph:  # static input buffers the graph reads from
                    ins = [None if t is None else t.clone() for t in ins]
                ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
                inp = _cabi.LgInputs(b, m, n, *[ptr(t) for t in ins[:10]], pruning_th, ptr(ins[10]), ptr(ins[11]))
                out = _cabi.LgOutputs(
                    ptr(io["m0"]), ptr(io["m1"]), ptr(io["ms0"]), ptr(io["ms1"]), io["meta"][0].data_ptr(), ptr(io["pr0"]),
                    ptr(io["pr1"]), io["meta"][1].data_ptr(), ptr(io["pairs"]), ptr(io["pscores"]), None,
                )
                if self.timing:
                    lib.lg_timing_enable(handle, 1)
                    self.timing = False

                def launch():
                    stream = torch.cuda.current_stream(device).cuda_stream
                    _cabi.check(
                        lib.lg_forward(handle, C.byref(inp), C.byref(out), ws.data_ptr(), ws.numel(), stream), "lg_forward"
                    )

                if use_graph:
                    side = torch.cuda.Stream(device)
                    side.wait_stream(torch.cuda.current_stream(device))
                    with torch.cuda.stream(side):
                        launch()  # warm-up: one-time function attributes / tensor-map cache
                    torch.cuda.current_stream(device).wait_stream(side)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        launch()
                    slot = (graph, ins, io, (inp, out, ws))
                    if len(self._graphs) > 16:
                        self._graphs.clear()
                    self._graphs[key] = slot
                else:
                    launch()
            if use_graph:
                graph, ins, io, _keep = slot
                for dst, src in zip(ins, [k0, k1, x0, x1, s0, s1, sc0, or0, sc1, or1, l0, l1]):
                    if dst is not None:
                        dst.copy_(src, non_blocking=True)
                graph.replay()
                io = {k: (None if v is None else v.clone()) for k, v in io.items()}  # results must not alias the graph's buffers
            m0, m1, ms0, ms1, meta = io["m0"], io["m1"], io["ms0"], io["ms1"], io["meta"]
            pr0, pr1, pairs, pscores = io["pr0"], io["pr1"], io["pairs"], io["pscores"]
            # the single device->host read-back (stop flags + match counts), asynchronous into pinned memory
            pool = self._meta_pool.get(b)
            if pool is None:  # pinned allocation is slow and synchronises the device: take a few buffers at once
                block = torch.empty(4, 2, b, dtype=torch.int32, pin_memory=True)
                pool = self._meta_pool[b] = [block[i] for i in range(4)]
            meta_h = pool.pop() if pool else torch.empty(2, b, dtype=torch.int32, pin_memory=True)
            meta_h.copy_(meta, non_blocking=True)
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream(device))
        return PendingMatch(self, done, meta_h, (b, m, n), prune, l0 is not None or l1 is not None,
                            dict(m0=m0, m1=m1, ms0=ms0, ms1=ms1, pr0=pr0, pr1=pr1, pairs=pairs, pscores=pscores))

    def _finish(self, meta_h, shape, prune, ragged, dev) -> dict:
        """Assemble the reference's output dict once the read-back buffer is valid."""
        b, m, n = shape
        m0, m1, ms0, ms1 = dev["m0"], dev["m1"], dev["ms0"], dev["ms1"]
        pr0, pr1, pairs, pscores = dev["pr0"], dev["pr1"], dev["pairs"], dev["pscores"]
        device = m0.device
        stop = int(meta_h[0].max())
        if m == 0 or n == 0:  # reference 568-588: tensors instead of lists
            matches = torch.empty(b, 0, 2, dtype=torch.int64, device=device)
            scores = torch.empty(b, 0, dtype=torch.float32, device=device)
        else:
            counts = meta_h[1].tolist()
            matches = [pairs[i, : counts[i]] for i in range(b)]
            scores = [pscores[i, : counts[i]] for i in range(b)]
        if prune:
            prune0, prune1 = pr0.to(torch.int64), pr1.to(torch.int64)  # reference 535-536: integer counters
        else:  # reference 616-617: float tensors filled with n_layers
            prune0 = torch.full((b, m), float(self.conf.n_layers), dtype=torch.float32, device=device)
            prune1 = torch.full((b, n), float(self.conf.n_layers), dtype=torch.float32, device=device)
        res = {
            "matches0": m0,
            "matches1": m1,
            "matching_scores0": ms0,
            "matching_scores1": ms1,
            "stop": stop,
            "matches": matches,
            "scores": scores,
            "prune0": prune0,
            "prune1": prune1,
        }
        if ragged or b > 1:  # per-pair exit layers (split_outputs of a ragged batch; a dense batch decides per pair too)
            res["stops"] = [int(v) for v in meta_h[0].tolist()]
        return res

    # ------------------------------------------------------------------ extras used by tests / bench
    def log_assignment_matrix(self, layer: int, desc0: torch.Tensor, desc1: torch.Tensor):
        """``MatchAssignment.forward`` + ``filter_matches`` (reference 287-296, 302-318) through
        ``lg_assign``: returns (scores [B, M+1, N+1], matches0, matches1, mscores0, mscores1)."""
        device = desc0.device
        b, m, _ = desc0.shape
        n = desc1.shape[1]
        with torch.cuda.device(device):
            handle = self._get_handle(device)
            lib = _cabi.load()
            ws = self._workspace(handle, device, b, m, n)
            x0 = desc0.detach().float().contiguous()
            x1 = desc1.detach().float().contiguous()
            cap = min(m, n)
            m0 = torch.empty(b, m, dtype=torch.int64, device=device)
            m1 = torch.empty(b, n, dtype=torch.int64, device=device)
            ms0 = torch.empty(b, m, dtype=torch.float32, device=device)
            ms1 = torch.empty(b, n, dtype=torch.float32, device=device)
            meta = torch.empty(2, b, dtype=torch.int32, device=device)
            pairs = torch.empty(b, cap, 2, dtype=torch.int64, device=device)
            pscores = torch.empty(b, cap, dtype=torch.float32, device=device)
            full = torch.empty(b, m + 1, n + 1, dtype=torch.float32, device=device)
            out = _cabi.LgOutputs(
                m0.data_ptr(), m1.data_ptr(), ms0.data_ptr(), ms1.data_ptr(), meta[0].data_ptr(), None, None,
                meta[1].data_ptr(), pairs.data_ptr(), pscores.data_ptr(), full.data_ptr(),
            )
            if self.timing:
                lib.lg_timing_enable(handle, 1)
                self.timing = False
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(
                lib.lg_assign(handle, layer, b, m, n, x0.data_ptr(), x1.data_ptr(), C.byref(out), ws.data_ptr(),
                              ws.numel(), stream),
                "lg_assign",
            )
        return full, m0, m1, ms0, ms1

    def attention(self, q0, k0, v0, q1, k1, v1, cross: bool = False):
        """Kernel-level entry (``lg_attention``): ``Attention.forward`` (reference 97-137) on projected / rotated
        heads ``[B, 4, M|N, 64]`` through the attention kernel of this matcher's precision mode.  Self
        (``cross=False``): each image attends to itself; cross: image 0 queries image 1's keys / values and vice
        versa (210-214).  Returns ``(ctx0 [B, M, 256], ctx1 [B, N, 256])`` fp32, heads concatenated h-major."""
        device = q0.device
        b, hh, m, dh = q0.shape
        n = q1.shape[2]
        assert hh == 4 and dh == 64 and k0.shape == q0.shape == v0.shape and k1.shape == q1.shape == v1.shape
        with torch.cuda.device(device):
            handle = self._get_handle(device)
            lib = _cabi.load()
            ws = self._workspace(handle, device, b, m, n)
            ts = [t.detach().to(device=device, dtype=torch.float32).contiguous() for t in (q0, k0, v0, q1, k1, v1)]
            c0 = torch.empty(b, m, 256, dtype=torch.float32, device=device)
            c1 = torch.empty(b, n, 256, dtype=torch.float32, device=device)
            if self.timing:
                lib.lg_timing_enable(handle, 1)
                self.timing = False
            stream = torch.cuda.current_stream(device).cuda_stream
            _cabi.check(
                lib.lg_attention(handle, b, m, n, int(bool(cross)), *[t.data_ptr() for t in ts], c0.data_ptr(), c1.data_ptr(),
                                 ws.data_ptr(), ws.numel(), stream),
                "lg_attention",
            )
        return c0, c1

    def forward_with_layers(self, data: dict):
        """Debug / block-level parity (``lg_debug_capture_layers``): one forward that also returns the residual stream
        after every transformer layer, ``[(desc0 [B, M, 256], desc1 [B, N, 256]), ...]`` -- what a forward hook on the
        reference's ``transformers[i]`` sees (lightglue.py:541).  Dense, non-pruned batches only."""
        k0, k1 = data["image0"]["keypoints"], data["image1"]["keypoints"]
        b, m, n = k0.shape[0], k0.shape[1], k1.shape[1]
        device = k0.device
        lib = _cabi.load()
        with torch.cuda.device(device):
            handle = self._get_handle(device)
            lp = int(lib.lg_padded_length(m, n))
            buf = torch.zeros(self.conf.n_layers, 2 * b, lp, DIM, dtype=torch.float32, device=device)
            _cabi.check(lib.lg_debug_capture_layers(handle, buf.data_ptr(), buf.numel()), "lg_debug_capture_layers")
            try:
                out = self.forward(data)
                torch.cuda.synchronize(device)
            finally:
                lib.lg_debug_capture_layers(handle, None, 0)
        layers = [(buf[i, :b, :m].clone(), buf[i, b:, :n].clone()) for i in range(int(out["stop"]))]
        return out, layers

    def kernel_times(self) -> dict:
        """Summed device milliseconds / launch counts per kernel class since timing was switched on."""
        if self._handle is None:
            return {}
        lib = _cabi.load()
        res = {}
        for name, kc in (("attention", 0), ("linear", 1), ("assign", 2), ("other", 3), ("assign_matrix", 4), ("qkv", 5),
                         ("ffn0", 6), ("ffn3", 7), ("assign_stage", 8)):
            ms, cnt = C.c_double(), C.c_int64()
            _cabi.check(lib.lg_kernel_time_ms(self._handle[0], kc, C.byref(ms), C.byref(cnt)), "lg_kernel_time_ms")
            res[name] = (ms.value, cnt.value)
        lib.lg_timing_enable(self._handle[0], 0)
        return res

    def debug_timeout_code(self) -> int:
        """0, or the site code of an in-kernel pipeline wait that timed out (debug aid; synchronises)."""
        if self._handle is None:
            return 0
        words = (C.c_uint32 * 32)()
        code = int(_cabi.load().lg_debug_timeout_code(self._handle[0], words))
        self.debug_words = [int(w) for w in words]
        return code

    def last_launch_count(self) -> int:
        return 0 if self._handle is None else int(_cabi.load().lg_last_launch_count(self._handle[0]))


class PendingMatch:
    """A forward that has been enqueued but whose host-side result (``stop``, list lengths) is not resolved yet.

    ``tensors`` are the device outputs (valid in stream order right away); ``result()`` waits for the read-back of
    the [stop | n_matches] words and returns the reference's output dict; it may be called more than once."""

    def __init__(self, matcher, done, meta_h, shape, prune, ragged, dev):
        self._matcher, self._done, self._meta, self._shape = matcher, done, meta_h, shape
        self._prune, self._ragged, self._dev, self._res = prune, ragged, dev, None

    @property
    def tensors(self) -> dict:
        d = self._dev
        return {"matches0": d["m0"], "matches1": d["m1"], "matching_scores0": d["ms0"], "matching_scores1": d["ms1"]}

    def done(self) -> bool:
        return self._res is not None or self._done.query()

    def result(self) -> dict:
        if self._res is None:
            self._done.synchronize()
            self._res = self._matcher._finish(self._meta, self._shape, self._prune, self._ragged, self._dev)
            self._matcher._meta_pool.setdefault(self._shape[0], []).append(self._meta)  # recycle the pinned buffer
            self._meta = None
        return self._res
