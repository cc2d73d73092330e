"""CPU oracle for the LightGlue matcher forward path  --  TEST INFRASTRUCTURE ONLY.

This file is a *restatement* (functional, state_dict-driven, plain torch CPU tensor arithmetic) of
the algorithm in the reference ``lightglue/lightglue.py``.  It is the checker the CUDA path is
compared against; it is never the thing measured or shipped.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may
import it.  The product package ``lightglue_b200`` does not import anything from ``oracle/``.

Parity status: the reference ships **no** tests, golden vectors or known-answer fixtures for this
path (SURVEY.md §4, §8c), so the oracle is pinned the other way the task allows: against outputs
of the reference itself.  ``oracle/make_golden.py`` imports ``/root/reference/lightglue/lightglue.py``
in the build container, runs it on seeded synthetic inputs/weights and commits the results under
``tests/golden/``; ``tests/test_oracle_golden.py`` checks this restatement against those fixtures
(identical match indices, |dscore| <= 2e-5).

Each function cites the reference lines it restates (paths relative to /root/reference).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

N_HEADS = 4
HEAD_DIM = 64
DIM = 256


def confidence_thresholds(n_layers: int = 9) -> np.ndarray:
    """lightglue/lightglue.py:631-634 -- clip(0.8 + 0.1*exp(-4 i / L), 0, 1), float64 -> float32 buffer (408-413)."""
    i = np.arange(n_layers, dtype=np.float64)
    return np.clip(0.8 + 0.1 * np.exp(-4.0 * i / n_layers), 0.0, 1.0).astype(np.float32)


def normalize_keypoints(kpts: torch.Tensor, size: Optional[torch.Tensor]) -> torch.Tensor:
    """lightglue/lightglue.py:31-43.  With no size: size = 1 + max - min, and the shift is size/2
    (NOT the bounding-box centre -- a quirk of the reference that is preserved)."""
    if size is None:
        size = 1 + kpts.amax(dim=-2) - kpts.amin(dim=-2)
    size = torch.as_tensor(size, dtype=kpts.dtype)
    half = size / 2
    scale = size.amax(dim=-1) / 2
    return (kpts - half.unsqueeze(-2)) / scale[..., None, None]


def fourier_encoding(pos: torch.Tensor, wr: torch.Tensor):
    """lightglue/lightglue.py:76-81.  Returns (cos, sin) each [B, N, 32]; the reference duplicates
    each over adjacent channel pairs (repeat_interleave(2)) -- kept implicit here."""
    proj = pos @ wr.t()
    return torch.cos(proj), torch.sin(proj)


def rope(t: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """lightglue/lightglue.py:58-65 on t [B, H, N, 64]:  (x0, x1) -> (x0 c - x1 s, x1 c + x0 s) per pair."""
    te, to = t[..., 0::2], t[..., 1::2]
    c, s = cos.unsqueeze(1), sin.unsqueeze(1)
    out = torch.empty_like(t)
    out[..., 0::2] = te * c - to * s
    out[..., 1::2] = to * c + te * s
    return out


def attention(q, k, v):
    """lightglue/lightglue.py:113-137: softmax(q k^T / sqrt(64)) v, no mask/bias; empty -> zeros (114-115)."""
    if q.shape[-2] == 0 or k.shape[-2] == 0:
        return q.new_zeros(*q.shape[:-1], v.shape[-1])
    s = (q @ k.transpose(-1, -2)) * (q.shape[-1] ** -0.5)
    return torch.softmax(s, dim=-1) @ v


def _ffn(w: Dict[str, torch.Tensor], p: str, x: torch.Tensor, msg: torch.Tensor) -> torch.Tensor:
    """lightglue/lightglue.py:152-157 / 187-192 and the residual at 172 / 228-229."""
    hcat = torch.cat([x, msg], dim=-1)
    h1 = F.linear(hcat, w[p + "ffn.0.weight"], w[p + "ffn.0.bias"])
    h1 = F.layer_norm(h1, (h1.shape[-1],), w[p + "ffn.1.weight"], w[p + "ffn.1.bias"], 1e-5)
    h1 = F.gelu(h1)  # exact erf form (nn.GELU default)
    return x + F.linear(h1, w[p + "ffn.3.weight"], w[p + "ffn.3.bias"])


def self_block(w, i: int, x: torch.Tensor, cos, sin) -> torch.Tensor:
    """lightglue/lightglue.py:159-172.  Wqkv output channel c = h*192 + d*3 + {0:q,1:k,2:v} (166)."""
    p = f"transformers.{i}.self_attn."
    b, n, _ = x.shape
    qkv = F.linear(x, w[p + "Wqkv.weight"], w[p + "Wqkv.bias"]).view(b, n, N_HEADS, HEAD_DIM, 3)
    q, k, v = (qkv[..., j].permute(0, 2, 1, 3) for j in range(3))
    ctx = attention(rope(q, cos, sin), rope(k, cos, sin), v)
    ctx = ctx.permute(0, 2, 1, 3).reshape(b, n, DIM)
    msg = F.linear(ctx, w[p + "out_proj.weight"], w[p + "out_proj.bias"])
    return _ffn(w, p, x, msg)


def cross_block(w, i: int, x0: torch.Tensor, x1: torch.Tensor):
    """lightglue/lightglue.py:201-230.  One shared projection serves as query AND key (204)."""
    p = f"transformers.{i}.cross_attn."

    def heads(t):
        return t.view(t.shape[0], t.shape[1], N_HEADS, HEAD_DIM).permute(0, 2, 1, 3)

    def merge(t):
        return t.permute(0, 2, 1, 3).reshape(t.shape[0], t.shape[2], DIM)

    qk0 = heads(F.linear(x0, w[p + "to_qk.weight"], w[p + "to_qk.bias"]))
    qk1 = heads(F.linear(x1, w[p + "to_qk.weight"], w[p + "to_qk.bias"]))
    v0 = heads(F.linear(x0, w[p + "to_v.weight"], w[p + "to_v.bias"]))
    v1 = heads(F.linear(x1, w[p + "to_v.weight"], w[p + "to_v.bias"]))
    m0 = merge(attention(qk0, qk1, v1))
    m1 = merge(attention(qk1, qk0, v0))
    m0 = F.linear(m0, w[p + "to_out.weight"], w[p + "to_out.bias"])
    m1 = F.linear(m1, w[p + "to_out.weight"], w[p + "to_out.bias"])
    return _ffn(w, p, x0, m0), _ffn(w, p, x1, m1)


def log_assignment(w, i: int, x0: torch.Tensor, x1: torch.Tensor) -> torch.Tensor:
    """lightglue/lightglue.py:287-296 + 265-277: the [B, M+1, N+1] log-assignment matrix."""
    p = f"log_assignment.{i}."
    b, m, _ = x0.shape
    n = x1.shape[1]
    p0 = F.linear(x0, w[p + "final_proj.weight"], w[p + "final_proj.bias"]) / DIM ** 0.25
    p1 = F.linear(x1, w[p + "final_proj.weight"], w[p + "final_proj.bias"]) / DIM ** 0.25
    sim = p0 @ p1.transpose(1, 2)
    z0 = F.linear(x0, w[p + "matchability.weight"], w[p + "matchability.bias"])  # [B, M, 1]
    z1 = F.linear(x1, w[p + "matchability.weight"], w[p + "matchability.bias"])
    out = sim.new_zeros(b, m + 1, n + 1)
    out[:, :m, :n] = (
        torch.log_softmax(sim, dim=2) + torch.log_softmax(sim, dim=1) + F.logsigmoid(z0) + F.logsigmoid(z1).transpose(1, 2)
    )
    out[:, :m, n] = F.logsigmoid(-z0.squeeze(-1))
    out[:, m, :n] = F.logsigmoid(-z1.squeeze(-1))
    return out


def matchability(w, i: int, x: torch.Tensor) -> torch.Tensor:
    """lightglue/lightglue.py:298-299."""
    p = f"log_assignment.{i}.matchability."
    return torch.sigmoid(F.linear(x, w[p + "weight"], w[p + "bias"])).squeeze(-1)


def token_confidence(w, i: int, x: torch.Tensor) -> torch.Tensor:
    """lightglue/lightglue.py:84-94."""
    p = f"token_confidence.{i}.token.0."
    return torch.sigmoid(F.linear(x, w[p + "weight"], w[p + "bias"])).squeeze(-1)


def filter_matches(scores: torch.Tensor, th: float):
    """lightglue/lightglue.py:302-318 (mutual nearest neighbour over the M x N core, then threshold)."""
    core = scores[:, :-1, :-1]
    max0, max1 = core.max(dim=2), core.max(dim=1)
    m0, m1 = max0.indices, max1.indices
    ar0 = torch.arange(m0.shape[1])[None]
    ar1 = torch.arange(m1.shape[1])[None]
    mutual0 = ar0 == m1.gather(1, m0)
    mutual1 = ar1 == m0.gather(1, m1)
    ms0 = torch.where(mutual0, max0.values.exp(), max0.values.new_zeros(()))
    ms1 = torch.where(mutual1, ms0.gather(1, m1), ms0.new_zeros(()))
    valid0 = mutual0 & (ms0 > th)
    valid1 = mutual1 & valid0.gather(1, m1)
    return torch.where(valid0, m0, -1), torch.where(valid1, m1, -1), ms0, ms1


def encodings(w: Dict[str, torch.Tensor], data: dict, add_scale_ori: bool = False):
    """lightglue/lightglue.py:491-501, 523-524: the rotary encodings ``(c0, s0, c1, s1)`` of both images' normalised
    keypoints (with scale and orientation appended when ``add_scale_ori``), in the dtype and on the device of
    ``w["posenc.Wr.weight"]``."""
    wr = w["posenc.Wr.weight"]
    enc = []
    for d in (data["image0"], data["image1"]):
        k = normalize_keypoints(d["keypoints"].to(wr), d.get("image_size"))
        if add_scale_ori:  # 495-501
            k = torch.cat([k, d["scales"].to(wr).unsqueeze(-1), d["oris"].to(wr).unsqueeze(-1)], -1)
        enc += fourier_encoding(k, wr)
    return tuple(enc)


def layer(w: Dict[str, torch.Tensor], i: int, x0: torch.Tensor, x1: torch.Tensor, enc):
    """lightglue/lightglue.py:541-543 (``TransformerLayer``, 233-253): transformer layer ``i`` (self blocks, then the cross block) on the residual
    streams ``x0``, ``x1`` with the encodings ``enc = encodings(...)`` of those rows; returns the new ``(x0, x1)``."""
    c0, s0, c1, s1 = enc
    x0 = self_block(w, i, x0, c0, s0)
    x1 = self_block(w, i, x1, c1, s1)
    return cross_block(w, i, x0, x1)


def forward(
    w: Dict[str, torch.Tensor],
    data: dict,
    *,
    n_layers: int = 9,
    depth_confidence: float = -1.0,
    width_confidence: float = -1.0,
    filter_threshold: float = 0.1,
    pruning_threshold: int = -1,
    add_scale_ori: bool = False,
    dtype: torch.dtype = torch.float32,
    return_layers: bool = False,
    return_decisions: bool = False,
) -> dict:
    """lightglue/lightglue.py:483-629 (``LightGlue._forward``), eager/unpadded path, any device -> CPU.

    ``pruning_threshold`` plays the role of ``pruning_min_kpts(device)`` (658-662): point pruning
    runs on an image only while it still has more keypoints than this.  The reference's adaptive
    bookkeeping (549, 554) is only meaningful for batch size 1; the oracle asserts that.

    ``return_decisions`` adds ``out["decisions"]``: one dict per executed layer below the last with the values its
    adaptive decisions were taken from -- ``thr`` and ``size`` (m + n, original sizes) always; with early exit on,
    ``tok0`` / ``tok1`` (token confidences of the live points) and ``below`` (how many are < ``thr``); for each image
    that is pruned at that layer, ``mat0`` / ``mat1`` (matchability of its live points).  ``certificate`` turns
    them into the pair's smallest margins.
    """
    w = {k: v.to(dtype) for k, v in w.items()}
    d0, d1 = data["image0"], data["image1"]
    b, m, _ = d0["keypoints"].shape
    n = d1["keypoints"].shape[1]
    x0 = d0["descriptors"].to(dtype)
    x1 = d1["descriptors"].to(dtype)
    if "input_proj.weight" in w:  # 388-391, 521-522
        x0 = F.linear(x0, w["input_proj.weight"], w["input_proj.bias"])
        x1 = F.linear(x1, w["input_proj.weight"], w["input_proj.bias"])
    else:
        assert x0.shape[-1] == DIM and x1.shape[-1] == DIM
    c0, s0, c1, s1 = encodings(w, data, add_scale_ori)

    early = depth_confidence > 0
    prune = width_confidence > 0
    if early or prune:
        assert b == 1, "adaptive depth/width follow the reference's batch-1 semantics"
    thr = torch.from_numpy(confidence_thresholds(n_layers)).to(dtype)
    ind0 = torch.arange(m)[None]
    ind1 = torch.arange(n)[None]
    pr0 = torch.ones(b, m, dtype=torch.long)
    pr1 = torch.ones(b, n, dtype=torch.long)
    layers: List[tuple] = []
    decisions: List[dict] = []
    last = 0
    tok0 = tok1 = None
    for i in range(n_layers):
        last = i
        if x0.shape[1] == 0 or x1.shape[1] == 0:  # 539-540
            break
        x0, x1 = layer(w, i, x0, x1, (c0, s0, c1, s1))
        if return_layers:
            layers.append((x0.clone(), x1.clone()))
        if i == n_layers - 1:  # 544-545
            continue
        dec = {"thr": float(thr[i]), "size": m + n}
        if return_decisions:
            decisions.append(dec)
        if early:  # 547-550, 645-656
            tok0, tok1 = token_confidence(w, i, x0), token_confidence(w, i, x1)
            below = (torch.cat([tok0, tok1], -1) < thr[i]).to(dtype).sum()
            dec.update(tok0=tok0[0], tok1=tok1[0], below=int(below))
            if 1.0 - below / (m + n) > depth_confidence:
                break
        if prune and x0.shape[1] > pruning_threshold:  # 551-558, 636-643
            dec["mat0"] = matchability(w, i, x0)[0]
            keep = dec["mat0"][None] > (1 - width_confidence)
            if tok0 is not None:
                keep |= tok0 <= thr[i]
            kk = torch.where(keep)[1]
            ind0, x0, c0, s0 = ind0[:, kk], x0[:, kk], c0[:, kk], s0[:, kk]
            pr0[:, ind0[0]] += 1
        if prune and x1.shape[1] > pruning_threshold:  # 559-566
            dec["mat1"] = matchability(w, i, x1)[0]
            keep = dec["mat1"][None] > (1 - width_confidence)
            if tok1 is not None:
                keep |= tok1 <= thr[i]
            kk = torch.where(keep)[1]
            ind1, x1, c1, s1 = ind1[:, kk], x1[:, kk], c1[:, kk], s1[:, kk]
            pr1[:, ind1[0]] += 1

    if x0.shape[1] == 0 or x1.shape[1] == 0:  # 568-588
        out = {
            "matches0": torch.full((b, m), -1, dtype=torch.long),
            "matches1": torch.full((b, n), -1, dtype=torch.long),
            "matching_scores0": torch.zeros(b, m, dtype=dtype),
            "matching_scores1": torch.zeros(b, n, dtype=dtype),
            "stop": last + 1,
            "matches": torch.empty(b, 0, 2, dtype=torch.long),
            "scores": torch.empty(b, 0, dtype=dtype),
            "prune0": pr0 if prune else torch.full((b, m), float(n_layers), dtype=dtype),
            "prune1": pr1 if prune else torch.full((b, n), float(n_layers), dtype=dtype),
        }
        if return_decisions:
            out["decisions"] = decisions
        return out

    scores = log_assignment(w, last, x0, x1)  # 591
    a0, a1, ms0, ms1 = filter_matches(scores, filter_threshold)  # 592
    matches, mscores = [], []
    for bi in range(b):  # 593-602
        valid = a0[bi] > -1
        i0 = torch.where(valid)[0]
        i1 = a0[bi][valid]
        if prune:
            i0, i1 = ind0[bi, i0], ind1[bi, i1]
        matches.append(torch.stack([i0, i1], -1))
        mscores.append(ms0[bi][valid])
    if prune:  # 605-614
        f0 = torch.full((b, m), -1, dtype=torch.long)
        f1 = torch.full((b, n), -1, dtype=torch.long)
        f0[:, ind0[0]] = torch.where(a0 == -1, -1, ind1.gather(1, a0.clamp(min=0)))
        f1[:, ind1[0]] = torch.where(a1 == -1, -1, ind0.gather(1, a1.clamp(min=0)))
        g0 = torch.zeros(b, m, dtype=dtype)
        g1 = torch.zeros(b, n, dtype=dtype)
        g0[:, ind0[0]] = ms0
        g1[:, ind1[0]] = ms1
        a0, a1, ms0, ms1 = f0, f1, g0, g1
        p0, p1 = pr0, pr1
    else:  # 616-617
        p0 = torch.full((b, m), float(n_layers), dtype=dtype)
        p1 = torch.full((b, n), float(n_layers), dtype=dtype)
    out = {
        "matches0": a0,
        "matches1": a1,
        "matching_scores0": ms0,
        "matching_scores1": ms1,
        "stop": last + 1,
        "matches": matches,
        "scores": mscores,
        "prune0": p0,
        "prune1": p1,
    }
    if return_layers:
        out["layers"] = layers
        out["log_assignment"] = scores
    if return_decisions:
        out["decisions"] = decisions
    return out


def certificate(decisions: List[dict], *, depth_confidence: float, width_confidence: float):
    """A pair's smallest decision margins over ``forward(..., return_decisions=True)["decisions"]``:
    ``(margin, slack)`` where

    * ``margin`` is the least of |token confidence - thr_i| over the live points and |matchability - (1 -
      width_confidence)| over the points a pruning step could drop (confidence > thr_i; every point when early exit
      is off);
    * ``slack`` is the least distance, in points, between the below-threshold count and the stop boundary
      (1 - depth_confidence)(m + n).  The stop ratio is evaluated in fp32 on both sides, so a count on the
      boundary has slack 0 and is never certified.

    Both are ``inf`` where no such decision was taken."""
    margin = slack = math.inf
    for d in decisions:
        thr = d["thr"]
        if "below" in d:
            for t in (d["tok0"], d["tok1"]):
                if t.numel():
                    margin = min(margin, float((t.double() - thr).abs().min()))
            slack = min(slack, abs((1.0 - depth_confidence) * d["size"] - d["below"]))
        for k, t in (("mat0", d.get("tok0")), ("mat1", d.get("tok1"))):
            if k not in d:
                continue
            mt = d[k].double()
            if t is not None:
                mt = mt[t > thr]
            if mt.numel():
                margin = min(margin, float((mt - (1.0 - width_confidence)).abs().min()))
    return margin, slack
