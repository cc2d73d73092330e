"""Keypoint matching between two SIFT outputs of one image (test infrastructure).

Keypoints are paired mutually by nearest position; a pair is matched when the positions are within 0.05 px, the sizes
within 0.1 % and the orientations within 0.2 degrees (circular)."""
from __future__ import annotations

import math

import torch

POS_TOL, SIZE_RTOL, ORI_TOL_DEG = 0.05, 1e-3, 0.2


def match(a: dict, b: dict):
    """(ia, ib) index tensors of the matched pairs between outputs a and b (dicts of one image)."""
    ka, kb = a["keypoints"].double(), b["keypoints"].double()
    if len(ka) == 0 or len(kb) == 0:
        return torch.zeros(0, dtype=torch.long), torch.zeros(0, dtype=torch.long)
    # several keypoints can share a position (orientations); pair by position, size and orientation together
    d = torch.cdist(ka, kb)
    ds = (a["scales"].double()[:, None] - b["scales"].double()[None]).abs() / b["scales"].double()[None].clamp_min(1e-9)
    do = (a["oris"].double()[:, None] - b["oris"].double()[None]).abs() % (2 * math.pi)
    do = torch.minimum(do, 2 * math.pi - do) * 180 / math.pi
    cost = d + ds + do * 1e-3
    nn_ab = cost.argmin(1)
    nn_ba = cost.argmin(0)
    ia = torch.arange(len(ka))
    mutual = nn_ba[nn_ab] == ia
    ok = mutual & (d[ia, nn_ab] <= POS_TOL) & (ds[ia, nn_ab] <= SIZE_RTOL) & (do[ia, nn_ab] <= ORI_TOL_DEG)
    return ia[ok], nn_ab[ok]


def rootsift(x: torch.Tensor, eps=1e-6) -> torch.Tensor:
    x = torch.nn.functional.normalize(x.double(), p=1, dim=-1, eps=eps)
    return torch.nn.functional.normalize(x.clip(min=eps).sqrt(), p=2, dim=-1, eps=eps)


def compare(test: dict, ref: dict, ordered: bool, is_rootsift: bool = True) -> dict:
    """Statistics of `test` against `ref` for one image.  Descriptors are compared as RootSIFT (raw SIFT descriptors
    are converted first)."""
    ia, ib = match(test, ref)
    nt, nr = len(test["keypoints"]), len(ref["keypoints"])
    st = {"n_test": nt, "n_ref": nr, "matched": len(ia),
          "frac_ref": len(ia) / max(nr, 1), "frac_test": len(ia) / max(nt, 1)}
    if len(ia):
        s_t, s_r = test["keypoint_scores"][ia].double(), ref["keypoint_scores"][ib].double()
        st["score_rel"] = float(((s_t - s_r).abs() / s_r.abs().clamp_min(1e-12)).max())
        dt, dr = test["descriptors"][ia].double(), ref["descriptors"][ib].double()
        if not is_rootsift:
            dt, dr = rootsift(dt), rootsift(dr)
        dd = (dt - dr).norm(dim=-1)
        st["desc_l2_max"] = float(dd.max())
        st["desc_l2_frac_le_0.02"] = float((dd <= 0.02).double().mean())
        if ordered:  # matched rows appear in the same order on both sides
            st["ordered"] = bool((ia.diff() > 0).all() and (ib.diff() > 0).all())
    else:
        st.update(score_rel=0.0, desc_l2_max=0.0, **{"desc_l2_frac_le_0.02": 1.0}, ordered=True)
    return st


def check(st: dict, ordered: bool) -> None:
    """The parity criteria: >= 99 % matched both ways, counts within 1 %, scores within 1e-4 relative, descriptor L2
    <= 0.02 on >= 99 % of the matched keypoints and <= 0.1 on all, the reference's order when uncapped."""
    assert st["frac_ref"] >= 0.99 and st["frac_test"] >= 0.99, st
    assert abs(st["n_test"] - st["n_ref"]) <= 0.01 * st["n_ref"], st
    assert st["score_rel"] <= 1e-4, st
    assert st["desc_l2_frac_le_0.02"] >= 0.99 and st["desc_l2_max"] <= 0.1, st
    if ordered:
        assert st["ordered"], st
