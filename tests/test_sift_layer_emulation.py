"""SIFT's stages against float64 (oracle/sift_oracle.py) on the host build's intermediates; no GPU needed.

The host build (oracle/sift_emul.cpp) runs the functors of csrc/sift_pipeline.h on a workspace carved as sift_forward
carves it, so ``sift_workspace_layout`` locates its intermediates as it does the GPU's.  Each stage check starts from
the captured input of that stage (tests/test_gpu_sift_layers.py runs the same checks on the GPU's workspace).

Tolerances (TOL) are at least 3x the fp32 error observed here, at least the allowance for the CUDA Math API's maximum
ulp errors the host build does not see (expf 2 ulp in the orientation and descriptor weights, sinf / cosf 2 ulp in the
descriptor rotation, powf 4 ulp in the candidate size: relative 2.4e-7 at most, far below the fp32 error of the steps
around them), and at most 1/3 of the deviation each listed defect causes.  Margins (``*_margin*``) exclude decisions
float64 cannot settle for fp32 (a candidate whose Newton step, contrast, edge or det test is that close to its
threshold, an orientation sample that close to a bin's rounding step or a peak test that close to its limit)."""
import math

import numpy as np
import pytest
import torch

from lightglue_b200.sift import SIFT
from oracle.sift_oracle import F32
from oracle import sift_emul, sift_oracle as so, sift_synth

TOL = {
    "gauss": 2e-6,          # max|d| / max|ref| per layer; observed 5.0e-7
    "cand_xy": 2e-4,        # octave pixels; observed 3.1e-5
    "cand_size": 2e-6,      # relative; observed 1.9e-7 (powf 4 ulp: 2.4e-7)
    "cand_response": 1e-4,  # relative; observed 3.1e-5
    "ori_angle": 2e-4,      # degrees; observed 3.4e-5
    "desc_abs": 1e-2,       # |q - v| - 1/2, uint8 units; observed 0
    "rootsift": 1e-6,       # absolute on unit rows; observed 1.6e-7
    "cand_margin_x": 1e-4,      # |x| < 0.5 and rounding steps, octave pixels (3x the x error)
    "cand_margin_rel": 1e-4,    # contrast, edge, det tests, relative
    "ori_margin_bin": 1e-5,     # bin units
    "ori_margin_peak": 1e-5,    # relative to the histogram maximum
    "desc_half": 1e-2,          # uint8 units: rint(v) is checked where v is this far from a half-integer
}
# stage -> the defects it must resolve; every other stage must pass under them
OWN = {"gauss0": ("reflect",), "gauss": ("reflect", "total_sigma"), "cand": ("swap_xc_xr",),
       "orient": ("smooth_nowrap",), "descriptor": ("descr_rot_sign", "clip_025"), "retain": ("retain_gt",),
       "dogfilter": ("dog_larger_angle",), "nms": ("nms_radius",)}


def assert_decided(info):
    """At most 1 % of the captured candidates fall outside the decided set.  Orientations may leave out up to 2 % (+1):
    a histogram sums about 500 samples at 768x1024's scales, each within ori_margin_bin of a rounding step with
    probability 2e-5, so about 1 % of the candidates hold one (49 of 4453 at 768x1024 on the host build and the GPU)."""
    if info["overflow"]:
        return
    assert info["cand_excluded"] <= 0.01 * info["cand_total"], info
    assert info.get("ori_undecided", 0) <= 0.02 * info["cand_total"] + 1, info


def lattice(n, step=4):
    """Bright dots every `step` pixels on a dark ground: each dot gives candidates at several scales and each of those
    four orientation peaks, so at 96x96 the raw keypoints outnumber the list (H W / 4 + 4096)."""
    yy, xx = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    return (0.1 + 0.8 * ((yy % step == 0) & (xx % step == 0)).float())[None, None].contiguous()


def tiled(h, w, period, seed):
    """A random patch tiled at `period` pixels: keypoints one period apart have bitwise equal responses."""
    patch = sift_synth.make_image(period, period, 1, seed)
    return patch.repeat(1, 1, -(-h // period), -(-w // period))[:, :, :h, :w].contiguous()


def tie_cut(kpt, tie=True):
    """An nfeatures that cuts the unique raw responses inside a run of equal values (tie) or between two distinct
    ones, about halfway down the list."""
    r = np.sort(np.unique(np.stack([kpt["x"], kpt["y"], kpt["size"], kpt["angle"], kpt["response"]], 1), axis=0)[:, 4])[::-1]
    at = np.nonzero((r[1:] == r[:-1]) if tie else (r[1:] < r[:-1]))[0]
    assert len(at), "no such cut"
    return int(at[len(at) // 2] + 1)


def run_emul(conf, image, sizes=None, defect=None, tol=TOL):
    """Host build -> (errs, fails, info, captured raw keypoints) of the batch's last image."""
    conf = {**SIFT.default_conf, **conf}
    outs, ws = sift_emul.forward_ws(conf, image, sizes)
    _, _, H, W = image.shape
    w, h = (int(sizes[-1][0]), int(sizes[-1][1])) if sizes is not None else (W, H)
    cap = so.capture(ws, so.layout(SIFT(**conf)._config(), H, W, h, w), h, w)
    errs, fails, info, sel = so.check_stages(cap, conf, image[-1], h, w, tol, defect)
    o = outs[-1]
    out = {"keypoints": o["keypoints"].numpy(), "scales": o["scales"].numpy(), "oris": o["oris"].numpy(),
           "scores": o["keypoint_scores"].numpy(), "descriptors": o["descriptors"].numpy(), "count": o["count"]}
    so.check_outputs(cap, conf, out, tol, defect, sel, errs, fails, info)
    return errs, fails, info, cap["kpt"]


needs_emul = pytest.mark.skipif(not sift_emul.available(), reason="oracle/_build/libsift_emul.so is not built")


def _cases():
    """(name, conf, image, image_size, regimes the case must reach)."""
    img = sift_synth.make_image(120, 160, 1, 21)
    return [
        ("natural", {}, img, None, ("multi_reflect", "pixel_dup_equal", "wrap_peak", "desc_border_clip")),
        ("nms3_plain", dict(nms_radius=3, rootsift=False), img, None, ("nms_suppression",)),
        ("tiny_8layers", dict(num_octaves=8), sift_synth.make_image(33, 47, 1, 22), None, ("multi_reflect",)),
        ("crop_1layer", dict(num_octaves=1), sift_synth.make_image(64, 80, 2, 23), [[80, 64], [71, 53]], ()),
    ]


CASES = _cases()


@needs_emul
@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_stages_of_the_host_build(i):
    name, conf, image, sizes, regimes = CASES[i]
    errs, fails, info, _ = run_emul(conf, image, sizes)
    assert not fails, (fails, errs)
    for r in regimes:
        assert info[r], (r, info)
    assert_decided(info)


@needs_emul
def test_tie_at_the_cut_and_top_k():
    """A tiled image with nfeatures inside a run of equal responses: retainBest keeps the whole tie, so without
    filter_dog_point the top-k applies, with ties in its order too."""
    img = tiled(128, 128, 32, 24)
    _, _, _, kpt = run_emul(dict(nms_radius=None), img)
    k = tie_cut(kpt)
    errs, fails, info, _ = run_emul(dict(nms_radius=None, max_num_keypoints=k), img)
    assert not fails, (fails, errs)
    assert info["cut_tie"] and info["topk"] and info["n_out"] == k, info


@needs_emul
def test_cut_between_distinct_responses():
    """nfeatures between two distinct responses: retainBest keeps exactly nfeatures."""
    img = sift_synth.make_image(120, 160, 1, 21)
    k = tie_cut(run_emul({}, img)[3], tie=False)
    errs, fails, info, _ = run_emul(dict(max_num_keypoints=k), img)
    assert not fails, (fails, errs)
    assert info["cut"] and not info["cut_tie"], info


@needs_emul
def test_overflow_reports_minus_one():
    """More raw keypoints than the list holds: counts = -1, and the ordering stages still run on the list's prefix."""
    errs, fails, info, _ = run_emul(dict(nms_radius=None), lattice(96))
    assert not fails, (fails, errs)
    assert info["overflow"] and info["count"] == -1, info


def _records(rows):
    from lightglue_b200 import _cabi

    k = np.zeros(len(rows), np.dtype(_cabi.SIFT_KPT_DTYPE))
    for i, (x, y, size, angle, resp) in enumerate(rows):
        k[i] = (x, y, size, angle, resp, 1 << 8, 1, 1)
    return k


@needs_emul
@pytest.mark.parametrize("nms_radius", [None, 0, 1, 2])
@pytest.mark.parametrize("max_kpts", [3, 100])
def test_filtering_of_constructed_records(nms_radius, max_kpts):
    """The ordering and filtering functors on records no image gives: at pixel (5, 10) two records with equal score and
    equal angle (filter_dog_point keeps both), one with that score and a larger angle and one with a lower score (both
    dropped); an exact duplicate (removed by the dedupe); a lower score two columns away (suppressed by NMS of radius
    2, kept at radius 1); a tie of scores at another pixel across the nfeatures cut."""
    k = _records([(10.2, 5.3, 3.0, 30.0, 0.05), (10.4, 5.3, 3.0, 30.0, 0.05), (10.1, 5.4, 2.5, 45.0, 0.05),
                  (10.3, 5.2, 2.0, 10.0, 0.04), (10.2, 5.3, 3.0, 30.0, 0.05), (12.0, 5.0, 2.0, 5.0, 0.03),
                  (40.0, 30.0, 2.0, 5.0, 0.05), (60.0, 30.0, 2.0, 5.0, 0.02)])
    w = 64
    got = sift_emul.filter_records(k, w, nms_radius, max_kpts)
    n = len(k)
    order = so.lex_order(k)
    assert np.array_equal(got["order"][:n], order)
    s = k[order]
    uniq, keep, cut = so.retain(s, max_kpts)
    pi, pj = so.pixels(s)
    fl = got["flags"][:n]
    assert np.array_equal(got["pix"][:n], pi * w + pj)
    assert np.array_equal(fl & 3, uniq * 1 + keep * 2) and bool(got["counters"][1]) == cut
    dup = so.dog_filter(s, keep, w) if nms_radius is not None else keep
    assert np.array_equal(fl & 4, dup * 4)
    alive = so.nms(s, dup, -1 if nms_radius is None else nms_radius)
    assert np.array_equal(fl & 8, alive * 8)
    out, _ = so.select(s, alive, cut, max_kpts)
    assert got["counters"][2] == len(out) and np.array_equal(got["out_src"][:len(out)], out)
    # the regimes: the equal-score, equal-angle pair at one pixel survives filter_dog_point together
    if nms_radius is not None and not cut:
        pair = [i for i in range(n) if s["angle"][i] == 30.0 and s["response"][i] == F32(0.05) and uniq[i]]
        assert len(pair) == 2 and all(fl[i] & 4 for i in pair), fl
        if nms_radius == 2:
            assert not fl[list(s["response"]).index(F32(0.03))] & 8


@needs_emul
def test_near_blank_image_has_no_keypoints():
    img = torch.full((1, 1, 64, 64), 0.5)
    img[0, 0, 30, 30] = 0.502
    errs, fails, info, _ = run_emul({}, img)
    assert not fails, (fails, errs)
    assert info["n_out"] == 0 and not info["overflow"], info


@needs_emul
@pytest.mark.parametrize("defect", so.DEFECTS)
def test_each_defect_fails_exactly_its_own_stage(defect):
    """Every stage check passes the host build with the correct oracle; with one defect switched on, the stages it
    belongs to fail even at 3x their tolerance and every other stage still passes."""
    own = {s for s, ds in OWN.items() if defect in ds}
    img = sift_synth.make_image(120, 160, 1, 21)
    runs = [({"nms_radius": 3} if defect == "nms_radius" else {}, img)]
    if defect == "retain_gt":
        t = tiled(128, 128, 32, 24)
        runs = [(dict(nms_radius=None, max_num_keypoints=tie_cut(run_emul(dict(nms_radius=None), t)[3])), t)]
    strict = {k: (v * 3 if k in TOL and not k.endswith(("margin_x", "margin_rel", "margin_bin", "margin_peak", "half"))
                  else v) for k, v in TOL.items()}
    failed = set()
    for conf, image in runs:
        errs, fails, _, _ = run_emul(conf, image, defect=defect, tol=strict)
        failed |= set(fails)
        _, loose, _, _ = run_emul(conf, image, defect=defect)
        assert set(loose) <= own, (defect, loose)
    assert failed == own, (defect, failed, errs)


def test_fast_atan2_polynomial_is_within_its_bound_of_atan2():
    """The polynomial's constants are OpenCV's: its distance from atan2 over the circle is 0.00955 degrees; a change
    of 0.1 % in any one constant moves it above 0.0104."""
    t = torch.linspace(0, 2 * math.pi, 200001, dtype=torch.float64)
    for rad in (1.0, 1e-3, 300.0):
        y, x = rad * torch.sin(t), rad * torch.cos(t)
        ref = torch.rad2deg(torch.atan2(y, x)) % 360
        d = (so.fast_atan2(y, x) - ref + 180) % 360 - 180
        assert float(d.abs().max()) < 0.0096
        assert float(d.abs().max()) > 0.001  # the polynomial, not atan2 itself


def test_reflect101_repeats_for_wide_kernels():
    p = np.arange(-9, 13)
    assert so.reflect(p, 4).tolist() == [3, 2, 1, 0, 1, 2, 3, 2, 1, 0, 1, 2, 3, 2, 1, 0, 1, 2, 3, 2, 1, 0]
    assert so.reflect(np.array([-2, -1, 4, 5]), 4, "reflect").tolist() == [1, 0, 3, 2]
