"""Keypoint selection without a GPU: every constructed SuperPoint case of ``oracle/keypoint_cases.py`` through the
post-processing functors on the host (``oracle/sp_emul.cpp`` ``sp_emul_post``, on a workspace laid out by
``sp_workspace_layout``), stage by stage against the oracle, and each case's regime; the DISK cases' regimes on the
oracle; the gates against the listed defects; and the host checks of ``sp_workspace_layout``, ``sp_post`` and
``disk_detect``.  The GPU run of the same cases is tests/test_gpu_keypoint_selection.py."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from lightglue_b200 import _cabi
from oracle import keypoint_cases as kc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SP_CASES = kc.sp_cases()
DISK_CASES = kc.disk_cases()


@pytest.fixture(scope="module")
def emul():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_build", "libsp_emul.so"))
    lib.sp_emul_post.restype = C.c_int
    return lib


def sp_config(case, thr, k, precision=0):
    return _cabi.SpConfig(_cabi.SP_ABI_VERSION, case.nms_radius, k, case.remove_borders, thr, precision)


def layout(cfg, b, h, w):
    n = _cabi.SP_LAYOUT_BUFFERS
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    total = _cabi.load().sp_workspace_layout(C.byref(cfg), b, h, w, off, size)
    return total, list(off), list(size)


def run_emulated(lib, case, thr, k):
    b, h, w = case.shape
    cfg = sp_config(case, thr, k)
    total, off, size = layout(cfg, b, h, w)
    cap = k if k > 0 else (h + case.nms_radius) // (case.nms_radius + 1) * ((w + case.nms_radius) // (case.nms_radius + 1))
    ws = torch.zeros(total, dtype=torch.uint8)
    kp, ks = torch.full((b, cap, 2), 7.0), torch.full((b, cap), 7.0)
    de, cnt = torch.full((b, cap, 256), 7.0), torch.full((b,), -5, dtype=torch.int32)
    lg, dn = case.logits.contiguous(), case.dense.contiguous()
    rc = lib.sp_emul_post(case.nms_radius, k, case.remove_borders, C.c_float(thr), C.c_void_p(lg.data_ptr()),
                          C.c_void_p(dn.data_ptr()), b, h, w, C.c_long(cap), C.c_void_p(kp.data_ptr()),
                          C.c_void_p(ks.data_ptr()), C.c_void_p(de.data_ptr()), C.c_void_p(cnt.data_ptr()),
                          C.c_void_p(ws.data_ptr()), C.c_size_t(total))
    assert rc == 0
    assert torch.equal(ws[off[0]:off[0] + size[0]].view(torch.float32).view_as(lg), lg), "the logits' copy"
    v = kc.sp_views(ws, off, size, b, h, w, cap)
    return kc.captured_stages(v, (kp, ks, de, cnt), thr, k)


def resolve(case, run):
    """The case's threshold and k, reading a first run where they depend on its captured stages."""
    thr, k = case.threshold, case.k
    if callable(thr) or callable(k):
        first = run(0.0005 if callable(thr) else thr, 0)
        thr = thr(first) if callable(thr) else thr
        k = k(first) if callable(k) else k
    return float(torch.tensor(thr, dtype=torch.float32)), int(k)


@pytest.mark.parametrize("case", SP_CASES, ids=[c.name for c in SP_CASES])
def test_sp_functors_on_host_stage_by_stage(emul, case):
    thr, k = resolve(case, lambda t, kk: run_emulated(emul, case, t, kk))
    st = run_emulated(emul, case, thr, k)
    print(f"{case.name}: {case.regime(st)}")
    worst = {}
    bad = kc.check_sp(case, st, worst)
    print("  deviation:", {n: f"{v:.1e}" for n, v in worst.items()})
    assert not bad, bad


@pytest.mark.parametrize("case", SP_CASES, ids=[c.name for c in SP_CASES])
def test_sp_gates_sit_below_the_listed_defects(emul, case):
    """Each gate is at most a third of every listed defect the case can show."""
    thr, k = resolve(case, lambda t, kk: run_emulated(emul, case, t, kk))
    defects = kc.sp_defects(case, run_emulated(emul, case, thr, k))
    gate = {"scores": kc.SCORE_TOL, "half-pixel shift": kc.DESC_TOL, "align_corners=False": kc.DESC_TOL}
    for name, d in defects.items():
        assert d >= 3 * gate[name], (name, d)


@pytest.mark.parametrize("case", DISK_CASES, ids=[c.name for c in DISK_CASES])
def test_disk_case_regimes_on_the_oracle(case):
    n = kc.disk_n(case)
    cands, sel = [], []
    for img in case.heat:
        cands.append(kc.disk_candidates(img, case.window, case.threshold).tolist())
        pos, _ = kc.disk_expected(img, case.window, case.threshold, n)
        w = img.shape[1]
        sel.append([(p % w, p // w) for p in pos.tolist()])
    print(f"{case.name}: {case.regime(cands, sel)}")


# ---------------------------------------------------------------------------------------------- host checks
@pytest.mark.parametrize("prec,k,r,b,h,w", [(0, 0, 4, 1, 8, 8), (1, 0, 4, 2, 203, 317), (0, 1024, 2, 3, 240, 320),
                                            (1, 4097, 0, 1, 1040, 16)])
def test_sp_workspace_layout(prec, k, r, b, h, w):
    """Buffers disjoint, 256-aligned and inside sp_workspace_bytes' total, each sized as sp_carve sizes it; the
    tensor-core part of precision 1 follows them."""
    cfg = _cabi.SpConfig(_cabi.SP_ABI_VERSION, r, k, 4, 0.0005, prec)
    total, off, size = layout(cfg, b, h, w)
    px, cells = b * h * w, b * (h // 8) * (w // 8)
    cap = k if k > 0 else -(-h // (r + 1)) * -(-w // (r + 1))
    want = dict(logits=65 * cells * 4, scores=px * 4, t0=px * 4, mask=px * 4, dense=256 * cells * 4, row_count=b * h * 4,
                row_start=b * h * 4, n_cand=b * 4, cand_pos=px * 4, cand_score=px * 4, sel_pos=b * cap * 4,
                sel_score=b * cap * 4, n_sel=b * 4)
    assert dict(zip(kc.SP_LAYOUT_NAMES, size)) == want
    spans = sorted(zip(off, size))
    assert all(o % 256 == 0 for o in off)
    for (o0, n0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + n0 <= o1
    end = (spans[-1][0] + spans[-1][1] + 255) // 256 * 256
    tc = _cabi.load().sp_tc_layout(b, h, w, None, None)
    assert tc > 0 and total == end + (tc if prec == 1 else 0)


def test_sp_workspace_layout_rejects_bad_arguments():
    lib = _cabi.load()
    cfg = _cabi.SpConfig(_cabi.SP_ABI_VERSION, 4, 0, 4, 0.0005, 0)
    assert lib.sp_workspace_layout(None, 1, 64, 64, None, None) == 0
    for b, h, w in ((0, 64, 64), (1, 7, 64), (1, 64, 7)):
        assert lib.sp_workspace_layout(C.byref(cfg), b, h, w, None, None) == 0
    for field, v in (("precision", 2), ("nms_radius", -1)):
        bad = _cabi.SpConfig(_cabi.SP_ABI_VERSION, 4, 0, 4, 0.0005, 0)
        setattr(bad, field, v)
        assert lib.sp_workspace_layout(C.byref(bad), 1, 64, 64, None, None) == 0
    assert lib.sp_workspace_layout(C.byref(cfg), 1, 64, 64, None, None) > 0


def test_null_handles_are_rejected_before_device_work():
    lib = _cabi.load()
    one = C.c_void_p(16)  # never dereferenced: the null handle is rejected first
    assert lib.sp_post(None, one, one, 1, 64, 64, 100, one, one, one, one, one, 1 << 30, None) != 0
    assert lib.lg_last_error().decode() == "sp_post: null argument"
    assert lib.disk_detect(None, one, 1, 64, 64, 100, one, one, one, one, 1 << 30, None) != 0
    assert lib.lg_last_error().decode() == "disk_detect: null argument"
