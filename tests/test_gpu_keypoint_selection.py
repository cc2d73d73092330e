"""Keypoint selection on the GPU: SuperPoint's post-processing (``sp_post``) and DISK's detection (``disk_detect``) on the
constructed inputs of ``oracle/keypoint_cases.py``, stage by stage against the oracle applied to the captured output of
the stage before (the NMS map, candidates and selection exactly; scores, the normalised map and descriptors within the
gates of keypoint_cases), for both SuperPoint handles: the functors (fp32) and the warp / block kernels of the
tensor-core mode (bf16x3).  Also: the two handles agree bit for bit on the keypoints of the same logits and dense map;
``sp_forward`` is ``sp_backbone`` then ``sp_post``; ``disk_detect`` on ``disk_heads``' heatmap is ``disk_forward``'s
detection; and the entries reject bad arguments."""
import ctypes as C

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.disk import DISK
from lightglue_b200.superpoint import SuperPoint
from oracle import keypoint_cases as kc
from oracle import superpoint_synth as sps

pytestmark = pytest.mark.gpu

SP_CASES = kc.sp_cases()
DISK_CASES = kc.disk_cases()
PRECISIONS = (0, 1)  # fp32 functors, tensor-core mode's kernels
WORST = {}
_handles = {}  # SpConfig bytes -> handle
_blob = []


@pytest.fixture(scope="module", autouse=True)
def report_and_release():
    yield
    print("\nworst deviation:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})
    lib = _cabi.load()
    for h in _handles.values():
        lib.sp_destroy(h)
    _handles.clear()


def blob():
    if not _blob:
        m = SuperPoint(weights=None)
        m.load_state_dict(sps.make_superpoint_state_dict(0))
        _blob.append(m._blob().cuda())
    return _blob[0]


def sp_handle(cfg):
    key = bytes(cfg)
    if key not in _handles:
        b = blob()
        h = C.c_void_p()
        lib = _cabi.load()
        _cabi.check(lib.sp_create(C.byref(cfg), b.data_ptr(), b.numel(), torch.cuda.current_stream().cuda_stream,
                                  C.byref(h)), "sp_create")
        torch.cuda.synchronize()
        _handles[key] = h
    return _handles[key]


def sp_cfg(r, k, borders, thr, prec):
    return _cabi.SpConfig(_cabi.SP_ABI_VERSION, r, k, borders, thr, prec)


def sp_run(cfg, logits, dense, b, h, w, image=None):
    """sp_post (or sp_forward on `image`) on a zero-filled workspace -> (views by layout name, outputs)."""
    lib = _cabi.load()
    handle = sp_handle(cfg)
    n = _cabi.SP_LAYOUT_BUFFERS
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    total = lib.sp_workspace_layout(C.byref(cfg), b, h, w, off, size)
    assert total == lib.sp_workspace_bytes(handle, b, h, w) > 0
    cap = int(lib.sp_max_keypoints(handle, h, w))
    ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
    kp, ks = torch.full((b, cap, 2), 7.0, device="cuda"), torch.full((b, cap), 7.0, device="cuda")
    de, cnt = torch.full((b, cap, 256), 7.0, device="cuda"), torch.full((b,), -5, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    tail = (cap, kp.data_ptr(), ks.data_ptr(), de.data_ptr(), cnt.data_ptr(), ws.data_ptr(), total, stream)
    if image is None:
        lg, dn = logits.cuda().contiguous(), dense.cuda().contiguous()
        lg0, dn0 = lg.clone(), dn.clone()
        _cabi.check(lib.sp_post(handle, lg.data_ptr(), dn.data_ptr(), b, h, w, *tail), "sp_post")
        torch.cuda.synchronize()
        assert torch.equal(lg, lg0) and torch.equal(dn, dn0), "sp_post modified its inputs"
    else:
        _cabi.check(lib.sp_forward(handle, image.data_ptr(), b, h, w, *tail), "sp_forward")
        torch.cuda.synchronize()
    return kc.sp_views(ws, list(off), list(size), b, h // 8 * 8, w // 8 * 8, cap), (kp, ks, de, cnt)


def resolve(case, run):
    thr, k = case.threshold, case.k
    if callable(thr) or callable(k):
        first = run(0.0005 if callable(thr) else thr, 0)
        thr = thr(first) if callable(thr) else thr
        k = k(first) if callable(k) else k
    return float(torch.tensor(thr, dtype=torch.float32)), int(k)


def run_case(case, prec, thr, k):
    b, h, w = case.shape
    v, out = sp_run(sp_cfg(case.nms_radius, k, case.remove_borders, thr, prec), case.logits, case.dense, b, h, w)
    return kc.captured_stages(v, out, thr, k)


@pytest.mark.parametrize("case", SP_CASES, ids=[c.name for c in SP_CASES])
def test_sp_post_stage_by_stage_both_handles(case):
    thr, k = resolve(case, lambda t, kk: run_case(case, 1, t, kk))
    st = {}
    for prec in PRECISIONS:
        st[prec] = run_case(case, prec, thr, k)
        print(f"[{'bf16x3' if prec else 'fp32'}] {case.name}: {case.regime(st[prec])}")
        worst = {}
        bad = kc.check_sp(case, st[prec], worst)
        for n, e in worst.items():
            WORST[n] = max(WORST.get(n, 0.0), e)
        assert not bad, (prec, bad)
    assert_same_keypoints(st[0]["out"], st[1]["out"])


def assert_same_keypoints(a, b):
    """The fp32 and bf16x3 handles on the same logits and dense map: counts, keypoints and scores bit for bit,
    descriptors within the sampling gate."""
    (kp0, ks0, de0, c0), (kp1, ks1, de1, c1) = a, b
    assert torch.equal(c0, c1) and torch.equal(kp0, kp1) and torch.equal(ks0, ks1)
    d = float((de0.double() - de1.double()).abs().max()) if de0.numel() else 0.0
    WORST["descriptors fp32 vs bf16x3"] = max(WORST.get("descriptors fp32 vs bf16x3", 0.0), d)
    assert d <= kc.DESC_TOL


def backbone(prec, image, r=4, k=0, borders=4, thr=0.0005):
    b, _, h, w = image.shape
    lib = _cabi.load()
    cfg = sp_cfg(r, k, borders, thr, prec)
    handle = sp_handle(cfg)
    ws = torch.zeros(lib.sp_workspace_bytes(handle, b, h, w), dtype=torch.uint8, device="cuda")
    lg = torch.empty(b, 65, h // 8, w // 8, device="cuda")
    dn = torch.empty(b, 256, h // 8, w // 8, device="cuda")
    _cabi.check(lib.sp_backbone(handle, image.data_ptr(), b, h, w, lg.data_ptr(), dn.data_ptr(), ws.data_ptr(), ws.numel(),
                                torch.cuda.current_stream().cuda_stream), "sp_backbone")
    torch.cuda.synchronize()
    return cfg, lg, dn


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("b,h,w,k", [(1, 67, 45, 0), (3, 64, 96, 50), (1, 240, 320, 0), (3, 240, 320, 300)])
def test_sp_forward_is_backbone_then_post(prec, b, h, w, k):
    image = sps.make_image(h, w, b, 300 + h).cuda().contiguous()
    cfg, lg, dn = backbone(prec, image, k=k)
    v0, out0 = sp_run(cfg, None, None, b, h, w, image=image)
    v1, out1 = sp_run(cfg, lg, dn, b, h, w)
    for x, y in zip(out0, out1):
        assert torch.equal(x, y)
    for name in kc.SP_LAYOUT_NAMES:
        assert torch.equal(v0[name], v1[name]), name
    assert int(out0[3].min()) > 0


@pytest.mark.parametrize("h,w,k", [(240, 320, 0), (768, 1024, 0), (768, 1024, 2048)])
def test_sp_handles_agree_on_backbone_outputs(h, w, k):
    """Real logits and dense maps (the tensor-core backbone's): both handles' post-processing, stage by stage and
    against each other."""
    image = sps.make_image(h, w, 1, 400 + h).cuda().contiguous()
    _, lg, dn = backbone(1, image)
    case = kc.SpCase(f"backbone {h}x{w}", lg.cpu(), dn.cpu(), lambda st: "", k=k)
    st = {}
    for prec in PRECISIONS:
        st[prec] = run_case(case, prec, 0.0005, k)
        worst = {}
        bad = kc.check_sp(case, st[prec], worst)
        for n, e in worst.items():
            WORST[n] = max(WORST.get(n, 0.0), e)
        assert not bad, (prec, bad)
    assert int(st[0]["n_sel"][0]) > 100
    assert_same_keypoints(st[0]["out"], st[1]["out"])


def test_sp_post_rejects_bad_arguments():
    lib = _cabi.load()
    cfg = sp_cfg(4, 0, 4, 0.0005, 1)
    h = sp_handle(cfg)
    b, hh, ww = 1, 64, 64
    cap = int(lib.sp_max_keypoints(h, hh, ww))
    need = lib.sp_workspace_bytes(h, b, hh, ww)
    t = torch.zeros(need, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    s = torch.cuda.current_stream().cuda_stream

    def call(*args):
        rc = lib.sp_post(*args)
        return rc, lib.lg_last_error().decode()

    good = [h, p, p, b, hh, ww, cap, p, p, p, p, p, need, s]
    for i in (0, 1, 2, 7, 8, 9, 10):
        a = list(good)
        a[i] = None
        rc, err = call(*a)
        assert rc != 0 and err == "sp_post: null argument", (i, err)
    for i, v, msg in ((4, 7, "H and W must be at least 8"), (5, 7, "H and W must be at least 8"),
                      (3, 0, "H and W must be at least 8"), (6, cap - 1, "output capacity below sp_max_keypoints()"),
                      (12, need - 1, "workspace too small"), (11, None, "workspace too small")):
        a = list(good)
        a[i] = v
        rc, err = call(*a)
        assert rc != 0 and err == f"sp_post: {msg}", (i, err)


# ---------------------------------------------------------------------------------------------- DISK
_disk = {}


def disk_model(window, n, thr):
    key = (window, n, thr)
    if key not in _disk:
        m = DISK(weights=None, nms_window_size=window, max_num_keypoints=n, detection_threshold=thr).cuda()
        _disk[key] = m
    return _disk[key]


def disk_detect(m, heat):
    lib = _cabi.load()
    heat = heat.cuda().contiguous()
    b, h, w = heat.shape
    handle = m._get_handle(heat.device)
    cap = int(lib.disk_max_keypoints(handle, h, w))
    ws = torch.zeros(lib.disk_workspace_bytes(handle, b, h, w), dtype=torch.uint8, device="cuda")
    pos = torch.full((b, cap), 7, dtype=torch.int32, device="cuda")
    sc = torch.full((b, cap), 7.0, device="cuda")
    cnt = torch.full((b,), -5, dtype=torch.int32, device="cuda")
    _cabi.check(lib.disk_detect(handle, heat.data_ptr(), b, h, w, cap, pos.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), "disk_detect")
    torch.cuda.synchronize()
    return pos.cpu(), sc.cpu(), cnt.cpu(), (handle, ws, cap)


@pytest.mark.parametrize("case", DISK_CASES, ids=[c.name for c in DISK_CASES])
def test_disk_detect_exactly(case):
    n = kc.disk_n(case)
    pos, sc, cnt, _ = disk_detect(disk_model(case.window, n, case.threshold), case.heat)
    cands, sel = [], []
    for i, img in enumerate(case.heat):
        w = img.shape[1]
        rp, rs = kc.disk_expected(img, case.window, case.threshold, n)
        k = int(cnt[i])
        assert k == rp.numel(), (i, k, rp.numel())
        assert torch.equal(pos[i, :k].long(), rp) and torch.equal(sc[i, :k], rs.float())
        assert not pos[i, k:].any() and not sc[i, k:].any()
        cands.append(kc.disk_candidates(img, case.window, case.threshold).tolist())
        sel.append([(p % w, p // w) for p in pos[i, :k].tolist()])
    print(f"{case.name}: {case.regime(cands, sel)}")


@pytest.mark.parametrize("b,h,w,n", [(1, 240, 320, None), (2, 200, 232, 300)])
def test_disk_detect_on_heads_is_forward(b, h, w, n):
    from oracle import disk_synth as ds

    m = DISK(weights=None, max_num_keypoints=n)
    m.model.load_state_dict(ds.make_disk_state_dict(0))
    m = m.cuda()
    lib = _cabi.load()
    image = ds.make_image(h, w, b, 7).cuda().contiguous()
    handle = m._get_handle(image.device)
    cap = int(lib.disk_max_keypoints(handle, h, w))
    ws = torch.zeros(lib.disk_workspace_bytes(handle, b, h, w), dtype=torch.uint8, device="cuda")
    heat = torch.empty(b, h, w, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.disk_heads(handle, image.data_ptr(), image.shape[1], b, h, w, None, 0, heat.data_ptr(), None,
                               ws.data_ptr(), ws.numel(), s), "disk_heads")
    kp = torch.zeros(b, cap, 2, device="cuda")
    sc = torch.zeros(b, cap, device="cuda")
    de = torch.zeros(b, cap, 128, device="cuda")
    cnt = torch.zeros(b, dtype=torch.int32, device="cuda")
    _cabi.check(lib.disk_forward(handle, image.data_ptr(), image.shape[1], b, h, w, cap, kp.data_ptr(), sc.data_ptr(),
                                 de.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), s), "disk_forward")
    torch.cuda.synchronize()
    pos, dsc, dcnt, _ = disk_detect(m, heat)
    assert torch.equal(dcnt, cnt.cpu()) and int(dcnt.min()) > 0
    xy = torch.stack([pos % w, pos // w], -1).float()
    for i in range(b):
        k = int(dcnt[i])
        assert torch.equal(xy[i, :k], kp[i, :k].cpu()) and torch.equal(dsc[i, :k], sc[i, :k].cpu())


def test_disk_detect_rejects_bad_arguments():
    m = disk_model(5, None, 0.0)
    heat = torch.zeros(1, 64, 64)
    _, _, _, (handle, ws, cap) = disk_detect(m, heat)
    lib = _cabi.load()
    p, n, s = ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream
    good = [handle, p, 1, 64, 64, cap, p, p, p, p, n, s]
    for i in (0, 1, 6, 7, 8):
        a = list(good)
        a[i] = None
        assert lib.disk_detect(*a) != 0 and lib.lg_last_error().decode() == "disk_detect: null argument"
    for i, v, msg in ((3, 16, "disk: the padded image needs at least two pixels at 1/16 resolution"),
                      (2, 0, "disk: B, H and W must be positive"),
                      (5, cap - 1, "disk_detect: output capacity below disk_max_keypoints()"),
                      (10, n - 1, "disk_detect: workspace too small"), (9, None, "disk_detect: workspace too small")):
        a = list(good)
        a[i] = v
        if i == 3:
            a[4] = 16
        assert lib.disk_detect(*a) != 0 and lib.lg_last_error().decode() == msg, (i, lib.lg_last_error())
