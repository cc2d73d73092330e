"""SIFT's CUDA stages against float64 from the kernels' own inputs (oracle/sift_oracle.py).

``sift_forward`` is called through the C ABI on a workspace the test owns; ``sift_workspace_layout`` says where the last
image's intermediates sit in it (include/sift_b200.h).  Exact: the gray crop, each octave's base as the decimation of
the previous octave, every DoG layer as the fp32 difference of the captured Gaussians, every Gaussian and DoG layer bit
for bit against the host build, the lexicographic order, the filtering flags, pixels, output slots and counters from the
captured raw keypoints, the output rows and counts.  Within the tolerances of tests/test_sift_layer_emulation.py: each
Gaussian from its captured predecessor (the first from the captured crop), the candidates from the captured DoG, the
raw keypoints' orientations from the captured candidates and Gaussians, the descriptors from the captured Gaussians and
selected keypoints, RootSIFT from the uint8 descriptors.  Every case asserts the regimes it claims to reach."""
import ctypes as C

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.sift import SIFT
from oracle import sift_emul, sift_oracle as so, sift_synth
from tests.test_sift_layer_emulation import TOL, assert_decided, lattice, tie_cut, tiled

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst deviation:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})


def run_gpu(conf, image, sizes=None):
    """sift_forward on image [B, C, H, W] -> (capture of the last image, its output rows as numpy, crop (h, w))."""
    conf = {**SIFT.default_conf, **conf}
    cfg = SIFT(**conf)._config()
    lib = _cabi.load()
    b, ch, H, W = image.shape
    w, h = (int(sizes[-1][0]), int(sizes[-1][1])) if sizes is not None else (W, H)
    lay = so.layout(cfg, H, W, h, w)
    handle = C.c_void_p()
    _cabi.check(lib.sift_create(C.byref(cfg), None, C.byref(handle)), "sift_create")
    try:
        total = lib.sift_workspace_bytes(handle, b, H, W)
        assert total == lay["total"] > 0
        ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
        k = cfg.max_num_keypoints
        img = image.cuda().contiguous()
        out = {"keypoints": torch.full((b, k, 2), 7.0, device="cuda"), "scales": torch.full((b, k), 7.0, device="cuda"),
               "oris": torch.full((b, k), 7.0, device="cuda"), "scores": torch.full((b, k), 7.0, device="cuda"),
               "descriptors": torch.full((b, k, 128), 7.0, device="cuda"),
               "count": torch.full((b,), -5, dtype=torch.int32, device="cuda")}
        sz = None if sizes is None else torch.as_tensor(sizes, dtype=torch.int32).contiguous()
        _cabi.check(lib.sift_forward(handle, img.data_ptr(), ch, None if sz is None else sz.data_ptr(), b, H, W, k,
                                     out["keypoints"].data_ptr(), out["scales"].data_ptr(), out["oris"].data_ptr(),
                                     out["scores"].data_ptr(), out["descriptors"].data_ptr(), out["count"].data_ptr(),
                                     ws.data_ptr(), total, torch.cuda.current_stream().cuda_stream), "sift_forward")
        torch.cuda.synchronize()
    finally:
        lib.sift_destroy(handle)
    base = (-ws.data_ptr()) % 256
    cap = so.capture(ws[base:], lay, h, w)
    return cap, {key: v[-1].cpu().numpy() for key, v in out.items()}, (h, w), conf


def check(conf, image, sizes=None, regimes=(), bitwise=True):
    cap, out, (h, w), conf = run_gpu(conf, image, sizes)
    errs, fails, info, sel = so.check_stages(cap, conf, image[-1], h, w, TOL)
    so.check_outputs(cap, conf, out, TOL, None, sel, errs, fails, info)
    for k, v in errs.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    assert not fails, (fails, errs, info)
    if bitwise and sift_emul.available():  # the pyramid has no libm call: both builds round the same
        _, ews = sift_emul.forward_ws(conf, image, sizes)
        emu = so.capture(ews, so.layout(SIFT(**conf)._config(), *image.shape[2:], h, w), h, w)
        for o in range(len(cap["gauss"])):
            for a, b in zip(cap["gauss"][o] + cap["dog"][o], emu["gauss"][o] + emu["dog"][o]):
                assert torch.equal(a.cpu(), b), o
    for r in regimes:
        assert info[r], (r, info)
    assert_decided(info)
    return cap, info


# (h, w, conf, regimes): octaves narrower than the kernel radius, odd sizes, thin strips, the default conf
SHAPES = [
    (8, 8, {}, ("multi_reflect",)),
    (16, 16, dict(num_octaves=8), ("multi_reflect",)),
    (17, 23, dict(num_octaves=1), ("multi_reflect",)),
    (33, 47, dict(nms_radius=None, rootsift=False), ("multi_reflect",)),
    (203, 317, dict(nms_radius=1), ("multi_reflect", "pixel_dup_equal", "desc_border_clip")),
    (32, 1024, dict(num_octaves=1, nms_radius=3), ("multi_reflect",)),
    (1024, 32, dict(num_octaves=8, rootsift=False), ("multi_reflect",)),
    (240, 320, dict(nms_radius=3), ("nms_suppression", "wrap_peak", "desc_border_clip")),
    (768, 1024, {}, ("pixel_dup_equal", "wrap_peak", "desc_border_clip")),
]


@pytest.mark.parametrize("h,w,conf,regimes", SHAPES, ids=[f"{s[0]}x{s[1]}" for s in SHAPES])
def test_stages_at_shape(h, w, conf, regimes):
    check(conf, sift_synth.make_image(h, w, 1, 31 + h + w), regimes=regimes)


def test_tie_at_the_cut_and_top_k():
    """A patch tiled at one deepest-octave pixel (32 px at 128x128): nfeatures inside a run of equal responses, so
    retainBest keeps the whole tie and, without filter_dog_point, the top-k applies with ties in its order."""
    img = tiled(128, 128, 32, 24)
    cap, _, _, _ = run_gpu(dict(nms_radius=None), img)
    k = tie_cut(cap["kpt"])
    _, info = check(dict(nms_radius=None, max_num_keypoints=k), img, regimes=("cut_tie", "topk"))
    assert info["n_out"] == k


def test_tie_at_the_cut_with_filtering():
    img = tiled(128, 160, 32, 26)
    cap, _, _, _ = run_gpu({}, img)
    check(dict(max_num_keypoints=tie_cut(cap["kpt"])), img, regimes=("cut_tie", "pixel_dup_equal"))


def test_cut_between_distinct_responses():
    img = sift_synth.make_image(240, 320, 1, 29)
    cap, _, _, _ = run_gpu({}, img)
    _, info = check(dict(max_num_keypoints=tie_cut(cap["kpt"], tie=False)), img, regimes=("cut",))
    assert not info["cut_tie"]


def test_batch_of_three_with_crops():
    img = sift_synth.make_image(96, 128, 3, 27)
    check(dict(max_num_keypoints=64), img, sizes=[[128, 96], [101, 77], [117, 83]])


def test_mirror_symmetric_image():
    half = sift_synth.make_image(96, 64, 1, 28)
    check({}, torch.cat([half, half.flip(3)], 3).contiguous(), regimes=("pixel_dup_equal",))


def test_overflow_reports_minus_one():
    """More raw keypoints than the list holds (a dot lattice at 96x96): counts = -1; the pyramid, ordering and
    filtering stages are still checked on what the lists hold."""
    _, info = check(dict(nms_radius=None), lattice(96), regimes=("overflow",))
    assert info["count"] == -1


def test_near_blank_image_has_no_keypoints():
    img = torch.full((1, 1, 64, 64), 0.5)
    img[0, 0, 30, 30] = 0.502
    _, info = check({}, img)
    assert info["n_out"] == 0 and info["cand_total"] == 0
