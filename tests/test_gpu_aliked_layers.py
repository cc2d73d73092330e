"""ALIKED's CUDA stages against float64 given the kernels' own inputs, at the padding, tail and offset edges.

``al_forward`` is called through the C ABI with a workspace the test owns; ``al_workspace_layout`` says where each
stage's output sits in it after the call (include/aliked_b200.h lists what each buffer holds then).  Each check applies
a float64 stage of ``oracle/aliked_oracle.py`` on the GPU to the captured input and compares the captured output:
max|delta| / max|ref| per image; keypoints relative to the image's extent max(w - 1, h - 1), keypoint scores and unit
descriptors absolute.  The tolerances
come from tests/test_aliked_layer_emulation.py.

* Encoder: x1 from the replicate-padded image (block1's first convolution is overwritten); p1, p2, p3 from their
  inputs; block2's d2 and t2 from p1 and x2 from the captured t2, d2; block3 / block4's d and t from p (t with the
  offsets in float64: the first offset convolution is overwritten), o (the second offset convolution) from the captured
  t, x from the captured t, o and d; a2 .. a4 from x2 .. x4.
* Head: s1 and invn at every padded pixel from the captured x1 and a2 .. a4; s2, s3 and the pre-crop score each from
  its captured predecessor; the cropped score bit for bit.
* DKD, exactly on the captured fp32 score: the NMS map with its borders and the threshold mask, the counts, the
  selected positions in output order, the top-k filler, zero rows past each count; the mean against float64, with the
  NMS decisions within MEAN_MARGIN of it excluded (and counted).
* After DKD: normalised keypoints, keypoints and scores from the float64 soft-argmax at the selected positions, and
  descriptors from float64 SDDH on the captured maps and normalised keypoints."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from lightglue_b200 import _cabi
from lightglue_b200.aliked import ALIKED
from oracle import aliked_oracle as alo
from oracle import aliked_synth as als
from tests.test_aliked_host_api import LAYOUT_NAMES
from tests.test_aliked_layer_emulation import TOL

pytestmark = pytest.mark.gpu

MEAN_TOL, MEAN_MARGIN = TOL["mean"], TOL["mean_margin"]  # relative to the float64 mean
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst deviation:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})


def rel(a, ref):
    """max|a - ref| / max|ref| per image (dim 0) -> the largest of them."""
    d = (a.double() - ref).abs().flatten(1).amax(1) / ref.abs().flatten(1).amax(1)
    return float(d.max())


def check(bad, name, err, tol):
    """Records the deviation; a failure goes to `bad`, so that one call reports every check it fails."""
    WORST[name] = max(WORST.get(name, 0.0), err)
    if not err <= tol:
        bad.append((name, err, tol))


def expect(bad, name, ok):
    if not ok:
        bad.append(name)


def run(model_name, sd, image, conf, image_size=None):
    """al_forward on `image` [B, 3, H, W] (CUDA) -> (views of the workspace buffers by name, outputs, config)."""
    m = ALIKED(model_name=model_name, weights=None, **conf)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    lib = _cabi.load()
    b, _, h, w = image.shape
    cfg = m._config()
    handle = m._get_handle(image.device)
    n = _cabi.AL_LAYOUT_BUFFERS
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    total = lib.al_workspace_layout(C.byref(cfg), b, h, w, off, size)
    assert total == lib.al_workspace_bytes(handle, b, h, w) > 0
    ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
    cap = int(lib.al_max_keypoints(handle, h, w))
    dim = cfg.dim
    out = {"keypoints": torch.full((b, cap, 2), 7.0, device="cuda"), "scores": torch.full((b, cap), 7.0, device="cuda"),
           "descriptors": torch.full((b, cap, dim), 7.0, device="cuda"),
           "counts": torch.full((b,), -5, dtype=torch.int32, device="cuda")}
    size_t = None if image_size is None else image_size.to("cuda", torch.float32).contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.al_forward(handle, image.data_ptr(), None if size_t is None else size_t.data_ptr(), b, h, w, cap,
                               out["keypoints"].data_ptr(), out["scores"].data_ptr(), out["descriptors"].data_ptr(),
                               out["counts"].data_ptr(), ws.data_ptr(), total, stream), "al_forward")
    torch.cuda.synchronize()
    bufs = {}
    for i, k in enumerate(LAYOUT_NAMES):
        dt = torch.int32 if k in ("cnt", "sel_pos", "n_sel") else torch.float32
        bufs[k] = ws[off[i]:off[i] + size[i]].view(dt)
    return bufs, out, cfg, cap


def check_forward(bad, model_name, sd, image, conf, image_size=None, run=run):
    """Every stage of one al_forward call -> {"counts", "maxima" (positive NMS values per image), "passed" (values
    above the threshold, threshold mode), "undecided"}."""
    torch.set_grad_enabled(False)
    bufs, out, cfg, cap = run(model_name, sd, image, conf, image_size)
    sd64 = {k: v.to(image.device, torch.float64) for k, v in sd.items() if v.is_floating_point()}
    b, _, h, w = image.shape
    hp, wp = -(-h // 32) * 32, -(-w // 32) * 32
    c1, c2, c3, c4, dim, _, M = alo.CFGS[model_name]
    q, p0 = dim // 4, b * hp * wp

    def fmap(name, c, s, n0=0):
        return bufs[name][n0:n0 + b * c * (hp // s) * (wp // s)].view(b, c, hp // s, wp // s)

    D = torch.Tensor.double
    # ---- encoder
    x1 = fmap("x1", c1, 1)
    check(bad, "x1", rel(x1, alo.block(sd64, 1, alo.pad(D(image)))), TOL["x1"])
    check(bad, "p1", rel(fmap("p1", c1, 2), alo.pool(D(x1), 2)), TOL["pool"])
    p1 = D(fmap("p1", c1, 2))
    t2, d2, x2 = fmap("t2", c2, 2), fmap("d2", c2, 2), fmap("x2", c2, 2)
    check(bad, "d2", rel(d2, alo.downsample(sd64, "block2", p1)), TOL["conv"])
    check(bad, "t2", rel(t2, F.selu(alo.conv_bn(sd64, "block2", 1, p1))), TOL["conv"])
    check(bad, "x2", rel(x2, alo.block_out(sd64, "block2", D(t2), D(d2))), TOL["conv"])
    xs = [x1, x2]
    for i, (ci, co, s) in ((3, (c2, c3, 8)), (4, (c3, c4, 32))):
        blk = f"block{i}"
        p = fmap(f"p{i - 1}", ci, s)
        check(bad, f"p{i - 1}", rel(p, alo.pool(D(xs[-1]), 4)), TOL["pool"])
        t, d, o, x = fmap(f"t{i}", co, s), fmap(f"d{i}", co, s), fmap(f"o{i}", 18, s), fmap(f"x{i}", co, s)
        check(bad, f"d{i}", rel(d, alo.downsample(sd64, blk, D(p))), TOL["conv"])
        check(bad, f"t{i}", rel(t, F.selu(alo.conv_bn(sd64, blk, 1, D(p)))), TOL["dcn"])
        check(bad, f"o{i}", rel(o, alo.offsets(sd64, f"{blk}.conv2", D(t))), TOL["offset"])
        check(bad, f"x{i}", rel(x, alo.block_out(sd64, blk, D(t), D(d), D(o))), TOL["conv"])
        xs.append(x)
    a = [None] + [fmap(f"a{i}", q, s) for i, s in ((2, 2), (3, 8), (4, 32))]
    for i in (2, 3, 4):
        check(bad, f"a{i}", rel(a[i - 1], alo.aggregate(sd64, i, D(xs[i - 1]))), TOL["conv"])
    # ---- head
    x1234 = alo.upsample([alo.aggregate(sd64, 1, D(x1))] + [D(v) for v in a[1:]])
    s1 = fmap("s1", 8, 1)
    check(bad, "s1", rel(s1, alo.score_layer(sd64, 0, x1234)), TOL["head"])
    check(bad, "invn", rel(bufs["invn"][:p0].view(b, hp, wp), alo.inv_norm(x1234)), TOL["head"])
    s2, s3, pre = fmap("ta", 4, 1), fmap("ta", 4, 1, 4 * p0), fmap("img", 1, 1)
    check(bad, "s2", rel(s2, alo.score_layer(sd64, 2, D(s1))), TOL["score"])
    check(bad, "s3", rel(s3, alo.score_layer(sd64, 4, D(s2))), TOL["score"])
    check(bad, "pre-crop score", rel(pre, alo.score_layer(sd64, 6, D(s3))), TOL["score"])
    score = bufs["score"][:b * h * w].view(b, 1, h, w)
    expect(bad, "score is the crop", torch.equal(score, alo.crop(pre, h, w)))
    # ---- DKD, exactly on the captured score
    r, thr, k = cfg.nms_radius, cfg.detection_threshold, cfg.max_num_keypoints
    topk = not thr > 0 and k > 0
    nms = alo.nms_borders(score.clone(), r, image_size)
    flat = nms.reshape(b, -1)
    nms_gpu = bufs["nms"][:b * h * w].view(b, h * w)
    n_sel = bufs["n_sel"][:b].cpu()
    undecided = 0
    thr_b = None
    if topk:
        expect(bad, "nms map", torch.equal(nms_gpu, flat))
    else:
        cnt = (flat > torch.tensor(thr, dtype=torch.float32)).sum(1).to(torch.int32)
        expect(bad, "cnt", torch.equal(bufs["cnt"][:b], cnt))
        mean = bufs["mean"][:b]
        mean64 = D(score).reshape(b, -1).mean(1)
        check(bad, "mean", float(((D(mean) - mean64).abs() / mean64).max()), MEAN_TOL)
        fallback = not (thr > 0 and int(cnt.sum()) > 0)
        thr_b = (mean if fallback else torch.full_like(mean, thr))[:, None]
        expect(bad, "nms map with the mask", torch.equal(nms_gpu, torch.where(flat > thr_b, flat, torch.full_like(flat, -1.0))))
        if fallback:  # the mask's decisions against the float64 mean, away from it
            near = (D(flat) - mean64[:, None]).abs() <= MEAN_MARGIN * mean64[:, None]
            undecided = int(near.sum())
            expect(bad, "mask decisions vs the float64 mean",
                   torch.equal((D(flat) > mean64[:, None])[~near], (nms_gpu > 0)[~near]))
    idx = alo.select(nms, score, thr, k, thr=thr_b)
    expect(bad, f"counts {n_sel.tolist()} vs {[len(v) for v in idx]}",
           n_sel.tolist() == [len(v) for v in idx] == out["counts"].cpu().tolist())
    sel_pos = bufs["sel_pos"][:b * cap].view(b, cap)
    sel_score = bufs["sel_score"][:b * cap].view(b, cap)
    kpn = bufs["kpn"][:b * cap * 2].view(b, cap, 2)
    gflat = nms_gpu if not topk else flat
    for i in range(b):
        n, pos = len(idx[i]), idx[i]
        expect(bad, f"image {i}: selected positions", torch.equal(sel_pos[i, :n].long(), pos))
        expect(bad, f"image {i}: selected scores", torch.equal(sel_score[i, :n], gflat[i, pos]))
        for name, t in (("kpn", kpn), ("keypoints", out["keypoints"]), ("scores", out["scores"]),
                        ("descriptors", out["descriptors"])):
            expect(bad, f"image {i}: {name} zero past the count", not t[i, n:].any())
        if n == 0:
            continue
        kp64, ks64, _ = alo.soft_argmax(D(score[i]), pos, r)
        px64, ext = alo.pixels(kp64, h, w), max(w - 1, h - 1)
        check(bad, "kpn", float((alo.pixels(D(kpn[i, :n]), h, w) - px64).abs().max()) / ext, TOL["kpt"])
        check(bad, "keypoints", float((D(out["keypoints"][i, :n]) - px64).abs().max()) / ext, TOL["kpt"])
        check(bad, "keypoint scores", float((D(out["scores"][i, :n]) - ks64).abs().max()), TOL["kscore"])
        l, _, t, _ = alo._pads(h, w)
        featp = F.normalize(x1234[i], dim=0)
        d64 = alo.sddh(sd64, featp, (t, l, h, w), D(kpn[i, :n]), M)
        check(bad, "descriptors", float((D(out["descriptors"][i, :n]) - d64).abs().max()), TOL["desc"])
    passed = (flat > thr_b).sum(1).tolist() if thr_b is not None else None
    return {"counts": n_sel.tolist(), "maxima": (flat > 0).sum(1).tolist(), "passed": passed, "undecided": undecided}


_sd = {}


def state_dict(model_name, variant=None):
    key = (model_name, variant)
    if key not in _sd:
        sd = als.make_aliked_state_dict(model_name, 0)
        if variant == "dcn":  # block3 / block4 offsets = exact binary fractions (constant per channel)
            for blk in ("block3", "block4"):
                for cv in (1, 2):
                    p = f"{blk}.conv{cv}.offset_conv"
                    sd[f"{p}.weight"] = torch.zeros_like(sd[f"{p}.weight"])
                    sd[f"{p}.bias"] = DCN_BIAS[cv - 1].clone()
        elif variant == "sddh":  # SDDH sample offsets = exact binary fractions
            sd["desc_head.offset_conv.2.weight"] = torch.zeros_like(sd["desc_head.offset_conv.2.weight"])
            r = sd["desc_head.offset_conv.2.bias"].numel() // 2 // len(SDDH_BIAS)  # M / 16
            sd["desc_head.offset_conv.2.bias"] = torch.cat([SDDH_BIAS.repeat(r), SDDH_BIAS.flip(0).repeat(r)])
        _sd[key] = sd
    return _sd[key]


# (dy, dx) of taps 0 .. 8: on integers, at +-0.5, just inside -1 (-1 + 2^-5 from row / column 0's first tap), exactly
# at -1 and at the far edge (outside: zero), one pixel past each edge, and beyond the clamp (+-1000)
DCN_BIAS = [torch.tensor([0.0, 0.0, 0.03125, -0.5, 0.5, 1.0, -1.0, 0.0, 0.0, 1000.0, -1000.0, 2.0, 1.0, -2.0, 0.5, 0.03125,
                          -0.96875, 1.5]),
            torch.tensor([0.0, 1.0, -1.0, 0.0, 0.5, 0.5, -0.5, -0.5, 2.0, -1000.0, 1000.0, 0.0, -0.96875, 0.03125, 1.0, 1.0,
                          -1.0, -1.0])]
# SDDH sample offsets dx (dy: the same values reversed): 0, +-0.25, +-0.5, +-1, +-2.5, +-3.25, +-7.75, 12 and +-1000
# (clamped to max(h, w) / 4)
SDDH_BIAS = torch.tensor([0.0, 0.5, -0.5, 1.0, -1.0, 2.5, -2.5, 7.75, -7.75, 1000.0, -1000.0, 3.25, -3.25, 0.25, -0.25,
                          12.0])


def level_dims(h, w, s):
    return -(-h // 32) * 32 // s, -(-w // 32) * 32 // s


# ------------------------------------------------------------------------------------------------ regimes
def _tiny(h, w):  # Hp = Wp = 32: the 1/32 level is one pixel, lim = 0.25
    assert level_dims(h, w, 32) == (1, 1)


def _no_pad(h, w):
    assert h % 32 == 0 and w % 32 == 0


def _odd_pads(h, w):
    assert (-h) % 32 % 2 == 1 and (-w) % 32 % 2 == 1


def _tail(n):
    def f(h, w):
        assert level_dims(h, w, 32)[1] % 4 == n
    return f


def _tall(h, w):  # the clamp at every level depends on H
    hh, ww = level_dims(h, w, 8)
    assert hh > ww and level_dims(h, w, 32)[0] > level_dims(h, w, 32)[1]


def _any(h, w):
    pass


DEFAULT = dict(max_num_keypoints=-1, detection_threshold=0.2, nms_radius=2)
SHAPES = [
    ("aliked-t16", 8, 8, dict(detection_threshold=-1, max_num_keypoints=4), _tiny),
    ("aliked-n16", 32, 32, {}, _no_pad),
    ("aliked-n16", 33, 47, {}, _odd_pads),
    ("aliked-n32", 203, 317, {}, _odd_pads),
    ("aliked-n16", 40, 150, {}, _tail(1)),
    ("aliked-t16", 40, 190, {}, _tail(2)),
    ("aliked-n32", 40, 200, {}, _tail(3)),
    ("aliked-n16", 200, 72, {}, _tall),
]


@pytest.mark.parametrize("model_name,h,w,conf,regime", SHAPES, ids=[f"{s[0][7:]}-{s[1]}x{s[2]}" for s in SHAPES])
def test_stages(model_name, h, w, conf, regime):
    regime(h, w)
    bad = []
    res = check_forward(bad, model_name, state_dict(model_name), als.make_image(h, w, 1, 500 + h + w).cuda(),
                        {**DEFAULT, **conf})
    assert res["counts"][0] > 0
    assert not bad, bad


def test_stages_768x1024_default_conf():
    """B = 1 at 768 x 1024 with the default conf: about 10 000 keypoints."""
    bad = []
    counts = check_forward(bad, "aliked-n16", state_dict("aliked-n16"), als.make_image(768, 1024, 1, 91).cuda(),
                           DEFAULT)["counts"]
    assert 5000 <= counts[0] <= 20000, counts
    assert not bad, bad


def test_stages_batch_with_image_size():
    """B = 3 at 240 x 320 with image_size crops, the last narrower than nms_radius (Python's negative-slice rule)."""
    size = torch.tensor([[320.0, 240.0], [200.0, 150.0], [1.0, 240.0]])
    bad = []
    counts = check_forward(bad, "aliked-n16", state_dict("aliked-n16"), als.make_image(240, 320, 3, 93).cuda(),
                           dict(DEFAULT, max_num_keypoints=400), size)["counts"]
    assert min(counts) > 0
    assert not bad, bad


MODES = [
    ("threshold", "aliked-n16", 96, 128, {}),
    ("threshold, n_limit below the count", "aliked-n16", 96, 128, dict(max_num_keypoints=20)),
    ("top-k, fewer maxima than k", "aliked-t16", 32, 32, dict(detection_threshold=-1, max_num_keypoints=600)),
    ("top-k", "aliked-n32", 64, 96, dict(detection_threshold=-1, max_num_keypoints=50)),
    ("mean fallback", "aliked-n16", 64, 96, dict(detection_threshold=0.9999999)),
    ("nms_radius 1", "aliked-n16", 67, 45, dict(nms_radius=1)),
    ("nms_radius 3", "aliked-t16", 96, 128, dict(nms_radius=3)),
    ("top-k, flat image", "aliked-n16", 64, 64, dict(detection_threshold=-1, max_num_keypoints=100)),
    ("top-k, nms_radius 0, k = 4096", "aliked-n16", 96, 96, dict(detection_threshold=-1, max_num_keypoints=4096, nms_radius=0)),
    ("top-k, nms_radius 0, k = 4097", "aliked-n16", 96, 96, dict(detection_threshold=-1, max_num_keypoints=4097, nms_radius=0)),
]


def mode_image(mode, h, w):
    if "flat" in mode:  # one grey level: a plateau of equal scores, and filler rows after its few maxima
        return torch.full((1, 3, h, w), 0.5)
    return als.make_image(h, w, 1, 700 + h)


@pytest.mark.parametrize("mode,model_name,h,w,conf", MODES, ids=[m[0] for m in MODES])
def test_dkd_modes(mode, model_name, h, w, conf):
    bad = []
    res = check_forward(bad, model_name, state_dict(model_name), mode_image(mode, h, w).cuda(), {**DEFAULT, **conf})
    assert not bad, bad
    assert res["counts"][0] > 0
    if "flat" in mode:
        assert 0 < res["maxima"][0] < res["counts"][0] == conf["max_num_keypoints"]
    if "4096" in mode or "4097" in mode:  # the block kernel and, above 4096, the functor, on 9216 NMS survivors
        assert res["counts"][0] == conf["max_num_keypoints"]
    if "n_limit" in mode:
        assert res["counts"][0] == 20 < res["passed"][0]
    if "fewer" in mode:  # filler rows follow the maxima
        assert 0 < res["maxima"][0] < res["counts"][0] == conf["max_num_keypoints"]
    if "mean" in mode:
        print(f"mean fallback: {res['undecided']} NMS values within {MEAN_MARGIN:g} of the mean")


def test_nms_radius_0_with_image_size():
    """r = 0: every pixel is a maximum; image_size with the full size zeroes no border (t[h - 0:] is empty)."""
    bad = []
    res = check_forward(bad, "aliked-n16", state_dict("aliked-n16"), als.make_image(32, 32, 1, 5).cuda(),
                        dict(DEFAULT, nms_radius=0), torch.tensor([[32.0, 32.0]]))
    assert res["maxima"][0] == 32 * 32 and res["counts"][0] > 20
    assert not bad, bad


def test_batch_where_only_one_image_passes():
    """B = 2, image 1 flat grey (no score above 0.2): image 0 passes, so there is no fallback and the counts differ."""
    img = torch.cat([als.make_image(64, 96, 1, 3), torch.full((1, 3, 64, 96), 0.7)]).cuda()
    bad = []
    counts = check_forward(bad, "aliked-n16", state_dict("aliked-n16"), img, DEFAULT)["counts"]
    assert counts[0] > 0 and counts[1] == 0, counts
    assert not bad, bad


# constructed offsets: every tap / sample position exact in fp32 and float64
@pytest.mark.parametrize("model_name,h,w", [("aliked-n16", 75, 111), ("aliked-t16", 200, 72), ("aliked-n32", 8, 8)])
def test_constructed_deformable_offsets(model_name, h, w):
    bad = []
    conf = DEFAULT if h > 8 else dict(DEFAULT, detection_threshold=-1, max_num_keypoints=4)
    check_forward(bad, model_name, state_dict(model_name, "dcn"), als.make_image(h, w, 1, 17).cuda(), conf)
    assert not bad, bad


@pytest.mark.parametrize("model_name,h,w", [("aliked-n16", 75, 111), ("aliked-n32", 203, 317)])
def test_constructed_sddh_offsets(model_name, h, w):
    """Odd sizes: samples past the crop land in the padded band, where the features are nonzero but SDDH reads 0."""
    assert (-h) % 32 and (-w) % 32
    bad = []
    check_forward(bad, model_name, state_dict(model_name, "sddh"), als.make_image(h, w, 1, 19).cuda(), DEFAULT)
    assert not bad, bad
