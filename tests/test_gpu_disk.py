"""DISK on the GPU against the torch restatement of kornia's DISK (oracle/disk_oracle.py) on synthetic weights.

* ``heads`` (``disk_heads``): the cropped heatmap and the raw 128-d descriptors at chosen pixels -- crop corners and
  edges, pixels next to the padded frame, random ones -- against the oracle in float64 on the GPU, held to 1e-4 of
  max|ref| per head (split-bf16 tensor-core convolutions, fp32 statistics): at least 3x the emulated rounding and at
  most 1/3 of a lost split-bf16 pass (tests/test_conv_layer_emulation.py).  A lost bias in down0 .. up2 is removed by
  the next instance norm and invisible here; tests/test_gpu_conv_layers.py checks each layer from its own input.
* ``forward``: against the oracle in fp32 (cuDNN, TF32 off).  The same keypoints in the same row-major order, except
  keypoints whose float64 NMS / threshold / top-k margin is below 1e-4 max|heatmap| (at most 0.5 % of them); on common
  keypoints scores within 1e-4 max|heatmap| and descriptors within 1e-4.
* batches equal single images, repeated calls are bit-identical, and the output feeds the matcher."""
import pytest
import torch
import torch.nn.functional as F

from lightglue_b200 import DISK, _cabi, synth
from oracle import disk_oracle as do
from oracle import disk_synth as ds
from tests.test_conv_layer_emulation import E2E_DISK

pytestmark = pytest.mark.gpu

_models = {}
_sd = {}


def sd_on(dtype):
    if dtype not in _sd:
        _sd[dtype] = {k: v.to("cuda", dtype) for k, v in ds.make_disk_state_dict(0).items()}
    return _sd[dtype]


def model(**conf):
    key = tuple(sorted(conf.items()))
    if key not in _models:
        m = DISK(weights=None, **conf)
        m.model.load_state_dict(ds.make_disk_state_dict(0), strict=True)
        _models[key] = m.cuda()
    return _models[key]


def image_of(b, h, w, seed=0):
    return ds.make_image(h, w, b, 300 + seed + h).cuda()


def rel(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("b,h,w", [(1, 16, 32), (1, 33, 47), (1, 203, 317), (1, 240, 320), (1, 768, 1024), (3, 33, 47)])
def test_heads_vs_float64(b, h, w):
    torch.set_grad_enabled(False)
    m = model()
    image = image_of(b, h, w)
    cap = int(_cabi.load().disk_max_keypoints(m._get_handle(image.device), h, w))
    g = torch.Generator().manual_seed(h * w)
    edge = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (h // 2, w - 1), (h - 1, w // 2), (h - 2, w - 2), (1, 1)]
    n_rand = max(0, min(cap, 200) - len(edge))
    ys = torch.randint(0, h, (n_rand,), generator=g).tolist()
    xs = torch.randint(0, w, (n_rand,), generator=g).tolist()
    pix = edge + list(zip(ys, xs))
    pos = torch.tensor([[y * w + x for y, x in pix]] * b, dtype=torch.int32)
    for i in range(1, b):  # other images: other pixels (rolled), so that seam-crossing taps of every image are read
        pos[i] = pos[0].roll(i)
    heat, desc = m.heads(image, pos)
    ref_heat, ref_desc = do.heads(sd_on(torch.float64), image.double())
    pc = pos.long().cuda()
    ref_d = torch.stack([ref_desc[i].flatten(1)[:, pc[i]].T for i in range(b)])
    eh, ed = rel(heat, ref_heat), rel(desc, ref_d)
    print(f"B={b} {h}x{w}: max rel error heatmap {eh:.2e} descriptors {ed:.2e} ({pos.shape[1]} pixels)")
    assert heat.shape == (b, h, w) and desc.shape == (b, pos.shape[1], 128)
    assert eh <= E2E_DISK and ed <= E2E_DISK, (eh, ed)


def _margins(h64, xy, conf, cand_vals):
    """float64 margins of keypoints xy [k, 2] on heatmap h64 [H, W]: NMS, threshold and top-k cut."""
    r = conf.get("nms_window_size", 5) // 2
    H, W = h64.shape
    pad = F.pad(h64[None, None], (r, r, r, r), value=float("inf"))[0, 0]
    out = []
    cut = None
    n = conf.get("max_num_keypoints")
    if n is not None and cand_vals.numel():
        v = cand_vals.sort(descending=True).values
        cut = float(v[min(n, v.numel() - 1)])
    for x, y in xy.tolist():
        x, y = int(x), int(y)
        v = float(h64[y, x])
        win = pad[y:y + 2 * r + 1, x:x + 2 * r + 1].clone()
        win[r, r] = float("inf")
        m = min(float((win - v).abs().min()), abs(v - conf.get("detection_threshold", 0.0)))
        if cut is not None:
            m = min(m, abs(v - cut))
        out.append(m)
    return out


CONFS = [
    ("default", 1, 240, 320, {}),
    ("top32", 1, 240, 320, dict(max_num_keypoints=32)),
    ("top2048", 1, 480, 640, dict(max_num_keypoints=2048)),
    ("nms3", 1, 240, 320, dict(nms_window_size=3)),
    ("nms7", 1, 240, 320, dict(nms_window_size=7)),
    ("thr", 1, 240, 320, dict(detection_threshold=0.5)),
    ("odd", 1, 203, 317, {}),
    ("gray", 1, 240, 320, {}),
    ("b3cap", 3, 160, 224, dict(max_num_keypoints=64)),
    ("nopad", 1, 192, 256, dict(pad_if_not_divisible=False)),
]


@pytest.mark.parametrize("name,b,h,w,conf", CONFS, ids=[c[0] for c in CONFS])
def test_forward_vs_fp32_oracle(name, b, h, w, conf):
    torch.set_grad_enabled(False)
    image = image_of(b, h, w, seed=len(name))
    if name == "gray":
        image = image.mean(1, keepdim=True)
    out = model(**conf)({"image": image})
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = do.forward(sd_on(torch.float32), image, conf)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    h64, _d = do.heads(sd_on(torch.float64), image.double(), conf.get("pad_if_not_divisible", True))
    total, odd = 0, 0
    for i in range(b):
        hmax = float(h64[i].abs().max())
        k_c = [tuple(p) for p in out["keypoints"][i].long().tolist()]
        k_r = [tuple(p) for p in ref["keypoints"][i].long().tolist()]
        sc, sr = set(k_c), set(k_r)
        common = [p for p in k_c if p in sr]
        assert common == [p for p in k_r if p in sc], "common keypoints in a different order"
        only = [p for p in k_c if p not in sr] + [p for p in k_r if p not in sc]
        keep = do.nms_mask(h64[i], conf.get("nms_window_size", 5)) & (h64[i] > conf.get("detection_threshold", 0.0))
        margins = _margins(h64[i], torch.tensor(only).reshape(-1, 2), conf, h64[i][keep])
        assert all(mg < 1e-4 * hmax for mg in margins), (name, only, margins)
        total += len(k_r)
        odd += len(only)
        ic = torch.tensor([k_c.index(p) for p in common], dtype=torch.long)
        ir = torch.tensor([k_r.index(p) for p in common], dtype=torch.long)
        ds_ = float((out["keypoint_scores"][i, ic].double().cpu() - ref["keypoint_scores"][i, ir].double().cpu()).abs().max()) \
            if len(common) else 0.0
        dd = float((out["descriptors"][i, ic].cpu() - ref["descriptors"][i, ir].cpu()).abs().max()) if len(common) else 0.0
        print(f"{name} image {i}: {len(k_c)} keypoints (oracle {len(k_r)}), one-sided {len(only)}, "
              f"max|dscore|/max|heat| {ds_ / hmax:.2e}, max|ddesc| {dd:.2e}")
        assert ds_ <= 1e-4 * hmax and dd <= 1e-4, (ds_, hmax, dd)
    assert total > 0 and odd <= 0.005 * total, (odd, total)
    assert out["keypoints"].dtype == out["descriptors"].dtype == out["keypoint_scores"].dtype == torch.float32


def test_batch_equals_single_images_and_repeats_are_bit_identical():
    torch.set_grad_enabled(False)
    m = model(max_num_keypoints=64)
    image = image_of(3, 160, 224, seed=9)
    first = m({"image": image})
    second = m({"image": image})
    for k in first:
        assert torch.equal(first[k], second[k]), k
    for i in range(3):
        single = m({"image": image[i:i + 1].contiguous()})
        for k in first:
            assert torch.equal(first[k][i:i + 1], single[k]), k


def test_zero_candidates_give_zero_rows():
    m = model(max_num_keypoints=16, detection_threshold=1e9)
    out = m({"image": image_of(1, 64, 64)})
    assert out["keypoints"].shape == (1, 0, 2) and out["descriptors"].shape == (1, 0, 128)


def test_bad_sizes_raise():
    with pytest.raises(ValueError):
        model(pad_if_not_divisible=False)({"image": image_of(1, 40, 64)})
    with pytest.raises(ValueError):
        model()({"image": image_of(1, 16, 16)})


def test_disk_feeds_the_matcher():
    """extract() -> LightGlue with 128-d descriptors: the two halves of match_pair run back to back on the device."""
    from lightglue_b200 import LightGlue
    from lightglue_b200.utils import match_pair

    dk = model(max_num_keypoints=256)
    lg = LightGlue(features=None, input_dim=128, precision="bf16x3", depth_confidence=-1, width_confidence=-1)
    lg.load_state_dict(synth.make_state_dict(input_dim=128), strict=False)
    lg = lg.eval().cuda()
    im0 = image_of(1, 240, 320, seed=81)[0]
    im1 = torch.roll(im0, shifts=(8, 16), dims=(1, 2))
    f0, f1, m01 = match_pair(dk, lg, im0, im1, device="cuda", resize=None)
    assert f0["keypoints"].shape[1] == 2 and f0["descriptors"].shape[1] == 128
    assert 0 < f0["keypoints"].shape[0] <= 256
    assert m01["matches0"].shape == (f0["keypoints"].shape[0],) and int((m01["matches0"] > -1).sum()) > 0
