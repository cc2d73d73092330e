"""The SuperPoint convolution stack alone (``SuperPoint.backbone_heads`` -> ``sp_backbone``): raw detector logits and the
un-normalised descriptor map, in both precision modes, against the oracle's ``heads`` computed in float64 on the GPU.

Error measure: max|delta| / max|ref| per head.  bf16x3 (tensor cores, split-bf16 operands) is held to 1e-4: its rounding
emulated in float64 stays within 3e-5 and a lost lo image of one layer moves a head by more than 1e-3
(tests/test_superpoint_bf16x3_emulation.py).  fp32 (CUDA cores) is held to 1e-5."""
import pytest
import torch

from lightglue_b200.superpoint import SuperPoint
from oracle import superpoint_oracle as spo
from oracle import superpoint_synth as sps

pytestmark = pytest.mark.gpu

TOL = {"bf16x3": 1e-4, "fp32": 1e-5}
SHAPES = [  # (B, H, W)
    (1, 8, 8), (1, 9, 15), (1, 17, 33),  # one tile sequence per level: the 1/4- and 1/8-resolution maps are the widest
    (1, 14, 14),                          # 256 padded rows: both 128-row sequences exactly full
    (1, 14, 30),                          # 512 rows: Lp = 256, exactly full
    (1, 63, 65), (1, 64, 64),             # either side of 64 x 64 pixels
    (1, 24, 131), (1, 67, 45),            # odd extents
    (3, 9, 15),                           # several images in one tile: taps across image seams
    (2, 203, 317),                        # batch with odd extents
    (1, 480, 640), (1, 768, 1024),        # many tiles
]
_ref_cache = {}


def rel(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


def image_of(b, h, w):
    return sps.make_image(h, w, b, 100 + h).cuda()


def reference(b, h, w):
    if (b, h, w) not in _ref_cache:
        w64 = {k: v.double().cuda() for k, v in sps.make_superpoint_state_dict(0).items()}
        _ref_cache[(b, h, w)] = spo.heads(w64, image_of(b, h, w).double())
    return _ref_cache[(b, h, w)]


@pytest.fixture(scope="module", params=["bf16x3", "fp32"])
def model(request):
    torch.set_grad_enabled(False)
    m = SuperPoint(weights=None, precision=request.param)
    m.load_state_dict(sps.make_superpoint_state_dict(0))
    return m.eval().cuda()


@pytest.mark.parametrize("b,h,w", SHAPES)
def test_backbone_heads_vs_float64(model, b, h, w):
    logits, dense = model.backbone_heads(image_of(b, h, w))
    ref_logits, ref_dense = reference(b, h, w)
    assert logits.shape == ref_logits.shape == (b, 65, h // 8, w // 8)
    assert dense.shape == ref_dense.shape == (b, 256, h // 8, w // 8)
    el, ed = rel(logits, ref_logits), rel(dense, ref_dense)
    print(f"[{model.conf.precision}] B={b} {h}x{w}: max rel error logits {el:.2e} dense {ed:.2e}")
    tol = TOL[model.conf.precision]
    assert el <= tol and ed <= tol, (el, ed)


@pytest.mark.parametrize("b,h,w", [(3, 9, 15), (2, 203, 317)])
def test_batched_heads_equal_single_image_heads(model, b, h, w):
    """A batch shares padded row tiles across its images; each image's heads must not depend on its neighbours."""
    image = image_of(b, h, w)
    heads = model.backbone_heads(image)
    for i in range(b):
        single = model.backbone_heads(image[i:i + 1].contiguous())
        for got, ref in zip(heads, single):
            assert rel(got[i:i + 1], ref.double()) <= 1e-6


@pytest.mark.parametrize("h,w", [(9, 15), (17, 33)])
def test_repeated_calls_are_bit_identical(model, h, w):
    """The convolutions have no atomics: two calls on the same input differ only if buffers race."""
    image = image_of(1, h, w)
    first = [t.clone() for t in model.backbone_heads(image)]
    second = model.backbone_heads(image)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
