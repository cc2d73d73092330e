"""Calibration of the tolerance the GPU head test (tests/test_gpu_sp_backbone.py) applies to the tensor-core convolutions:
the float64 emulation of their split-bf16 arithmetic (``oracle.superpoint_oracle.heads_split_bf16``) against the exact
float64 heads, with the synthetic weights.  Correct rounding stays within 3e-5 of the heads' largest magnitude; a lost lo
image of one layer (what a buffer overrun or a race on the lo half does) moves a head by more than 1e-3.  The GPU gate of
1e-4 sits between the two."""
import pytest
import torch

from oracle import superpoint_oracle as spo
from oracle import superpoint_synth as sps

ROUNDING = 3e-5
LOST_LO = 1e-3


def rel(a, ref):
    return float((a - ref).abs().max() / ref.abs().max())


@pytest.fixture(scope="module")
def weights():
    return sps.make_superpoint_state_dict(0)


def exact(w, image):
    return spo.heads({k: v.double() for k, v in w.items()}, image.double())


@pytest.mark.parametrize("h,w", [(9, 15), (17, 33), (67, 45), (240, 320)])
def test_split_bf16_rounding_stays_within_calibrated_bound(weights, h, w):
    torch.set_grad_enabled(False)
    image = sps.make_image(h, w, 1, 100 + h)
    el, ed = exact(weights, image)
    sl, sd = spo.heads_split_bf16(weights, image)
    assert sl.shape == el.shape == (1, 65, h // 8, w // 8) and sd.shape == ed.shape == (1, 256, h // 8, w // 8)
    assert 0 < rel(sl, el) <= ROUNDING and 0 < rel(sd, ed) <= ROUNDING, (rel(sl, el), rel(sd, ed))


@pytest.mark.parametrize("h,w", [(9, 15), (17, 33), (67, 45)])
@pytest.mark.parametrize("layer,heads", [("conv4b", (0, 1)), ("convPa", (0,)), ("convDa", (1,))])
def test_a_lost_lo_image_exceeds_the_bound(weights, h, w, layer, heads):
    """conv4b feeds both heads, convPa the logits, convDa the descriptor map."""
    torch.set_grad_enabled(False)
    image = sps.make_image(h, w, 1, 100 + h)
    ref = exact(weights, image)
    lost = spo.heads_split_bf16(weights, image, drop_lo=(layer,))
    for i in heads:
        assert rel(lost[i], ref[i]) > LOST_LO, (layer, i, rel(lost[i], ref[i]))
