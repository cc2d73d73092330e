"""The linears write their outputs as 64-row boxes staged in shared memory (TMA stores), and the ffn.3 residual is
loaded the same way.  In one ragged bf16x3 batch whose lengths straddle the 64-row box, 128-row tile and 256-column
edges, every pair must give what it gives alone: a box landing in a neighbour's rows, or a residual read from them,
would change that neighbour's result."""
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.ragged import match_ragged

pytestmark = pytest.mark.gpu

LENS = [1, 31, 33, 127, 128, 129, 255, 257, 2047]
SIZES = [(m, LENS[(i + 4) % len(LENS)]) for i, m in enumerate(LENS)]


def test_ragged_batch_is_bit_identical_to_each_pair_alone():
    sd = synth.make_state_dict()
    pairs = []
    for i, (m, n) in enumerate(SIZES):
        data, _ = synth.make_pair(max(m, n), d=256, b=1, seed=300 + i, m=m)
        f0 = {k: v[:, :m].contiguous() if v.dim() == 3 else v for k, v in data["image0"].items()}
        f1 = {k: v[:, :n].contiguous() if v.dim() == 3 else v for k, v in data["image1"].items()}
        pairs.append({k: {kk: vv.cuda() for kk, vv in f.items()} for k, f in (("image0", f0), ("image1", f1))})
    m = LightGlue(features=None, precision="bf16x3", depth_confidence=-1, width_confidence=-1)
    m.load_state_dict(sd, strict=False)
    m = m.eval().cuda()
    with torch.no_grad():
        batch = match_ragged(m, pairs)
        matched = 0
        for (mm, nn), p, got in zip(SIZES, pairs, batch):
            alone = match_ragged(m, [p])[0]
            assert got["matches0"].shape == (1, mm) and got["matches1"].shape == (1, nn)
            for k in ("matches0", "matches1"):
                assert torch.equal(got[k].cpu(), alone[k].cpu()), ((mm, nn), k)
            for k in ("matching_scores0", "matching_scores1"):
                if min(mm, nn) > 1:
                    assert torch.equal(got[k].cpu(), alone[k].cpu()), ((mm, nn), k)
                else:  # an image of one keypoint: its scores move by ~4e-6 between batch and alone (the direct-store
                    # kernel too)
                    assert float((got[k] - alone[k]).abs().max()) <= 1e-5, ((mm, nn), k)
            matched += int((got["matches0"] > -1).sum())
    assert matched > 100  # the batch is doing real matching
