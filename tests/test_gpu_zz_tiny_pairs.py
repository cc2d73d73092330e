"""Pairs far below one 128-row tile through the tensor-core path against the oracle."""
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from oracle import lightglue_oracle as oracle

pytestmark = pytest.mark.gpu


def to_cuda(data):
    return {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}


@pytest.mark.parametrize("m,n", [(5, 3), (1, 1), (130, 2), (127, 129)])
def test_tiny_pairs_on_the_tensor_core_path(m, n):
    """Pairs far below one 128-row tile (Lp = 128 / 256) through the bf16x3 path against the oracle."""
    sd = synth.make_state_dict()
    data, _ = synth.make_pair(max(m, n), b=1, seed=300 + m, m=m)
    data["image1"] = {k: (v[:, :n].contiguous() if v.dim() == 3 else v) for k, v in data["image1"].items()}
    ref = oracle.forward(sd, data)
    mod = LightGlue(features=None, precision="bf16x3", depth_confidence=-1, width_confidence=-1)
    mod.load_state_dict(sd, strict=False)
    out = mod.eval().cuda()(to_cuda(data))
    assert out["matches0"].shape == (1, m) and out["matches1"].shape == (1, n)
    assert torch.equal(out["matches0"].cpu(), ref["matches0"]) and torch.equal(out["matches1"].cpu(), ref["matches1"])
    assert float((out["matching_scores0"].cpu() - ref["matching_scores0"]).abs().max()) < 1e-3
