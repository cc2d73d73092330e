"""Pairs/s of the resident forward against the batch size (bf16, N=2048, pruning off): does keeping the
per-layer activations inside the 50 MB L2 (smaller batches) beat fuller waves (larger batches)?"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightglue_b200 import LightGlue, synth  # noqa: E402

m = LightGlue(features=None, precision=sys.argv[1] if len(sys.argv) > 1 else "bf16", depth_confidence=-1, width_confidence=-1)
m.load_state_dict(synth.make_state_dict(), strict=False)
m = m.eval().cuda()
for b in (8, 12, 16, 20, 24, 28, 32, 37, 48, 64):
    data, _ = synth.make_pair(2048, b=min(b, 8), seed=1)
    rep = (b + 7) // 8
    data = {k: {kk: torch.cat([vv] * rep)[:b].cuda() for kk, vv in v.items()} for k, v in data.items()}
    for _ in range(3):
        m(data)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        m(data)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(f"B={b:3d}  {ms:7.3f} ms/forward  {b / ms * 1e3:7.1f} pairs/s", flush=True)
