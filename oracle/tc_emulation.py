"""The tensor-core kernels' operand rounding, emulated on the CPU matcher oracle  --  TEST INFRASTRUCTURE ONLY.

``emulated(sd, pmap)`` swaps the arithmetic of ``oracle/lightglue_oracle.py`` for the duration of a ``with`` block:
each Linear class named in ``pmap`` runs with its operands rounded the way ``tc_linear_kernel`` rounds them (bf16 or
fp16 single pass, or split hi + lo products, fp32 accumulation), attention takes fp16 q, k, v and an fp16 P for the
numerator with fp32 scores and softmax statistics (``k_tc_attn.cu``), and the assignment's ``final_proj`` and
similarity follow ``pmap["final"]`` / ``pmap["sim"]``.  Everything else (token confidence, matchability, LayerNorm,
residual) stays fp32, as in the kernels.  ``tools/precision_study.py`` compares operand maps with it and
``tests/test_adaptive_margins.py`` calibrates the adaptive decisions' certificate with it.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from . import lightglue_oracle as oracle

# precision="bf16x3": every linear and the similarity as three split-bf16 products (DESIGN.md §3)
BF16X3 = dict(qkv="bf16x3", out="bf16x3", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3")


def rnd(x: torch.Tensor, bits: int) -> torch.Tensor:
    """round-to-nearest-even to `bits` explicit mantissa bits (7 = bf16, 10 = fp16 ignoring its range)."""
    if bits == 7:
        return x.to(torch.bfloat16).to(torch.float32)
    if bits == 10:
        return x.to(torch.float16).to(torch.float32)
    raise ValueError(bits)


def split(x, bits):
    hi = rnd(x, bits)
    return hi, rnd(x - hi, bits)


def gemm(a, w, mode):
    """a [.., K] x w [N, K]^T with the operand formats of `mode`."""
    if mode == "f32":
        return a @ w.t()
    if mode in ("bf16", "fp16"):
        b = 7 if mode == "bf16" else 10
        return rnd(a, b) @ rnd(w, b).t()
    b = 7 if mode.startswith("bf16") else 10
    ah, al = split(a, b)
    wh, wl = split(w, b)
    if mode.endswith("x3"):
        return al @ wh.t() + ah @ wl.t() + ah @ wh.t()
    if mode.endswith("x2a"):  # activations split, weights hi only
        return al @ wh.t() + ah @ wh.t()
    if mode.endswith("x2w"):  # weights split, activations hi only
        return ah @ wl.t() + ah @ wh.t()
    raise ValueError(mode)


class Shim:
    """Stands in for torch.nn.functional inside the oracle: routes F.linear by weight name."""

    def __init__(self, sd, pmap):
        self.cls = {}
        for k, v in sd.items():
            if not k.endswith("weight"):
                continue
            c = None
            if "Wqkv" in k or "to_qk" in k or "to_v" in k:
                c = "qkv"
            elif "out_proj" in k or "to_out" in k:
                c = "out"
            elif "ffn.0" in k:
                c = "ffn0"
            elif "ffn.3" in k:
                c = "ffn3"
            elif "final_proj" in k:
                c = "final"
            elif "input_proj" in k:
                c = "qkv"
            if c:
                self.cls[id(v)] = c
        self.pmap = pmap

    def linear(self, x, w, b=None):
        c = self.cls.get(id(w))
        if c == "ffn0" and self.pmap.get("msg") == "hi":  # msg half of cat([x, msg]) kept as a single 16-bit image
            mode = self.pmap.get(c, "f32")
            x = torch.cat([x[..., :256], rnd(x[..., 256:], 7 if mode.startswith("bf16") else 10)], -1)
        y = gemm(x, w, self.pmap.get(c, "f32")) if c else x @ w.t()
        return y if b is None else y + b

    def __getattr__(self, name):
        return getattr(F, name)


def attention_fp16(q, k, v):
    """fp16 q, k, v operands, fp32 scores / softmax statistics, fp16 P for the numerator (k_tc_attn.cu)."""
    q, k, v = rnd(q, 10), rnd(k, 10), rnd(v, 10)
    s = (q @ k.transpose(-1, -2)) * 0.125
    e = torch.exp(s - s.amax(-1, keepdim=True))
    return (rnd(e, 10) @ v) / e.sum(-1, keepdim=True)


def make_log_assignment(pmap):
    def log_assignment(w, i, x0, x1):
        p = f"log_assignment.{i}."
        b, m, _ = x0.shape
        n = x1.shape[1]
        fm = pmap.get("final", "f32")
        p0 = (gemm(x0, w[p + "final_proj.weight"], fm) + w[p + "final_proj.bias"]) / 4.0
        p1 = (gemm(x1, w[p + "final_proj.weight"], fm) + w[p + "final_proj.bias"]) / 4.0
        sm = pmap.get("sim", "f32")
        sim = torch.stack([gemm(p0[i_], p1[i_], sm) for i_ in range(b)])
        z0 = F.linear(x0, w[p + "matchability.weight"], w[p + "matchability.bias"])
        z1 = F.linear(x1, w[p + "matchability.weight"], w[p + "matchability.bias"])
        out = sim.new_zeros(b, m + 1, n + 1)
        out[:, :m, :n] = (torch.log_softmax(sim, 2) + torch.log_softmax(sim, 1) + F.logsigmoid(z0)
                          + F.logsigmoid(z1).transpose(1, 2))
        out[:, :m, n] = F.logsigmoid(-z0.squeeze(-1))
        out[:, m, :n] = F.logsigmoid(-z1.squeeze(-1))
        return out
    return log_assignment


@contextlib.contextmanager
def emulated(sd, pmap):
    """Run ``oracle.forward(sd, ...)`` (fp32) with the operand rounding of `pmap` inside the block; the oracle's own
    arithmetic is restored on exit.  `sd` must be the fp32 state_dict passed to ``forward``: the shim recognises
    the linears by the identity of its weight tensors."""
    saved = oracle.F, oracle.attention, oracle.log_assignment
    oracle.F, oracle.attention, oracle.log_assignment = Shim(sd, pmap), attention_fp16, make_log_assignment(pmap)
    try:
        yield
    finally:
        oracle.F, oracle.attention, oracle.log_assignment = saved
