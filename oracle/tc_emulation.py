"""The tensor-core kernels' operand rounding, emulated on the CPU matcher oracle  --  TEST INFRASTRUCTURE ONLY.

``emulated(sd, pmap)`` swaps the arithmetic of ``oracle/lightglue_oracle.py`` for the duration of a ``with`` block:
each Linear class named in ``pmap`` runs with its operands rounded the way ``tc_linear_kernel`` rounds them (bf16 or
fp16 single pass, or split hi + lo products, fp32 accumulation), attention takes fp16 q, k, v and an fp16 P for the
numerator with fp32 scores and softmax statistics (``k_tc_attn.cu``), and the assignment's ``final_proj`` and
similarity follow ``pmap["final"]`` / ``pmap["sim"]``.  Everything else (token confidence, matchability, LayerNorm,
residual) stays fp32, as in the kernels.  ``tools/precision_study.py`` compares operand maps with it and
``tests/test_adaptive_margins.py`` calibrates the adaptive decisions' certificate with it.

Further keys of ``pmap``:

* ``fold=True``: out_proj / to_out folded into ffn.0 as ``lg_create`` does (``fold_out_proj``): ffn.0 runs once over
  ``cat[x, ctx]`` with ``W1f = [W1[:, :256] | W1[:, 256:]·Wo]`` and ``b1f = b1 + W1[:, 256:]·bo``, formed in double and
  stored as fp32, and the ``msg`` tensor is never formed;
* ``nobias``: Linear classes ("qkv", "ffn0", "ffn3", ...) whose bias is dropped;
* ``gelu="tanh"``: the tanh approximation of GELU in place of the erf form;
* ``rope="swap"``: each rotary pair read and written as ``(x1, x0)``, i.e. rotated by ``-θ``.

The last three, and the ``bf16x2a`` / ``bf16x2w`` modes (one split-bf16 pass lost), express kernel defects:
``tests/test_matcher_layer_emulation.py`` checks that the GPU layer tolerances sit between the correct arithmetic's
error and each defect's.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from . import lightglue_oracle as oracle

# precision="bf16x3": every linear and the similarity as three split-bf16 products (DESIGN.md §3)
BF16X3 = dict(qkv="bf16x3", out="bf16x3", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3")


def rnd(x: torch.Tensor, bits: int) -> torch.Tensor:
    """round-to-nearest-even to `bits` explicit mantissa bits (7 = bf16, 10 = fp16 ignoring its range), same dtype."""
    if bits == 7:
        return x.to(torch.bfloat16).to(x.dtype)
    if bits == 10:
        return x.to(torch.float16).to(x.dtype)
    raise ValueError(bits)


def fold_out_proj(sd, key):
    """``(W1f, b1f)`` of the ffn.0 weight ``sd[key]`` (DESIGN.md §3, "Out-projection fusion"): double products, fp32."""
    p = key[: -len("ffn.0.weight")]
    o = p + ("out_proj." if p + "out_proj.weight" in sd else "to_out.")
    w1, b1 = sd[key].double(), sd[p + "ffn.0.bias"].double()
    wo, bo = sd[o + "weight"].double(), sd[o + "bias"].double()
    w1f = torch.cat([w1[:, :256], w1[:, 256:] @ wo], 1)
    return w1f.float(), (b1 + w1[:, 256:] @ bo).float()


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
        self.folded = {id(v): fold_out_proj(sd, k) for k, v in sd.items() if k.endswith("ffn.0.weight")} \
            if pmap.get("fold") else {}

    def linear(self, x, w, b=None):
        c = self.cls.get(id(w))
        if c == "out" and self.folded:  # ctx goes to ffn.0 unprojected: the fold carries out_proj
            return x
        if c == "ffn0" and self.folded:
            w, b = self.folded[id(w)]
        if c == "ffn0" and self.pmap.get("msg") == "hi":  # msg half of cat([x, msg]) kept as a single 16-bit image
            mode = self.pmap.get(c, "f32")
            x = torch.cat([x[..., :256], rnd(x[..., 256:], 7 if mode.startswith("bf16") else 10)], -1)
        y = gemm(x, w, self.pmap.get(c, "f32")) if c else x @ w.t()
        return y if b is None or c in self.pmap.get("nobias", ()) else y + b

    def gelu(self, x):
        return F.gelu(x, approximate=self.pmap.get("gelu", "none"))

    def __getattr__(self, name):
        return getattr(F, name)


def attention_fp16(q, k, v):
    """fp16 q, k, v operands, fp32 scores / softmax statistics, fp16 P for the numerator (k_tc_attn.cu)."""
    q, k, v = rnd(q, 10), rnd(k, 10), rnd(v, 10)
    s = (q @ k.transpose(-1, -2)) * 0.125
    e = torch.exp(s - s.amax(-1, keepdim=True))
    return (rnd(e, 10) @ v) / e.sum(-1, keepdim=True)


def attention_online(q, k, v, block=64, p_bits=10):
    """``tc_attention_kernel``'s arithmetic in fp32: fp16 q, k, v; per block of 64 keys fp32 scores, the running row
    maximum m, P = exp(s - m) summed in fp32 and rounded to fp16 (``p_bits``) for P·V, earlier blocks rescaled by
    exp(m_old - m)."""
    q, k, v = rnd(q.float(), 10), rnd(k.float(), 10), rnd(v.float(), 10)
    m = q.new_full(q.shape[:-1] + (1,), float("-inf"))
    l = q.new_zeros(q.shape[:-1] + (1,))
    o = q.new_zeros(q.shape[:-1] + (v.shape[-1],))
    for j in range(0, k.shape[-2], block):
        s = (q @ k[..., j:j + block, :].transpose(-1, -2)) * 0.125
        mx = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp(m - mx)
        e = torch.exp(s - mx)
        l = l * alpha + e.sum(-1, keepdim=True)
        o = o * alpha + rnd(e, p_bits) @ v[..., j:j + block, :]
        m = mx
    return o / l


_ROPE = oracle.rope
_SWAP = [i ^ 1 for i in range(oracle.HEAD_DIM)]


def rope_swapped(t, cos, sin):
    """``oracle.rope`` with each pair read and written as (x1, x0): a rotation by -θ."""
    return _ROPE(t[..., _SWAP], cos, sin)[..., _SWAP]


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
    saved = oracle.F, oracle.attention, oracle.log_assignment, oracle.rope
    oracle.F, oracle.attention, oracle.log_assignment = Shim(sd, pmap), attention_fp16, make_log_assignment(pmap)
    if pmap.get("rope") == "swap":
        oracle.rope = rope_swapped
    try:
        yield
    finally:
        oracle.F, oracle.attention, oracle.log_assignment, oracle.rope = saved
