"""The tolerances of ``tests/test_gpu_matcher_layers.py``, derived on the CPU from the kernels' emulated arithmetic
(``oracle/tc_emulation.py``) so that each one has room above the arithmetic it accepts and teeth against the defects it
must catch.

For every precision mode and every checked quantity -- a transformer layer's output from its own float64 input, the
attention output from given q, k, v, the log-assignment matrix -- the emulated arithmetic's deviation from float64 is
measured, and so is the deviation of each single defect: a lost split-bf16 pass or a lost bias in QKV, ffn.0 or ffn.3,
a tanh-GELU, RoPE pairs read in the wrong order, a key block or padding key handled wrongly, an assignment sweep without
its lo pass.  Each tolerance must be at least 3x its mode's own error and at most a third of every defect's deviation
that the mode can resolve.  Deviations are max|Δ| / max(max|ref|, 1), the largest over images, layers and shapes."""
import functools

import pytest
import torch

from lightglue_b200 import synth
from oracle import lightglue_oracle as oracle
from oracle import tc_emulation as tce

# tolerances of tests/test_gpu_matcher_layers.py (relative deviations, see above; the assignment's is absolute).  The
# layer tolerance has two tiers: a pair with an image of fewer than SMALL keypoints attends over too few keys to average
# the fp16 rounding of v out, so in bf16x3 its layers deviate up to 7.5e-5 against 1.1e-5 for larger pairs.
SMALL = 64
LAYER_TOL = {"large": {"fp32": 2e-5, "bf16x3": 5e-5, "bf16": 1.6e-2}, "small": {"fp32": 2e-5, "bf16x3": 2.5e-4, "bf16": 1.6e-2}}
LAYER_SHAPES = {"large": [(257, 300)], "small": [(1, 1), (5, 300)]}  # (M, N) of the B = 1 pairs each tier is set on
ATTN_TOL = {"fp32": 1e-5, "bf16x3": 4e-4, "bf16": 7e-3}
ASSIGN_TOL = {"fp32": 5e-5, "bf16x3": 5e-4}

BF16X3 = dict(tce.BF16X3, fold=True)  # the tensor-core modes fold out_proj into ffn.0 (lg_create)
BF16 = dict(qkv="bf16", out="bf16", ffn0="bf16", ffn3="bf16", final="bf16", sim="bf16", fold=True)
MODES = {"fp32": None, "bf16x3": BF16X3, "bf16": BF16}

DEFECTS = {
    "qkv A_lo·W_hi lost": {"qkv": "bf16x2w"},
    "qkv A_hi·W_lo lost": {"qkv": "bf16x2a"},
    "ffn.0 A_lo·W_hi lost": {"ffn0": "bf16x2w"},
    "ffn.0 A_hi·W_lo lost": {"ffn0": "bf16x2a"},
    "ffn.3 A_lo·W_hi lost": {"ffn3": "bf16x2w"},
    "ffn.3 A_hi·W_lo lost": {"ffn3": "bf16x2a"},
    "qkv bias lost": {"nobias": ("qkv",)},
    "ffn.0 bias lost": {"nobias": ("ffn0",)},
    "ffn.3 bias lost": {"nobias": ("ffn3",)},
    "tanh GELU": {"gelu": "tanh"},
    "RoPE pairs swapped": {"rope": "swap"},
}
BIAS = ["qkv bias lost", "ffn.0 bias lost", "ffn.3 bias lost"]
# The defects each mode's layer tolerance resolves.  fp32 has no lo passes; bf16's own operand rounding (~4e-3) hides
# everything but a lost bias.  In bf16x3 a lost A_lo·W_hi pass of QKV moves a layer of a large pair by only ~3x the
# mode's own error (2-3e-5 against 1e-5): q, k and v are rounded to fp16 for the attention right after it.  In small
# pairs the larger tolerance leaves QKV's lost passes (4.5-5.3e-4) and the tanh-GELU (3e-4) unresolved as well.
NOT_QKV_LO = [d for d in DEFECTS if d != "qkv A_lo·W_hi lost"]
RESOLVES = {
    "large": {"fp32": BIAS + ["tanh GELU", "RoPE pairs swapped"], "bf16x3": NOT_QKV_LO, "bf16": BIAS},
    "small": {"fp32": BIAS + ["tanh GELU", "RoPE pairs swapped"],
              "bf16x3": [d for d in NOT_QKV_LO if not d.startswith("qkv A") and d != "tanh GELU"], "bf16": BIAS},
}
LAYERS = (0, 4, 8)


def rel_dev(a, ref):
    return float((a.double() - ref).abs().max()) / max(float(ref.abs().max()), 1.0)


@functools.lru_cache(maxsize=None)
def _stream(m, n):
    """One B = 1 pair: the float64 residual stream that enters layers 0, 4 and 8, and both encodings."""
    sd = synth.make_state_dict()
    data, _ = synth.make_pair(n, m=m, seed=1000 + m + n)
    w64 = {k: v.double() for k, v in sd.items()}
    layers = oracle.forward(sd, data, dtype=torch.float64, return_layers=True, n_layers=max(LAYERS))["layers"]
    inputs = [(data["image0"]["descriptors"].double(), data["image1"]["descriptors"].double())] + layers
    return sd, w64, oracle.encodings(sd, data), oracle.encodings(w64, data), inputs


@functools.lru_cache(maxsize=None)
def layer_dev(pmap_key, tier):
    """Largest deviation over LAYERS and the tier's shapes of one layer run in fp32 (pmap None) or under the emulation
    of ``pmap``."""
    pmap = None if pmap_key is None else dict(pmap_key)
    worst = 0.0
    for m, n in LAYER_SHAPES[tier]:
        sd, w64, enc32, enc64, inputs = _stream(m, n)
        for i in LAYERS:
            x0, x1 = inputs[i]
            r0, r1 = oracle.layer(w64, i, x0, x1, enc64)
            if pmap is None:
                a0, a1 = oracle.layer(sd, i, x0.float(), x1.float(), enc32)
            else:
                with tce.emulated(sd, pmap):
                    a0, a1 = oracle.layer(sd, i, x0.float(), x1.float(), enc32)
            worst = max(worst, rel_dev(a0, r0), rel_dev(a1, r1))
    return worst


def _key(pmap):
    return None if pmap is None else tuple(sorted(pmap.items()))


@pytest.mark.parametrize("tier", list(LAYER_SHAPES))
@pytest.mark.parametrize("mode", list(MODES))
def test_layer_tolerance_sits_between_error_and_defects(mode, tier):
    err = layer_dev(_key(MODES[mode]), tier)
    base = BF16 if mode == "bf16" else BF16X3  # fp32's defects are measured on bf16x3 arithmetic, 100x below them
    shown = DEFECTS if mode == "bf16x3" else RESOLVES[tier][mode]
    devs = {d: layer_dev(_key(dict(base, **DEFECTS[d])), tier) for d in shown}
    tol = LAYER_TOL[tier][mode]
    print(f"[{mode}, {tier} pairs] layer: emulated error {err:.2e}, tolerance {tol:.1e}; defects: "
          + ", ".join(f"{d} {v:.2e}" for d, v in devs.items()))
    assert tol >= 3 * err
    for d in RESOLVES[tier][mode]:
        assert tol <= devs[d] / 3, (d, devs[d])


# ------------------------------------------------------------------------------------------------ attention
ATTN_SHAPES = [(65, 129), (128, 65), (129, 127)]  # every key count ends in a partial 64-key block
# fp16 P: a last-bit difference in a score flips the rounding of a P near 1 now and then, which costs ~1e-3 of |v|
# (the kernel's error against attention_fp16 in float64 is 1.3e-4 of max|v|, the same against a float64 restatement of
# its online schedule), so in the tensor-core modes the attention check resolves a lost key, not a padding key counted
# (6e-4) or P in bf16 (1e-3)
ATTN_RESOLVES = {"fp32": ["last partial key block dropped", "a padding key counted"],
                 "bf16x3": ["last partial key block dropped"], "bf16": ["last partial key block dropped"]}


def _qkv(m, n, seed):
    g = torch.Generator().manual_seed(seed)
    mk = lambda l, s: torch.randn(1, 4, l, 64, generator=g, dtype=torch.float64) * s  # noqa: E731
    return mk(m, 2.0), mk(n, 2.0), mk(n, 1.0)  # logits spread ~ +-12 as in the GPU test


def _attn_fp32(q, k, v):
    return oracle.attention(q.float(), k.float(), v.float())


def _out(o, mode):
    """The context the kernel writes: bf16 hi (bf16) or hi + lo (bf16x3)."""
    if mode == "bf16":
        return tce.rnd(o, 7)
    hi = tce.rnd(o, 7)
    return hi + tce.rnd(o - hi, 7)


def _attn_mode(mode, partial=True, pad=False, p_bits=10):
    def run(q, k, v):
        if not partial:  # keys of the last, partial 64-key block ignored
            k, v = k[..., : k.shape[-2] // 64 * 64, :], v[..., : v.shape[-2] // 64 * 64, :]
        if pad:  # one padding key (zero key, zero value) counted in the soft-max
            k = torch.cat([k, torch.zeros_like(k[..., :1, :])], -2)
            v = torch.cat([v, torch.zeros_like(v[..., :1, :])], -2)
        if mode == "fp32":
            return _attn_fp32(q, k, v)
        return _out(tce.attention_online(q, k, v, p_bits=p_bits), mode)
    return run


def attn_dev(run, mode):
    worst = 0.0
    for m, n in ATTN_SHAPES:
        q, k, v = _qkv(m, n, m * 7 + n)
        ref = tce.attention_fp16(q, k, v) if mode != "fp32" else oracle.attention(q, k, v)
        worst = max(worst, rel_dev(run(q, k, v), ref))
    return worst


@pytest.mark.parametrize("mode", list(MODES))
def test_attention_tolerance_sits_between_error_and_defects(mode):
    err = attn_dev(_attn_mode(mode), mode)
    defects = {"last partial key block dropped": _attn_mode(mode, partial=False),
               "a padding key counted": _attn_mode(mode, pad=True)}
    if mode != "fp32":
        defects["P rounded to bf16"] = _attn_mode(mode, p_bits=7)
    devs = {d: attn_dev(r, mode) for d, r in defects.items()}
    tol = ATTN_TOL[mode]
    print(f"[{mode}] attention: emulated error {err:.2e}, tolerance {tol:.1e}; defects: "
          + ", ".join(f"{d} {v:.2e}" for d, v in devs.items()))
    assert tol >= 3 * err
    for d in ATTN_RESOLVES[mode]:
        assert tol <= devs[d] / 3, (d, devs[d])


# ----------------------------------------------------------------------------------------------- assignment
ASSIGN_SHAPES = [(100, 127), (129, 200), (255, 257)]


def assign_dev(mode, sim=None):
    sd = synth.make_state_dict()
    w64 = {k: v.double() for k, v in sd.items()}
    worst = 0.0
    for m, n in ASSIGN_SHAPES:
        g = torch.Generator().manual_seed(m + n)
        x0, x1 = torch.randn(1, m, 256, generator=g), torch.randn(1, n, 256, generator=g)
        ref = oracle.log_assignment(w64, 3, x0.double(), x1.double())
        if mode == "fp32":
            got = oracle.log_assignment(sd, 3, x0, x1)
        else:
            got = tce.make_log_assignment(dict(final="bf16x3", sim=sim or "bf16x3"))(sd, 3, x0, x1)
        worst = max(worst, float((got.double() - ref).abs().max()))
    return worst


@pytest.mark.parametrize("mode", list(ASSIGN_TOL))
def test_assignment_tolerance_sits_between_error_and_defects(mode):
    """Absolute deviation of the log-assignment matrix; defect: a similarity sweep without one of its lo passes."""
    err = assign_dev(mode)
    devs = {"sim A_lo·W_hi lost": assign_dev("bf16x3", "bf16x2w"), "sim A_hi·W_lo lost": assign_dev("bf16x3", "bf16x2a")}
    tol = ASSIGN_TOL[mode]
    print(f"[{mode}] assignment: emulated error {err:.2e}, tolerance {tol:.1e}; defects: "
          + ", ".join(f"{d} {v:.2e}" for d, v in devs.items()))
    assert tol >= 3 * err
    for d, v in devs.items():
        assert tol <= v / 3, (d, v)
