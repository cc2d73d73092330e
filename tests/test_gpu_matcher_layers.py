"""The matcher's kernels against float64 given their own inputs, at the tile and persistent-schedule edges.

* Layers: ``forward_with_layers`` captures the residual stream after every layer; layer i's output is compared with
  ``oracle.layer`` run in float64 on the GPU from the captured output of layer i - 1 (layer 0 from the float64 input
  projection), per layer, pair and image, so an error cannot hide behind the accumulated stream.
* Attention: ``attention`` against ``tc_emulation.attention_fp16`` in float64 (fp32: plain float64) at every 64-key
  block and 128-query tile edge.
* Assignment: ``log_assignment_matrix`` on both sides of Lp = 256 (below it the tensor-core modes take the CUDA-core
  assignment) against float64 ``log_assignment``; matches on every row whose decision margins exceed the tolerance.

The tolerances come from ``tests/test_matcher_layer_emulation.py``, which places each between its mode's emulated
error and the defects it must catch.  Each shape asserts the schedule it is there for."""
import pytest
import torch

from lightglue_b200 import LightGlue, _cabi, synth
from oracle import lightglue_oracle as oracle
from oracle import tc_emulation as tce
from tests.test_matcher_layer_emulation import ASSIGN_TOL, ATTN_TOL, LAYER_TOL, SMALL

pytestmark = pytest.mark.gpu

TBM = 128  # rows per linear tile
_sd = {}


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def state_dict(input_dim, scale_ori):
    key = (input_dim, scale_ori)
    if key not in _sd:
        sd = synth.make_state_dict(input_dim=input_dim, add_scale_ori=scale_ori)
        _sd[key] = (sd, {k: v.to("cuda", torch.float64) for k, v in sd.items()})
    return _sd[key]


def rel_dev(a, ref):
    return float((a.double() - ref).abs().max()) / max(float(ref.abs().max()), 1.0)


# (B, M, N, input_dim, add_scale_ori, what the shape reaches); row_tiles = 2 B Lp / 128 over both images' sequences
def _one_row(b, m, n, lp, tiles):
    assert m == n == 1 and tiles == 2


def _skipped(b, m, n, lp, tiles):
    assert -(-m // TBM) < lp // TBM  # image 0's sequence has tiles without a row


def _box_edge(b, m, n, lp, tiles):
    assert lp == TBM and {m % 64, n % 64} <= {63, 0, 1} and min(m, n) in (63, 64)


def _lp256(b, m, n, lp, tiles):
    assert lp == 256


def _partial(b, m, n, lp, tiles):
    assert lp == 384 and m % TBM and n % TBM


def _qkv_ffn0_wrap(b, m, n, lp, tiles):
    assert 3 * tiles > sms() and tiles > sms() // 2 and tiles <= sms()  # QKV and ffn.0 take a second tile, ffn.3 not


def _all_wrap(b, m, n, lp, tiles):
    assert tiles > sms() and tiles % sms()  # every linear takes a second tile, the last round partly


def _any(b, m, n, lp, tiles):
    pass


LAYER_CASES = [
    (1, 1, 1, 256, False, _one_row),
    (1, 5, 300, 256, False, _skipped),
    (1, 63, 65, 256, False, _box_edge),
    (1, 64, 64, 256, False, _box_edge),
    (1, 65, 63, 256, False, _box_edge),
    (1, 127, 129, 256, False, _lp256),
    (2, 255, 257, 256, False, _partial),
    (3, 2047, 2049, 256, False, _qkv_ffn0_wrap),
    (5, 2048, 2048, 256, False, _all_wrap),
    (1, 700, 513, 128, False, _any),  # tc_input_proj
    (2, 300, 301, 256, True, _any),  # pos_dim 4
]
PRECISIONS = ["fp32", "bf16x3", "bf16"]


def _inputs(data, w64):
    """float64 copies of the pair's inputs, and layer 0's input (the input projection) in float64."""
    d64 = {k: {kk: vv.to("cuda", torch.float64) for kk, vv in v.items()} for k, v in data.items()}
    xs = []
    for im in ("image0", "image1"):
        x = d64[im]["descriptors"]
        if "input_proj.weight" in w64:
            x = torch.nn.functional.linear(x, w64["input_proj.weight"], w64["input_proj.bias"])
        xs.append(x)
    return d64, xs


def check_layers(mod, data, w64, scale_ori, prec, label, lengths=None):
    """Every captured layer against float64 ``layer`` from the captured previous one, per pair against the tolerance
    of its tier (an image with fewer than SMALL keypoints: "small")."""
    cd = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    out, layers = mod.forward_with_layers(cd)
    assert len(layers) == 9
    b, m = data["image0"]["keypoints"].shape[:2]
    n = data["image1"]["keypoints"].shape[1]
    for p in range(b):
        l0, l1 = (m, n) if lengths is None else (int(lengths[0][p]), int(lengths[1][p]))
        rows = {"image0": l0, "image1": l1}  # the pair's real rows
        sub = {k: {kk: vv[p:p + 1] if kk == "image_size" else vv[p:p + 1, : rows[k]]
                   for kk, vv in v.items() if kk != "num_keypoints"} for k, v in data.items()}
        d64, (x0, x1) = _inputs(sub, w64)
        enc = oracle.encodings(w64, d64, scale_ori)
        row = []
        for i, (a0, a1) in enumerate(layers):
            a0, a1 = a0[p:p + 1, :l0], a1[p:p + 1, :l1]
            r0, r1 = oracle.layer(w64, i, x0, x1, enc)
            row.append(max(rel_dev(a0, r0), rel_dev(a1, r1)))
            x0, x1 = a0.double(), a1.double()
        tier = "small" if min(l0, l1) < SMALL else "large"
        tol = LAYER_TOL[tier][prec]
        print(f"[{prec}] {label} pair {p} ({tier}): worst {max(row):.2e} (tolerance {tol:.1e}); per layer "
              + " ".join(f"{v:.1e}" for v in row))
        assert max(row) <= tol, (prec, p, row)


@pytest.mark.parametrize("b,m,n,d,scale_ori,regime", LAYER_CASES,
                         ids=[f"b{c[0]}_m{c[1]}_n{c[2]}_d{c[3]}{'_so' if c[4] else ''}" for c in LAYER_CASES])
def test_layers_from_their_own_inputs(b, m, n, d, scale_ori, regime):
    torch.set_grad_enabled(False)
    lp = int(_cabi.load().lg_padded_length(m, n))
    regime(b, m, n, lp, 2 * b * lp // TBM)
    sd, w64 = state_dict(d, scale_ori)
    data, _ = synth.make_pair(n, m=m, d=d, b=b, seed=1000 + m + n, scale_ori=scale_ori)
    for prec in PRECISIONS:
        mod = LightGlue(features=None, input_dim=d, add_scale_ori=scale_ori, precision=prec, depth_confidence=-1,
                        width_confidence=-1)
        mod.load_state_dict(sd, strict=False)
        check_layers(mod.eval().cuda(), data, w64, scale_ori, prec, f"B={b} {m}x{n}")


def test_layers_ragged_batch():
    """Lengths 1, 129 and 2047 in one batch padded to 2047: each pair's rows against float64 from its own inputs."""
    torch.set_grad_enabled(False)
    sd, w64 = state_dict(256, False)
    data, _ = synth.make_pair(2047, b=3, seed=4711)
    lengths = (torch.tensor([1, 129, 2047]), torch.tensor([2047, 1, 129]))
    data["image0"]["num_keypoints"], data["image1"]["num_keypoints"] = lengths
    for prec in PRECISIONS:
        mod = LightGlue(features=None, precision=prec, depth_confidence=-1, width_confidence=-1)
        mod.load_state_dict(sd, strict=False)
        check_layers(mod.eval().cuda(), data, w64, False, prec, "ragged 1/129/2047", lengths)


ATTN_SIZES = [1, 63, 64, 65, 127, 128, 129, 2049]


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("cross", [False, True])
def test_attention_at_block_edges(prec, cross):
    torch.set_grad_enabled(False)
    mod = LightGlue(features=None, precision=prec, depth_confidence=-1, width_confidence=-1).eval().cuda()
    worst, b = 0.0, 2
    for m in ATTN_SIZES:
        for n in ATTN_SIZES:
            g = torch.Generator(device="cuda").manual_seed(m * 7919 + n)
            mk = lambda l, s: torch.randn(b, 4, l, 64, device="cuda", generator=g) * s  # noqa: E731
            q0, k0, v0, q1, k1, v1 = mk(m, 2.0), mk(m, 2.0), mk(m, 1.0), mk(n, 2.0), mk(n, 2.0), mk(n, 1.0)
            c0, c1 = mod.attention(q0, k0, v0, q1, k1, v1, cross=cross)
            att = oracle.attention if prec == "fp32" else tce.attention_fp16
            merge = lambda o: o.transpose(1, 2).flatten(-2)  # noqa: E731
            r0 = merge(att(q0.double(), (k1 if cross else k0).double(), (v1 if cross else v0).double()))
            r1 = merge(att(q1.double(), (k0 if cross else k1).double(), (v0 if cross else v1).double()))
            e = max(max(rel_dev(c0[i], r0[i]), rel_dev(c1[i], r1[i])) for i in range(b))
            assert torch.isfinite(c0).all() and torch.isfinite(c1).all()
            worst = max(worst, e)
            assert e <= ATTN_TOL[prec], (prec, cross, m, n, e)
    print(f"[{prec}] attention cross={cross}: worst {worst:.2e} over {len(ATTN_SIZES) ** 2} shapes "
          f"(tolerance {ATTN_TOL[prec]:.1e})")


def decided(ref, tol):
    """Rows of image 0 and columns of image 1 whose matches0 / matches1 cannot change under a matrix error <= tol:
    arg-max margins over 2 tol for the row (column) and for the column (row) it points at, and the mutual best score
    more than tol from log(filter_threshold)."""
    core = ref[:, :-1, :-1]

    def margin(t, dim):
        if t.shape[dim] < 2:
            return torch.full(t.select(dim, 0).shape, float("inf"), dtype=t.dtype, device=t.device)
        top = t.topk(2, dim=dim).values
        return top.select(dim, 0) - top.select(dim, 1)

    mr, mc = margin(core, 2), margin(core, 1)  # [B, M], [B, N]
    a0, a1 = core.argmax(2), core.argmax(1)
    best0 = core.amax(2)
    th = torch.log(torch.tensor(0.1, dtype=ref.dtype))
    ok0 = (mr > 2 * tol) & (mc.gather(1, a0) > 2 * tol) & ((best0 - th).abs() > tol)
    ok1 = (mc > 2 * tol) & (mr.gather(1, a1) > 2 * tol) & ((best0.gather(1, a1) - th).abs() > tol)
    return ok0, ok1


ASSIGN_CASES = [(100, 127), (128, 128), (129, 200), (255, 257), (1, 600)]


@pytest.mark.parametrize("prec", ["bf16x3", "fp32"])
@pytest.mark.parametrize("m,n", ASSIGN_CASES)
def test_assignment_both_sides_of_lp256(prec, m, n):
    torch.set_grad_enabled(False)
    lp = int(_cabi.load().lg_padded_length(m, n))
    print(f"Lp = {lp}: {'tensor-core sweeps' if prec != 'fp32' and lp >= 256 else 'CUDA-core assignment'}")
    assert (lp < 256) == ((m, n) == (100, 127) or (m, n) == (128, 128))
    sd, w64 = state_dict(256, False)
    mod = LightGlue(features=None, precision=prec, depth_confidence=-1, width_confidence=-1)
    mod.load_state_dict(sd, strict=False)
    mod = mod.eval().cuda()
    g = torch.Generator(device="cuda").manual_seed(m * 131 + n)
    x0 = torch.randn(3, m, 256, device="cuda", generator=g)
    x1 = torch.randn(3, n, 256, device="cuda", generator=g)
    tol = ASSIGN_TOL[prec]
    full, m0, m1, _, _ = mod.log_assignment_matrix(5, x0, x1)
    ref = oracle.log_assignment(w64, 5, x0.double(), x1.double())
    err = float((full.double() - ref).abs().max())
    ref, m0, m1 = ref.cpu(), m0.cpu(), m1.cpu()
    r0, r1, _, _ = oracle.filter_matches(ref, 0.1)
    ok0, ok1 = decided(ref, tol)
    excl = 1.0 - float(torch.cat([ok0.flatten(), ok1.flatten()]).double().mean())
    print(f"[{prec}] B=3 {m}x{n}: max|Δ| {err:.2e} (tolerance {tol:.1e}); {excl:.2%} of rows undecided")
    assert err <= tol
    assert excl < 0.01
    assert torch.equal(m0[ok0], r0[ok0]) and torch.equal(m1[ok1], r1[ok1])
