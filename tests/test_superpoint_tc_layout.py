"""The workspace plan of the SuperPoint tensor-core backbone (csrc/sp_tc.cu, exported host-only as ``sp_tc_layout``)
against the writes the backbone makes, restated here from the kernels:

* every feature map is a zero-padded NHWC matrix whose rows are rounded up to two sequences of ``Lp`` rows, ``Lp`` a
  multiple of the 128-row tile (``level()``), and conv1a, the 2x2 poolings and every tensor-core convolution write ALL
  ``2 Lp`` rows of their level (padding rows as zeros) with ``Cout`` channels, as a bf16 hi and a bf16 lo image;
* the two fp32 heads write ``2 Lp`` rows at 1/8 resolution with row strides 96 (logits) and 256 (descriptors);
* the maps ping-pong between the buffers X, Y and F in the order of ``sp_tc_backbone``.

On small images every level pads up to the same 256 rows, so the 128- and 256-channel maps at 1/4 and 1/8 resolution are
the largest writes; a plan sized for the full-resolution 64-channel map only is overrun there (8x8, 9x15, 17x33)."""
import ctypes as C

import pytest

from lightglue_b200 import _cabi
from lightglue_b200.superpoint import LAYERS

TILE = 128
COUT = {name: co for name, co, _, _ in LAYERS}
CIN = {name: ci for name, _, ci, _ in LAYERS}
BUFFERS = ("XH", "XL", "YH", "YL", "FH", "FL", "logits", "dense", "state")  # sp_tc_layout's order (superpoint_b200.h)
MAPS = {"X": ("XH", "XL"), "Y": ("YH", "YL"), "F": ("FH", "FL"), "image": (), "logits": ("logits",), "dense": ("dense",)}
# (step, level written, map read, map written, channels (row stride) written, bytes per element) in sp_tc_backbone's
# order; a pooling writes level l + 1 from the level-l map it reads
SCHEDULE = (
    ("conv1a", 0, "image", "X", COUT["conv1a"], 2),
    ("conv1b", 0, "X", "Y", COUT["conv1b"], 2),
    ("pool1", 1, "Y", "X", COUT["conv1b"], 2),
    ("conv2a", 1, "X", "Y", COUT["conv2a"], 2),
    ("conv2b", 1, "Y", "X", COUT["conv2b"], 2),
    ("pool2", 2, "X", "Y", COUT["conv2b"], 2),
    ("conv3a", 2, "Y", "X", COUT["conv3a"], 2),
    ("conv3b", 2, "X", "Y", COUT["conv3b"], 2),
    ("pool3", 3, "Y", "X", COUT["conv3b"], 2),
    ("conv4a", 3, "X", "Y", COUT["conv4a"], 2),
    ("conv4b", 3, "Y", "F", COUT["conv4b"], 2),
    ("convPa", 3, "F", "X", COUT["convPa"], 2),
    ("convPb", 3, "X", "logits", 96, 4),   # fp32, 65 channels in a row stride of 96
    ("convDa", 3, "F", "Y", COUT["convDa"], 2),
    ("convDb", 3, "Y", "dense", COUT["convDb"], 4),
)
SIZES = [(h, w) for h in range(8, 161) for w in range(8, 161)] + [(480, 640), (768, 1024)]


def rows(B, H, W):
    """level(): the padded pixels of the batch as two sequences of Lp rows, Lp a multiple of the tile."""
    used = B * (H + 2) * (W + 2)
    lp = ((used + 1) // 2 + TILE - 1) // TILE * TILE
    return 2 * lp


def level_rows(B, H, W):
    return [rows(B, H >> i, W >> i) for i in range(4)]


def parent_total(B, H, W):
    """The plan before the 1/4- and 1/8-resolution maps were accounted for: X / Y sized for the full-resolution map."""
    r = level_rows(B, H, W)
    n = 0
    for size in [r[0] * 64 * 2] * 4 + [r[3] * 128 * 2] * 2 + [r[3] * 96 * 4, r[3] * 256 * 4, 64 * 4]:
        n = (n + 1023) // 1024 * 1024 + size
    return (n + 1023) // 1024 * 1024


def layout(lib, B, H, W):
    off, size = (C.c_int64 * _cabi.SP_TC_BUFFERS)(), (C.c_int64 * _cabi.SP_TC_BUFFERS)()
    total = lib.sp_tc_layout(B, H, W, off, size)
    return dict(zip(BUFFERS, off)), dict(zip(BUFFERS, size)), total


def problems(lib, B, H, W):
    off, size, total = layout(lib, B, H, W)
    out = []
    spans = sorted((off[b], off[b] + size[b], b) for b in BUFFERS)
    if spans[0][0] < 0 or spans[-1][1] > total:
        out.append(f"buffers outside the workspace of {total} bytes")
    for (_, end, a), (start, _, b) in zip(spans, spans[1:]):
        if end > start:
            out.append(f"{a} overlaps {b}")
    r = level_rows(B, H, W)
    for step, lvl, src, dst, ch, elt in SCHEDULE:
        if set(MAPS[src]) & set(MAPS[dst]):
            out.append(f"{step} writes the map it reads")
        need = r[lvl] * ch * elt
        for b in MAPS[dst]:
            if need > size[b]:
                out.append(f"{step} writes {need} bytes into {b} of {size[b]}")
    return out


def test_schedule_restates_the_layer_table():
    """The schedule above runs the twelve layers in order, and every step reads its map at the level and channel count
    the map's last writer left it with."""
    convs = [s for s in SCHEDULE if not s[0].startswith("pool")]
    assert [s[0] for s in convs] == [name for name, *_ in LAYERS]
    for i, (step, lvl, src, _, ch, _) in enumerate(SCHEDULE):
        if src == "image":
            continue
        last = [s for s in SCHEDULE[:i] if s[3] == src][-1]
        pool = step.startswith("pool")
        assert last[1] == (lvl - 1 if pool else lvl), (step, last)
        assert last[4] == (ch if pool else CIN[step]), (step, last)


@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_every_backbone_write_fits_its_buffer(B):
    """B in {1, 2, 3, 8}, every 8 <= H, W <= 160, 480 x 640 and 768 x 1024: each step's write fits the buffer it writes,
    no step writes the map it reads, the buffers are disjoint and inside the workspace."""
    lib = _cabi.load()
    bad = {}
    for H, W in SIZES:
        p = problems(lib, B, H, W)
        if p:
            bad[(H, W)] = p
    shown = {k: bad[k] for k in list(bad)[:3]}
    assert not bad, f"{len(bad)} sizes at B={B}, e.g. {shown}"


@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_plan_is_unchanged_from_64x64_up(B):
    """Images of at least 64 x 64 pixels never had a 1/4- or 1/8-resolution map larger than the full-resolution one: their
    workspace is what it always was, e.g. 429 196 288 bytes at 768 x 1024."""
    lib = _cabi.load()
    assert lib.sp_tc_layout(1, 768, 1024, None, None) == 429196288
    for H, W in SIZES:
        if H >= 64 and W >= 64:
            assert lib.sp_tc_layout(B, H, W, None, None) == parent_total(B, H, W), (B, H, W)


def test_layout_rejects_images_below_one_cell():
    lib = _cabi.load()
    assert lib.sp_tc_layout(0, 64, 64, None, None) == 0
    assert lib.sp_tc_layout(1, 7, 64, None, None) == 0
    assert lib.sp_tc_layout(1, 64, 7, None, None) == 0
    assert lib.sp_tc_layout(1, 8, 8, None, None) > 0
