"""DISK's and HardNet's convolutions against float64 given the kernels' own inputs, at the row-plan and chunk edges.

The C ABI is called with a workspace the test owns; ``disk_workspace_layout`` / ``dhn_workspace_layout`` say where each
layer's output sits in it after the call.  Each check applies the float64 oracle (``disk_oracle.layer`` / ``prepare``,
``doghardnet_oracle.hardnet_conv``) on the GPU to the captured input and compares the captured output, on interior
pixels and live rows only: max|delta| / max|ref| per image (HardNet: over the live patches of the last chunk).  The
tolerances come from tests/test_conv_layer_emulation.py.

* DISK (``disk_heads``): down0 from the image, down1 .. up2 from ``raw``, x3 from raw[7] and raw[0], the heatmap from
  x3, the descriptor GEMM from its gathered rows; the gathered rows themselves exactly from x3.
* HardNet (``dhn_describe``, the last chunk of the last image): conv 1 from the float64 conv 0 of the oracle's patch
  (conv 0's output is overwritten by conv 1's phase images, so conv 1's tolerance covers conv 0 and the patch sampling
  in fp32), conv 2 from the phase images of conv 1's output, conv 3 .. 5 from their captured inputs, conv 6 for every
  live row; exactly: padding pixels of every live frame and row 0 / column 0 of every phase frame are zero."""
import ctypes as C

import pytest
import torch

from lightglue_b200 import DISK, DoGHardNet, _cabi
from oracle import disk_oracle as do
from oracle import disk_synth as ds
from oracle import doghardnet_oracle as dho
from oracle import doghardnet_synth as dhs
from oracle import sift_synth
from oracle.superpoint_oracle import _split as split
from tests.test_conv_layer_emulation import TOL

pytestmark = pytest.mark.gpu

TILE = 128
LEVEL = [0, 1, 2, 3, 4, 3, 2, 1]  # level of raw[l]
COUT = [16, 32, 64, 64, 64, 64, 64, 64]
NP, RA, RB, RC = 256, 34 * 34, 18 * 18, 10 * 10
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst max|delta| / max|ref|:", {k: f"{v:.2e}" for k, v in sorted(WORST.items())})


def tc_rows(used):
    lp = max(TILE, ((used + 1) // 2 + TILE - 1) // TILE * TILE)
    return lp, 2 * lp


def rel(a, ref):
    """max|a - ref| / max|ref| per image (dim 0) -> the largest of them."""
    d = (a.double() - ref).abs().flatten(1).amax(1) / ref.abs().flatten(1).amax(1)
    return float(d.max())


def check(bad, name, a, ref, tol):
    """Records the deviation; a failure goes to `bad`, so that one call reports every check it fails."""
    e = rel(a, ref)
    WORST[name] = max(WORST.get(name, 0.0), e)
    if not e <= tol:
        bad.append((name, e, tol))


def expect(bad, name, ok):
    if not ok:
        bad.append(name)


def layout(fn, *args, n):
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    total = fn(*args, off, size)
    assert total > 0
    assert all(off[i] % 256 == 0 and off[i] + size[i] <= total for i in range(n))
    return list(off), list(size), total


def buf(ws, off, size, dtype, n_elems=None):
    t = ws[off:off + size].view(dtype)
    return t if n_elems is None else t[:n_elems]


def pair(ws, lay, i, n):
    """bf16 hi / lo buffers i, i + 1 -> their sum (float64) over the first n elements."""
    (off, size) = lay
    return buf(ws, off[i], size[i], torch.bfloat16, n).double() + buf(ws, off[i + 1], size[i + 1], torch.bfloat16, n).double()


# ------------------------------------------------------------------------------------------------------------ DISK
_disk = {}


def disk_model(pad):
    if pad not in _disk:
        m = DISK(weights=None, pad_if_not_divisible=pad)
        m.model.load_state_dict(ds.make_disk_state_dict(0), strict=True)
        _disk[pad] = (m.cuda(), {k: v.to("cuda", torch.float64) for k, v in ds.make_disk_state_dict(0).items()})
    return _disk[pad]


def disk_run(b, h, w, pad, p, seed=0):
    """disk_heads at P = p random pixels per image -> (workspace, layout, image, pos, heatmap, descriptors)."""
    m, _ = disk_model(pad)
    lib = _cabi.load()
    image = ds.make_image(h, w, b, 400 + seed + h).cuda()
    handle = m._get_handle(image.device)
    off, size, total = layout(lib.disk_workspace_layout, handle, b, h, w, n=_cabi.DISK_LAYOUT_BUFFERS)
    assert total == lib.disk_workspace_bytes(handle, b, h, w)
    ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
    g = torch.Generator().manual_seed(seed + p)
    pos = torch.stack([torch.randperm(h * w, generator=g)[:p] for _ in range(b)]).to(torch.int32).cuda()
    heat = torch.empty(b, h, w, device="cuda")
    desc = torch.empty(b, p, 128, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.disk_heads(handle, image.data_ptr(), image.shape[1], b, h, w, pos.data_ptr(), p, heat.data_ptr(),
                               desc.data_ptr(), ws.data_ptr(), total, stream), "disk_heads")
    torch.cuda.synchronize()
    return ws, (off, size), image, pos, heat, desc


def padded_map(ws, lay, i, b, h, w, c):
    """Buffer i as [B, C, h + 4, w + 4] float64 (fp32 values)."""
    off, size = lay
    return buf(ws, off[i], size[i], torch.float32, b * (h + 4) * (w + 4) * c).view(b, h + 4, w + 4, c).permute(0, 3, 1, 2).double()


# shapes: (B, H, W, pad_if_not_divisible, regime check on the level plans)
def _smallest(b, hp, wp):
    assert -(-hp // 16) * -(-wp // 16) == 2


def _both_full(b, hp, wp):
    for lv in range(3):  # levels 0 .. 2: both 128-row sequences exactly full
        used = b * ((hp >> lv) + 4) * ((wp >> lv) + 4)
        assert used == tc_rows(used)[1] and used // 2 % TILE == 0


def _seam(b, hp, wp):
    r = ((hp >> 2) + 4) * ((wp >> 2) + 4)  # level 2: image 1 starts at row Lp, the second sequence
    assert b == 2 and r == tc_rows(2 * r)[0]


def _any(b, hp, wp):
    pass


DISK_SHAPES = [
    (1, 16, 32, True, _smallest),
    (1, 33, 47, True, _any),
    (1, 48, 64, False, _any),
    (16, 32, 48, True, _both_full),
    (2, 16, 112, True, _seam),
    (1, 768, 1024, True, _any),
]


@pytest.mark.parametrize("b,h,w,pad,regime", DISK_SHAPES, ids=[f"{s[0]}x{s[1]}x{s[2]}{'' if s[3] else '-nopad'}" for s in DISK_SHAPES])
def test_disk_layers(b, h, w, pad, regime):
    torch.set_grad_enabled(False)
    hp, wp = (-(-h // 16) * 16, -(-w // 16) * 16) if pad else (h, w)
    regime(b, hp, wp)
    m, sd64 = disk_model(pad)
    cap = int(_cabi.load().disk_max_keypoints(m._get_handle(torch.device("cuda")), h, w))
    p = min(cap, 200)
    ws, lay, image, pos, heat, desc = disk_run(b, h, w, pad, p)
    raw = [padded_map(ws, lay, l, b, hp >> LEVEL[l], wp >> LEVEL[l], COUT[l]) for l in range(8)]
    inner = [r[:, :, 2:-2, 2:-2] for r in raw]
    bad = []
    check(bad, "disk down0", inner[0], do.layer(sd64, 0, do.network_input(image.double(), pad)), TOL["disk_down0"])
    for l in range(1, 8):
        check(bad, f"disk layer {l}", inner[l], do.layer(sd64, l, inner), TOL["disk_tc"])
    x3p = padded_map(ws, lay, 8, b, hp, wp, 80)
    x3 = x3p[:, :, 2:-2, 2:-2].contiguous()
    ring = x3p.clone()
    ring[:, :, 2:-2, 2:-2] = 0
    expect(bad, "x3 padding zero", not ring.any())  # the prepare pass zeroes x3's padding
    check(bad, "disk x3", x3, do.prepare(sd64, 8, inner), TOL["disk_x3"])
    _, w8, b8 = do.params(sd64, 8)
    check(bad, "disk heatmap", heat, torch.nn.functional.conv2d(x3, w8[128:], b8[128:], padding=2)[:, 0, :h, :w],
          TOL["disk_heat"])
    _disk_gemm(bad, ws, lay, b, w, p, sd64, x3, pos)
    assert not bad, bad


def _disk_gemm(bad, ws, lay, b, w, p, sd64, x3, pos):
    """The gathered rows exactly from x3 [B, 80, Hp, Wp] (the windows reach into the 16-padding), the GEMM on them
    (live rows b P + j) and its length words."""
    off, size = lay
    rows = b * p
    gh = buf(ws, off[9], size[9], torch.bfloat16, rows * 2048).view(rows, 2048)
    gl = buf(ws, off[10], size[10], torch.bfloat16, rows * 2048).view(rows, 2048)
    cols = torch.nn.functional.unfold(x3, 5, padding=2).view(b, 80, 25, -1).permute(0, 3, 2, 1).reshape(b, -1, 2000)
    at = (pos // w * x3.shape[-1] + pos % w).long()
    want = torch.cat([cols[i, at[i]] for i in range(b)])
    wh, wl = split(want)
    expect(bad, "gathered rows", torch.equal(gh[:, :2000].double(), wh) and torch.equal(gl[:, :2000].double(), wl)
           and not gh[:, 2000:].any())
    _, w8, b8 = do.params(sd64, 8)
    ref = (gh[:, :2000].double() + gl[:, :2000].double()) @ w8[:128].permute(0, 2, 3, 1).reshape(128, -1).T + b8[:128]
    out = buf(ws, off[11], size[11], torch.float32, rows * 128).view(rows, 128)
    check(bad, "disk descriptor GEMM", out.view(b, p, 128), ref.view(b, p, 128), TOL["disk_desc"])
    words = buf(ws, off[12], size[12], torch.int32).cpu()
    lp, _ = tc_rows(rows)
    # the length words of the plan the GEMM runs on, tc_rows(B P): len <= Lp
    expect(bad, f"GEMM length words {words[20:22].tolist()} for Lp {lp}", words[20:22].tolist() == [lp, lp])


@pytest.mark.parametrize("p", [1, 127, 128, 129, 256, 257, -1])
def test_disk_descriptor_gemm_row_edges(p):
    """B = 1: P rows in the GEMM; -1: disk_max_keypoints (594 at 64 x 80)."""
    torch.set_grad_enabled(False)
    m, sd64 = disk_model(True)
    h, w = 64, 80
    if p < 0:
        p = int(_cabi.load().disk_max_keypoints(m._get_handle(torch.device("cuda")), h, w))
    ws, lay, image, pos, heat, desc = disk_run(1, h, w, True, p, seed=p)
    x3 = padded_map(ws, lay, 8, 1, h, w, 80)[:, :, 2:-2, 2:-2]
    bad = []
    _disk_gemm(bad, ws, lay, 1, w, p, sd64, x3.contiguous(), pos)
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------ HardNet
_dhn = {}


def dhn_model(mnk):
    if mnk not in _dhn:
        sd = dhs.make_state_dict(0)
        m = DoGHardNet(weights=None, max_num_keypoints=mnk)
        m.laf_desc.descriptor.load_state_dict(sd, strict=True)
        _dhn[mnk] = (m.cuda(), {k: v.to("cuda", torch.float64) for k, v in sd.items()})
    return _dhn[mnk]


def keypoints(b, n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    kp = torch.rand(b, n, 2, generator=g) * torch.tensor([w - 1.0, h - 1.0])
    sc = 3.0 + 10 * torch.rand(b, n, generator=g)
    ori = (torch.rand(b, n, generator=g) - 0.5) * 6.28
    return kp.cuda(), sc.cuda(), ori.cuda()


def frames(t, n, side, c):
    return t[:n * side * side * c].view(n, side, side, c).permute(0, 3, 1, 2)


def dhn_check(mnk, counts, cap, seed=0):
    """dhn_describe on B = len(counts) 240 x 320 images with counts[b] random keypoints, capacity cap; checks the last
    chunk of the last image."""
    torch.set_grad_enabled(False)
    m, sd64 = dhn_model(mnk)
    lib = _cabi.load()
    b, h, w = len(counts), 240, 320
    image = sift_synth.make_image(h, w, b, 50 + seed).cuda()
    handle = m._get_handle(image.device)
    off, size, total = layout(lib.dhn_workspace_layout, handle, h, w, n=_cabi.DHN_LAYOUT_BUFFERS)
    assert total == lib.dhn_workspace_bytes(handle, b, h, w)
    ws = torch.zeros(total, dtype=torch.uint8, device="cuda")
    kp, sc, ori = keypoints(b, cap, h, w, seed)
    cnt = torch.tensor(counts, dtype=torch.int32).cuda()
    desc = torch.empty(b, cap, 128, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.dhn_describe(handle, image.data_ptr(), 1, None, b, h, w, cap, kp.data_ptr(), sc.data_ptr(),
                                 ori.data_ptr(), cnt.data_ptr(), desc.data_ptr(), ws.data_ptr(), total, stream), "dhn_describe")
    torch.cuda.synchronize()
    lay = (off, size)
    n = counts[-1]
    nchunk = -(-cap // NP)
    k0 = (nchunk - 1) * NP
    live = n - k0
    assert 1 <= live <= NP, (n, cap)  # the last chunk holds live patches
    # the row plans of the last chunk, as the device wrote them from the count
    words = buf(ws, off[15], size[15], torch.int32).cpu().view(-1, 4)
    for lvl, rpp in enumerate((RA, RB, RC)):
        lp, _ = tc_rows(NP * rpp)
        used = live * rpp
        assert words[(nchunk - 1) * 3 + lvl, :2].tolist() == [min(used, lp), max(0, used - lp)]
    lpd, _ = tc_rows(mnk)
    assert words[nchunk * 3, :2].tolist() == [min(n, lpd), max(0, n - lpd)]
    # float64 from the oracle's patches of the live keypoints
    img = image[-1].double()
    laf = dho.laf_from_center_scale_ori(kp[-1:, k0:n].double(), 6.0 * sc[-1:, k0:n].double().reshape(1, -1, 1, 1),
                                        torch.rad2deg(ori[-1:, k0:n].double()).reshape(1, -1, 1))
    ref = dho.hardnet_layers(sd64, dho.extract_patches(img[None], laf[0]))
    # conv 1's output from its phase images
    _, rows_b = tc_rows(NP * RB)
    ph = pair(ws, lay, 0, 4 * rows_b * 64).view(4, rows_b, 64)[:, :NP * RB].reshape(4, NP, 18, 18, 64)[:, :live]
    bad = []
    expect(bad, "phase frames: row 0 / column 0 zero", not ph[:, :, 0].any() and not ph[:, :, :, 0].any())
    c1 = torch.zeros(live, 34, 34, 64, dtype=torch.float64, device="cuda")
    for q in range(4):
        c1[:, q >> 1::2, q & 1::2] = ph[q][:, 1:, 1:]
    c1 = c1.permute(0, 3, 1, 2)
    outs = {1: c1}
    for i, (li, side, c) in zip((4, 6, 8, 10), ((2, 18, 64), (3, 18, 64), (4, 10, 128), (5, 10, 128))):
        _, rows = tc_rows(NP * side * side)
        outs[li] = frames(pair(ws, lay, i, rows * c), live, side, c)
    for li, o in outs.items():
        ring = o.clone()
        ring[:, :, 1:-1, 1:-1] = 0
        expect(bad, f"conv {li}: padding pixels zero", not ring.any())
    expect(bad, "conv 1: channels 32 .. 63 zero", not c1[:, 32:].any())
    check(bad, "hardnet conv 1", c1[None, :, :32, 1:-1, 1:-1], ref[1][None], TOL["hn_conv1"])  # [None]: one set of patches
    check(bad, "hardnet conv 2", outs[2][None, :, :, 1:-1, 1:-1], dho.hardnet_conv(sd64, 2, c1[:, :32, 1:-1, 1:-1])[None],
          TOL["hn_conv"])
    for li in (3, 4, 5):
        check(bad, f"hardnet conv {li}", outs[li][None, :, :, 1:-1, 1:-1],
              dho.hardnet_conv(sd64, li, outs[li - 1][:, :, 1:-1, 1:-1])[None], TOL["hn_conv"])
    # conv 6 on every live row of the image, and its input rows of this chunk exactly from conv 5's output
    _, rows_d = tc_rows(mnk)
    gh = buf(ws, off[12], size[12], torch.bfloat16, n * 8192).view(n, 8192)
    gl = buf(ws, off[13], size[13], torch.bfloat16, n * 8192).view(n, 8192)
    g = gh.double() + gl.double()
    expect(bad, "conv 6 rows", torch.equal(g[k0:n], outs[5][:, :, 1:-1, 1:-1].permute(0, 2, 3, 1).reshape(live, -1)))
    w6, b6 = dho.folded(sd64, 6, g)
    out6 = buf(ws, off[14], size[14], torch.float32, n * 128).view(n, 128)
    check(bad, "hardnet conv 6", out6[None], (g @ w6.permute(0, 2, 3, 1).reshape(128, -1).T + b6)[None], TOL["hn_conv6"])
    assert not bad, bad


# (max_num_keypoints, totals): every total the cap holds, last chunks of 1, 128, 129, 255 and 256 live patches
HN_CASES = [(256, t) for t in (1, 128, 129, 255, 256)] + [(257, t) for t in (1, 128, 129, 255, 256, 257)] + \
           [(2048, t) for t in (1, 128, 129, 255, 256, 257, 384, 385, 512)]


@pytest.mark.parametrize("mnk,total", HN_CASES, ids=[f"max{m}-n{t}" for m, t in HN_CASES])
def test_hardnet_layers(mnk, total):
    dhn_check(mnk, [total], total, seed=total)


def test_hardnet_later_image_with_fewer_keypoints():
    """Image 1 has fewer keypoints than image 0: the dead slots of its last chunk hold image 0's patches."""
    dhn_check(2048, [300, 270], 300, seed=7)
