"""Calibration of the per-layer tolerances of tests/test_gpu_conv_layers.py (DISK's U-Net and descriptor GEMM, HardNet's
seven convolutions) and of the end-to-end gates of tests/test_gpu_disk.py and tests/test_gpu_doghardnet.py.

Each check compares a kernel's output with float64 applied to the kernel's own input.  ``oracle/conv_emulation.py``
emulates the kernels' arithmetic on that input; each tolerance must be at least 3x the emulated error and at most 1/3 of
every defect listed for it.  Measure: max|delta| / max|ref| per image (HardNet: per set of patches); the HardNet
end-to-end gate is absolute, on unit descriptors.

Defects below every check: a nonzero operand channel past Cin (DISK's 16 / 32 / 96 -> 64 / 64 / 128, HardNet's 32 -> 64)
meets a zero packed weight column, so it changes no output; and a stride-1 layer cannot read phases transposed.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_emulation as ce
from oracle import disk_oracle as do
from oracle import disk_synth as ds
from oracle import doghardnet_oracle as dho
from oracle import doghardnet_synth as dhs
from oracle import sift_synth

TOL = {
    "disk_tc": 5e-5,     # down1 .. up2 on the tensor cores
    "disk_down0": 1e-5,  # fp32 on the CUDA cores, from the image
    "disk_x3": 1e-5,     # up3's input, from raw[7] and raw[0]
    "disk_heat": 1e-5,   # the heatmap channel, from x3
    "disk_desc": 5e-5,   # the descriptor GEMM, from the gathered rows
    "hn_conv1": 5e-5,    # from the float64 patch: includes conv 0 and the patch normalisation in fp32
    "hn_conv": 5e-5,     # convs 2 .. 5, from the captured input
    "hn_conv6": 5e-5,    # from the gathered rows
}
E2E_DISK = 1e-4  # tests/test_gpu_disk.py::test_heads_vs_float64, relative per head
E2E_HN = 1e-4    # tests/test_gpu_doghardnet.py, absolute on unit descriptors
LOST = {"a_lo": dict(lost={"a_lo"}), "w_lo": dict(lost={"w_lo"})}


def rel(a, ref):
    return float((a - ref).abs().max() / ref.abs().max())


def assert_between(tol, emulated, defects):
    assert 3 * emulated <= tol, (emulated, tol)
    for name, dev in defects.items():
        assert dev >= 3 * tol, (name, dev, tol)


# --------------------------------------------------------------------------------------------------------------- DISK
@pytest.fixture(scope="module")
def disk():
    torch.set_grad_enabled(False)
    sd = ds.make_disk_state_dict(0)
    sd64 = {k: v.double() for k, v in sd.items()}
    img = do.network_input(ds.make_image(48, 64, 1, 348).double())
    raw = [do.layer(sd64, 0, img)]
    for l in range(1, 8):
        raw.append(do.layer(sd64, l, raw))
    return sd, sd64, img.float().double(), [r.float().double() for r in raw]  # the fp32 values the kernels store


def _pre_split_unet(sd, x):
    """disk_oracle.unet as it was written before it was split into layers."""
    def conv(x, a, w, b):
        return F.conv2d(F.prelu(F.instance_norm(x, eps=1e-5), a), w, b, padding=w.shape[-1] // 2)

    feats = []
    for i in range(5):
        if i:
            x = F.avg_pool2d(x, 2)
        p = f"unet.path_down.{i}.1"
        x = conv(x, sd[f"{p}.1.weight"], sd[f"{p}.3.weight"], sd[f"{p}.3.bias"])
        feats.append(x)
    bot = feats[4]
    for i in range(4):
        up = F.interpolate(bot, scale_factor=2, mode="bilinear", align_corners=False)
        p = f"unet.path_up.{i}.conv"
        bot = conv(torch.cat([up, feats[3 - i]], 1), sd[f"{p}.1.weight"], sd[f"{p}.3.weight"], sd[f"{p}.3.bias"])
    return bot


def test_disk_layers_compose_to_the_pre_split_unet(disk):
    sd, sd64, _, _ = disk
    image = ds.make_image(33, 47, 2, 5)
    for s, x in ((sd, image), (sd64, image.double())):
        x = do.network_input(x)
        assert torch.equal(do.unet(s, x), _pre_split_unet(s, x))


@pytest.mark.parametrize("l", range(1, 8))
def test_disk_tensor_core_layer(disk, l):
    sd, sd64, _, raw = disk
    ref = do.layer(sd64, l, raw)
    defects = {k: rel(ce.disk_layer(sd, l, raw, **v), ref) for k, v in LOST.items()}
    defects["nobias"] = rel(ce.disk_layer(sd, l, raw, nobias=True), ref)
    defects["row stride W + 2"] = rel(ce.disk_layer(sd, l, raw, row_stride=True), ref)
    if l >= 5:
        defects["align_corners"] = rel(ce.disk_layer(sd, l, raw, align_corners=True), ref)
    assert_between(TOL["disk_tc"], rel(ce.disk_layer(sd, l, raw), ref), defects)


def test_disk_down0(disk):
    sd, sd64, img, _ = disk
    ref = do.layer(sd64, 0, img)
    assert_between(TOL["disk_down0"], rel(ce.disk_layer(sd, 0, img), ref),
                   {"nobias": rel(ce.disk_layer(sd, 0, img, nobias=True), ref)})


def test_disk_x3_and_heatmap(disk):
    sd, sd64, _, raw = disk
    x3 = do.prepare(sd64, 8, raw)
    assert_between(TOL["disk_x3"], rel(ce.disk_prepare(sd, 8, raw), x3),
                   {"align_corners": rel(ce.disk_prepare(sd, 8, raw, align_corners=True), x3)})
    x3 = x3.float().double()
    _, w, b = do.params(sd64, 8)
    heat = F.conv2d(x3, w[128:], b[128:], padding=2)[:, 0]
    assert_between(TOL["disk_heat"], rel(ce.disk_heat(sd, x3), heat), {"nobias": rel(ce.disk_heat(sd, x3, nobias=True), heat)})


@pytest.mark.parametrize("p", [129, 200])
def test_disk_descriptor_gemm(disk, p):
    sd, sd64, _, raw = disk
    x3 = ce.disk_prepare(sd, 8, raw)
    pos = torch.randperm(48 * 64, generator=torch.Generator().manual_seed(p))[:p][None]
    gh, gl = ce.split(ce.im2col(x3, pos))
    w, b = ce.desc_weight(sd64)
    ref = (gh + gl) @ w.T + b
    defects = {k: rel(ce.gemm_rows(gh, gl, w.float(), b, **v), ref) for k, v in LOST.items()}
    defects["nobias"] = rel(ce.gemm_rows(gh, gl, w.float(), b, nobias=True), ref)
    defects["last partial tile dropped"] = rel(ce.gemm_rows(gh, gl, w.float(), b, drop_tile=True), ref)
    assert_between(TOL["disk_desc"], rel(ce.gemm_rows(gh, gl, w.float(), b), ref), defects)


def _disk_heads(sd, img, pos, defects):
    raw = []
    for l in range(8):
        raw.append(ce.disk_layer(sd, l, img if l == 0 else raw, **defects.get(l, {})))
    x3 = ce.disk_prepare(sd, 8, raw)
    w, b = ce.desc_weight(sd)
    return ce.disk_heat(sd, x3), ce.gemm_rows(*ce.split(ce.im2col(x3, pos)), w, b)


def test_disk_end_to_end_gate(disk):
    """The heads after nine layers: a lost pass in any tensor-core layer moves them by >= 6e-4; a lost bias in layers
    0 .. 7 is removed by the next instance norm and stays invisible (the per-layer checks see it)."""
    sd, sd64, img, _ = disk
    pos = torch.randperm(48 * 64, generator=torch.Generator().manual_seed(0))[:200][None]
    heat64, desc64 = do.heads(sd64, img[:, :, :48, :64])
    ref = (heat64, desc64[0].flatten(1)[:, pos[0]].T)
    err = max(rel(a, r) for a, r in zip(_disk_heads(sd, img, pos, {}), ref))
    defects = {}
    for l in (1, 4, 7):
        for k, v in LOST.items():
            defects[f"layer {l} {k}"] = max(rel(a, r) for a, r in zip(_disk_heads(sd, img, pos, {l: v}), ref))
    assert_between(E2E_DISK, err, defects)
    hidden = max(rel(a, r) for a, r in zip(_disk_heads(sd, img, pos, {3: dict(nobias=True)}), ref))
    assert hidden < E2E_DISK


# --------------------------------------------------------------------------------------------------------------- HardNet
@pytest.fixture(scope="module")
def hardnet():
    torch.set_grad_enabled(False)
    sd = dhs.make_state_dict(0)
    sd64 = {k: v.double() for k, v in sd.items()}
    image = sift_synth.make_image(120, 160, 1, 31).double()
    g = torch.Generator().manual_seed(0)
    n = 16
    kp = torch.rand(n, 2, generator=g, dtype=torch.float64) * torch.tensor([159.0, 119.0])
    sc = 1.5 + 10 * torch.rand(n, generator=g, dtype=torch.float64)
    ori = (torch.rand(n, generator=g, dtype=torch.float64) - 0.5) * 6.28
    laf = dho.laf_from_center_scale_ori(kp[None], 6.0 * sc.reshape(1, -1, 1, 1), torch.rad2deg(ori).reshape(1, -1, 1))
    patches = dho.extract_patches(image[0:1], laf[0])
    return sd, sd64, patches, dho.hardnet_layers(sd64, patches), ce.hn_layers(sd, patches.float().double())


def val(pair):
    return (pair[0] + pair[1])[:, :, 1:-1, 1:-1]


def test_hardnet_layers_end_in_hardnet(hardnet):
    sd, sd64, patches, layers, _ = hardnet
    assert [tuple(t.shape[1:]) for t in layers] == [(32, 32, 32), (32, 32, 32), (64, 16, 16), (64, 16, 16),
                                                     (128, 8, 8), (128, 8, 8), (128,)]
    torch.testing.assert_close(F.normalize(layers[-1], dim=1), dho.hardnet(sd64, patches), rtol=0, atol=1e-13)


def test_hardnet_conv1_from_the_patch(hardnet):
    sd, _, _, layers, emu = hardnet
    x0 = ce.framed(emu[0])
    defects = {k: rel(val(ce.hn_conv(sd, 1, x0, **v)), layers[1]) for k, v in LOST.items()}
    defects["nobias"] = rel(val(ce.hn_conv(sd, 1, x0, nobias=True)), layers[1])
    assert_between(TOL["hn_conv1"], rel(val(emu[1]), layers[1]), defects)


@pytest.mark.parametrize("li", [2, 3, 4, 5])
def test_hardnet_conv(hardnet, li):
    sd, sd64, _, _, emu = hardnet
    x = emu[li - 1]
    ref = dho.hardnet_conv(sd64, li, val(x))
    defects = {k: rel(val(ce.hn_conv(sd, li, x, **v)), ref) for k, v in LOST.items()}
    defects["nobias"] = rel(val(ce.hn_conv(sd, li, x, nobias=True)), ref)
    if dho.STRIDES[li] == 2:
        defects["phases transposed"] = rel(val(ce.hn_conv(sd, li, x, phase_swap=True)), ref)
    # conv li - 1 leaving its padding ring as computed: conv li reads it, the float64 check reads zeros
    bad = ce.hn_conv(sd, li - 1, emu[li - 2] if li > 2 else ce.framed(emu[0]), ring=True)
    defects["input ring not re-zeroed"] = rel(val(ce.hn_conv(sd, li, bad)), dho.hardnet_conv(sd64, li, val(bad)))
    assert_between(TOL["hn_conv"], rel(val(ce.hn_conv(sd, li, x)), ref), defects)


def test_hardnet_conv6(hardnet):
    sd, sd64, _, _, emu = hardnet
    gh, gl = ce.hn_rows6(emu[5])
    w, b = ce.hn_weight6(sd)
    w64, b64 = dho.folded(sd64, 6, gh)
    ref = (gh + gl) @ w64.permute(0, 2, 3, 1).reshape(128, -1).T + b64
    defects = {k: rel(ce.gemm_rows(gh, gl, w, b, **v), ref) for k, v in LOST.items()}
    defects["nobias"] = rel(ce.gemm_rows(gh, gl, w, b, nobias=True), ref)
    defects["last partial tile dropped"] = rel(ce.gemm_rows(gh, gl, w, b, drop_tile=True), ref)  # 16 of 128 rows live
    assert_between(TOL["hn_conv6"], rel(ce.gemm_rows(gh, gl, w, b), ref), defects)


def test_hardnet_end_to_end_gate(hardnet):
    sd, _, patches, layers, emu = hardnet
    want = F.normalize(layers[-1], dim=1)

    def err(out):
        return float((F.normalize(out[-1], dim=1) - want).abs().max())

    defects = {f"conv {li} {k}": err(ce.hn_layers(sd, patches.float().double(), {li: v}))
               for li in (1, 3, 6) for k, v in LOST.items()}
    assert_between(E2E_HN, err(emu), defects)
