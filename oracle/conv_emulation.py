"""The arithmetic of DISK's and HardNet's convolutions on the GPU, emulated on the CPU  --  TEST INFRASTRUCTURE ONLY.

The tensor-core layers (``tc_conv``) read split-bf16 operands: every stored activation and every packed fp32 weight
becomes a bf16 pair hi = bf16(v), lo = bf16(v - hi), and each product is A_hi W_hi + A_hi W_lo + A_lo W_hi.  Here the
three products of one tap and one 64-channel block are summed exactly (float64) and accumulated in fp32 over the
blocks, as the kernel's MMAs accumulate; the bias is added in fp32.  What runs on the CUDA cores (DISK's statistics,
prepare pass, down0 and heatmap channel; HardNet's patch normalisation and conv 0) runs here in torch float32.

The switches express defects the GPU checks (tests/test_gpu_conv_layers.py) claim to resolve:

* ``lost``: a set of {"a_lo", "w_lo"}: the A_lo W_hi or the A_hi W_lo pass is missing;
* ``nobias``: the fp32 epilogue's bias is missing;
* ``row_stride``: DISK's 5x5 taps step rows by W + 2 instead of W + 4;
* ``align_corners``: DISK's upsampling with align_corners=True;
* ``phase_swap``: a stride-2 HardNet layer reads the polyphase images (py, px) transposed;
* ``ring``: a HardNet layer leaves its output's padding ring as computed instead of re-zeroing it;
* ``drop_tile``: a descriptor GEMM loses the last partial 128-row tile of its live rows.

Values are float64 tensors holding fp32 (or bf16) values.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import disk_oracle as do
from . import doghardnet_oracle as dho
from .superpoint_oracle import _split as split

BK = 64     # channels per K block of tc_conv
TILE = 128  # rows per GEMM tile


def _products(ah, al, wh, wl, lost, eq):
    p = torch.einsum(eq, ah, wh)
    if "w_lo" not in lost:
        p = p + torch.einsum(eq, ah, wl)
    if "a_lo" not in lost:
        p = p + torch.einsum(eq, al, wh)
    return p


def _bias(acc, b, nobias, shape):
    return acc if nobias else acc + b.to(torch.float32).view(shape)


# ------------------------------------------------------------------------------------------------------------- DISK
def rows_of(x, q):
    """[B, C, h, w] -> zero-padded NHWC rows [B (h + 2q)(w + 2q), C] (tc_conv's operand layout)."""
    return F.pad(x, (q, q, q, q)).permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def interior(rows, b, h, w, q):
    """The inverse of ``rows_of``: [B (h + 2q)(w + 2q), C] -> [B, C, h, w]."""
    return rows.reshape(b, h + 2 * q, w + 2 * q, -1)[:, q:q + h, q:q + w].permute(0, 3, 1, 2)


def _shift(a, off):
    out = torch.zeros_like(a)
    if off >= 0:
        out[:a.shape[0] - off] = a[off:]
    else:
        out[-off:] = a[:a.shape[0] + off]
    return out


def conv_rows(ah, al, w, b, width, q, lost=(), nobias=False, row_stride=None):
    """tc_conv on padded rows: output row r = sum over taps of A[r + (dy - q) S + dx - q] W_tap, S = width + 2q
    (``row_stride`` overrides it), split-bf16 products per (tap, 64-channel block), fp32 accumulation -> fp32 [R, Cout]."""
    wh, wl = split(w)
    k = w.shape[-1]
    stride = row_stride or width + 2 * q
    acc = torch.zeros(ah.shape[0], w.shape[0], dtype=torch.float32)
    for dy in range(k):
        for dx in range(k):
            off = (dy - q) * stride + dx - q
            sh, sl = _shift(ah, off), _shift(al, off)
            for c0 in range(0, w.shape[1], BK):
                c = slice(c0, c0 + BK)
                acc += _products(sh[:, c], sl[:, c], wh[:, c, dy, dx], wl[:, c, dy, dx], lost, "rc,oc->ro").float()
    return _bias(acc, b, nobias, (1, -1)).double()


def disk_prepare(sd, l, inputs, align_corners=False):
    """``disk_oracle.prepare`` in fp32 (the prepare pass): gathered input, per-image channel statistics, PReLU."""
    x = do.gather(l, inputs, align_corners).float()
    var, mean = torch.var_mean(x, dim=(2, 3), keepdim=True, unbiased=False)
    return F.prelu((x - mean) * (1.0 / torch.sqrt(var + 1e-5)), do.params(sd, l)[0].float()).double()


def disk_layer(sd, l, inputs, lost=(), nobias=False, row_stride=False, align_corners=False):
    """Layer l's raw output [B, Cout, h, w] as the kernels compute it from ``inputs`` (fp32 values, see
    ``disk_oracle.gather``): down0 in fp32 on the CUDA cores, down1 .. up2 on the tensor cores."""
    x = disk_prepare(sd, l, inputs, align_corners)
    _, w, b = do.params(sd, l)
    if l == 0:
        return F.conv2d(x.float(), w.float(), None if nobias else b.float(), padding=2).double()
    bs, _, h, wd = x.shape
    ah, al = split(rows_of(x, 2))
    y = conv_rows(ah, al, w.float(), b, wd, 2, lost, nobias, wd + 2 if row_stride else None)
    return interior(y, bs, h, wd, 2)


def disk_heat(sd, x3, nobias=False):
    """The heatmap channel: fp32 5x5x80 dot with the padded x3 [B, 80, h, w] -> [B, h, w]."""
    _, w, b = do.params(sd, 8)
    return F.conv2d(x3.float(), w[128:].float(), None if nobias else b[128:].float(), padding=2)[:, 0].double()


def im2col(x3, pos):
    """The descriptor GEMM's rows: the 5x5x80 window of x3 [B, 80, h, w] around each flat pixel pos [B, P] (y w + x),
    column tap 80 + ci -> [B P, 2000]."""
    bs, c, h, w = x3.shape
    cols = F.unfold(x3, 5, padding=2).view(bs, c, 25, h * w).permute(0, 3, 2, 1).reshape(bs, h * w, 25 * c)
    return torch.cat([cols[i, pos[i].long()] for i in range(bs)])


def desc_weight(sd):
    """up3's 128 descriptor channels as the packed [128, 2000] matrix (column tap 80 + ci) and bias [128]."""
    _, w, b = do.params(sd, 8)
    return w[:128].permute(0, 2, 3, 1).reshape(128, -1), b[:128]


def gemm_rows(gh, gl, w, b, lost=(), nobias=False, drop_tile=False):
    """A 1x1 tc_conv (descriptor heads) on gathered split rows [R, K] -> fp32 [R, Cout]; ``drop_tile`` zeroes the last
    partial 128-row tile of the R rows."""
    wh, wl = split(w)
    acc = torch.zeros(gh.shape[0], w.shape[0], dtype=torch.float32)
    for c0 in range(0, w.shape[1], BK):
        c = slice(c0, c0 + BK)
        acc += _products(gh[:, c], gl[:, c], wh[:, c], wl[:, c], lost, "rc,oc->ro").float()
    y = _bias(acc, b, nobias, (1, -1)).double()
    if drop_tile and y.shape[0] % TILE:
        y[y.shape[0] // TILE * TILE:] = 0.0
    return y


# ------------------------------------------------------------------------------------------------------------- HardNet
def hn_conv0(sd, patches):
    """Patch normalisation and conv 0 (folded BatchNorm, ReLU) in fp32 from patches [N, 1, 32, 32] -> [N, 32, 32, 32]."""
    p = patches.float()
    sp, mp = torch.std_mean(p, dim=(1, 2, 3), keepdim=True)
    w, b = dho.folded(sd, 0, p)
    return F.relu(F.conv2d((p - mp) / (sp + 1e-6), w, b, padding=1)).double()


def framed(x):
    """An activation [N, C, h, w] as the kernels store it: the (hi, lo) pair in its padded frame, zero ring."""
    return tuple(F.pad(t, (1, 1, 1, 1)) for t in split(x))


def hn_conv(sd, li, pair, lost=(), nobias=False, phase_swap=False, ring=False):
    """HardNet conv li = 1 .. 5 (3x3, stride 1 or 2 by phase split, folded BatchNorm, ReLU) on the framed input pair
    [N, C, h + 2, w + 2] -> the framed output pair.  Its padding ring is zero, or with ``ring`` what the GEMM computes
    there."""
    w, b = dho.folded(sd, li, torch.empty(0, dtype=torch.float64))
    w = w.float()
    wh, wl = split(w)
    s = dho.STRIDES[li]
    n, _, hp, wp = pair[0].shape
    ho, wo = (hp - 2) // s, (wp - 2) // s
    xh, xl = (F.pad(t, (s, s, s, s)) for t in pair)  # frame position Y reads rows s Y + dy
    acc = torch.zeros(n, w.shape[0], ho + 2, wo + 2, dtype=torch.float32)
    for dy in range(3):
        for dx in range(3):
            if s == 1:
                ys, xs = dy, dx
            else:
                py, px = (dx & 1, dy & 1) if phase_swap else (dy & 1, dx & 1)
                ys, xs = 2 * (dy >> 1) + py, 2 * (dx >> 1) + px
            sl = (slice(None), slice(None), slice(ys, ys + s * (ho + 2), s), slice(xs, xs + s * (wo + 2), s))
            for c0 in range(0, w.shape[1], BK):
                c = slice(c0, c0 + BK)
                acc += _products(xh[sl][:, c], xl[sl][:, c], wh[:, c, dy, dx], wl[:, c, dy, dx], lost,
                                 "nchw,oc->nohw").float()
    y = F.relu(_bias(acc, b, nobias, (1, -1, 1, 1))).double()
    if not ring:
        y = F.pad(y[:, :, 1:-1, 1:-1], (1, 1, 1, 1))
    return split(y)


def hn_rows6(pair):
    """conv 6's input rows: the 8 x 8 interior of the framed conv 5 output pair, column (ky 8 + kx) 128 + ci."""
    return tuple(t[:, :, 1:-1, 1:-1].permute(0, 2, 3, 1).reshape(t.shape[0], -1) for t in pair)


def hn_weight6(sd):
    w, b = dho.folded(sd, 6, torch.empty(0, dtype=torch.float64))
    return w.float().permute(0, 2, 3, 1).reshape(128, -1), b


def hn_layers(sd, patches, defects=None):
    """The whole stack from fp32 patches: conv 0's output, the framed pairs of convs 1 .. 5 and conv 6's fp32 rows.
    ``defects``: {layer: dict of hn_conv / gemm_rows switches}."""
    defects = defects or {}
    out = [hn_conv0(sd, patches)]
    x = framed(out[0])
    for li in range(1, 6):
        x = hn_conv(sd, li, x, **defects.get(li, {}))
        out.append(x)
    w6, b6 = hn_weight6(sd)
    out.append(gemm_rows(*hn_rows6(x), w6, b6, **defects.get(6, {})))
    return out
