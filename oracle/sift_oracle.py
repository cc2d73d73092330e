"""Float64 stages of the SIFT extractor (include/sift_b200.h), written from the semantics the headers state, and the
checks of a captured workspace against them.  Test infrastructure only.

Each stage takes the kernels' own inputs read back from the workspace (``capture``: ``sift_workspace_layout`` locates
the last image's intermediates) and computes its output in float64 (torch, on the inputs' device):

* gray and 8-bit quantisation: float32 emulation, exact;  upsample x2 and decimation: exact;
* Gaussian taps: ``getGaussianKernel`` in double, rounded to float (the taps are part of the definition); separable
  blur with REFLECT_101 (repeated reflection when the kernel is wider than the image) in float64; DoG as the fp32
  difference of the Gaussians;
* extremum test (exact on the fp32 DoG) and ``adjustLocalExtrema`` with a float64 solve, returning the margin of every
  decision: the |x| < 0.5 convergence test, the rounding steps, contrast, edge and det <= 0;
* orientation: the 36-bin histogram with fastAtan2's polynomial in float64, the wrapped smoothing, the 0.8 peak rule and
  the parabolic bin, with margins for the bin rounding and the peak tests;
* ordering and filtering, exact on the raw keypoint records: KeyPoint_LessThan, removeDuplicatedSorted, retainBest,
  filter_dog_point as the reference does it (highest score per pixel, then lowest |angle|, then max-pool NMS), top-k;
* descriptor: the float64 values before rounding (after the 0.2 clip and the x512 renormalisation), then RootSIFT.

``DEFECT`` names a deliberately wrong variant of one stage; the tests use them to show that each stage check resolves
it (see tests/test_sift_layer_emulation.py)."""
from __future__ import annotations

import ctypes as C
import math
from collections import Counter

import numpy as np
import torch

F32 = np.float32
D64 = torch.float64
BORDER = 5
ORI_BINS, ORI_PEAK, DESC_W, DESC_BINS = 36, 0.8, 4, 8
DEFECTS = ("reflect", "total_sigma", "swap_xc_xr", "smooth_nowrap", "descr_rot_sign", "clip_025", "retain_gt",
           "dog_larger_angle", "nms_radius")
# fastAtan2's polynomial (OpenCV's v_atan_f32), coefficients in degrees; evaluated in float64 here
ATAN_P = tuple(c * 180 / math.pi for c in (0.9997878412794807, -0.3258083974640975, 0.1555786518463281,
                                             -0.04432655554792128))


# --------------------------------------------------------------------------------------------------------- capture
def layout(cfg, H, W, h, w):
    """sift_workspace_layout -> {"off", "bytes", "n_oct", "dims", "gauss", "dog", "total"}."""
    from lightglue_b200 import _cabi

    n, mo, L = _cabi.SIFT_LAYOUT_BUFFERS, _cabi.SIFT_LAYOUT_MAX_OCTAVES, cfg.num_octave_layers
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    n_oct, dims = C.c_int32(), (C.c_int32 * (2 * mo))()
    g, d = (C.c_int64 * (mo * (L + 3)))(), (C.c_int64 * (mo * (L + 2)))()
    total = _cabi.load().sift_workspace_layout(C.byref(cfg), H, W, h, w, off, size, C.byref(n_oct), dims, g, d)
    no = n_oct.value
    return {"off": list(off), "bytes": list(size), "n_oct": no, "dims": [(dims[2 * o], dims[2 * o + 1]) for o in range(no)],
            "gauss": [[g[o * (L + 3) + i] for i in range(L + 3)] for o in range(no)],
            "dog": [[d[o * (L + 2) + i] for i in range(L + 2)] for o in range(no)], "total": total, "L": L}


BUFFERS = ("counters", "q", "tmp", "pyr", "cand", "kpt", "order", "flags", "pix", "out_src")


def capture(ws, lay, h, w):
    """Views of a workspace (uint8 tensor starting at the carve's aligned base) by the layout: torch fp32 maps on the
    workspace's device for q / gauss / dog, numpy copies of the lists and counters."""
    from lightglue_b200 import _cabi

    def buf(name):
        i = BUFFERS.index(name)
        return ws[lay["off"][i]:lay["off"][i] + lay["bytes"][i]]

    def plane(o_bytes, hh, ww):
        return ws[o_bytes:o_bytes + 4 * hh * ww].view(torch.float32).view(hh, ww)

    cap = {"counters": buf("counters").view(torch.int32).cpu().numpy().copy()}
    cap["q"] = buf("q")[:4 * h * w].view(torch.float32).view(h, w)
    cap["gauss"] = [[plane(o, *lay["dims"][k]) for o in lay["gauss"][k]] for k in range(lay["n_oct"])]
    cap["dog"] = [[plane(o, *lay["dims"][k]) for o in lay["dog"][k]] for k in range(lay["n_oct"])]
    raw = lay["bytes"][BUFFERS.index("order")] // 4
    nc, nk = (min(int(cap["counters"][i]), raw) for i in (4, 5))
    cap["cand"] = buf("cand").cpu().numpy().view(np.dtype(_cabi.SIFT_CAND_DTYPE))[:nc].copy()
    cap["kpt"] = buf("kpt").cpu().numpy().view(np.dtype(_cabi.SIFT_KPT_DTYPE))[:nk].copy()
    for k in ("order", "flags", "pix", "out_src"):
        cap[k] = buf(k).view(torch.int32).cpu().numpy().copy()
    cap["raw_cap"] = raw
    return cap


# --------------------------------------------------------------------------------------------------------- pyramid
def gray_q(image, h, w):
    """image [C, H, W] fp32 -> the 8-bit gray crop as fp32 [h, w], float32 arithmetic as the kernels do it (exact)."""
    x = image[:, :h, :w].detach().cpu().numpy().astype(F32)
    g = x[0] if x.shape[0] == 1 else (F32(0.299) * x[0] + F32(0.587) * x[1]) + F32(0.114) * x[2]
    return torch.from_numpy((g * F32(255)).astype(np.int32).astype(np.uint8).astype(F32))


def upsample(q):
    """cv::resize 2x INTER_LINEAR (half-pixel centres, clamped ends), float64 (exact for 8-bit inputs)."""
    def taps(n):
        d = np.arange(2 * n)
        src = (d + 0.5) / 2 - 0.5
        s0 = np.floor(src).astype(int)
        a1 = src - s0
        lo, hi = np.clip(s0, 0, n - 1), np.clip(s0 + 1, 0, n - 1)
        a1 = np.where(s0 < 0, 0.0, np.where(s0 + 1 > n - 1, 0.0, a1))
        return lo, hi, 1 - a1, a1

    q = q.to(D64)
    h, w = q.shape
    ylo, yhi, ay0, ay1 = taps(h)
    xlo, xhi, ax0, ax1 = taps(w)
    t = lambda a: torch.as_tensor(a, device=q.device)  # noqa: E731
    rows = q[:, t(xlo)] * t(ax0) + q[:, t(xhi)] * t(ax1)
    return rows[t(ylo)] * t(ay0)[:, None] + rows[t(yhi)] * t(ay1)[:, None]


def gaussian_taps(sigma):
    """cv::getGaussianKernel(ksize = round(8 sigma + 1) | 1, sigma) in double, rounded to float."""
    ks = min(int(np.rint(sigma * 8 + 1)) | 1, 127)
    t = [math.exp(-0.5 / (sigma * sigma) * (i - (ks - 1) * 0.5) ** 2) for i in range(ks)]
    s = 0.0
    for v in t:
        s += v
    return np.array([v / s for v in t], dtype=F32)


def layer_sigmas(L, defect=None):
    """(initial blur sigma, [sigma of layer i from layer i - 1 for i in 1 .. L + 2]): sigma 1.6 as float, the initial
    blur in float arithmetic, the incremental sigmas in double."""
    s = F32(1.6)
    sig0 = float(np.sqrt(np.maximum(s * s - F32(1.0), F32(0.01))))
    k = 2.0 ** (1.0 / L)
    out = []
    for i in range(1, L + 3):
        prev = k ** (i - 1) * float(s)
        total = prev * k
        out.append(total if defect == "total_sigma" else math.sqrt(total * total - prev * prev))
    return sig0, out


def reflect(p, n, defect=None):
    """cv::borderInterpolate for BORDER_REFLECT_101 (REFLECT with defect "reflect"), repeated for wide kernels."""
    if n == 1:
        return np.zeros_like(p)
    p = p.copy()
    while True:
        bad = (p < 0) | (p >= n)
        if not bad.any():
            return p
        if defect == "reflect":
            p = np.where(p < 0, -p - 1, np.where(p >= n, 2 * n - 1 - p, p))
        else:
            p = np.where(p < 0, -p, np.where(p >= n, 2 * n - 2 - p, p))


def blur(img, taps, defect=None):
    """Separable Gaussian blur of img [h, w] with the fp32 taps, REFLECT_101, float64."""
    img = img.to(D64)
    h, w = img.shape
    ks, r = len(taps), len(taps) // 2
    k = [float(v) for v in taps]
    dev = img.device
    ix = torch.as_tensor(reflect(np.arange(w)[:, None] - r + np.arange(ks)[None], w, defect), device=dev)
    iy = torch.as_tensor(reflect(np.arange(h)[:, None] - r + np.arange(ks)[None], h, defect), device=dev)
    row = torch.zeros_like(img)
    for t in range(ks):
        row += k[t] * img[:, ix[:, t]]
    out = torch.zeros_like(img)
    for t in range(ks):
        out += k[t] * row[iy[:, t]]
    return out


def multiple_reflection(h, w, L):
    """True when some blur of an octave of size h x w reads past a border by more than the octave's size (the border
    is reflected more than once)."""
    sig0, sig = layer_sigmas(L)
    r = max(len(gaussian_taps(s)) // 2 for s in [sig0] + sig)
    return r > min(h, w) - 1


# -------------------------------------------------------------------------------------------------------- detection
def _half_dist(x):
    """Distance of x to the nearest half-integer (where round-half-even changes its result)."""
    return (x - (torch.floor(x) + 0.5)).abs()


def candidates(dogs, o, L, contrast, edge, threshold, defect=None):
    """3x3x3 extrema of DoG layers 1..L of one octave (exact on the fp32 DoG), refined by adjustLocalExtrema in float64.

    -> dict of per-extremum tensors: alive, o, layer, r, c (final), x, y, size, response (cv::KeyPoint before the
    first-octave halving), m_x (smallest margin of the |x| < 0.5 tests and the rounding steps, in octave pixels) and
    m_rel (smallest relative margin of the contrast, edge and det tests)."""
    D = torch.stack([d.to(D64) for d in dogs])  # [L + 2, h, w]
    _, h, w = D.shape
    dev = D.device
    empty = {k: torch.zeros(0, device=dev) for k in ("x", "y", "size", "response", "m_x", "m_rel")}
    empty.update({k: torch.zeros(0, dtype=torch.long, device=dev) for k in ("o", "layer", "r", "c")})
    empty["alive"] = torch.zeros(0, dtype=torch.bool, device=dev)
    if h - 2 * BORDER <= 0 or w - 2 * BORDER <= 0:
        return empty
    found = []
    for layer in range(1, L + 1):
        val = D[layer, BORDER:h - BORDER, BORDER:w - BORDER]
        ok = val.abs() > threshold
        pos, neg = ok & (val > 0), ok & ~(val > 0)
        for s in (layer - 1, layer, layer + 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    nb = D[s, BORDER + dy:h - BORDER + dy, BORDER + dx:w - BORDER + dx]
                    pos &= val >= nb
                    neg &= val <= nb
        rr, cc = torch.nonzero(pos | neg, as_tuple=True)
        found.append(torch.stack([torch.full_like(rr, layer), rr + BORDER, cc + BORDER], 1))
    lrc = torch.cat(found)
    n = lrc.shape[0]
    if n == 0:
        return empty
    lay, r, c = lrc[:, 0].clone(), lrc[:, 1].clone(), lrc[:, 2].clone()
    alive = torch.ones(n, dtype=torch.bool, device=dev)
    done = torch.zeros(n, dtype=torch.bool, device=dev)
    m_x = torch.full((n,), math.inf, dtype=D64, device=dev)
    X = torch.zeros(n, 3, dtype=D64, device=dev)

    def at(s, dy, dx):
        return D[lay + s, r + dy, c + dx]

    def derivs():
        v2 = at(0, 0, 0) * 2
        g = torch.stack([at(0, 0, 1) - at(0, 0, -1), at(0, 1, 0) - at(0, -1, 0), at(1, 0, 0) - at(-1, 0, 0)], 1) * 0.5
        dxx, dyy, dss = at(0, 0, 1) + at(0, 0, -1) - v2, at(0, 1, 0) + at(0, -1, 0) - v2, at(1, 0, 0) + at(-1, 0, 0) - v2
        dxy = (at(0, 1, 1) - at(0, 1, -1) - at(0, -1, 1) + at(0, -1, -1)) * 0.25
        dxs = (at(1, 0, 1) - at(1, 0, -1) - at(-1, 0, 1) + at(-1, 0, -1)) * 0.25
        dys = (at(1, 1, 0) - at(1, -1, 0) - at(-1, 1, 0) + at(-1, -1, 0)) * 0.25
        Hm = torch.stack([torch.stack([dxx, dxy, dxs], 1), torch.stack([dxy, dyy, dys], 1),
                          torch.stack([dxs, dys, dss], 1)], 1)
        return g / 255, Hm / 255, dxx / 255, dyy / 255, dxy / 255

    for _ in range(5):
        act = alive & ~done
        if not bool(act.any()):
            break
        g, Hm, *_ = derivs()
        det = torch.linalg.det(Hm)
        sol = torch.zeros_like(g)
        nz = det != 0
        sol[nz] = torch.linalg.solve(Hm[nz], g[nz].unsqueeze(-1)).squeeze(-1)
        xn = -sol[:, [2, 1, 0]]  # (xi, xr, xc)
        if defect == "swap_xc_xr":
            xn = xn[:, [0, 2, 1]]
        X = torch.where(act[:, None], xn, X)
        mx = X.abs().amax(1)
        m_x = torch.where(act, torch.minimum(m_x, (mx - 0.5).abs()), m_x)
        conv = act & (mx < 0.5)
        done |= conv
        mv = act & ~conv
        m_x = torch.where(mv, torch.minimum(m_x, _half_dist(X).amin(1)), m_x)
        step = torch.round(X).long()
        lay = torch.where(mv, lay + step[:, 0], lay)
        r = torch.where(mv, r + step[:, 1], r)
        c = torch.where(mv, c + step[:, 2], c)
        out = (lay < 1) | (lay > L) | (c < BORDER) | (c >= w - BORDER) | (r < BORDER) | (r >= h - BORDER)
        alive &= ~(mv & out)
        lay, r, c = torch.where(alive, lay, 1), torch.where(alive, r, BORDER), torch.where(alive, c, BORDER)
    alive &= done
    g, _, dxx, dyy, dxy = derivs()
    xi, xr, xc = X[:, 0], X[:, 1], X[:, 2]
    contr = at(0, 0, 0) / 255 + (g * X[:, [2, 1, 0]]).sum(1) * 0.5
    tr, det = dxx + dyy, dxx * dyy - dxy * dxy
    s_con = (contr.abs() * L - contrast) / contrast  # >= 0: passes
    lhs, rhs = tr * tr * edge, (edge + 1) ** 2 * det
    s_edge = (rhs - lhs) / torch.maximum(lhs.abs(), rhs.abs()).clamp_min(1e-300)  # > 0: passes
    s_det = det / ((dxx * dyy).abs() + dxy * dxy).clamp_min(1e-300)  # > 0: passes
    terms = torch.stack([s_con, s_edge, s_det], 1)
    passed = (s_con >= 0) & (s_edge > 0) & (s_det > 0)
    # margin of the conjunction: the smallest true term if it holds, the largest false term's size if not
    m_rel = torch.where(passed, terms.abs().amin(1), torch.where(terms <= 0, terms.abs(), torch.zeros_like(terms)).amax(1))
    m_rel = torch.where(done, m_rel, torch.full_like(m_rel, math.inf))
    alive &= passed
    sc = float(1 << o)
    return {"alive": alive, "o": torch.full_like(lay, o), "layer": lay, "r": r, "c": c, "x": (c + xc) * sc,
            "y": (r + xr) * sc, "size": 1.6 * torch.pow(2.0, (lay + xi) / L) * sc * 2, "response": contr.abs(),
            "m_x": m_x, "m_rel": m_rel}


# ------------------------------------------------------------------------------------------------------ orientation
def fast_atan2(y, x):
    """fastAtan2's polynomial in degrees, [0, 360), evaluated in float64."""
    ax, ay = x.abs(), y.abs()
    cc_ = torch.minimum(ax, ay) / (torch.maximum(ax, ay) + float(F32(np.finfo(np.float64).eps)))
    c2 = cc_ * cc_
    a = (((ATAN_P[3] * c2 + ATAN_P[2]) * c2 + ATAN_P[1]) * c2 + ATAN_P[0]) * cc_
    a = torch.where(ax >= ay, a, 90.0 - a)
    a = torch.where(x < 0, 180.0 - a, a)
    return torch.where(y < 0, 360.0 - a, a)


def _window(R, dev):
    a = torch.arange(-R, R + 1, device=dev)
    return a[:, None].expand(-1, 2 * R + 1).reshape(-1), a[None, :].expand(2 * R + 1, -1).reshape(-1)


def orientations(img, r, c, scl_octv, defect=None):
    """calcOrientationHist + the peak loop for keypoints at (r, c) of one Gaussian layer img [rows, cols] with octave
    scale scl_octv (float64 tensors of one radius group) -> (angles: list of float lists, m_bin: smallest distance of a
    sample's bin to a rounding step, m_peak: smallest relative margin of a peak decision, wrap: a peak at bin 0 or 35)."""
    img = img.to(D64)
    rows, cols = img.shape
    dev = img.device
    n, K = ORI_BINS, r.shape[0]
    radius = torch.round(4.5 * scl_octv).long()
    R = int(radius.max())
    a, j = _window(R, dev)
    y, x = r[:, None] + a[None], c[:, None] + j[None]
    ok = (a[None].abs() <= radius[:, None]) & (j[None].abs() <= radius[:, None])
    ok &= (y > 0) & (y < rows - 1) & (x > 0) & (x < cols - 1)
    yc, xc = y.clamp(1, rows - 2), x.clamp(1, cols - 2)
    dx = img[yc, xc + 1] - img[yc, xc - 1]
    dy = img[yc - 1, xc] - img[yc + 1, xc]
    sig = 1.5 * scl_octv
    wt = torch.exp((a * a + j * j)[None].to(D64) * (-1.0 / (2 * sig * sig))[:, None])
    ori = fast_atan2(dy, dx)
    fb = ori * (n / 360.0)
    m_bin = torch.where(ok, _half_dist(fb), torch.full_like(fb, math.inf)).amin(1)
    b = torch.round(fb).long() % n
    th = torch.zeros(K, n, dtype=D64, device=dev)
    th.scatter_add_(1, b, torch.where(ok, wt * torch.sqrt(dx * dx + dy * dy), torch.zeros_like(wt)))
    if defect == "smooth_nowrap":
        z = torch.zeros(K, 2, dtype=D64, device=dev)
        ext = torch.cat([z, th, z], 1)
    else:
        ext = torch.cat([th[:, -2:], th, th[:, :2]], 1)
    hist = (ext[:, :-4] + ext[:, 4:]) / 16 + (ext[:, 1:-3] + ext[:, 3:-1]) * (4 / 16) + ext[:, 2:-2] * (6 / 16)
    omax = hist.amax(1, keepdim=True).clamp_min(1e-300)
    hl, hr = hist.roll(1, 1), hist.roll(-1, 1)
    terms = torch.stack([hist - hl, hist - hr, hist - ORI_PEAK * omax], 2) / omax[..., None]
    peak = (terms[..., 0] > 0) & (terms[..., 1] > 0) & (terms[..., 2] >= 0)
    margin = torch.where(peak, terms.abs().amin(2), torch.where(terms < 0, terms.abs(), torch.zeros_like(terms)).amax(2))
    m_peak = margin.amin(1)
    binf = torch.arange(n, device=dev, dtype=D64)[None] + 0.5 * (hl - hr) / (hl - 2 * hist + hr)
    binf = torch.where(binf < 0, binf + n, torch.where(binf >= n, binf - n, binf))
    ang = 360.0 - (360.0 / n) * binf
    ang = torch.where((ang - 360.0).abs() < float(np.finfo(F32).eps), torch.zeros_like(ang), ang)
    angles = [ang[k][peak[k]].tolist() for k in range(K)]
    wrap = bool((peak[:, 0] | peak[:, n - 1]).any())
    return angles, m_bin, m_peak, wrap


# ------------------------------------------------------------------------------------------ ordering and filtering
def lex_order(k):
    """KeyPoint_LessThan over raw records k (x, y asc, size desc, angle asc, response desc, octave desc, index)."""
    idx = np.arange(len(k))
    return np.lexsort((idx, -k["octave_packed"].astype(np.int64), -k["response"].astype(np.float64), k["angle"],
                       -k["size"].astype(np.float64), k["y"], k["x"]))


def pixels(s):
    """filter_dog_point's pixel of records s: np.round(pt - 0.5) on float32, half to even -> (row, column)."""
    return np.rint(s["y"] - F32(0.5)).astype(np.int64), np.rint(s["x"] - F32(0.5)).astype(np.int64)


def retain(s, nfeatures, defect=None):
    """removeDuplicatedSorted + retainBest(nfeatures) on records s in lexicographic order -> (unique, kept, cut)."""
    n = len(s)
    same = np.zeros(n, bool)
    if n > 1:
        same[1:] = (s["x"][1:] == s["x"][:-1]) & (s["y"][1:] == s["y"][:-1]) & (s["size"][1:] == s["size"][:-1]) & (
            s["angle"][1:] == s["angle"][:-1])
    uniq = ~same
    resp = s["response"].astype(np.float64)
    cut = nfeatures > 0 and int(uniq.sum()) > nfeatures
    keep = uniq.copy()
    if cut:
        thr = np.sort(resp[uniq])[::-1][nfeatures - 1]
        keep &= (resp > thr) if defect == "retain_gt" else (resp >= thr)
    return uniq, keep, cut


def dog_filter(s, keep, w, defect=None):
    """filter_dog_point's duplicate removal among the kept records: the highest score per pixel, then the lowest
    |angle| (radians, float32 as np.deg2rad gives it); ties are all kept."""
    pi, pj = pixels(s)
    pix = pi * w + pj
    resp = s["response"].astype(np.float64)
    oabs = np.abs(s["angle"].astype(F32) * (F32(np.pi) / F32(180))).astype(np.float64)
    best, pick = {}, {}
    for i in np.nonzero(keep)[0]:
        best[pix[i]] = max(best.get(pix[i], -np.inf), resp[i])
    dup = keep & np.array([resp[i] == best.get(pix[i]) for i in range(len(s))], bool)
    for i in np.nonzero(dup)[0]:
        v = pick.get(pix[i])
        pick[pix[i]] = oabs[i] if v is None else (max(v, oabs[i]) if defect == "dog_larger_angle" else min(v, oabs[i]))
    return dup & np.array([oabs[i] == pick.get(pix[i]) for i in range(len(s))], bool)


def nms(s, dup, radius, defect=None):
    """filter_dog_point's max-pool NMS (radius > 0) over the surviving pixels' scores: a record survives unless one
    within Chebyshev distance `radius` (in pixels) has a higher score."""
    if radius <= 0:
        return dup.copy()
    rad = radius + (1 if defect == "nms_radius" else 0)
    pi, pj = pixels(s)
    resp = s["response"].astype(np.float64)
    live = np.nonzero(dup)[0]
    out = dup.copy()
    for i in live:
        near = live[(np.abs(pi[live] - pi[i]) <= rad) & (np.abs(pj[live] - pj[i]) <= rad)]
        out[i] = not (resp[near] > resp[i]).any()
    return out


def select(s, alive_mask, cut, max_kpts):
    """Top-k and output order -> (lexicographic positions of the output rows, top-k applied): descending score with
    ties in lexicographic order when the nfeatures cut or the top-k applied, lexicographic order otherwise."""
    alive = np.nonzero(alive_mask)[0]
    topk = len(alive) > max_kpts
    if topk or cut:
        alive = alive[np.lexsort((alive, -s["response"][alive].astype(np.float64)))]
    return alive[:max_kpts], topk


# -------------------------------------------------------------------------------------------------------- descriptor
def descriptors(img, kp, defect=None):
    """calcSIFTDescriptor for raw records kp (one octave and layer, equal window radius) on img [rows, cols] -> float64
    [K, 128], the values before uint8 rounding; and whether a window crosses the image border."""
    img = img.to(D64)
    rows, cols = img.shape
    dev = img.device
    d, n = DESC_W, DESC_BINS
    o = int(kp["o"][0])
    scale = 2.0 ** (1 - o)
    size, ptx, pty = (torch.as_tensor(kp[f].astype(np.float64), device=dev) * scale for f in ("size", "x", "y"))
    ang = 360.0 - torch.as_tensor(kp["angle"].astype(np.float64), device=dev)
    ang = torch.where((ang - 360.0).abs() < float(np.finfo(F32).eps), torch.zeros_like(ang), ang)
    px, py = torch.round(ptx).long(), torch.round(pty).long()
    hw = 3.0 * size * 0.5
    radius = torch.round(hw * math.sqrt(2) * (d + 1) * 0.5).long().clamp_max(int(math.sqrt(cols * cols + rows * rows)))
    R = int(radius.max())
    cos_t, sin_t = torch.cos(ang * math.pi / 180) / hw, torch.sin(ang * math.pi / 180) / hw
    i, j = _window(R, dev)
    i, j = i[None].to(D64), j[None].to(D64)
    if defect == "descr_rot_sign":
        sin_t = -sin_t
    c_rot = j * cos_t[:, None] - i * sin_t[:, None]
    r_rot = j * sin_t[:, None] + i * cos_t[:, None]
    rbin, cbin = r_rot + d / 2 - 0.5, c_rot + d / 2 - 0.5
    rr, cc = py[:, None] + i.long(), px[:, None] + j.long()
    inwin = (i.abs() <= radius[:, None]) & (j.abs() <= radius[:, None])
    ok = inwin & (rbin > -1) & (rbin < d) & (cbin > -1) & (cbin < d)
    clipped = bool((ok & ~((rr > 0) & (rr < rows - 1) & (cc > 0) & (cc < cols - 1))).any())
    ok &= (rr > 0) & (rr < rows - 1) & (cc > 0) & (cc < cols - 1)
    yc, xc = rr.clamp(1, rows - 2), cc.clamp(1, cols - 2)
    dx = img[yc, xc + 1] - img[yc, xc - 1]
    dy = img[yc - 1, xc] - img[yc + 1, xc]
    mag = torch.sqrt(dx * dx + dy * dy) * torch.exp((c_rot * c_rot + r_rot * r_rot) * (-1.0 / (d * d * 0.5)))
    mag = torch.where(ok, mag, torch.zeros_like(mag))
    obin = (fast_atan2(dy, dx) - ang[:, None]) * (n / 360.0)
    r0, c0, o0 = torch.floor(rbin), torch.floor(cbin), torch.floor(obin)
    fr, fc, fo = rbin - r0, cbin - c0, obin - o0
    K = len(kp)
    hist = torch.zeros(K, (d + 2) * (d + 2) * n, dtype=D64, device=dev)
    for dr in (0, 1):
        for dc in (0, 1):
            for do in (0, 1):
                wgt = mag * (fr if dr else 1 - fr) * (fc if dc else 1 - fc) * (fo if do else 1 - fo)
                cell = ((r0.long() + 1 + dr).clamp(0, d + 1) * (d + 2) + (c0.long() + 1 + dc).clamp(0, d + 1)) * n
                hist.scatter_add_(1, cell + (o0.long() + do) % n, wgt)
    v = hist.view(K, d + 2, d + 2, n)[:, 1:d + 1, 1:d + 1].reshape(K, d * d * n)
    thr = v.norm(dim=1, keepdim=True) * (0.25 if defect == "clip_025" else 0.2)
    v = torch.minimum(v, thr)
    v = v * (512.0 / v.norm(dim=1, keepdim=True).clamp_min(float(np.finfo(F32).eps)))
    return v, clipped


def rootsift(q):
    """sift_to_rootsift in float64 on the uint8-valued descriptors q [K, 128]."""
    x = q.to(D64)
    x = x / x.abs().sum(1, keepdim=True).clamp_min(1e-6)
    x = x.clamp_min(1e-6).sqrt()
    return x / x.norm(dim=1, keepdim=True).clamp_min(1e-6)


def recover_q(d):
    """The uint8 descriptors behind RootSIFT rows d [K, 128], up to a common factor per row.  d^2 is q / |q|_1 up to a
    final normalisation within 128e-6 of 1, and zeros sit at the 1e-6 clip, so q = d^2 / m * q_min with m the smallest
    d^2 of a nonzero entry.  RootSIFT is the same for q and g q, so d only gives q / gcd(q): this returns the row with
    the smallest q_min in 1 .. 255 that makes every entry an integer (zeros round back to 0), and -1 where none does."""
    d2 = d.to(D64) ** 2
    nz = d2 > 1e-5  # a zero entry gives about 1e-6, a nonzero one at least 1 / (128 * 255)
    m = torch.where(nz, d2, torch.full_like(d2, math.inf)).amin(1, keepdim=True)
    q = torch.full_like(d2, -1.0)
    for qmin in range(255, 0, -1):
        t = torch.where(nz, d2 / m * qmin, torch.zeros_like(d2))
        fit = ((t - torch.round(t)).abs() < 0.05).all(1, keepdim=True) & (t <= 255.5).all(1, keepdim=True)
        q = torch.where(fit, torch.round(t), q)
    return q


def nearest_multiple(q0, v):
    """The multiple g q0 (g = 1, 2, ... while every entry stays <= 255) of each primitive row q0 [K, 128] that is
    nearest the float64 descriptor values v in max |g q0 - min(v, 255)|."""
    vc = v.clamp_max(255)
    top = q0.amax(1, keepdim=True).clamp_min(1)
    best, err = q0.clone(), (q0 - vc).abs().amax(1, keepdim=True)
    for g in range(2, 256):
        cand = q0 * g
        e = (cand - vc).abs().amax(1, keepdim=True)
        better = (e < err) & (top * g <= 255)
        best, err = torch.where(better, cand, best), torch.where(better, e, err)
    return best


# -------------------------------------------------------------------------------------------------- stage checks
def _rel(a, ref):
    return float((a.to(D64) - ref).abs().max() / ref.abs().max().clamp_min(1e-300)) if a.numel() else 0.0


def check_stages(cap, conf, image, h, w, tol, defect=None, skip_pyramid=False):
    """Every stage check of one captured image -> (errs {stage: deviation}, fails [stage names], info).

    conf: the extractor conf; image [C, H, W] fp32; (h, w) its crop.  A stage fails when its deviation exceeds tol or
    an exact comparison differs; info holds the regimes the image reached and the counts of undecided items."""
    L = int(conf["num_octaves"])
    contrast, edge = float(F32(conf["detection_threshold"])), float(F32(conf["edge_threshold"]))
    threshold = math.floor(0.5 * conf["detection_threshold"] / L * 255)
    max_kpts = int(conf["max_num_keypoints"])
    nms_radius = -1 if conf["nms_radius"] is None else int(conf["nms_radius"])
    errs, fails, info = {}, [], {}

    def err(stage, e, t):
        errs[stage] = max(errs.get(stage, 0.0), e)
        if not e <= t and stage not in fails:
            fails.append(stage)

    def exact(stage, ok):
        errs.setdefault(stage, 0.0)
        if not ok and stage not in fails:
            fails.append(stage)

    q = cap["q"]
    G, Dg = cap["gauss"], cap["dog"]
    n_oct = len(G)
    dev = q.device
    # ---- pyramid
    exact("q", torch.equal(q.cpu(), gray_q(image, h, w)))
    sig0, sig = layer_sigmas(L, defect)
    info["multi_reflect"] = any(multiple_reflection(*G[o][0].shape, L) for o in range(n_oct))
    if not skip_pyramid:
        err("gauss0", _rel(G[0][0], blur(upsample(q.to(D64)), gaussian_taps(sig0), defect)), tol["gauss"])
        for o in range(n_oct):
            if o > 0:
                exact("decimate", torch.equal(G[o][0], G[o - 1][L][::2, ::2][:G[o][0].shape[0], :G[o][0].shape[1]]))
            for i in range(1, L + 3):
                err("gauss", _rel(G[o][i], blur(G[o][i - 1], gaussian_taps(sig[i - 1]), defect)), tol["gauss"])
                exact("dog", torch.equal(Dg[o][i - 1], G[o][i] - G[o][i - 1]))
    # ---- candidates
    cand = cap["cand"]
    ov = cap["counters"]
    info["overflow"] = bool(ov[3])
    key = lambda o, l, r, c: (int(o), int(l), int(r), int(c))  # noqa: E731
    got = Counter(key(k["octave_packed"] & 255, k["layer"], k["r"], k["c"]) for k in cand)
    want, n_und, vals = Counter(), 0, {}
    for o in range(n_oct):
        cd = candidates(Dg[o], o, L, contrast, edge, threshold, defect)
        und = (cd["m_x"] < tol["cand_margin_x"]) | (cd["m_rel"] < tol["cand_margin_rel"])
        n_und += int(und.sum())
        sel = cd["alive"] & ~und
        for idx in torch.nonzero(sel).flatten().tolist():
            k = key(o, cd["layer"][idx], cd["r"][idx], cd["c"][idx])
            want[k] += 1
            vals[k] = tuple(float(cd[f][idx]) for f in ("x", "y", "size", "response"))
    # excluded: captured candidates outside the decided set (each needs an undecided extremum to account for it)
    info["cand_undecided"], info["cand_total"] = n_und, len(cand)
    info["cand_excluded"] = sum((got - want).values())
    if not info["overflow"]:
        exact("cand", not (want - got) and info["cand_excluded"] <= n_und)
        dx = ds = dr = 0.0
        for k in cand:
            kk = key(k["octave_packed"] & 255, k["layer"], k["r"], k["c"])
            if kk in vals:
                x, y, s, rsp = vals[kk]
                sc = float(1 << kk[0])
                dx = max(dx, abs(k["x"] - x) / sc, abs(k["y"] - y) / sc)
                ds, dr = max(ds, abs(k["size"] / s - 1)), max(dr, abs(k["response"] / rsp - 1))
        err("cand", dx, tol["cand_xy"])
        err("cand", ds, tol["cand_size"])
        err("cand", dr, tol["cand_response"])
    # ---- orientations: raw keypoints grouped by their candidate
    kpt = cap["kpt"]
    if not info["overflow"] and len(cand):
        by_key = {}
        for k in kpt:
            kk = (float(k["x"]), float(k["y"]), float(k["size"]), float(k["response"]), int(k["o"]), int(k["layer"]))
            by_key.setdefault(kk, []).append(float(k["angle"]))
        ck = [(float(F32(c["x"]) * F32(0.5)), float(F32(c["y"]) * F32(0.5)), float(F32(c["size"]) * F32(0.5)),
               float(c["response"]), int(c["octave_packed"] & 255), int(c["layer"])) for c in cand]
        mult = Counter(ck)
        dang, n_und_o, wrap, ok_all = 0.0, 0, False, True
        groups = {}
        for i, c in enumerate(cand):
            groups.setdefault((int(c["octave_packed"] & 255), int(c["layer"])), []).append(i)
        for (o, layer), idx in groups.items():
            sub = cand[idx]
            t = lambda a: torch.as_tensor(a, device=dev)  # noqa: E731
            scl = t((sub["size"].astype(F32) * F32(0.5) / F32(1 << o)).astype(np.float64))
            angs, m_bin, m_peak, wr = orientations(G[o][layer], t(sub["r"].astype(np.int64)), t(sub["c"].astype(np.int64)),
                                                   scl, defect)
            und = ((m_bin < tol["ori_margin_bin"]) | (m_peak < tol["ori_margin_peak"])).tolist()
            rad_und = np.abs(4.5 * scl.cpu().numpy() - np.floor(4.5 * scl.cpu().numpy()) - 0.5) < 1e-5
            for m, i in enumerate(idx):
                if und[m] or rad_und[m]:
                    n_und_o += 1
                    continue
                kk = ck[i]
                gs = sorted(by_key.get(kk, []))
                ws_ = sorted(angs[m] * mult[kk])
                if len(gs) != len(ws_):
                    ok_all = False
                    continue
                for a, b in zip(gs, ws_):
                    dang = max(dang, abs((a - b + 180.0) % 360.0 - 180.0))
            wrap |= wr
        info["ori_undecided"], info["wrap_peak"] = n_und_o, wrap
        exact("orient", ok_all)
        err("orient", dang, tol["ori_angle"])
    # ---- ordering and filtering, exact on the captured raw records
    n = int(ov[0])
    exact("counters", n == min(int(ov[5]), cap["raw_cap"]) and bool(ov[3]) == (int(ov[5]) > cap["raw_cap"] or
                                                                          int(ov[4]) > cap["raw_cap"]))
    k = kpt[:n]
    exact("order", np.array_equal(cap["order"][:n], lex_order(k)))
    order = cap["order"][:n]
    s = k[order]
    fl = cap["flags"][:n]
    pi, pj = pixels(s)
    exact("pix", np.array_equal(cap["pix"][:n], pi * w + pj))
    uniq, keep, cut = retain(s, max_kpts, defect)
    exact("retain", np.array_equal(fl & 1, uniq * 1) and np.array_equal(fl & 2, keep * 2) and bool(ov[1]) == cut)
    if nms_radius >= 0:
        dup = dog_filter(s, (fl & 2) > 0, w, defect)
    else:
        dup = (fl & 2) > 0
    exact("dogfilter", np.array_equal(fl & 4, dup * 4))
    alive = nms(s, (fl & 4) > 0, nms_radius, defect)
    exact("nms", np.array_equal(fl & 8, alive * 8))
    out, topk = select(s, (fl & 8) > 0, bool(ov[1]), max_kpts)
    n_out = int(ov[2])
    exact("select", n_out == len(out) and np.array_equal(cap["out_src"][:n_out], out))
    info["cut"] = cut
    info["cut_tie"] = cut and int(keep.sum()) > max_kpts
    dup_pairs = Counter((int(p), float(r)) for p, r, f in zip(pi * w + pj, s["response"], fl) if f & 2)
    info["pixel_dup_equal"] = any(v > 1 for v in dup_pairs.values())
    info["nms_suppression"] = bool(((fl & 4) > 0).sum() > ((fl & 8) > 0).sum())
    info["topk"] = topk
    info["n_out"] = n_out
    return errs, fails, info, (k, order)


def check_outputs(cap, conf, out, tol, defect, sel, errs, fails, info):
    """Output rows and descriptors of one captured image.  out: this image's rows as numpy (keypoints [cap, 2], scales,
    oris, scores, descriptors [cap, 128], count); sel: check_stages' (raw records, order, filter state)."""
    k, order = sel
    G = cap["gauss"]
    dev = G[0][0].device
    n_out = int(cap["counters"][2])

    def err(stage, e, t):
        errs[stage] = max(errs.get(stage, 0.0), e)
        if not e <= t and stage not in fails:
            fails.append(stage)

    def exact(stage, ok):
        errs.setdefault(stage, 0.0)
        if not ok and stage not in fails:
            fails.append(stage)

    want_count = -1 if cap["counters"][3] else n_out
    info["count"] = int(out["count"])
    exact("counts", int(out["count"]) == want_count)
    if cap["counters"][3]:
        return
    rows = k[order[cap["out_src"][:n_out]]] if n_out else k[:0]
    exact("rows", np.array_equal(out["keypoints"][:n_out, 0], rows["x"]) and np.array_equal(
        out["keypoints"][:n_out, 1], rows["y"]) and np.array_equal(out["scales"][:n_out], rows["size"]) and np.array_equal(
        out["scores"][:n_out], rows["response"]) and np.array_equal(
        out["oris"][:n_out], (rows["angle"].astype(F32) * F32(np.float32(math.pi) / F32(180))).astype(F32)))
    exact("rows", not out["keypoints"][n_out:].any() and not out["descriptors"][n_out:].any())
    if not n_out:
        return
    desc = torch.as_tensor(out["descriptors"][:n_out], device=dev)
    dq, dv, dr, n_half, sat, clipped = 0.0, 0.0, 0.0, 0, False, False
    groups = {}
    for m in range(n_out):
        groups.setdefault((int(rows["o"][m]), int(rows["layer"][m])), []).append(m)
    for (o, layer), idx in groups.items():
        v, cl = descriptors(G[o][layer], rows[idx], defect)
        clipped |= cl
        d = desc[idx]
        q = d.to(D64)
        if conf["rootsift"]:  # RootSIFT from the primitive row; the descriptor check takes the multiple nearest v
            q0 = recover_q(d)
            exact("rootsift", bool((q0 >= 0).all()))
            dr = max(dr, float((rootsift(q0) - d.to(D64)).abs().max()))
            q = nearest_multiple(q0, v)
        exact("descriptor", bool(((q >= 0) & (q <= 255) & (q == torch.round(q))).all()))
        dq = max(dq, float((q - v.clamp_max(255)).abs().max()))
        far = _half_dist(v) > tol["desc_half"]
        n_half += int((~far).sum())
        exact("descriptor", bool((q[far & (v < 255)] == torch.round(v[far & (v < 255)])).all()))
        exact("descriptor", bool((q[v >= 255 + tol["desc_half"]] == 255).all()))
        sat |= bool((v >= 255).any())
    err("descriptor", max(dq - 0.5, 0.0), tol["desc_abs"])
    err("rootsift", dr, tol["rootsift"])
    info["desc_border_clip"], info["desc_saturated"], info["desc_near_half"] = clipped, sat, n_half
