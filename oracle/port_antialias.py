"""fp64 restatement of crop generation at antialias factors 5..16 (warp_crops_aa_kernel in metrabs_b200/csrc/multiperson.cuh),
written from the reference's `_get_crops` (metrabs_pytorch/multiperson/multiperson_model.py:295-318): the res*f render of
port_multiperson (source_coords + sample), shrunk by torchvision's resize(BILINEAR, antialias=True), which is
F.interpolate(mode='bilinear', align_corners=False, antialias=True), then the gamma.  With a per-element error bound for
the fp32 kernel.  Plain torch in float64; imports nothing from the reference, so GPU tests can use it.

The resize, per axis from n_in = res * f to res (ATen's _compute_weights_aa with scale and support f): output i takes
the taps j in [lo, lo + n), lo = max(int(c - f + 0.5), 0), lo + n = min(int(c + f + 0.5), n_in), c = f (i + 0.5), with
weight max(0, 1 - |j - c + 0.5| / f), renormalised over the taps that remain inside [0, n_in)."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import port_multiperson as pm

F64 = torch.float64
U32 = pm.U32
MAX_FACTOR = 16


def golden_frames(n=2, h=360, w=640):
    """uint8 [n,3,h,w] frames of the antialias goldens (oracle/gen_golden_antialias.py): per channel the sum of two
    triangle waves along oblique directions, at most 5 grey levels per pixel, in 16..246: no black, where the gamma
    encoding x ** (gamma / 2.2) would magnify last-bit differences of the linear crops without bound.  Integer arithmetic
    only, so every host regenerates them bit for bit and the goldens need not store them."""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    out = np.empty((n, 3, h, w), np.uint8)
    for i in range(n):
        for c in range(3):
            k = 3 * i + c
            t1 = x * (1 + k % 3) + y * (2 + k % 2) + 37 * k
            t2 = x * (3 - k % 2) - y * (1 + k % 3) + 4 * w + 91 * k
            p1, p2 = 170 + 23 * k, 130 + 17 * k
            v1 = np.abs(t1 % (2 * p1) - p1) * 130 // p1
            v2 = np.abs(t2 % (2 * p2) - p2) * 100 // p2
            out[i, c] = (16 + v1 + v2).astype(np.uint8)
    return torch.from_numpy(out)


def aa_matrix(n_in, n_out, device=None):
    """[n_out, n_in] fp64 weights of the antialiased bilinear shrink along one axis (scale n_in / n_out >= 1)."""
    f = n_in / n_out
    i = torch.arange(n_out, dtype=F64, device=device)
    c = f * (i + 0.5)
    lo = torch.clamp((c - f + 0.5).trunc(), min=0)
    hi = torch.clamp((c + f + 0.5).trunc(), max=n_in)
    j = torch.arange(n_in, dtype=F64, device=device)
    w = torch.clamp(1 - (j[None] - c[:, None] + 0.5).abs() / f, min=0)
    w = torch.where((j[None] >= lo[:, None]) & (j[None] < hi[:, None]), w, torch.zeros_like(w))
    return w / w.sum(1, keepdim=True)


def shrink(img, res):
    """[..., H, W] -> [..., res, res]: the width pass, then the height pass."""
    wx = aa_matrix(img.shape[-1], res, img.device)
    wy = aa_matrix(img.shape[-2], res, img.device)
    return wy @ (img.to(F64) @ wx.T)


def support_max(x, f):
    """Per output element of shrink(): the largest of x [C,H,W] over a window that covers its taps in both axes."""
    return F.max_pool2d(x[None], 3 * f, f, padding=f)[0]


def warp(levels, K_box, invproj, dist_box, crop_levels, gamma_exp, res, image_ids, num_aug, af, with_bound=False,
         invproj_err=None):
    """All num_aug * n crops at antialias factor af in 5..16, as port_multiperson.warp (same arguments and results) with
    the antialiased resize in place of avg_pool2d.

    bound: per output element, in LINEAR light, of the fp32 kernel (same fp32 matrices and gamma exponents) against
    `linear`.  Per render sample, port_multiperson.warp's bound `per` (coordinate error through the tap neighbourhood,
    24 u of the largest tap for the value), carried through the filter's fp64 weights.  Per pass, the fp32 weights lie
    within (2f + 16) u of the fp64 ones in sum (|t| fl(1/f) and 1 - x: 3 u each; the running total of 2f weights near f:
    (2f + 6) u relative; the division: u), and the ascending sum of at most 2f products adds (2f + 1) u of the largest
    term, so each pass adds (4f + 20) u of M, the largest sample value plus its bound over the output's support.  The
    powf of the gamma as in port_multiperson.warp."""
    if not 5 <= af <= MAX_FACTOR:
        raise ValueError(f'antialias factor {af}: this restatement covers 5..{MAX_FACTOR}')
    n = K_box.shape[0]
    d12 = pm.pad12(dist_box).to(K_box.device)
    lev = torch.as_tensor(crop_levels).long().to(K_box.device)
    kl = pm.level_intrinsics(K_box.repeat(num_aug, 1, 1), lev)
    out_lin, bound, worst = [], [], 0.0
    for c in range(num_aug * n):
        b = c % n
        img = levels[int(lev[c])][int(image_ids[b])]
        hl, wl = img.shape[-2:]
        u, v, eu, ev = pm.source_coords(invproj[c], kl[c], d12[b], (hl, wl), af, res,
                                        invproj_err[c] if invproj_err is not None else None)
        out_lin.append(shrink(pm.sample(img, u, v), res))
        if with_bound:
            worst = max(worst, float(torch.maximum(eu, ev).max()))
            dmax, vmax = pm.neighbourhood(img, u, v)
            per = dmax * (eu + ev)[None] + 24 * U32 * vmax
            bound.append(shrink(per, res) + 2 * (4 * af + 20) * U32 * support_max(vmax + per, af))
    lin = torch.stack(out_lin)
    ge = torch.as_tensor(gamma_exp).to(F64).to(lin.device).repeat_interleave(n)[:, None, None, None]
    crops = lin ** ge
    if not with_bound:
        return crops, lin, None
    warp.last_coord_bound = worst
    assert worst < 0.5, f'coordinate bound {worst:.3g} px: past 0.5 px the 3x3 tap neighbourhood no longer covers the sample'
    pw = (1 + pm.POWF_REL + U32) ** (1 / ge) - 1
    return crops, lin, torch.stack(bound) + pw * lin + 1e-300
