"""fp64 restatement of the stages either side of the crop model (metrabs_b200/csrc/multiperson.cuh), written from the
reference's formulas (metrabs_pytorch/multiperson/{warping,multiperson_model,plausibility_check}.py), with per-element
error bounds for the fp32 device kernels.  Plain torch in float64; runs on the CPU or on a CUDA device, imports nothing
from the reference, so GPU tests can use it.

  pyramid              (u8 / 255) ** 2.2, then two avg_pool2d(2, 2) levels with floor sizes
  crop_setup           undistorted box points, look-at rotation, box scale; per augmentation new_K, R, inv(new_K @ R)
                       (@ the antialias scaling), level clip(floor(-log2(scale * af)), 0, 2)
  warp                 the reference's way: a render of res*af by grid_sample(align_corners=True, zeros) on the level
                       image with the level intrinsics and 12-coefficient distortion, avg_pool2d(af), then the gamma
  tta_merge            mirror swap, poses @ R, joint transform, distorted projection, inverse extrinsics, skeleton, mean
  filter_decisions     plausibility checks + pose NMS, with every decision's margin to its threshold

Crop order everywhere: flat index = aug * n_box + box."""
import math

import torch
import torch.nn.functional as F

F64 = torch.float64
U32 = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)
# CUDA's powf: at most 4 ulp (CUDA C Programming Guide, single-precision mathematical functions); one ulp <= 2 U32 relative
POWF_REL = 8 * U32


# ------------------------------------------------------------------------------------------------------------- pyramid
def pyramid(images_u8):
    """u8 [N,3,H,W] -> [level0, level1, level2] fp64 in linear light (level k: floor(H / 2**k) x floor(W / 2**k))."""
    l0 = (images_u8.to(F64) / 255) ** 2.2
    l1 = F.avg_pool2d(l0, 2, 2)
    return [l0, l1, F.avg_pool2d(l1, 2, 2)]


# ---------------------------------------------------------------------------------------------------------- distortion
def pad12(d):
    d = torch.as_tensor(d).to(F64)
    return F.pad(d, (0, 12 - d.shape[-1]))


def dist_parts(x, y, d):
    """(a, b, cx, cy) of the distortion model (k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4); d [..., 12] broadcasts
    against x, y with its last axis dropped."""
    d = [d[..., i] for i in range(12)]
    r2 = x * x + y * y
    a = (((d[4] * r2 + d[1]) * r2 + d[0]) * r2 + 1) / (((d[7] * r2 + d[6]) * r2 + d[5]) * r2 + 1)
    b = 2 * (x * d[3] + y * d[2])
    cx = (d[9] * r2 + d[3] + d[8]) * r2
    cy = (d[11] * r2 + d[2] + d[10]) * r2
    return a, b, cx, cy


def distort(x, y, d):
    a, b, cx, cy = dist_parts(x, y, d)
    return x * (a + b) + cx, y * (a + b) + cy


def undistort(x, y, d):
    ux, uy = x, y
    for _ in range(5):
        a, b, cx, cy = dist_parts(ux, uy, d)
        ux, uy = (x - cx - ux * b) / a, (y - cy - uy * b) / a
    return ux, uy


def distort_bound(x, y, ex, ey, d):
    """Bound on |fl32(distort(x~, y~)) - distort(x, y)| where |x~ - x| <= ex, |y~ - y| <= ey: the input error through the
    fp64 Jacobian (central differences, 1 % margin) plus the fp32 rounding of the evaluation.  Rounding: each of P, Q (the
    cubic numerator / denominator in r2) is within 16 u of its absolute-value evaluation P_abs (three Horner steps, r2 itself
    2 u off and raised to the third power), b within 4 u of b_abs, c within 10 u of c_abs; then s = a + b and x s + c."""
    h = 1e-7 * torch.clamp(torch.maximum(x.abs(), y.abs()), min=1.0)
    xp, yp = distort(x + h, y, d)
    xm, ym = distort(x - h, y, d)
    jxx, jyx = (xp - xm) / (2 * h), (yp - ym) / (2 * h)
    xp, yp = distort(x, y + h, d)
    xm, ym = distort(x, y - h, d)
    jxy, jyy = (xp - xm) / (2 * h), (yp - ym) / (2 * h)
    prop_x = 1.01 * (jxx.abs() * ex + jxy.abs() * ey)
    prop_y = 1.01 * (jyx.abs() * ex + jyy.abs() * ey)
    da = [d[..., i].abs() for i in range(12)]
    r2 = x * x + y * y
    p = ((d[..., 4] * r2 + d[..., 1]) * r2 + d[..., 0]) * r2 + 1
    q = ((d[..., 7] * r2 + d[..., 6]) * r2 + d[..., 5]) * r2 + 1
    p_abs = ((da[4] * r2 + da[1]) * r2 + da[0]) * r2 + 1
    q_abs = ((da[7] * r2 + da[6]) * r2 + da[5]) * r2 + 1
    a = p / q
    e_a = a.abs() * (16 * U32 * p_abs / p.abs() + 16 * U32 * q_abs / q.abs() + U32)
    b = 2 * (x * d[..., 3] + y * d[..., 2])
    e_b = 4 * U32 * 2 * (x.abs() * da[3] + y.abs() * da[2])
    s = a + b
    e_s = e_a + e_b + U32 * s.abs()
    cx_abs = (da[9] * r2 + da[3] + da[8]) * r2
    cy_abs = (da[11] * r2 + da[2] + da[10]) * r2
    _, _, cx, cy = dist_parts(x, y, d)
    rx = x.abs() * e_s + 10 * U32 * cx_abs + 2 * U32 * ((x * s).abs() + cx.abs())
    ry = y.abs() * e_s + 10 * U32 * cy_abs + 2 * U32 * ((y * s).abs() + cy.abs())
    return prop_x + rx, prop_y + ry


# ---------------------------------------------------------------------------------------------------------- crop setup
def corner_aligned_scale_mat(factor, device=None):
    s = (factor - 1) / 2
    return torch.tensor([[factor, 0, s], [0, factor, s], [0, 0, 1]], dtype=F64, device=device)


def lookat_matrix(forward, up):
    z = forward / torch.linalg.norm(forward, dim=-1, keepdim=True)
    x = torch.linalg.cross(z, up.expand_as(z))
    alt = torch.stack([z[:, 2], torch.zeros_like(z[:, 2]), -z[:, 0]], dim=1)
    x = torch.where(torch.linalg.norm(x, dim=-1, keepdim=True) == 0, alt, x)
    x = x / torch.linalg.norm(x, dim=-1, keepdim=True)
    return torch.stack([x, torch.linalg.cross(z, x), z], dim=1)


def crop_setup(boxes, K, dist, up, rotflip, aug_scales, res, af=1, dtype=F64):
    """Per box [n]: K [n,3,3], dist [n,<=12], up [n,3]; per augmentation [A]: rotflip [A,3,3], aug_scales [A].
    -> new_K [A,n,3,3], R [A,n,3,3], invproj [A*n,3,3], log_level [A*n] = -log2(crop_scale * af) and
    level [A*n] = clip(floor(log_level), 0, 2).  dtype=torch.float32 evaluates the same formulas in fp32 (the two 3x3
    inverses in fp64, rounded, as the kernel does): an fp32 setup in an operation order of its own, for the tests."""
    boxes, K, up, rotflip, aug_scales = (torch.as_tensor(t).to(dtype) for t in (boxes, K, up, rotflip, aug_scales))
    d = pad12(dist).to(K.device, dtype)

    def inv3(m):
        return torch.linalg.inv(m.to(F64)).to(dtype)
    x, y, w, h = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    pts = torch.stack([torch.stack([x + w / 2, y + h / 2], 1), torch.stack([x + w / 2, y], 1), torch.stack([x + w, y + h / 2], 1),
                       torch.stack([x + w / 2, y + h], 1), torch.stack([x, y + h / 2], 1)], 1)
    cam = torch.einsum('bpc,bCc->bpC', F.pad(pts, (0, 1), value=1.0), inv3(K))
    ux, uy = undistort(cam[..., 0], cam[..., 1], d[:, None])
    cam = torch.stack([ux, uy, torch.ones_like(ux)], -1)
    r0 = lookat_matrix(cam[:, 0], up)
    side = torch.einsum('bpc,bCc->bpC', cam[:, 1:], K @ r0)
    side = side[..., :2] / side[..., 2:]
    size = torch.maximum(torch.linalg.norm(side[:, 0] - side[:, 2], dim=-1), torch.linalg.norm(side[:, 1] - side[:, 3], dim=-1))
    box_scale = res / size
    cs = aug_scales[:, None] * box_scale[None]  # [A, n]
    A, n = cs.shape
    new_k = torch.zeros(A, n, 3, 3, dtype=dtype, device=K.device)
    new_k[..., :2, :2] = K[None, :, :2, :2] * cs[..., None, None]
    new_k[..., :2, 2] = res / 2
    new_k[..., 2, 2] = 1
    R = rotflip[:, None] @ r0[None]
    inv = inv3(new_k @ R)
    if af > 1:
        inv = inv @ corner_aligned_scale_mat(1 / af, K.device).to(dtype)
    log_level = -torch.log2(cs * af).reshape(-1)
    return new_k, R, inv.reshape(-1, 3, 3), log_level, torch.clip(torch.floor(log_level), 0, 2).long()


class _Rounding:
    """First-order rounding model of an fp32 computation evaluated in fp64: `r(t)` stands for one rounded operation,
    t (1 + delta) with delta = 0 and a gradient.  For an output O, |fl32(O) - O| <= u sum_i |dO/d delta_i| + O(u^2); each
    delta carries its box axis so that one backward pass over all boxes gives every box its own sum."""

    def __init__(self):
        self.deltas = []

    def __call__(self, t, box_axis=0):
        d = torch.zeros_like(t, requires_grad=True)
        self.deltas.append((d, box_axis))
        return t * (1 + d)

    def bound(self, out_sum):
        grads = torch.autograd.grad(out_sum, [d for d, _ in self.deltas], retain_graph=True, allow_unused=True)
        tot = 0.0
        for g, (d, ax) in zip(grads, self.deltas):
            if g is not None:
                g = g.abs().movedim(ax, 0)
                tot = tot + g.reshape(g.shape[0], -1).sum(1)
        return U32 * tot


def crop_setup_bound(boxes, K, dist, up, rotflip, aug_scales, res, af=1):
    """Per-entry bounds on |device - fp64| of crop_setup's new_K [A,n,3,3], R [A,n,3,3] and invproj [A*n,3,3], for the fp32
    crop_setup_kernel on the same fp32 inputs.  The kernel's operations are restated in its own order, each rounded once
    (_Rounding: a fused multiply-add rounds once where this counts two, so the bound covers it): K^-1 from the fp64 closed
    form rounded to fp32, the five box points through K^-1, five undistortion iterations, the look-at rotation, the side
    points through K R0, the box scale, new_K, R = rotflip R0, new_K R, its fp64 closed-form inverse rounded to fp32, and
    the antialias scaling.  First order in u; the result is doubled to cover the second-order terms with a wide margin."""
    out_dev = torch.as_tensor(K).device  # small tensors: the many backward passes run on the host
    K, boxes, up, rotflip, aug_scales = (torch.as_tensor(t).detach().to('cpu', F64) for t in (K, boxes, up, rotflip, aug_scales))
    dv = K.device
    d = pad12(torch.as_tensor(dist).detach().cpu())
    r = _Rounding()
    n, A = K.shape[0], aug_scales.shape[0]

    def dot(a, b):  # a0 b0 + a1 b1 + a2 b2, left to right
        return r(r(r(a[0] * b[0]) + r(a[1] * b[1])) + r(a[2] * b[2]))

    def parts(x, y):
        dd = [d[:, None, i] for i in range(12)]
        r2 = r(r(x * x) + r(y * y))
        num = r(r(r(r(r(r(dd[4] * r2) + dd[1]) * r2) + dd[0]) * r2) + 1)
        den = r(r(r(r(r(r(dd[7] * r2) + dd[6]) * r2) + dd[5]) * r2) + 1)
        b = r(2 * r(r(x * dd[3]) + r(y * dd[2])))
        cx = r(r(r(r(dd[9] * r2) + dd[3]) + dd[8]) * r2)
        cy = r(r(r(r(dd[11] * r2) + dd[2]) + dd[10]) * r2)
        return r(num / den), b, cx, cy

    kinv = r(torch.linalg.inv(K))
    x, y, w, h = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    hw, hh = w / 2, h / 2  # exact
    px = torch.stack([r(x + hw), r(x + hw), r(x + w), r(x + hw), x], 1)
    py = torch.stack([r(y + hh), y, r(y + hh), r(y + h), r(y + hh)], 1)
    cx0 = r(r(r(kinv[:, 0, 0:1] * px) + r(kinv[:, 0, 1:2] * py)) + kinv[:, 0, 2:3])
    cy0 = r(r(r(kinv[:, 1, 0:1] * px) + r(kinv[:, 1, 1:2] * py)) + kinv[:, 1, 2:3])
    ux, uy = cx0, cy0
    for _ in range(5):
        a, b, cx, cy = parts(ux, uy)
        ux, uy = r(r(r(cx0 - cx) - r(ux * b)) / a), r(r(r(cy0 - cy) - r(uy * b)) / a)
    f = [ux[:, 0], uy[:, 0], torch.ones_like(ux[:, 0])]
    fn = r(torch.sqrt(dot(f, f)))
    z = [r(c / fn) for c in f]
    u = [up[:, i] for i in range(3)]
    xv = [r(r(z[1] * u[2]) - r(z[2] * u[1])), r(r(z[2] * u[0]) - r(z[0] * u[2])), r(r(z[0] * u[1]) - r(z[1] * u[0]))]
    xn = r(torch.sqrt(dot(xv, xv)))
    xv = [r(c / xn) for c in xv]
    yv = [r(r(z[1] * xv[2]) - r(z[2] * xv[1])), r(r(z[2] * xv[0]) - r(z[0] * xv[2])), r(r(z[0] * xv[1]) - r(z[1] * xv[0]))]
    R0 = torch.stack([torch.stack(xv, -1), torch.stack(yv, -1), torch.stack(z, -1)], 1)  # [n,3,3]
    M = torch.stack([torch.stack([dot([K[:, i, 0], K[:, i, 1], K[:, i, 2]], [R0[:, 0, j], R0[:, 1, j], R0[:, 2, j]])
                                  for j in range(3)], -1) for i in range(3)], 1)
    sx, sy = [], []
    for i in range(1, 5):
        q = [ux[:, i], uy[:, i], torch.ones_like(ux[:, i])]
        aa, bq, c = (dot([M[:, k, 0], M[:, k, 1], M[:, k, 2]], q) for k in range(3))
        sx.append(r(aa / c))
        sy.append(r(bq / c))

    def dist2(i, j):
        ddx, ddy = r(sx[i] - sx[j]), r(sy[i] - sy[j])
        return r(torch.sqrt(r(r(ddx * ddx) + r(ddy * ddy))))
    box_scale = r(res / torch.maximum(dist2(0, 2), dist2(1, 3)))
    cs = r(aug_scales[:, None] * box_scale[None], 1)  # [A,n]
    Kx = K[None].expand(A, n, 3, 3)
    nK = torch.zeros(A, n, 3, 3, dtype=F64, device=dv)
    nK[..., 0, 0], nK[..., 0, 1] = r(Kx[..., 0, 0] * cs, 1), r(Kx[..., 0, 1] * cs, 1)
    nK[..., 1, 0], nK[..., 1, 1] = r(Kx[..., 1, 0] * cs, 1), r(Kx[..., 1, 1] * cs, 1)
    nK[..., :2, 2], nK[..., 2, 2] = res / 2, 1

    def mat(a, b, ax):  # [A,n,3,3] @ [A,n,3,3] in mat3_mul's order
        return torch.stack([torch.stack([r(r(r(a[..., i, 0] * b[..., 0, j], ax) + r(a[..., i, 1] * b[..., 1, j], ax), ax)
                                           + r(a[..., i, 2] * b[..., 2, j], ax), ax) for j in range(3)], -1) for i in range(3)], -2)
    R = mat(rotflip[:, None].expand(A, n, 3, 3), R0[None].expand(A, n, 3, 3), 1)
    inv = r(torch.linalg.inv(mat(nK, R, 1)), 1)
    if af > 1:
        inv = mat(inv, corner_aligned_scale_mat(1 / af, dv).expand(A, n, 3, 3), 1)
    out = []
    for t in (nK, R, inv):
        e = torch.zeros(A, n, 3, 3, dtype=F64, device=dv)
        for a in range(A):
            for i in range(3):
                for j in range(3):
                    if t[a, :, i, j].requires_grad:
                        e[a, :, i, j] = 2 * r.bound(t[a, :, i, j].sum())
        out.append(e.to(out_dev))
    return out[0], out[1], out[2].reshape(-1, 3, 3)


# ----------------------------------------------------------------------------------------------------------------- warp
def level_intrinsics(K, level):
    """corner_aligned_scale_mat(2 ** -level) @ K, per crop."""
    f = 2.0 ** -level.to(F64)
    s = (f - 1) / 2
    kl = K.to(F64).clone()
    kl[:, :2, :] = f[:, None, None] * K[:, :2, :].to(F64) + s[:, None, None] * K[:, 2:3, :].to(F64)
    return kl


def source_coords(invproj, k_level, d, size, af, res, invproj_err=None):
    """fp64 source coordinates (gx, gy) in level pixels of the res*af render grid of ONE crop: invproj [3,3], k_level [3,3],
    d [12], size (H_l, W_l).  Also the bound of the fp32 kernel chain on them (homography: 3 u per dot product of absolute
    values, plus invproj_err [3,3] times |(x, y, 1)| when the kernel's matrix is only known to lie within invproj_err of
    invproj; division; distortion (distort_bound); the level affine with its fp32 entries: 5 u of the absolute sum;
    normalise / unnormalise by (size - 1): 6 u of (|u| + size))."""
    dev = invproj.device
    r = torch.arange(res * af, dtype=F64, device=dev)
    ny, nx = torch.meshgrid(r, r, indexing='ij')
    M = invproj.to(F64)
    h = [M[i, 0] * nx + M[i, 1] * ny + M[i, 2] for i in range(3)]
    habs = [M[i, 0].abs() * nx + M[i, 1].abs() * ny + M[i, 2].abs() for i in range(3)]
    qx, qy = h[0] / h[2], h[1] / h[2]
    eh = [3 * U32 * a for a in habs]
    if invproj_err is not None:
        E = invproj_err.to(F64)
        eh = [eh[i] + E[i, 0] * nx + E[i, 1] * ny + E[i, 2] for i in range(3)]
    eqx = (eh[0] + qx.abs() * eh[2]) / h[2].abs() + U32 * qx.abs()
    eqy = (eh[1] + qy.abs() * eh[2]) / h[2].abs() + U32 * qy.abs()
    dx, dy = distort(qx, qy, d)
    edx, edy = distort_bound(qx, qy, eqx, eqy, d)
    k = k_level.to(F64)
    u = k[0, 0] * dx + k[0, 1] * dy + k[0, 2]
    v = k[1, 0] * dx + k[1, 1] * dy + k[1, 2]
    eu = k[0, 0].abs() * edx + k[0, 1].abs() * edy + 5 * U32 * ((k[0, 0] * dx).abs() + (k[0, 1] * dy).abs() + k[0, 2].abs())
    ev = k[1, 0].abs() * edx + k[1, 1].abs() * edy + 5 * U32 * ((k[1, 0] * dx).abs() + (k[1, 1] * dy).abs() + k[1, 2].abs())
    hl, wl = size
    eu = eu + 6 * U32 * (u.abs() + wl)
    ev = ev + 6 * U32 * (v.abs() + hl)
    return u, v, eu, ev


def sample(img, gx, gy):
    """grid_sample(align_corners=True, bilinear, zeros) of img [3,H,W] at pixel coordinates gx, gy [h,w] -> [3,h,w]."""
    hl, wl = img.shape[-2:]
    grid = torch.stack([gx / (wl - 1) * 2 - 1, gy / (hl - 1) * 2 - 1], -1)
    return F.grid_sample(img[None], grid[None], mode='bilinear', padding_mode='zeros', align_corners=True)[0]


def neighbourhood(img, gx, gy):
    """(largest difference of adjacent taps, largest tap) over the 3x3 taps around round(g), zero outside the image:
    a coordinate within 0.5 px of g samples only cells whose corners are among these taps.  -> [3,h,w] each."""
    hl, wl = img.shape[-2:]
    pad = F.pad(img, (2, 2, 2, 2))
    rx = torch.round(gx).clamp(-2, wl + 1).long() + 2
    ry = torch.round(gy).clamp(-2, hl + 1).long() + 2
    taps = torch.stack([torch.stack([pad[:, (ry + j).clamp(0, hl + 3), (rx + i).clamp(0, wl + 3)] for i in (-1, 0, 1)], -1)
                        for j in (-1, 0, 1)], -2)  # [3,h,w,3,3]
    dh = (taps[..., :, 1:] - taps[..., :, :-1]).abs().flatten(-2).amax(-1)
    dv = (taps[..., 1:, :] - taps[..., :-1, :]).abs().flatten(-2).amax(-1)
    return torch.maximum(dh, dv), taps.abs().flatten(-2).amax(-1)


def warp(levels, K_box, invproj, dist_box, crop_levels, gamma_exp, res, image_ids, num_aug, af=1, with_bound=False,
         coord_shift=None, invproj_err=None):
    """All num_aug * n crops, the reference's way, in fp64.  levels: pyramid(); K_box [n,3,3], dist_box [n,<=12],
    image_ids [n] per box; invproj [A*n,3,3], crop_levels [A*n], gamma_exp [A] per crop / augmentation.
    -> (crops [A*n,3,res,res] gamma-encoded, linear [A*n,3,res,res] before the gamma, bound [A*n,3,res,res] or None).

    bound: per output element, in LINEAR light, of the fp32 kernel (same fp32 matrices, same gamma exponents) against
    `linear`.  Per render sample s with source coordinate g_s and fp32 coordinate error bound (ex_s, ey_s)
    (source_coords): a sample within 0.5 px of g_s interpolates between taps of the 3x3 neighbourhood of round(g_s), so its
    value moves by at most D_s (ex_s + ey_s) with D_s the largest adjacent-tap difference there.  Value rounding per
    sample: the decoded tap within 17 u of the largest tap V_s (the table's powf 8 u and i/255 2.2 u, then up to two fp32
    box-filter levels of 3 u each), the bilinear blend (weight products, products, three additions) 5 u of V_s: 24 u.  The af^2 samples average with af^2 u of the largest tap; 1/af^2 is exact.
    The device output is gamma-encoded, out = powf(lin, e) with e = gamma_exp; taken back to linear light as
    out^(1/e) in fp64 its powf error becomes (1 + POWF_REL + U32)^(1/e) - 1 relative.
    invproj_err [A*n,3,3]: the kernel ran on matrices within that of `invproj` (crop_setup_bound), carried through
    source_coords.  The neighbourhood argument needs every coordinate bound under 0.5 px: asserted, the largest returned
    as `warp.last_coord_bound`.  coord_shift (dx, dy) px serves the tests."""
    n = K_box.shape[0]
    d12 = pad12(dist_box).to(K_box.device)
    lev = torch.as_tensor(crop_levels).long().to(K_box.device)
    kl = level_intrinsics(K_box.repeat(num_aug, 1, 1), lev)
    out_lin, bound, worst = [], [], 0.0
    for c in range(num_aug * n):
        b = c % n
        img = levels[int(lev[c])][int(image_ids[b])]
        hl, wl = img.shape[-2:]
        u, v, eu, ev = source_coords(invproj[c], kl[c], d12[b], (hl, wl), af, res,
                                     invproj_err[c] if invproj_err is not None else None)
        if coord_shift is not None:
            u, v = u + coord_shift[0], v + coord_shift[1]
        lin = sample(img, u, v)
        if af > 1:
            lin = F.avg_pool2d(lin[None], af, af)[0]
        out_lin.append(lin)
        if with_bound:
            worst = max(worst, float(torch.maximum(eu, ev).max()))
            dmax, vmax = neighbourhood(img, u, v)
            per = dmax * (eu + ev)[None] + 24 * U32 * vmax
            e = F.avg_pool2d(per[None], af, af)[0] if af > 1 else per
            vm = F.max_pool2d(vmax[None], af, af)[0] if af > 1 else vmax
            bound.append(e + af * af * U32 * vm)
    lin = torch.stack(out_lin)
    ge = torch.as_tensor(gamma_exp).to(F64).to(lin.device).repeat_interleave(n)[:, None, None, None]
    crops = lin ** ge
    if not with_bound:
        return crops, lin, None
    warp.last_coord_bound = worst
    assert worst < 0.5, f'coordinate bound {worst:.3g} px: past 0.5 px the 3x3 tap neighbourhood no longer covers the sample'
    pw = (1 + POWF_REL + U32) ** (1 / ge) - 1
    return crops, lin, torch.stack(bound) + pw * lin + 1e-300


def to_linear(crops, gamma_exp, n_box):
    """Gamma-encoded crops (any dtype) -> fp64 linear light, inverting `crops ** gamma_exp` per augmentation."""
    ge = torch.as_tensor(gamma_exp).to(F64).to(crops.device).repeat_interleave(n_box)[:, None, None, None]
    return crops.to(F64).clamp_min(0) ** (1 / ge)


# ------------------------------------------------------------------------------------------------------------ TTA merge
def tta_merge(poses, R, flip, mirror, jt, skel, K_box, dist_box, ext_inv_box, average, with_bound=False):
    """poses [A*n,J,3] crop-model output, R [A*n,3,3] (or [A,n,3,3]), flip [A] bool, mirror [J], jt [J,J2] or None,
    skel indices into J2 or None, per box K [n,3,3], dist [n,<=12], ext_inv [n,4,4].
    -> poses3d [n,(A,)Js,3], poses2d [n,(A,)Js,2] (and their bounds for the fp32 kernel on the same fp32 inputs).

    Bounds: camera-space c = sum_n t_n (q_n R) accumulates J2 + 4 roundings at most, so |c~ - c| <= (J + 4) u sum_n |t_n|
    |q_n| |R| (3 u |q| |R| without a transform).  World w = E [c, 1]: |E| e_c + 4 u |E| [|c|, 1].  2D: x = c0 / c2 has
    error (e_c0 + |x| e_c2) / |c2| + u |x| (the 1/|z| conditioning; unbounded where e_c2 >= |c2| / 2), then the distortion
    (distort_bound) and K: |K| e_q + 3 u |K| [|q|, 1].  The mean over A (A - 1 additions, the rounded 1/A and the product) adds (A + 2) u of the
    mean absolute value."""
    dev = poses.device
    P = poses.to(F64)
    A = len(flip)
    n = K_box.shape[0]
    J = P.shape[1]
    P = P.reshape(A, n, J, 3)
    Rm = R.to(F64).reshape(A, n, 3, 3)
    mirror = torch.as_tensor(mirror, dtype=torch.long, device=dev)
    flip = torch.as_tensor(flip, dtype=torch.bool, device=dev)
    P = torch.where(flip[:, None, None, None], P[:, :, mirror], P)
    cam = P @ Rm  # [A,n,J,3]
    cam_abs = P.abs() @ Rm.abs()
    if jt is not None:
        jt = torch.as_tensor(jt).to(F64).to(dev)
        c = torch.einsum('ankc,kN->anNc', cam, jt)
        c_err = (J + 4) * U32 * torch.einsum('ankc,kN->anNc', cam_abs, jt.abs())
    else:
        c, c_err = cam, 3 * U32 * cam_abs
    E = ext_inv_box.to(F64)
    w = torch.einsum('anjc,nrc->anjr', c, E[:, :3, :3]) + E[None, :, None, :3, 3]
    w_err = torch.einsum('anjc,nrc->anjr', c_err, E[:, :3, :3].abs()) + 4 * U32 * (
        torch.einsum('anjc,nrc->anjr', c.abs(), E[:, :3, :3].abs()) + E[None, :, None, :3, 3].abs())
    z = c[..., 2]
    qx, qy = c[..., 0] / z, c[..., 1] / z
    eqx = (c_err[..., 0] + qx.abs() * c_err[..., 2]) / z.abs() + U32 * qx.abs()
    eqy = (c_err[..., 1] + qy.abs() * c_err[..., 2]) / z.abs() + U32 * qy.abs()
    ill = c_err[..., 2] >= z.abs() / 2
    d12 = pad12(dist_box).to(dev)[None, :, None]
    dx, dy = distort(qx, qy, d12)
    K = K_box.to(F64)[None, :, None]
    u = dx * K[..., 0, 0] + dy * K[..., 0, 1] + K[..., 0, 2]
    v = dx * K[..., 1, 0] + dy * K[..., 1, 1] + K[..., 1, 2]
    p2 = torch.stack([u, v], -1)
    out3, out2 = w, p2
    if with_bound:
        edx, edy = distort_bound(qx, qy, eqx, eqy, d12)
        eu = K[..., 0, 0].abs() * edx + K[..., 0, 1].abs() * edy + 3 * U32 * ((K[..., 0, 0] * dx).abs() + (K[..., 0, 1] * dy).abs() + K[..., 0, 2].abs())
        ev = K[..., 1, 0].abs() * edx + K[..., 1, 1].abs() * edy + 3 * U32 * ((K[..., 1, 0] * dx).abs() + (K[..., 1, 1] * dy).abs() + K[..., 1, 2].abs())
        e2 = torch.where(ill[..., None], torch.full_like(p2, math.inf), torch.stack([eu, ev], -1))
        e3 = w_err
    if skel is not None:
        s = torch.as_tensor(skel, dtype=torch.long, device=dev)
        out3, out2 = out3[:, :, s], out2[:, :, s]
        if with_bound:
            e3, e2 = e3[:, :, s], e2[:, :, s]
    out3, out2 = out3.transpose(0, 1), out2.transpose(0, 1)  # [n,A,Js,k]
    if with_bound:
        e3, e2 = e3.transpose(0, 1), e2.transpose(0, 1)
    if average:
        if with_bound:
            e3 = e3.mean(1) + (A + 2) * U32 * out3.abs().mean(1)
            e2 = e2.mean(1) + (A + 2) * U32 * out2.abs().mean(1)
        out3, out2 = out3.mean(1), out2.mean(1)
    return (out3, out2, e3, e2) if with_bound else (out3, out2)


# ----------------------------------------------------------------------------------------------- plausibility + NMS
def filter_decisions(poses3d, poses2d, boxes, n_per_image, bones, mean_bones):
    """The three plausibility checks and pose NMS per image (threshold 0.4), in fp64.  poses3d [n,A,J,3], poses2d
    [n,A,J,2], boxes [n,>=5], bones [nb,2] joint pairs, mean_bones [nb] mm.
    -> dict(plausible, keep [n] bool, margin [n]: the smallest distance of any decision of that box to its threshold, in
    the decision's own unit relative to the threshold (bone 0.1x / 3x ratio and 300 mm difference, per-joint stdev of
    200 mm, in-box area ratio 0.5, similarity 0.4 for every pair of valid boxes of an image), and the parts)."""
    p3, p2, bx = poses3d.to(F64), poses2d.to(F64), boxes.to(F64)
    mb = torch.as_tensor(mean_bones).to(F64).to(p3.device)
    bones = torch.as_tensor(bones, dtype=torch.long, device=p3.device).reshape(-1, 2)
    n, A, J, _ = p3.shape
    mean3, mean2 = p3.mean(1), p2.mean(1)
    ln = torch.linalg.norm(mean3[:, bones[:, 0]] - mean3[:, bones[:, 1]], dim=-1)  # [n, nb]
    rel, ad = ln / mb, (ln - mb).abs()
    big, small, far = rel > 3, rel < 0.1, ad > 300
    m_big, m_small, m_far = (rel / 3 - 1).abs(), (rel / 0.1 - 1).abs(), (ad / 300 - 1).abs()
    # margin of a boolean: a true OR holds while one true part holds, a false one needs every part; AND the other way round
    off = big | small
    m_off = torch.where(off, torch.maximum(torch.where(big, m_big, 0), torch.where(small, m_small, 0)), torch.minimum(m_big, m_small))
    bad = off & far
    m_bad = torch.where(bad, torch.minimum(m_off, m_far),
                        torch.maximum(torch.where(off, 0, m_off), torch.where(far, 0, m_far)))
    plaus = ~bad.any(-1)
    m_bone = torch.where(plaus, m_bad.amin(-1), torch.where(bad, m_bad, 0).amax(-1))
    sq = p3.square().mean((-2, -1), keepdim=True)
    aligned = p3 * torch.sqrt(sq.mean(1, keepdim=True) / sq)
    std = torch.sqrt(aligned.var(1).sum(-1))  # [n, J]
    cons = (std < 200).sum(-1) > J // 4
    m_std = (std / 200 - 1).abs().amin(-1)
    lo, hi = mean2.amin(1), mean2.amax(1)
    ist = torch.maximum(bx[:, :2], lo)
    ien = torch.minimum(bx[:, :2] + bx[:, 2:4], hi)
    inter = torch.relu(ien - ist).prod(-1)
    area = bx[:, 2:4].prod(-1)
    inbox = inter > 0.5 * area
    m_box = (inter / (0.5 * area) - 1).abs()
    valid = plaus & cons & inbox
    keep = torch.zeros(n, dtype=torch.bool, device=p3.device)
    m_sim = torch.full((n,), math.inf, dtype=F64, device=p3.device)
    s0 = 0
    k = J // 4
    for cnt in [int(c) for c in n_per_image]:
        idx = torch.nonzero(valid[s0:s0 + cnt]).flatten() + s0
        if len(idx):
            P = mean3[idx]
            ss = P.square().mean((-2, -1))
            ms = (ss[None] + ss[:, None]) / 2
            f1 = torch.sqrt(ms / ss[None])[..., None, None]
            f2 = torch.sqrt(ms / ss[:, None])[..., None, None]
            dist = torch.linalg.norm(f1 * P[None] - f2 * P[:, None], dim=-1)
            sim = torch.relu(1 - torch.topk(dist, k, dim=-1).values / 300).mean(-1)
            off = ~torch.eye(len(idx), dtype=torch.bool, device=p3.device)
            msim = torch.where(off, (sim / 0.4 - 1).abs(), torch.full_like(sim, math.inf))
            m_sim[idx] = msim.amin(1)
            order = torch.argsort(bx[idx, 4], stable=True, descending=True).tolist()
            supp = [False] * len(idx)
            for oi, i in enumerate(order):
                if supp[i]:
                    continue
                for j in order[oi + 1:]:
                    if not supp[j] and sim[i, j] > 0.4:
                        supp[j] = True
            keep[idx[[i for i in range(len(idx)) if not supp[i]]]] = True
        s0 += cnt
    margin = torch.minimum(torch.minimum(m_bone, m_std), torch.minimum(m_box, m_sim))
    return dict(plausible=valid, keep=keep, plausible_bones=plaus, consistent=cons, in_box=inbox, margin=margin,
                margin_bone=m_bone, margin_stdev=m_std, margin_box=m_box, margin_similarity=m_sim)
