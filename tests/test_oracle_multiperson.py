"""CPU: the fp64 restatement of the frames -> poses stages (oracle/port_multiperson.py) against the goldens of the
unmodified reference (tests/golden/multiperson_*.npz, same bars as test_gpu_multiperson.py), and its error bounds: they
hold for fp32 evaluations of the same chains in two operation orders, and reject a 0.05 px coordinate shift, the wrong
pyramid level, a dropped distortion term, a dropped mirror swap and a transposed rotation."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from metrabs_b200.multiperson.multiperson_model import aug_parameters
from oracle import port_multiperson as pm

F64 = torch.float64


@pytest.fixture(scope='module')
def G(golden_dir):
    return np.load(os.path.join(golden_dir, 'multiperson_pipeline.npz'), allow_pickle=False)


def _per_box(G):
    boxes = [torch.from_numpy(G[f'boxes_{i}']) for i in range(int(G['n_images']))]
    n_box = torch.tensor([len(b) for b in boxes])
    intr, dist, ext, up = (torch.from_numpy(G[k]) for k in ('intrinsics', 'distortion', 'extrinsics', 'world_up'))
    k_box = torch.repeat_interleave(intr, n_box, dim=0)
    d_box = torch.repeat_interleave(dist, n_box, dim=0)
    cam_up = torch.repeat_interleave(torch.einsum('c,bCc->bC', up, ext[..., :3, :3]), n_box, dim=0)
    ext_inv = torch.repeat_interleave(torch.linalg.inv(ext), n_box, dim=0)
    return torch.from_numpy(G['images']), torch.cat(boxes), k_box, d_box, cam_up, ext_inv, torch.repeat_interleave(torch.arange(2), n_box)


def _rel(a, b):
    a, b = torch.as_tensor(a).to(F64), torch.as_tensor(b).to(F64)
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize('num_aug,af', [(5, 1), (5, 2), (2, 1), (2, 2)])
def test_crops_reproduce_reference(G, num_aug, af):
    images, boxes, k_box, d_box, up, _, ids = _per_box(G)
    gam, sc, fl, rf = aug_parameters(num_aug)
    new_k, R, inv, log_lev, lev = pm.crop_setup(boxes, k_box, d_box, up, rf, sc, 64, af)
    tag = f'crops_a{num_aug}_af{af}'
    assert _rel(new_k, G[tag + '_newk']) < 2e-6
    assert float((R - torch.from_numpy(G[tag + '_rot']).to(F64)).abs().max()) < 2e-6
    assert max(_rel(inv[i], G[tag + '_invproj'][i]) for i in range(len(inv))) < 1e-4
    crops, lin, _ = pm.warp(pm.pyramid(images), k_box, torch.from_numpy(G[tag + '_invproj']), d_box, lev, gam / 2.2, 64, ids,
                            num_aug, af)
    ref = torch.from_numpy(G[tag]).to(F64)
    assert float((pm.to_linear(crops, gam / 2.2, len(boxes)) - pm.to_linear(ref, gam / 2.2, len(boxes))).abs().max()) < 5e-5
    assert float((crops - ref).abs().max()) < 5e-4


def test_twelve_coefficient_crops(G):
    images, boxes, k_box, d_box, up, _, ids = _per_box(G)
    lev = torch.clip(torch.floor(-torch.log2(torch.from_numpy(G['d12_scales']).to(F64))), 0, 2).long()
    crops, _, _ = pm.warp(pm.pyramid(images), k_box, torch.from_numpy(G['d12_invproj']), torch.from_numpy(G['d12_coeffs']), lev,
                          torch.tensor([1.0]), 64, ids, 1, 1)
    # the device kernel meets 1e-5 against these fp32 reference crops; fp64 differs from them by the reference's own fp32
    # coordinate rounding, measured 1.01e-5
    assert float((crops - torch.from_numpy(G['d12_crops'])).abs().max()) < 1.5e-5


def _merge_inputs(G):
    images, boxes, k_box, d_box, up, ext_inv, ids = _per_box(G)
    gam, sc, fl, rf = aug_parameters(5)
    _, R, _, _, _ = pm.crop_setup(boxes, k_box, d_box, up, rf, sc, 64, 1)
    return torch.from_numpy(G['merge_table']), R, fl, G['mirror'], torch.from_numpy(G['joint_transform']), k_box, d_box, ext_inv


def test_merge_reproduces_reference(G):
    table, R, fl, mirror, jt, k_box, d_box, ext_inv = _merge_inputs(G)
    skels = {'all': None, 'upper': [5, 6, 7, 9, 0]}
    for avg in (True, False):
        for sk, idx in skels.items():
            p3, p2 = pm.tta_merge(table, R, fl, mirror, jt, idx, k_box, d_box, ext_inv, avg)
            tag = f'merge_avg{int(avg)}_{sk}'
            for i, sl in enumerate((slice(0, 3), slice(3, 5))):
                assert _rel(p3[sl], G[f'{tag}_p3d_{i}']) < 1e-5, (tag, i)
                assert _rel(p2[sl], G[f'{tag}_p2d_{i}']) < 1e-5, (tag, i)


def _emulated_merge(table, R, fl, mirror, jt, k_box, d_box, ext_inv, order):
    """The merge in fp32, in the kernel's order (0) or with matmuls / einsums (1)."""
    A, n = len(fl), len(k_box)
    P = table.float().reshape(A, n, -1, 3)
    P = torch.where(fl[:, None, None, None], P[:, :, torch.as_tensor(mirror)], P)
    Rf = R.float().reshape(A, n, 3, 3)
    if order == 0:
        cam = sum(P[..., k:k + 1] * Rf[:, :, None, k, :] for k in range(3))
        c = sum(cam[:, :, j:j + 1, :] * jt.float()[j][None, None, :, None] for j in range(P.shape[2]))
    else:
        c = torch.einsum('anjk,jN->anNk', P @ Rf, jt.float())
    x, y = c[..., 0] / c[..., 2], c[..., 1] / c[..., 2]
    dx, dy = pm.distort(x, y, pm.pad12(d_box).float()[None, :, None])
    K = k_box.float()[None, :, None]
    p2 = torch.stack([dx * K[..., 0, 0] + dy * K[..., 0, 1] + K[..., 0, 2], dx * K[..., 1, 0] + dy * K[..., 1, 1] + K[..., 1, 2]], -1)
    E = ext_inv.float()
    p3 = torch.einsum('anjc,nrc->anjr', c, E[:, :3, :3]) + E[None, :, None, :3, 3]
    return p3.transpose(0, 1).mean(1), p2.transpose(0, 1).mean(1)


def test_merge_bound_holds_and_rejects(G):
    table, R, fl, mirror, jt, k_box, d_box, ext_inv = _merge_inputs(G)
    R32 = R.float()
    p3, p2, e3, e2 = pm.tta_merge(table, R32, fl, mirror, jt, None, k_box, d_box, ext_inv, True, with_bound=True)
    for order in (0, 1):
        q3, q2 = _emulated_merge(table, R32, fl, mirror, jt, k_box, d_box, ext_inv, order)
        r3, r2 = float(((q3 - p3).abs() / e3).max()), float(((q2 - p2).abs() / e2).max())
        print(f'merge, fp32 order {order}: worst |fp32 - fp64| / bound: 3D {r3:.3f}, 2D {r2:.3f}')
        assert r3 <= 1 and r2 <= 1
    no_swap = _emulated_merge(table, R32, torch.zeros_like(fl), mirror, jt, k_box, d_box, ext_inv, 0)
    transposed = _emulated_merge(table, R32.transpose(-1, -2).contiguous(), fl, mirror, jt, k_box, d_box, ext_inv, 0)
    for name, (q3, q2) in (('no mirror swap', no_swap), ('transposed R', transposed)):
        r3, r2 = float(((q3 - p3).abs() / e3).max()), float(((q2 - p2).abs() / e2).max())
        print(f'merge, {name}: worst ratio 3D {r3:.3g}, 2D {r2:.3g}')
        assert r3 > 100 and r2 > 100


def _noise_scene(h, w, seed=3):
    g = torch.Generator().manual_seed(seed)
    images = torch.randint(0, 256, (2, 3, h, w), generator=g, dtype=torch.uint8)
    boxes = torch.tensor([[10., 5., 30., 50., 1.], [-15., 20., 60., 60., 1.], [w - 20., h - 25., 40., 45., 1.], [3., 3., w - 6., h - 6., 1.]])
    k = torch.tensor([[w * 0.9, 0., w / 2], [0., w * 0.9, h / 2], [0., 0., 1.]]).repeat(4, 1, 1)
    d12 = torch.tensor([-0.1, 0.03, 0.001, -0.002, 0.004, 0.02, -0.01, 0.003, 0.0005, -0.0004, 0.0003, 0.0002]).repeat(4, 1)
    up = torch.tensor([0., -1., 0.]).repeat(4, 1)
    return images, boxes, k, d12, up, torch.tensor([0, 1, 0, 1])


def _emulated_warp(images, K, inv, d12, lev, gexp, res, ids, A, af, order):
    """The warp chain in fp32, in the kernel's order (0) or with einsums and the distortion regrouped (1), sampled with
    fp32 grid_sample on an fp32 pyramid; -> gamma-encoded fp32 crops."""
    l0 = (images.float() / 255) ** 2.2
    levels = [l0, F.avg_pool2d(l0, 2, 2)]
    levels.append(F.avg_pool2d(levels[1], 2, 2))
    n = len(K)
    kl = pm.level_intrinsics(K.repeat(A, 1, 1), lev).float()
    r = torch.arange(res * af, dtype=torch.float32)
    ny, nx = torch.meshgrid(r, r, indexing='ij')
    out = []
    for c in range(A * n):
        M, d = inv[c].float(), d12[c % n].float()
        if order == 0:
            hx, hy, hz = (M[i, 0] * nx + M[i, 1] * ny + M[i, 2] for i in range(3))
        else:
            hx, hy, hz = torch.einsum('ij,jhw->ihw', M, torch.stack([nx, ny, torch.ones_like(nx)]))
        qx, qy = hx / hz, hy / hz
        if order == 0:
            dx, dy = pm.distort(qx, qy, d)
        else:
            r2 = qy * qy + qx * qx
            a = (1 + r2 * (d[0] + r2 * (d[1] + r2 * d[4]))) / (1 + r2 * (d[5] + r2 * (d[6] + r2 * d[7])))
            b = 2 * qy * d[2] + 2 * qx * d[3]
            dx = qx * a + qx * b + r2 * (d[3] + d[8] + r2 * d[9])
            dy = qy * a + qy * b + r2 * (d[2] + d[10] + r2 * d[11])
        u = kl[c, 0, 0] * dx + kl[c, 0, 1] * dy + kl[c, 0, 2]
        v = kl[c, 1, 0] * dx + kl[c, 1, 1] * dy + kl[c, 1, 2]
        img = levels[int(lev[c])][int(ids[c % n])]
        s = pm.sample(img, u, v)
        out.append(F.avg_pool2d(s[None], af, af)[0] if af > 1 else s)
    ge = torch.as_tensor(gexp).float().repeat_interleave(n)[:, None, None, None]
    return torch.stack(out) ** ge


@pytest.mark.parametrize('h,w,af', [(61, 83, 1), (64, 96, 2)])
def test_warp_bound_holds_for_fp32_chains(h, w, af):
    images, boxes, K, d12, up, ids = _noise_scene(h, w)
    gam, sc, fl, rf = aug_parameters(2)
    _, _, inv, _, lev = pm.crop_setup(boxes, K, d12, up, rf, sc, 24, af)
    inv32 = inv.float()
    ge = (gam / 2.2).float()
    _, lin, bound = pm.warp(pm.pyramid(images), K, inv32, d12, lev, ge, 24, ids, 2, af, with_bound=True)
    assert len(set(lev.tolist())) >= 2
    for order in (0, 1):
        dev = pm.to_linear(_emulated_warp(images, K, inv32, d12, lev, ge, 24, ids, 2, af, order), ge, len(boxes))
        ratio = float(((dev - lin).abs() / bound).max())
        print(f'{h}x{w} af={af} fp32 order {order}: worst |fp32 - fp64| / bound {ratio:.3f}, median bound {float(bound.median()):.2e}')
        assert ratio <= 1


def test_warp_bound_rejects_wrong_warps():
    images, boxes, K, d12, up, ids = _noise_scene(61, 83)
    gam, sc, fl, rf = aug_parameters(2)
    _, _, inv, _, lev = pm.crop_setup(boxes, K, d12, up, rf, sc, 24, 1)
    inv32, ge, pyr = inv.float(), (gam / 2.2).float(), pm.pyramid(images)
    _, lin, bound = pm.warp(pyr, K, inv32, d12, lev, ge, 24, ids, 2, 1, with_bound=True)
    wrong = {'0.05 px shift': pm.warp(pyr, K, inv32, d12, lev, ge, 24, ids, 2, 1, coord_shift=(0.05, 0.0))[1],
             'wrong pyramid level': pm.warp(pyr, K, inv32, d12, (lev + 1) % 3, ge, 24, ids, 2, 1)[1],
             'dropped k1': pm.warp(pyr, K, inv32, torch.cat([torch.zeros(4, 1), d12[:, 1:]], 1), lev, ge, 24, ids, 2, 1)[1]}
    for name, x in wrong.items():
        ratio = float(((x - lin).abs() / bound).max())
        print(f'warp, {name}: worst ratio {ratio:.3g}')
        assert ratio > 10, name


def _shift_crop_px(inv, dx):
    """invproj of crops whose principal point is off by dx crop pixels along x (the render samples x + dx)."""
    T = torch.eye(3, dtype=inv.dtype)
    T[0, 2] = dx
    return inv @ T


@pytest.mark.parametrize('af', [1, 2])
def test_setup_bound_holds_and_rejects(af):
    """new_K, R and invproj of an fp32 setup (torch's operation order, not the kernel's) lie within crop_setup_bound of
    the fp64 setup; the fp64 warp on the fp64 setup, with that bound carried to the coordinates, holds the fp32 chain; an
    invproj off by 0.05 crop px fails both."""
    images, boxes, K, d12, up, ids = _noise_scene(61, 83)
    gam, sc, fl, rf = aug_parameters(2)
    nk, R, inv, _, lev = pm.crop_setup(boxes, K, d12, up, rf, sc, 24, af)
    nk32, R32, inv32, _, lev32 = pm.crop_setup(boxes, K, d12, up, rf, sc, 24, af, dtype=torch.float32)
    ek, er, ei = pm.crop_setup_bound(boxes, K, d12, up, rf, sc, 24, af)
    assert torch.equal(lev, lev32)
    ratios = {name: float(((a.to(F64) - b).abs() / (e + 1e-300)).max())
              for name, a, b, e in (('new_K', nk32, nk, ek), ('R', R32, R, er), ('invproj', inv32, inv, ei))}
    shifted = _shift_crop_px(inv32, 0.05)
    ratios['invproj shifted 0.05 px'] = float(((shifted.to(F64) - inv).abs() / ei).max())
    print(f'af={af} setup, worst |fp32 - fp64| / bound: ' + ', '.join(f'{k} {v:.3g}' for k, v in ratios.items()))
    assert ratios['new_K'] <= 1 and ratios['R'] <= 1 and ratios['invproj'] <= 1
    assert ratios['invproj shifted 0.05 px'] > 10
    ge = (gam / 2.2).float()
    _, lin, bound = pm.warp(pm.pyramid(images), K, inv, d12, lev, ge, 24, ids, 2, af, with_bound=True, invproj_err=ei)
    chain = pm.to_linear(_emulated_warp(images, K, inv32, d12, lev, ge, 24, ids, 2, af, 0), ge, len(boxes))
    wrong = pm.to_linear(_emulated_warp(images, K, shifted, d12, lev, ge, 24, ids, 2, af, 0), ge, len(boxes))
    r_chain, r_wrong = float(((chain - lin).abs() / bound).max()), float(((wrong - lin).abs() / bound).max())
    print(f'af={af} warp on the fp64 setup: fp32 chain {r_chain:.3g}, invproj shifted 0.05 px {r_wrong:.3g}, '
          f'largest coordinate bound {pm.warp.last_coord_bound:.2e} px')
    assert r_chain <= 1 and r_wrong > 10


def _filter_check(poses3d, poses2d, boxes, n_per_image, bones, mean_bones, plausible, keep):
    d = pm.filter_decisions(torch.from_numpy(poses3d), torch.from_numpy(poses2d), torch.from_numpy(boxes), n_per_image, bones,
                            mean_bones)
    assert d['plausible'].tolist() == plausible.tolist()
    assert d['keep'].tolist() == keep.tolist()
    return d


def test_filter_reproduces_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, 'multiperson_filter.npz'), allow_pickle=False)
    _filter_check(g['poses3d'], g['poses2d'], g['boxes'], g['n_per_image'], g['bones'], g['mean_bones'],
                  g['plausible_bones'] & g['consistent'] & g['in_box'], g['keep'])


@pytest.mark.parametrize('group', ['crowd', 'wide'])
def test_filter_reproduces_reference_crowd(golden_dir, group):
    g = np.load(os.path.join(golden_dir, 'multiperson_filter_crowd.npz'), allow_pickle=False)
    d = _filter_check(*(g[f'{group}_{k}'] for k in ('poses3d', 'poses2d', 'boxes', 'n_per_image', 'bones', 'mean_bones',
                                                    'plausible', 'keep')))
    assert float(d['margin'].min()) > 1e-3
    if group == 'crowd':  # the golden exercises every decision past box 128 of its first image
        keep, plaus = g['crowd_keep'][128:170], g['crowd_plausible'][128:170]
        assert keep.any() and not keep.all() and not plaus.all() and (plaus & ~keep).any()
