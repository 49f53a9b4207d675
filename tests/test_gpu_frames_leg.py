"""GPU: every stage of the frames -> poses leg that bench.py times (frames_leg: 8 noise frames of 720x1280, 51 boxes x 5
augmentations = 255 crops of 256x256, EfficientNetV2-L bf16, J = 24, no joint transform) against the fp64 restatement
oracle/port_multiperson.py, element by element within its derived bounds; then the edges the bench does not reach (odd
frame sizes, boxes outside the frame, every pyramid level, antialias 1 / 2 / 4, 0 / 5 / 8 / 12 distortion coefficients,
1 / 2 / 16 augmentations, J = 122 with a mirror swap, a joint transform and a skeleton, with and without the mean); and the
plausibility filter on crowded images (tests/golden/multiperson_filter_crowd.npz, from the unmodified reference)."""
import math
import os
import time
import types

import numpy as np
import pytest
import torch

from oracle import port_multiperson as pm

pytestmark = pytest.mark.gpu
F64 = torch.float64


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')


def _ratio(d, r, b):
    return float(((d.to(F64) - r).abs() / b).max())


def _bench_scene(dev):
    """bench.py frames_leg, seed for seed."""
    g = torch.Generator().manual_seed(11)
    n_img, h, w = 8, 720, 1280
    frames = torch.randint(0, 256, (n_img, 3, h, w), generator=g, dtype=torch.uint8).to(dev)
    counts = [7, 6, 7, 6, 6, 7, 6, 6]
    boxes = []
    for c in counts:
        xy = torch.rand(c, 2, generator=g) * torch.tensor([w - 400., h - 500.])
        wh = torch.tensor([180., 400.]) * (0.6 + 0.8 * torch.rand(c, 2, generator=g))
        boxes.append(torch.cat([xy, wh, torch.rand(c, 1, generator=g)], dim=1))
    kw = dict(intrinsic_matrix=torch.tensor([[[1100., 0, w / 2], [0, 1100., h / 2], [0, 0, 1]]]),
              distortion_coeffs=torch.tensor([[-0.05, 0.01, 0.0005, -0.0005, 0.001]]),
              extrinsic_matrix=torch.eye(4)[None], world_up_vector=torch.tensor([0., -1., 0.]), default_fov_degrees=55,
              internal_batch_size=0, antialias_factor=1, num_aug=5, average_aug=True, skeleton='', suppress_implausible_poses=False)
    return frames, boxes, counts, kw


def _check_pyramid(frames, l1, l2):
    """Levels 1 and 2 within 20 u of fp64: the decode table's powf (4 ulp, 8 u) and i/255 rounding (2.2 u), then three
    additions and the exact * 0.25 per level."""
    ref = pm.pyramid(frames)
    worst = 0.0
    for d, r in ((l1, ref[1]), (l2, ref[2])):
        assert d.shape == r.shape
        worst = max(worst, _ratio(d, r, 20 * pm.U32 * r + 1e-300))
    assert worst <= 1, worst
    return ref, worst


def _check_setup(boxes, k_box, d_box, up, rf, sc, res, af, new_k, rot, inv, lev, tol=1e-4):
    """Device matrices within the derived element-wise bounds of pm.crop_setup_bound around the fp64 setup; levels equal
    except where -log2(scale * af) lies within `tol` of an integer (fp32 and fp64 may round to either side there).
    -> (fp64 setup, invproj bound, exception mask, worst ratios)."""
    nk, R, iv, log_lev, lv = pm.crop_setup(boxes.to(F64), k_box, d_box, up, rf, sc, res, af)
    ek, er, ei = pm.crop_setup_bound(boxes, k_box, d_box, up, rf, sc, res, af)
    ratios = {name: _ratio(a, b, e + 1e-300) for name, a, b, e in (('new_K', new_k, nk, ek), ('R', rot, R, er), ('invproj', inv, iv, ei))}
    near = (log_lev - torch.round(log_lev)).abs() < tol
    mismatch = lev.long() != lv
    assert not (mismatch & ~near).any(), (log_lev[mismatch & ~near], lev[mismatch & ~near], lv[mismatch & ~near])
    assert all(v <= 1 for v in ratios.values()), ratios
    return (nk, R, iv, lv), ei, mismatch, ratios


def _check_warp(frames, pyr_dev, levels64, k_box, d_box, inv_dev, lev_dev, gam, res, ids, num_aug, af, setup64=None, inv_err=None,
                mismatch=None, crops=None):
    """The kernel on the device's own matrices vs fp64 on the same fp32 matrices; with setup64, also the device chain vs
    fp64 on the fp64 setup, the kernel's matrices known only to lie within inv_err of it (the device level where the two
    levels legitimately differ).  crops: the device crops to judge (default: the kernel on inv_dev).  -> (crops, ratios)."""
    from metrabs_b200.multiperson import warping
    ge = (gam / 2.2).float()
    if crops is None:
        crops = warping.warp_images_with_pyramid(frames, pyr_dev, k_box.float(), inv_dev, d_box.float(), lev_dev, ge, res, ids,
                                                 num_aug, af)
    n = k_box.shape[0]
    lin_dev = pm.to_linear(crops, ge, n)
    out = {}
    if inv_dev is not None:
        _, lin, bound = pm.warp(levels64, k_box, inv_dev, d_box, lev_dev, ge, res, ids, num_aug, af, with_bound=True)
        out['warp_kernel'] = _ratio(lin_dev, lin, bound)
        out['coord_bound_px'] = pm.warp.last_coord_bound
        del lin, bound
    if setup64 is not None:
        _, _, inv64, lev64 = setup64
        lev_c = torch.where(mismatch, lev_dev.long(), lev64)
        _, lin, bound = pm.warp(levels64, k_box, inv64, d_box, lev_c, ge, res, ids, num_aug, af, with_bound=True, invproj_err=inv_err)
        out['warp_chain'] = _ratio(lin_dev, lin, bound)
        out['chain_coord_bound_px'] = pm.warp.last_coord_bound
    return crops, out


def _check_merge(est, poses, rot, flip, k_box, d_box, ext_inv, skel, average, jt=None):
    """The device merge against the fp64 merge of the same poses; 2D elements whose projection is ill-conditioned (the
    bound is infinite: |z| within twice its own rounding of 0) are counted, not compared.  -> (worst 3D, worst 2D, #ill)."""
    n, A = k_box.shape[0], len(flip)
    js = len(skel) if skel is not None else (jt.shape[1] if jt is not None else poses.shape[1])
    shape = (n, js, 3) if average else (n, A, js, 3)
    o3 = torch.empty(shape, device=poses.device)
    o2 = torch.empty(shape[:-1] + (2,), device=poses.device)
    est._tta_merge(poses, rot, flip, k_box, d_box, ext_inv, skel, average, o3, o2)
    r3, r2, e3, e2 = pm.tta_merge(poses, rot, flip, est.joint_info.mirror_mapping, jt, skel, k_box, d_box, ext_inv, average,
                                  with_bound=True)
    ok2 = torch.isfinite(e2)
    w3 = _ratio(o3, r3, e3)
    w2 = float(((o2.to(F64) - r2).abs() / e2)[ok2].max()) if ok2.any() else 0.0
    assert torch.isfinite(o3).all() and w3 <= 1 and w2 <= 1, (w3, w2)
    return w3, w2, int((~ok2).sum())


def test_frames_leg_at_benchmark_shape(dev):
    import bench
    from metrabs_b200.multiperson import Pose3dEstimator, warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    t0 = time.perf_counter()
    args = types.SimpleNamespace(size='l', side=256, precision='bf16', stride=32, depth=8, joints=24)
    model = bench.build_model(args, dev)
    j = args.joints
    model.joint_names = [f'j{i}' for i in range(j)]
    model.joint_edges = [[0, 1]]
    est = Pose3dEstimator(model, {'': dict(indices=list(range(j)), names=model.joint_names, edges=[[0, 1]])}, None)
    frames, boxes, counts, kw = _bench_scene(dev)
    res_all = est._estimate_poses_batched(frames, boxes, **kw)
    n = sum(counts)
    k_box = kw['intrinsic_matrix'].repeat(n, 1, 1).to(dev)
    d_box = kw['distortion_coeffs'].repeat(n, 1).to(dev)
    up = torch.tensor([[0., -1., 0.]]).repeat(n, 1).to(dev)
    ext_inv = torch.eye(4).repeat(n, 1, 1).to(dev)
    ids = torch.repeat_interleave(torch.arange(8), torch.tensor(counts)).to(dev)
    bx = torch.cat(boxes).to(dev)
    gam, sc, fl, rf = aug_parameters(5)
    worst = {}
    pyr = warping.build_pyramid(frames)
    levels64, worst['pyramid'] = _check_pyramid(frames, *pyr)
    new_k, rot, inv, lev = warping.crop_setup(bx, k_box, d_box, up, rf, sc, 256, 1)
    setup64, inv_err, mismatch, w = _check_setup(bx, k_box.to(F64), d_box, up, rf.to(dev), sc.to(dev), 256, 1, new_k, rot, inv, lev)
    worst.update(w)
    print(f'crop setup: {int(mismatch.sum())} of {len(lev)} levels differ from fp64, all where -log2 lies within 1e-4 of an integer')
    crops, w = _check_warp(frames, pyr, levels64, k_box.to(F64), d_box.to(F64), inv, lev, gam, 256, ids, 5, 1, setup64, inv_err, mismatch)
    assert w['warp_kernel'] <= 1 and w['warp_chain'] <= 1, w
    worst.update(w)
    # negative control: a setup whose principal point is off by 0.05 crop px fails the invproj bound and the chain check
    T = torch.eye(3, device=dev)
    T[0, 2] = 0.05
    inv_off = (inv @ T).contiguous()
    r_inv = _ratio(inv_off, setup64[2], inv_err)
    off = warping.warp_images_with_pyramid(frames, pyr, k_box, inv_off, d_box, lev, (gam / 2.2).float(), 256, ids, 5, 1)
    _, w_off = _check_warp(frames, pyr, levels64, k_box.to(F64), d_box.to(F64), None, lev, gam, 256, ids, 5, 1, setup64, inv_err,
                           mismatch, crops=off)
    print(f'invproj off by 0.05 crop px: invproj ratio {r_inv:.3g}, warp chain ratio {w_off["warp_chain"]:.3g}')
    assert r_inv > 10 and w_off['warp_chain'] > 10
    del off
    # the crop model on those crops, and the staged calls against the pipeline, bit for bit
    poses = model((crops, new_k.reshape(-1, 3, 3)))
    p3 = torch.empty(n, j, 3, device=dev)
    p2 = torch.empty(n, j, 2, device=dev)
    est._tta_merge(poses, rot, fl, k_box, d_box, ext_inv, None, True, p3, p2)
    assert torch.equal(torch.cat(res_all['poses3d']), p3) and torch.equal(torch.cat(res_all['poses2d']), p2)
    # merge: jt == nullptr (what the bench runs), then a joint transform + skeleton on the same poses, mean and per-aug
    w3, w2, ill = _check_merge(est, poses, rot, fl, k_box, d_box, ext_inv, None, True)
    assert ill == 0  # every 2D element compared
    worst.update(merge3d=w3, merge2d=w2)
    g = torch.Generator().manual_seed(5)
    jt = torch.cat([torch.eye(j), torch.rand(j, 6, generator=g) / j], 1)
    est_jt = Pose3dEstimator(model, {'': dict(indices=list(range(j + 6)), names=[], edges=[])}, jt)
    skel = list(range(0, j + 6, 2))
    for avg in (True, False):
        w3, w2, ill2 = _check_merge(est_jt, poses, rot, fl, k_box, d_box, ext_inv, skel, avg, jt)
        assert ill2 == 0
        worst[f'merge3d_jt_avg{int(avg)}'], worst[f'merge2d_jt_avg{int(avg)}'] = w3, w2
    torch.cuda.synchronize()
    print('worst |dev - fp64| / bound per stage: ' + ', '.join(f'{k} {v:.3g}' for k, v in worst.items()))
    print(f'wall time {time.perf_counter() - t0:.1f} s')


EDGES = [  # (H, W, af, n_dist, num_aug, res)
    (719, 1279, 1, 5, 5, 64),
    (37, 53, 2, 12, 2, 8),
    (64, 90, 4, 0, 1, 8),
    (720, 1280, 1, 8, 16, 48),
]


@pytest.mark.parametrize('h,w,af,n_dist,num_aug,res', EDGES)
def test_crop_stages_edges(dev, h, w, af, n_dist, num_aug, res):
    from metrabs_b200.multiperson import warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    g = torch.Generator().manual_seed(h * 7 + w)
    frames = torch.randint(0, 256, (2, 3, h, w), generator=g, dtype=torch.uint8).to(dev)
    boxes = torch.tensor([
        [0.3 * w, 0.3 * h, 0.4 * w, 0.5 * h, 1.],     # inside
        [-0.2 * w, 0.1 * h, 0.4 * w, 0.5 * h, 1.],    # partly outside
        [1.2 * w, 1.3 * h, 0.2 * w, 0.2 * h, 1.],     # wholly outside
        [0.5 * w, 0.5 * h, res / 4, res / 3, 1.],     # small: level 0, upsampled
        [w / 2 - 3 * res * af, h / 2 - 3 * res * af, 6 * res * af, 6 * res * af, 1.],  # large: level 2
    ]).to(dev)
    n = len(boxes)
    # fp32 values, held in fp64: the device and the fp64 restatement see the same inputs
    k = torch.tensor([[0.8 * w, 0., w / 2 - 0.3], [0., 0.8 * w, h / 2 + 0.4], [0., 0., 1.]]).to(F64)
    d12 = torch.tensor([-0.08, 0.02, 0.001, -0.0015, 0.003, 0.01, -0.005, 0.002, 0.0004, -0.0003, 0.0002, 0.0001]).to(F64)
    k_box = k.repeat(n, 1, 1).to(dev)
    d_box = d12[:n_dist].repeat(n, 1).to(dev)
    up = torch.tensor([[0., -1., 0.]]).repeat(n, 1).to(dev)
    ids = torch.tensor([0, 1, 0, 1, 1], device=dev)
    gam, sc, fl, rf = aug_parameters(num_aug)
    pyr = warping.build_pyramid(frames)
    levels64, wp = _check_pyramid(frames, *pyr)
    new_k, rot, inv, lev = warping.crop_setup(boxes, k_box.float(), d_box.float(), up, rf, sc, res, af)
    setup64, inv_err, mismatch, ws = _check_setup(boxes, k_box, d_box, up, rf.to(dev), sc.to(dev), res, af, new_k, rot, inv, lev)
    assert {0, 2} <= set(lev.tolist())
    _, ww = _check_warp(frames, pyr, levels64, k_box, d_box, inv, lev, gam, res, ids, num_aug, af, setup64, inv_err, mismatch)
    assert ww['warp_kernel'] <= 1 and ww['warp_chain'] <= 1, ww
    print(f'{h}x{w} af={af} n_dist={n_dist} A={num_aug}: pyramid {wp:.3g}, ' + ', '.join(f'{k} {v:.3g}' for k, v in {**ws, **ww}.items())
          + f'; levels {sorted(set(lev.tolist()))}, {int(mismatch.sum())} near-integer level differences')


@pytest.mark.parametrize('average', [True, False])
@pytest.mark.parametrize('num_aug', [2, 16])
def test_merge_edges_j122(dev, average, num_aug):
    """J = 122 joints named l.../r... (a real mirror swap), a joint transform to 130 joints, a 40-joint skeleton."""
    from metrabs_b200.multiperson import Pose3dEstimator
    from metrabs_b200.multiperson.joint_info import JointInfo
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    J, n = 122, 3
    names = ['pelv'] + [f'{s}j{i}' for i in range(60) for s in 'lr'] + ['neck']
    ji = JointInfo(names, [(0, 1)])
    assert ji.mirror_mapping[1:3] == [2, 1]
    g = torch.Generator().manual_seed(num_aug)
    poses = torch.cat([600 * torch.randn(num_aug * n, J, 2, generator=g), 2000 + 2000 * torch.rand(num_aug * n, J, 1, generator=g)], -1)
    jt = torch.cat([torch.eye(J), torch.rand(J, 8, generator=g) * (torch.rand(J, 8, generator=g) < 0.1)], 1)
    skel = torch.randperm(J + 8, generator=g)[:40].tolist()

    class Table(torch.nn.Module):
        joint_names, joint_edges, input_resolution, device = names, [(0, 1)], np.int32(64), 'cuda'
    est = Pose3dEstimator(Table(), {'': dict(indices=skel, names=[], edges=[])}, jt, joint_info=ji)
    gam, sc, fl, rf = aug_parameters(num_aug)
    a = torch.rand(num_aug * n, generator=g) * 2 * math.pi
    rot = torch.stack([torch.stack([a.cos(), -a.sin(), 0 * a], -1), torch.stack([a.sin(), a.cos(), 0 * a], -1),
                       torch.tensor([0., 0., 1.]).expand(num_aug * n, 3)], -2)
    k_box = torch.tensor([[1000., 0, 640], [0, 1000., 360], [0, 0, 1]]).repeat(n, 1, 1)
    d_box = torch.tensor([-0.1, 0.02, 0.001, -0.001, 0.002, 0.01, -0.004, 0.001, 0.0002, -0.0001, 0.0001, 0.00005]).repeat(n, 1)
    ext = torch.eye(4).repeat(n, 1, 1)
    ext[:, :3, 3] = torch.tensor([100., -200., 50.])
    t = [x.to(dev).contiguous() for x in (poses, rot.reshape(num_aug, n, 3, 3), k_box, d_box, ext)]
    w3, w2, ill = _check_merge(est, t[0], t[1], fl, t[2], t[3], t[4], skel, average, jt.to(dev))
    assert ill == 0
    # a dropped swap must show: the same merge with every flip off exceeds the bound
    if fl.any():
        o3 = torch.empty((n, 40, 3) if average else (n, num_aug, 40, 3), device=dev)
        o2 = torch.empty(o3.shape[:-1] + (2,), device=dev)
        est._tta_merge(t[0], t[1], torch.zeros_like(fl), t[2], t[3], t[4], skel, average, o3, o2)
        r3, _, e3, _ = pm.tta_merge(t[0], t[1], fl, ji.mirror_mapping, jt.to(dev), skel, t[2], t[3], t[4], average, with_bound=True)
        assert _ratio(o3, r3, e3) > 100
    print(f'J=122 A={num_aug} average={average}: merge 3D {w3:.3g}, 2D {w2:.3g}')


@pytest.mark.parametrize('group', ['crowd', 'wide'])
def test_pose_filter_crowd_vs_reference(dev, golden_dir, group):
    """Image 0 of `crowd` has 170 boxes: every box past the 128th must be judged like the others."""
    from metrabs_b200.multiperson import plausibility_check
    g = np.load(os.path.join(golden_dir, 'multiperson_filter_crowd.npz'), allow_pickle=False)
    p3, p2, boxes = (torch.from_numpy(g[f'{group}_{k}']).to(dev) for k in ('poses3d', 'poses2d', 'boxes'))
    plausible, keep = plausibility_check.filter_poses(p3, p2, boxes, g[f'{group}_n_per_image'].tolist(), g[f'{group}_bones'],
                                                      g[f'{group}_mean_bones'])
    want_p, want_k = g[f'{group}_plausible'], g[f'{group}_keep']
    bad = np.nonzero((plausible.cpu().numpy() != want_p) | (keep.cpu().numpy() != want_k))[0]
    assert len(bad) == 0, f'boxes judged unlike the reference: {bad.tolist()}'


def test_pose_filter_too_many_boxes_raises(dev):
    from metrabs_b200 import _lib
    from metrabs_b200.multiperson import plausibility_check
    n = 20000  # 14 B each: more than one block's shared memory holds
    p3 = torch.zeros(n, 2, 4, 3, device=dev)
    with pytest.raises(_lib.MetrabsB200Error, match='shared memory'):
        plausibility_check.filter_poses(p3, torch.zeros(n, 2, 4, 2, device=dev), torch.ones(n, 5, device=dev), [n], [(0, 1)], [100.])
