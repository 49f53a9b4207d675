"""GPU: crop generation at antialias factors 5..16 (warp_crops_aa_kernel) against the fp64 restatement
oracle/port_antialias.py element by element within its derived bound, and against goldens of the unmodified reference
(tests/golden/multiperson_antialias.npz: _get_crops and _estimate_poses_batched at f = 5 and 8); crops bit-identical
from run to run and whatever other crops share the launch; the refused factors; and no res*f render in device memory."""
import os

import numpy as np
import pytest
import torch

from metrabs_b200._lib import MetrabsB200Error
from oracle import port
from oracle import port_antialias as pa
from oracle import port_multiperson as pm

pytestmark = pytest.mark.gpu
F64 = torch.float64


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def G(golden_dir):
    return np.load(os.path.join(golden_dir, 'multiperson_antialias.npz'), allow_pickle=False)


def _scene(G, dev):
    images = pa.golden_frames().to(dev)
    boxes = [torch.from_numpy(G[f'boxes_{i}']) for i in range(int(G['n_images']))]
    return images, boxes, torch.from_numpy(G['intrinsics']), torch.from_numpy(G['distortion']), \
        torch.from_numpy(G['extrinsics']), torch.from_numpy(G['world_up'])


def _per_box(G, dev):
    images, boxes, intr, dist, ext, up = _scene(G, dev)
    n_box = torch.tensor([len(b) for b in boxes])
    k_box = torch.repeat_interleave(intr, n_box, dim=0)
    d_box = torch.repeat_interleave(dist, n_box, dim=0)
    cam_up = torch.repeat_interleave(torch.einsum('c,bCc->bC', up, ext[..., :3, :3]), n_box, dim=0)
    ids = torch.repeat_interleave(torch.arange(len(boxes)), n_box)
    return images, torch.cat(boxes).to(dev), k_box.to(dev), d_box.to(dev), cam_up.to(dev), ids


def _crops(images, pyr, boxes, k_box, d_box, cam_up, ids, num_aug, res, af):
    from metrabs_b200.multiperson import warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    gam, sc, fl, rf = aug_parameters(num_aug)
    new_k, rot, inv, lev = warping.crop_setup(boxes, k_box, d_box, cam_up, rf, sc, res, af)
    ge = (gam / 2.2).float()
    crops = warping.warp_images_with_pyramid(images, pyr, k_box, inv, d_box, lev, ge, res, ids, num_aug, af)
    return crops, inv, lev, ge


@pytest.mark.parametrize('af', [5, 6, 8, 16])
def test_crops_within_bound_of_fp64(dev, G, af):
    """The kernel on the device's own fp32 matrices against fp64 on the same matrices; res 44 is not a multiple of the
    8-pixel tile."""
    from metrabs_b200.multiperson import warping
    images, boxes, k_box, d_box, cam_up, ids = _per_box(G, dev)
    pyr = warping.build_pyramid(images)
    res, num_aug = 44, 5
    crops, inv, lev, ge = _crops(images, pyr, boxes, k_box, d_box, cam_up, ids, num_aug, res, af)
    _, lin, bound = pa.warp(pm.pyramid(images), k_box, inv, d_box, lev, ge, res, ids, num_aug, af, with_bound=True)
    ratio = float(((pm.to_linear(crops, ge, len(boxes)) - lin).abs() / bound).max())
    print(f'af={af}: worst |device - fp64| / bound {ratio:.3f}, median bound {float(bound.median()):.2e}, largest coordinate '
          f'bound {pa.warp.last_coord_bound:.2e} px, levels {sorted(set(lev.tolist()))}')
    assert ratio <= 1
    assert torch.isfinite(crops).all()


@pytest.mark.parametrize('af,res', [(5, 36), (8, 32)])
def test_crops_vs_reference(dev, G, af, res):
    """Bars as for factors 1 and 2 (test_gpu_multiperson.py): on the reference's own inverse projections 5e-5 in linear
    light, with the device's setup 1e-4; 5e-4 gamma-encoded where the linear value is at least 1e-3.  Below that the
    encoding x ** (gamma / 2.2) has a slope past 40: the filter's 2f taps give the pixels along the frame border linear
    values down to 1e-7, where the two fp32 setups' last-bit coordinate differences become 7e-4 gamma-encoded."""
    from metrabs_b200.multiperson import warping
    images, boxes, k_box, d_box, cam_up, ids = _per_box(G, dev)
    pyr = warping.build_pyramid(images)
    tag = f'crops_r{res}_af{af}'
    crops, inv, lev, ge = _crops(images, pyr, boxes, k_box, d_box, cam_up, ids, 5, res, af)
    inv_ref = torch.from_numpy(G[tag + '_invproj']).to(dev).contiguous()
    crops_ref_inv = warping.warp_images_with_pyramid(images, pyr, k_box, inv_ref, d_box, lev, ge, res, ids, 5, af)
    ref = torch.from_numpy(G[tag]).to(dev)
    n = len(boxes)
    for name, c, bar in (('reference matrices', crops_ref_inv, 5e-5), ('device setup', crops, 1e-4)):
        lin_ref = pm.to_linear(ref, ge, n)
        e_lin = float((pm.to_linear(c, ge, n) - lin_ref).abs().max())
        e = float((c - ref).abs()[lin_ref >= 1e-3].max())
        print(f'{tag}, {name}: max abs crop error linear {e_lin:.2e}, gamma-encoded {e:.2e}')
        assert e_lin < bar and e < 5e-4, name


def _device_estimator(G, golden_dir):
    from metrabs_b200.multiperson import Pose3dEstimator
    from metrabs_b200.multiperson.joint_info import JointInfo
    from tests import helpers
    g = np.load(os.path.join(golden_dir, 'tiny_s64_j8.npz'), allow_pickle=False)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith('sd/')}
    m = helpers.device_model('efficientnetv2-tiny', port.PathConfig(proc_side=64), 8, sd, precision='fp32')
    m.joint_names, m.joint_edges = G['joint_names'], G['joint_edges']
    ji = JointInfo(G['joint_names'], G['joint_edges'])
    assert ji.mirror_mapping == G['mirror'].tolist()
    skel = {'': dict(indices=list(range(10)), names=[f'k{i}' for i in range(10)], edges=[[0, 1]])}
    return Pose3dEstimator(m, skel, G['joint_transform'], joint_info=ji)


@pytest.mark.parametrize('af', [8, 5])
def test_estimate_poses_vs_reference(dev, G, golden_dir, af):
    """frames + boxes -> poses3d through this package's Pose3dEstimator at antialias_factor f against the reference's
    _estimate_poses_batched on the same weights (bars as test_gpu_multiperson.py: 1e-3 on poses3d)."""
    est = _device_estimator(G, golden_dir)
    images, boxes, intr, dist, ext, up = _scene(G, dev)
    res = est.estimate_poses_batched(images, [b[:, :4] for b in boxes], intr, dist, ext, up, 55, 64, antialias_factor=af)
    for i in range(2):
        e3 = port.relative_error(res['poses3d'][i].float().cpu(), torch.from_numpy(G[f'pipe_af{af}_p3d_{i}']))
        print(f'af={af} image {i}: poses3d relative error vs the reference caller {e3:.2e}')
        assert res['poses3d'][i].shape == G[f'pipe_af{af}_p3d_{i}'].shape
        assert e3 < 1e-3


def test_crops_do_not_depend_on_the_launch(dev, G):
    """Two runs give the same bits, and each crop of a box rendered alone equals its crop in the full launch."""
    from metrabs_b200.multiperson import warping
    images, boxes, k_box, d_box, cam_up, ids = _per_box(G, dev)
    pyr = warping.build_pyramid(images)
    n, A, res = len(boxes), 5, 44
    for af in (5, 8, 16):
        crops, inv, lev, ge = _crops(images, pyr, boxes, k_box, d_box, cam_up, ids, A, res, af)
        again = warping.warp_images_with_pyramid(images, pyr, k_box, inv, d_box, lev, ge, res, ids, A, af)
        assert torch.equal(crops, again), af
        for b in range(n):
            rows = torch.arange(A, device=dev) * n + b
            alone = warping.warp_images_with_pyramid(images, pyr, k_box[b:b + 1], inv[rows].contiguous(), d_box[b:b + 1],
                                                     lev[rows].contiguous(), ge, res, ids[b:b + 1], A, af)
            assert torch.equal(alone, crops[rows]), (af, b)


@pytest.mark.parametrize('af', [3, 17, 0])
def test_refused_factors(dev, G, af):
    from metrabs_b200.multiperson import warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    images, boxes, k_box, d_box, cam_up, ids = _per_box(G, dev)
    gam, sc, fl, rf = aug_parameters(2)
    with pytest.raises(MetrabsB200Error, match=r'5\.\.16'):
        warping.crop_setup(boxes, k_box, d_box, cam_up, rf, sc, 32, af)
    _, _, inv, lev = warping.crop_setup(boxes, k_box, d_box, cam_up, rf, sc, 32, 1)
    with pytest.raises(MetrabsB200Error, match=r'5\.\.16'):
        warping.warp_images_with_pyramid(images, warping.build_pyramid(images), k_box, inv, d_box, lev, gam / 2.2, 32, ids, 2, af)


def test_no_render_in_device_memory(dev):
    """256 crops of 384 x 384 at f = 8 from a 3840 x 2160 frame: the res*f render would be 29 GB; the launch allocates
    no more than the crops and the pyramid (plus the per-crop matrices and 1 MB for the small argument tensors)."""
    from metrabs_b200.multiperson import warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    g = torch.Generator().manual_seed(5)
    h, w, n, A, res, af = 2160, 3840, 64, 4, 384, 8
    frames = torch.randint(0, 256, (1, 3, h, w), generator=g, dtype=torch.uint8).to(dev)
    xy = torch.rand(n, 2, generator=g) * torch.tensor([w - 800., h - 1000.])
    wh = torch.tensor([400., 900.]) * (0.5 + torch.rand(n, 2, generator=g))
    boxes = torch.cat([xy, wh], 1).to(dev)
    k_box = torch.tensor([[2000., 0, w / 2], [0, 2000., h / 2], [0, 0, 1]]).repeat(n, 1, 1).to(dev)
    d_box = torch.tensor([[-0.05, 0.01, 0.0005, -0.0005, 0.001]]).repeat(n, 1).to(dev)
    up = torch.tensor([0., -1., 0.]).repeat(n, 1).to(dev)
    ids = torch.zeros(n, dtype=torch.int32)
    gam, sc, fl, rf = aug_parameters(A)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    pyr = warping.build_pyramid(frames)
    _, _, inv, lev = warping.crop_setup(boxes, k_box, d_box, up, rf, sc, res, af)
    crops = warping.warp_images_with_pyramid(frames, pyr, k_box, inv, d_box, lev, gam / 2.2, res, ids, A, af)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    crop_bytes = crops.numel() * 4
    pyr_bytes = sum(t.numel() * 4 for t in pyr)
    print(f'peak allocation {peak / 2**20:.1f} MiB: crops {crop_bytes / 2**20:.1f} MiB, pyramid {pyr_bytes / 2**20:.1f} MiB')
    assert crops.shape == (A * n, 3, res, res) and torch.isfinite(crops).all()
    assert peak <= crop_bytes + pyr_bytes + 2 ** 20
