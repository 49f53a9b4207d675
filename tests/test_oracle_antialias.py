"""CPU: the fp64 restatement of crop generation at antialias factors 5..16 (oracle/port_antialias.py).  Its filter is
F.interpolate(bilinear, antialias=True) for every factor; with it the crops and poses reproduce the unmodified reference
(tests/golden/multiperson_antialias.npz, oracle/gen_golden_antialias.py); its error bound holds for an fp32 evaluation of
the chain and rejects a shifted render and the wrong filter; and the C header and the ctypes binding still agree."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from metrabs_b200 import _lib
from metrabs_b200.multiperson.multiperson_model import aug_parameters
from oracle import port
from oracle import port_antialias as pa
from oracle import port_multiperson as pm

F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def G(golden_dir):
    return np.load(os.path.join(golden_dir, 'multiperson_antialias.npz'), allow_pickle=False)


def _per_box(G):
    boxes = [torch.from_numpy(G[f'boxes_{i}']) for i in range(int(G['n_images']))]
    n_box = torch.tensor([len(b) for b in boxes])
    intr, dist, ext, up = (torch.from_numpy(G[k]) for k in ('intrinsics', 'distortion', 'extrinsics', 'world_up'))
    k_box = torch.repeat_interleave(intr, n_box, dim=0)
    d_box = torch.repeat_interleave(dist, n_box, dim=0)
    cam_up = torch.repeat_interleave(torch.einsum('c,bCc->bC', up, ext[..., :3, :3]), n_box, dim=0)
    ext_inv = torch.repeat_interleave(torch.linalg.inv(ext), n_box, dim=0)
    ids = torch.repeat_interleave(torch.arange(len(boxes)), n_box)
    return pa.golden_frames(), torch.cat(boxes), k_box, d_box, cam_up, ext_inv, ids


@pytest.mark.parametrize('f', list(range(5, 17)))
def test_filter_is_torch_antialiased_bilinear(f):
    g = torch.Generator().manual_seed(f)
    for res in (13, 21):  # neither a multiple of the kernel's 8-pixel tile
        x = torch.rand(2, 3, res * f, res * f, generator=g, dtype=F64)
        ref = F.interpolate(x, size=(res, res), mode='bilinear', align_corners=False, antialias=True)
        assert float((pa.shrink(x, res) - ref).abs().max()) < 1e-12, (f, res)


@pytest.mark.parametrize('af,res', [(5, 36), (8, 32)])
def test_crops_reproduce_reference(G, af, res):
    """Same bars as the factors 1 and 2 (test_oracle_multiperson.py): 5e-5 in linear light, 5e-4 gamma-encoded where the
    linear value is at least 1e-3 (test_gpu_antialias.py: along the frame border the filter gives linear values down to
    1e-7, where x ** (gamma / 2.2) magnifies last-bit differences without bound)."""
    images, boxes, k_box, d_box, up, _, ids = _per_box(G)
    gam, sc, fl, rf = aug_parameters(5)
    new_k, R, inv, _, lev = pm.crop_setup(boxes, k_box, d_box, up, rf, sc, res, af)
    tag = f'crops_r{res}_af{af}'
    assert float(((new_k - torch.from_numpy(G[tag + '_newk']).to(F64)).abs() / new_k.abs().max()).max()) < 2e-6
    assert float((R - torch.from_numpy(G[tag + '_rot']).to(F64)).abs().max()) < 2e-6
    crops, _, _ = pa.warp(pm.pyramid(images), k_box, torch.from_numpy(G[tag + '_invproj']), d_box, lev, gam / 2.2, res, ids, 5, af)
    ref = torch.from_numpy(G[tag]).to(F64)
    lin_ref = pm.to_linear(ref, gam / 2.2, len(boxes))
    e_lin = float((pm.to_linear(crops, gam / 2.2, len(boxes)) - lin_ref).abs().max())
    e = float((crops - ref).abs()[lin_ref >= 1e-3].max())
    print(f'{tag}: levels {sorted(set(lev.tolist()))}, max abs error linear {e_lin:.2e}, gamma-encoded {e:.2e}')
    assert e_lin < 5e-5 and e < 5e-4


@pytest.mark.parametrize('af', [5, 8])
def test_poses_reproduce_reference(G, golden_dir, af):
    """Restated crops -> the restated tiny crop model -> the restated TTA merge, against the reference's
    _estimate_poses_batched on the same weights (bar 1e-3, the joint tolerance)."""
    images, boxes, k_box, d_box, up, ext_inv, ids = _per_box(G)
    gam, sc, fl, rf = aug_parameters(5)
    new_k, R, inv, _, lev = pm.crop_setup(boxes, k_box, d_box, up, rf, sc, 64, af)
    crops, _, _ = pa.warp(pm.pyramid(images), k_box, inv, d_box, lev, gam / 2.2, 64, ids, 5, af)
    w = np.load(os.path.join(golden_dir, 'tiny_s64_j8.npz'), allow_pickle=False)
    sd = {k[3:]: torch.from_numpy(w[k]) for k in w.files if k.startswith('sd/')}
    with torch.inference_mode():
        poses = port.metrabs_forward(sd, port.effnet_spec('efficientnetv2-tiny'), port.PathConfig(proc_side=64), 8,
                                     crops.float(), new_k.reshape(-1, 3, 3).float())
    p3, _ = pm.tta_merge(poses, R, fl, G['mirror'], torch.from_numpy(G['joint_transform']), None, k_box, d_box, ext_inv, True)
    for i, sl in enumerate((slice(0, 3), slice(3, 5))):
        e = port.relative_error(p3[sl].float(), torch.from_numpy(G[f'pipe_af{af}_p3d_{i}']))
        print(f'af={af} image {i}: poses3d relative error {e:.2e}')
        assert e < 1e-3


def _fp32_chain(images, K, inv, d12, lev, gexp, res, ids, A, af, shift=0.0, shrink=None):
    """The chain in fp32: the render with fp32 coordinates on an fp32 pyramid, then torch's own fp32 antialiased resize
    (or `shrink`), then the gamma."""
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
        hx, hy, hz = (M[i, 0] * nx + M[i, 1] * ny + M[i, 2] for i in range(3))
        dx, dy = pm.distort(hx / hz, hy / hz, d)
        u = kl[c, 0, 0] * dx + kl[c, 0, 1] * dy + kl[c, 0, 2] + shift
        v = kl[c, 1, 0] * dx + kl[c, 1, 1] * dy + kl[c, 1, 2]
        s = pm.sample(levels[int(lev[c])][int(ids[c % n])], u, v)[None]
        out.append((shrink(s) if shrink else F.interpolate(s, size=(res, res), mode='bilinear', antialias=True))[0])
    ge = torch.as_tensor(gexp).float().repeat_interleave(n)[:, None, None, None]
    return torch.stack(out) ** ge


@pytest.mark.parametrize('af', [5, 16])
def test_bound_holds_for_fp32_chain_and_rejects_wrong_warps(af):
    g = torch.Generator().manual_seed(3)
    h, w = 61, 83
    images = torch.randint(0, 256, (2, 3, h, w), generator=g, dtype=torch.uint8)
    boxes = torch.tensor([[10., 5., 30., 50., 1.], [-15., 20., 60., 60., 1.], [3., 3., w - 6., h - 6., 1.]])
    K = torch.tensor([[w * 0.9, 0., w / 2], [0., w * 0.9, h / 2], [0., 0., 1.]]).repeat(3, 1, 1)
    d12 = torch.tensor([-0.1, 0.03, 0.001, -0.002, 0.004, 0.02, -0.01, 0.003, 0.0005, -0.0004, 0.0003, 0.0002]).repeat(3, 1)
    up, ids = torch.tensor([0., -1., 0.]).repeat(3, 1), torch.tensor([0, 1, 0])
    gam, sc, fl, rf = aug_parameters(2)
    res = 7  # the whole frame onto 7 pixels: levels 0 and 1 at f = 5
    _, _, inv, _, lev = pm.crop_setup(boxes, K, d12, up, rf, sc, res, af)
    inv32, ge = inv.float(), (gam / 2.2).float()
    _, lin, bound = pa.warp(pm.pyramid(images), K, inv32, d12, lev, ge, res, ids, 2, af, with_bound=True)
    assert af > 5 or len(set(lev.tolist())) >= 2
    chain = pm.to_linear(_fp32_chain(images, K, inv32, d12, lev, ge, res, ids, 2, af), ge, 3)
    ratio = float(((chain - lin).abs() / bound).max())
    print(f'af={af}: worst |fp32 chain - fp64| / bound {ratio:.3f}, median bound {float(bound.median()):.2e}')
    assert ratio <= 1
    wrong = {'0.05 px shift': _fp32_chain(images, K, inv32, d12, lev, ge, res, ids, 2, af, shift=0.05),
             'box filter': _fp32_chain(images, K, inv32, d12, lev, ge, res, ids, 2, af, shrink=lambda s: F.avg_pool2d(s, af, af))}
    for name, x in wrong.items():
        r = float(((pm.to_linear(x, ge, 3) - lin).abs() / bound).max())
        print(f'af={af}, {name}: worst ratio {r:.3g}')
        assert r > 10, name


def test_restatement_refuses_factors_outside_its_range():
    for af in (4, 17):
        with pytest.raises(ValueError):
            pa.warp(None, torch.zeros(1, 3, 3), None, torch.zeros(1, 5), [0], [1.0], 8, [0], 1, af)


def test_header_and_binding_agree():
    """The antialias factor stays an int32 field of both argument structs; the ABI version is unchanged."""
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    flat = re.sub(r'\s+', ' ', re.sub(r'/\*.*?\*/', '', src, flags=re.S))
    assert re.search(r'#define MTB_ABI_VERSION (\d+)', src).group(1) == str(_lib.MTB_ABI_VERSION) == '2'
    for struct, cls in (('mtb_crop_setup_args', _lib.MtbCropSetupArgs), ('mtb_warp_args', _lib.MtbWarpArgs)):
        body = re.search(r'typedef struct \{([^}]*)\} ' + struct + ';', flat).group(1)
        names = [n for decl in body.split(';') if decl.strip() for n in re.findall(r'\*?\s*(\w+)\s*(?:,|$)', decl.strip())]
        assert names == [f for f, _ in cls._fields_], struct
        assert dict(cls._fields_)['antialias_factor'] is C.c_int32
    assert 'int mtb_warp_crops(const mtb_warp_args* args, void* stream);' in flat
    assert 'int mtb_crop_setup(const mtb_crop_setup_args* args, void* stream);' in flat

