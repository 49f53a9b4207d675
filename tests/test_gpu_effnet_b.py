"""GPU: EfficientNet-B0..B7 (metrabs_b200.backbones.efficientnet.efficientnet_bN) and the pooling 16-bit 5x5 depthwise
kernel (dwconv5x5_16b_kernel with SE pooling, mtb_kernel DW_5X5_POOL_16B).

* fp32 and tf32x3: B0, B3@384 (no centered stride) and B5 against the goldens the unmodified reference produced
  (tests/golden/effnetb*.npz) and against the restatement (oracle/port_effnet_b.py); all eight variants in fp32 against the
  restatement.  Features and joints within 1e-3.
* bf16, bf16_simt, fp16, fp16_simt: every distinct op of B0, B3@384 and B5 element by element against fp64 conv2d at the
  mode's rounding points (port_effnet_b.layer_bound, port_ops.check_bound), at batch 1 and 3, with the kernel class and
  the depthwise kernel asserted: every 5x5 op on DW_5X5_POOL_16B in the tensor-core modes.
* The pooling 5x5 kernel against dwconv_kernel: every distinct 5x5 op of B0, B3, B5 and B7 (stride 1 and 2, the
  bottom-right shift, the odd 7x7 maps of S=224, widths 144 to 2304) at batch 1, 3 and 5 in 'bf16' vs 'bf16_simt' and
  'fp16' vs 'fp16_simt': torch.equal.
* SE pooling on the forward: fc1 behind every fused 5x5 pool against act(W1 mean(D) + b1) on the depthwise output D the
  device stored; no pool_mean_kernel launch in a bf16 / fp16 B0 forward, one per SE block in fp32.
* BatchNorm eps 1e-5 (B0-B4): a folded conv against conv2d + BN where some running variances are ~1e-4.
* Determinism (two bf16 forwards bit-identical) and the Pose3dEstimator pipeline on a B0 crop model in fp16."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from oracle import port, port_effnet_b, port_ops
from tests.test_gpu_ops16_vs_conv2d import MODES, POOL_SLICES, expected_class, op_classes, operands, se_fc_key

pytestmark = pytest.mark.gpu

GOLDENS = [('efficientnet-b0', 256, True, 'effnetb0_s256_j24.npz'),
           ('efficientnet-b3', 384, False, 'effnetb3_s384_j24_nocenter.npz'),
           ('efficientnet-b5', 256, True, 'effnetb5_s256_j24.npz')]


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def device_model(H, name, pcfg, n_joints, sd, precision='fp32'):
    """Metrabs(Sequential(PreprocLayer(), efficientnet_bN().features), ji), as the reference assembles it."""
    import metrabs_b200
    from metrabs_b200.backbones import efficientnet as E
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    bb = getattr(E, 'efficientnet_' + name.split('-')[1])()
    m = Metrabs(torch.nn.Sequential(E.PreprocLayer(), bb.features), H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def model(name, side, centered=True, j=8, calib_batch=1):
    pcfg = port.PathConfig(proc_side=side, centered_stride=centered)
    spec = port_effnet_b.effnet_b_spec(name, centered_stride=centered)
    return pcfg, spec, port_effnet_b.make_state_dict(spec, pcfg, j, seed=0, calib_batch=calib_batch)


def is_se(name):
    return name.endswith(('.avgpool', '.fc1', '.fc2'))


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name,side,centered,fname', GOLDENS)
def test_goldens_and_oracle(H, golden_dir, name, side, centered, fname, precision):
    import numpy as np
    import os
    g = np.load(os.path.join(golden_dir, fname), allow_pickle=False)
    j, batch = int(g['n_joints']), int(g['batch'])
    pcfg = port.PathConfig(proc_side=side, centered_stride=centered)
    spec = port_effnet_b.effnet_b_spec(name, centered_stride=centered)
    sd = port_effnet_b.make_state_dict(spec, pcfg, j, seed=int(g['seed']))
    crops, k = port.synthetic_inputs(batch, side, seed=int(g['seed']))
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    m = device_model(H, name, pcfg, j, sd, precision)
    eng = m.engine()
    feats = eng.backbone(crops.cuda()).permute(0, 3, 1, 2)
    out = m((crops.cuda(), k.cuda()))
    e_feat, e_out = H.rel_err(feats, stages['features']), H.rel_err(out, ref)
    e_gfeat = H.rel_err(feats.reshape(batch, -1)[:, ::int(g['feature_stride'])], g['features'])
    e_gold = H.rel_err(out, g['coords3d_abs'])
    print(f'{name}@{side} [{precision}]: vs oracle features {e_feat:.2e} joints {e_out:.2e}; vs reference goldens features '
          f'{e_gfeat:.2e} joints {e_gold:.2e}; {eng.last_launch_count} launches')
    assert e_feat < 1e-3 and e_out < 1e-3 and e_gfeat < 1e-3 and e_gold < 1e-3


@pytest.mark.parametrize('v', range(8))
def test_every_variant_fp32(H, v):
    name = f'efficientnet-b{v}'
    pcfg, spec, sd = model(name, 256, j=24, calib_batch=2)
    crops, k = port.synthetic_inputs(2, 256, seed=3)
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, 24, crops, k, stages=stages)
    m = device_model(H, name, pcfg, 24, sd, 'fp32')
    eng = m.engine()
    e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
    e_out = H.rel_err(m((crops.cuda(), k.cuda())), ref)
    print(f'{name} [fp32]: features {e_feat:.2e}, joints {e_out:.2e}, {eng.backbone_flops_per_crop / 1e9:.2f} GFLOP/crop')
    assert e_feat < 1e-3 and e_out < 1e-3


def dw_expected(op, precision):
    from metrabs_b200 import _lib
    if precision not in ('bf16', 'fp16'):
        return {_lib.DW_GENERIC}
    if op['kernel'] == 5:
        return {_lib.DW_5X5_POOL_16B}
    return {_lib.DW_STRIP_16B} if op['stride'] == 2 else {_lib.DW_TMA, _lib.DW_STRIP_16B}


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name,side,centered', [('efficientnet-b0', 256, True), ('efficientnet-b3', 384, False),
                                                ('efficientnet-b5', 256, True)])
def test_ops16_vs_conv2d(H, name, side, centered, batch):
    from metrabs_b200 import _lib
    pcfg, spec, sd = model(name, side, centered)
    table = port_effnet_b.op_table(spec)
    for precision in MODES:
        eng = device_model(H, name, pcfg, 8, sd, precision).engine()
        classes = op_classes(eng, side)
        st = port_ops.MODES[precision][0]
        g = torch.Generator().manual_seed(side + batch)
        seen, feats, worst = set(), set(), {}
        for i, nm in enumerate(eng.op_names()):
            if is_se(nm):
                continue
            op, io = table[nm], eng.op_io(i)
            sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], op['stride'], op['shift'], op['act'],
                   op['kernel'], op['depthwise'], op['stem'])
            if sig in seen:
                continue
            seen.add(sig)
            assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
            kind = classes[nm]
            if op['depthwise']:
                dk = eng.op_kernel(i)
                assert dk in dw_expected(op, precision), (nm, precision, dk)
                kind += f'/{dk}'
            feats |= {kind, ('shift', op['shift']), ('k', op['kernel'])}
            x, res, sc = operands(io, batch, st, g, i == 0)
            out = eng.debug_run_op(i, x, res, sc)
            ref, tol = port_effnet_b.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), sc,
                                                 precision)
            assert out.shape == ref.shape, (nm, tuple(out.shape), tuple(ref.shape))
            r, bad = port_ops.check_bound(out, ref, tol, precision)
            assert bad == 0, f'{nm} [{precision}] batch {batch}: {bad} elements outside the bound (worst |dev-ref|/tol {r:.2f})'
            worst[kind] = max(worst.get(kind, 0.0), r)
        assert ('k', 5) in feats and (('shift', 1) in feats) == centered
        if precision in ('bf16', 'fp16'):
            assert f'dwconv_kernel/{_lib.DW_5X5_POOL_16B}' in feats and 'tc_conv_kernel' in feats
        print(f'{name}@{side} x{batch} [{precision}]: {len(seen)} ops, worst |dev-ref|/tol {worst}')
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize('side', [256, 224])
@pytest.mark.parametrize('v', [0, 3, 5, 7])
def test_dw5x5_pool_bit_equal_to_the_generic_kernel(H, v, side):
    from metrabs_b200 import _lib
    name = f'efficientnet-b{v}'
    pcfg, spec, sd = model(name, side)
    table = port_effnet_b.op_table(spec)
    g = torch.Generator().manual_seed(31 + v)
    reached = set()
    for tc_mode, simt_mode in (('bf16', 'bf16_simt'), ('fp16', 'fp16_simt')):
        tc = device_model(H, name, pcfg, 8, sd, tc_mode).engine()
        simt = device_model(H, name, pcfg, 8, sd, simt_mode).engine()
        st = port_ops.MODES[tc_mode][0]
        seen = set()
        for i, nm in enumerate(tc.op_names()):
            if nm not in table or not table[nm]['depthwise'] or table[nm]['kernel'] != 5:
                continue
            op, io = table[nm], tc.op_io(i)
            sig = (io['in_shape'], io['out_shape'], op['stride'], op['shift'])
            if sig in seen:
                continue
            seen.add(sig)
            assert tc.op_kernel(i) == _lib.DW_5X5_POOL_16B and simt.op_kernel(i) == _lib.DW_GENERIC, nm
            for batch in (1, 3, 5):
                x = (3 * torch.randn((batch,) + io['in_shape'], generator=g)).to(st).float().cuda()
                a, b = tc.debug_run_op(i, x), simt.debug_run_op(i, x)
                assert torch.isfinite(a).all()
                assert torch.equal(a, b), (nm, tc_mode, batch, int((a != b).sum()))
            reached |= {('stride', op['stride']), ('shift', op['shift']), ('odd', io['out_shape'][0] % 2),
                        ('width', io['out_shape'][2])}
        print(f'{name}@{side} [{tc_mode} vs {simt_mode}]: {len(seen)} distinct 5x5 ops bit-equal at batch 1, 3, 5')
        del tc, simt
        torch.cuda.empty_cache()
    assert {('stride', 1), ('stride', 2), ('shift', 1)} <= reached, reached
    widths = {w for k, w in reached if k == 'width'}
    if v == 0:
        assert min(widths) == 144
    if v == 7:
        assert max(widths) == 2304
    if side == 224:
        assert ('odd', 1) in reached  # the 7x7 maps


@pytest.mark.parametrize('precision', MODES + ['fp32'])
@pytest.mark.parametrize('name,side,centered,batch', [('efficientnet-b0', 256, True, 2),
                                                      ('efficientnet-b3', 224, False, 3)])
def test_se_pool_on_the_forward(H, precision, name, side, centered, batch):
    """fc1 behind every fused 5x5 pool against act(W1 mean(D) + b1) in fp64, D the depthwise output the device stored:
    the kernel pools the stored (rounded) values, so the only error left is the fp32 summation (se_fc_bound's n_in)."""
    from metrabs_b200 import _lib
    pcfg, spec, sd = model(name, side, centered)
    eng = device_model(H, name, pcfg, 8, sd, precision).engine()
    names = eng.op_names()
    crops = port.synthetic_inputs(batch, side, seed=14)[0].cuda()
    checked, worst = 0, 0.0
    for i, nm in enumerate(names):
        if not nm.endswith('.avgpool') or eng.op_kernel(i - 1) != _lib.DW_5X5_POOL_16B:
            continue
        hh, ww, _c = eng.op_io(i - 1)['out_shape']
        d = eng.debug_run_ops(crops, i).double()
        f1 = eng.debug_run_ops(crops, i + 2)[:, 0, 0].double()
        key = se_fc_key(sd, names[i + 1])
        w, b = sd[key + '.weight'], sd[key + '.bias']
        ref, tol = port_ops.se_fc_bound(d.mean(dim=(1, 2)), d.abs().mean(dim=(1, 2)), hh * ww + POOL_SLICES + 2, w, b, 'silu')
        err = (f1[:, :w.shape[0]] - ref).abs()
        assert bool((err <= tol).all()), f'{names[i + 1]} [{precision}]: |dev-ref|/tol {float((err / tol).max()):.2f}'
        assert not f1[:, w.shape[0]:].any()
        worst = max(worst, float((err / tol).max()))
        checked += 1
    assert (checked > 0) == (precision in ('bf16', 'fp16'))
    eng.profile_begin()
    eng.backbone(crops)
    prof = eng.profile_end()
    pools = prof.get('pool_mean_kernel', {}).get('launches', 0)
    if precision in ('bf16', 'fp16'):
        assert pools == 0, prof.get('pool_mean_kernel')
    else:
        assert pools == sum(n.endswith('.avgpool') for n in names)
    print(f'{name}@{side} x{batch} [{precision}]: {checked} fused 5x5 pools, worst fc1 |dev-ref|/tol {worst:.2f}, '
          f'{pools} pool_mean_kernel launches')


def test_bn_eps_1e5_is_folded(H):
    """B0 keeps torchvision's BatchNorm eps 1e-5.  With running_var ~1e-4 on some channels, folding with 1e-3 would
    shrink those channels' outputs by sqrt(1.1e-3 / 1.1e-4) = 3.2x."""
    name = 'efficientnet-b0'
    pcfg, spec, sd = model(name, 256)
    nm = 'backbone.1.2.0.block.3'  # a projection: conv + BN, no activation
    bn = nm + '.1'
    sd = dict(sd)
    for k in ('running_var', 'running_mean', 'bias'):
        sd[f'{bn}.{k}'] = sd[f'{bn}.{k}'].clone()
    sd[f'{bn}.running_var'][:8] = 1e-4
    sd[f'{bn}.running_mean'][:8] = 0.0
    sd[f'{bn}.bias'][:8] = 0.0
    eng = device_model(H, name, pcfg, 8, sd, 'fp32').engine()
    i = eng.op_names().index(nm)
    io = eng.op_io(i)
    x = torch.randn((2,) + io['in_shape'], generator=torch.Generator().manual_seed(5))
    out = eng.debug_run_op(i, x.cuda(), None, torch.ones(2, io['in_shape'][2]).cuda()).cpu().double()  # SE scale 1

    def conv_bn(eps):
        z = F.conv2d(x.permute(0, 3, 1, 2).double(), sd[nm + '.0.weight'].double())
        y = F.batch_norm(z, sd[f'{bn}.running_mean'].double(), sd[f'{bn}.running_var'].double(), sd[f'{bn}.weight'].double(),
                         sd[f'{bn}.bias'].double(), training=False, eps=eps)
        return y.permute(0, 2, 3, 1)
    ref5, ref3 = conv_bn(1e-5), conv_bn(1e-3)
    e5 = port.relative_error(out, ref5)
    ratio = float(ref5[..., :8].abs().max() / ref3[..., :8].abs().max())
    e3 = port.relative_error(out, ref3)
    print(f'folded conv vs conv2d + BN: eps 1e-5 {e5:.2e}, eps 1e-3 {e3:.2e}; low-variance channels {ratio:.2f}x')
    assert e5 < 1e-5 and ratio > 2.0 and e3 > 0.5


def test_determinism_and_pipeline(H):
    name = 'efficientnet-b0'
    pcfg, spec, sd = model(name, 256, j=8)
    crops, k = port.synthetic_inputs(5, 256, seed=6)
    m = device_model(H, name, pcfg, 8, sd, 'bf16')
    eng = m.engine()
    f1, f2 = eng.backbone(crops.cuda()).clone(), eng.backbone(crops.cuda()).clone()
    o1, o2 = m((crops.cuda(), k.cuda())), m((crops.cuda(), k.cuda()))
    assert torch.equal(f1, f2) and torch.equal(o1, o2) and torch.isfinite(o1).all()
    del m, eng
    m = device_model(H, name, pcfg, 8, sd, 'fp16')
    from metrabs_b200.multiperson import Pose3dEstimator
    m.joint_names, m.joint_edges = [f'j{i}' for i in range(8)], [[0, 1]]
    est = Pose3dEstimator(m, {'': dict(indices=list(range(8)), names=m.joint_names, edges=[[0, 1]])}, None)
    frames = torch.randint(0, 256, (1, 3, 240, 320), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    res = est.estimate_poses_batched(frames.cuda(), [torch.tensor([[40., 20., 120., 180.], [150., 40., 100., 160.]])],
                                     num_aug=3)
    torch.cuda.synchronize()
    assert res['poses3d'][0].shape == (2, 8, 3) and torch.isfinite(res['poses3d'][0]).all()
