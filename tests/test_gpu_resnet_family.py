"""GPU: ResNet-18, -34, -101 and -152 (V1, metrabs_b200.backbones.resnet) against this build's torch restatement of the
Keras code (oracle/port_resnet.py ResNetSpec; the reference has no test, golden or importable implementation of
these backbones, so parity is "this build's restatement vs this build's kernels").

* fp32 and tf32x3: every layer within 1e-4 of the restatement on the restatement's own operands, features within 1e-3,
  joints within 1e-3 (5e-3 for ResNet-152, see below), at output strides 32 and 8; the basic nets also with stride_train
  32 at stride_test 8 (the mixed dilations of the second 3x3 of block1 in conv4 / conv5) and once without the centered
  stride.
* bf16, bf16_simt, fp16, fp16_simt: every distinct op element by element against fp64 conv2d at the mode's rounding
  points (port_resnet.layer_bound, port_ops.check_bound), with its kernel class asserted: every GEMM-type op on
  tc_conv_kernel in the tensor-core modes.  The cases include the basic block's dense 3x3 stride-2 conv with the bottom-right shift
  (begin pad 0), its 64->64 3x3 convs at 64x64 with an identity residual before ReLU, dilated 3x3 convs with a residual
  before ReLU and the mixed dilations.
* a 16-bit end-to-end forward of each depth (finite joints, deviation from fp32 printed), and the host-buffer,
  pipelined and Pose3dEstimator entry points on the new nets."""
import dataclasses

import pytest
import torch

from oracle import port, port_ops, port_resnet
from oracle import port_tf_backbones as tfb
from tests.test_gpu_ops16_vs_conv2d import MODES, expected_class, op_classes, operands

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def device_model(H, depth, pcfg, n_joints, sd, precision='fp32'):
    import metrabs_b200
    from metrabs_b200.backbones import resnet
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    m = Metrabs(getattr(resnet, f'resnet{depth}')(), H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def layer_operands(spec, tap, crops):
    """op name -> (input NCHW, residual NCHW or None): each layer's operands taken from the restatement's own tensors, so
    that every layer is checked on its own rather than through the fp32 drift of the layers before it."""
    p = 'backbone.'
    ops = {p + 'conv1_conv': (crops, None), p + 'pool1_pool': (tap[p + 'conv1_conv'], None)}
    x = tap[p + 'pool1_pool']
    for b in port_resnet.resnet_blocks(spec.cfg, spec.depth):
        n = p + b['name']
        if b['conv_shortcut']:
            ops[n + '_0_conv'] = (x, None)
        sc = tap[n + '_0_conv'] if b['conv_shortcut'] else x
        ops[n + '_1_conv'] = (x, None)
        if spec.basic:
            ops[n + '_2_conv'] = (tap[n + '_1_conv'], sc)
            x = tap[n + '_2_conv']
        else:
            ops[n + '_2_conv'] = (tap[n + '_1_conv'], None)
            ops[n + '_3_conv'] = (tap[n + '_2_conv'], sc)
            x = tap[n + '_3_conv']
    return ops


def check_all_ops(eng, sd, spec, side, precision, batch, seed):
    """every distinct op (stem and max pool included) on random 16-bit operands, element by element against
    port_resnet.layer_bound -> (ops checked, features seen, worst |dev-ref|/tol per kernel class)"""
    table = port_resnet.op_table(spec)
    classes = op_classes(eng, side)
    st = port_ops.MODES[precision][0]
    g = torch.Generator().manual_seed(seed)
    seen, feats, worst = set(), set(), {}
    for i, nm in enumerate(eng.op_names()):
        op, io = table[nm], eng.op_io(i)
        sig = (io['in_shape'], io['out_shape'], io['residual'], op['stride'], op['shift'], op['dil'], op['act'],
               op['kernel'], op['maxpool'], op['stem'], op['res_first'])
        if sig in seen:
            continue
        seen.add(sig)
        assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
        kind = classes[nm]
        feats |= {kind, ('act', op['act']), ('dil', op['dil']), ('shift', op['shift']), ('res_first', op['res_first'])}
        x, res, _ = operands(io, batch, st, g, i == 0)
        out = eng.debug_run_op(i, x, res)
        ref, tol = port_resnet.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), precision)
        assert out.shape == ref.shape, (nm, tuple(out.shape), tuple(ref.shape))
        r, bad = port_ops.check_bound(out, ref, tol, precision)
        assert bad == 0, f'{nm} [{precision}]: {bad} elements outside the bound (worst |dev-ref|/tol {r:.2f})'
        worst[kind] = max(worst.get(kind, 0.0), r)
    return seen, feats, worst


PARITY = [(d, dict(proc_side=256, stride_test=32, stride_train=32, depth=8)) for d in (18, 34, 101, 152)]
PARITY += [(d, dict(proc_side=256, stride_test=8, stride_train=8, depth=32)) for d in (18, 34, 101, 152)]
PARITY += [(d, dict(proc_side=256, stride_test=8, stride_train=32, depth=32)) for d in (18, 34)]  # mixed dilations
PARITY += [(d, dict(proc_side=256, stride_test=32, stride_train=32, depth=8, centered_stride=False)) for d in (18, 34)]


@pytest.mark.parametrize('depth,cfgkw', PARITY)
def test_resnet_family_fp32_and_tf32x3(H, depth, cfgkw):
    j, batch = 24, 2
    pcfg = port.PathConfig(**cfgkw)
    spec = port_resnet.ResNetSpec(pcfg, depth)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
    tap, stages = {}, {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    for precision in ('fp32', 'tf32x3'):
        m = device_model(H, depth, pcfg, j, sd, precision)
        eng = m.engine()
        names = eng.op_names()
        assert set(names) == set(tap)
        operands = layer_operands(spec, tap, crops)
        nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).cuda()  # noqa: E731
        bad = []
        for i, name in enumerate(names):
            x, res = operands[name]
            out = eng.debug_run_op(i, x.cuda() if i == 0 else nhwc(x), nhwc(res)).permute(0, 3, 1, 2).cpu()
            err = port.relative_error(out, tap[name])
            if not err < 1e-4:
                bad.append((name, err))
        assert not bad, f'{precision}: first diverging layers: {bad[:5]}'
        out = m((crops.cuda(), k.cuda()))
        e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
        e_out = H.rel_err(out, ref)
        print(f'resnet{depth} {cfgkw} [{precision}]: features {e_feat:.2e}, joints {e_out:.2e}, '
              f'{eng.backbone_flops_per_crop / 1e9:.2f} GFLOP/crop, {eng.last_launch_count} launches')
        # ResNet-152: every layer above is within 1e-4 on its own, and the features stay within 1e-3, but two fp32
        # evaluations drift apart over its 155 convs and the peaked soft-argmax of the head amplifies that in the joints
        # (up to 3.2e-3 measured on an H100)
        assert e_feat < 1e-3 and e_out < (5e-3 if depth == 152 else 1e-3)
        del m, eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize('depth', [18, 34, 101, 152])
@pytest.mark.parametrize('side,stride,stride_train,centered,batch', [(256, 8, 32, True, 2), (256, 32, 32, False, 3)])
def test_resnet_family_ops16_vs_conv2d(H, depth, side, stride, stride_train, centered, batch):
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, stride_train=stride_train, centered_stride=centered, depth=8)
    spec = port_resnet.ResNetSpec(pcfg, depth)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    table = port_resnet.op_table(spec)
    for precision in MODES:
        eng = device_model(H, depth, pcfg, 8, sd, precision).engine()
        seen, feats, worst = check_all_ops(eng, sd, spec, side, precision, batch, seed=stride)
        assert ('res_first', True) in feats and 'other' in feats and 'stem_conv_kernel' in feats
        gemm = 'tc_conv_kernel' if precision in ('bf16', 'fp16') else 'conv_igemm_kernel'
        assert gemm in feats and not feats & {'fmb_kernel', 'conv_igemm_kernel', 'tc_conv_kernel'} - {gemm}
        if stride < 32:
            assert ('dil', 2) in feats and ('dil', 4) in feats
            if spec.basic:  # block1 of conv5: dilation 4 then 8
                assert ('dil', 8) in feats
        if centered:
            assert ('shift', 1) in feats
        if spec.basic:
            # the shapes no other test runs: the bottom-right 3x3 stride-2 conv (begin pad 0), 64->64 3x3 at 64x64 with
            # the identity residual before ReLU, and a dilated 3x3 with the residual before ReLU
            ios = {nm: eng.op_io(i) for i, nm in enumerate(eng.op_names())}
            c3 = table['backbone.conv3_block1_1_conv']
            assert (c3['kernel'], c3['stride'], c3['shift'] if centered else 0) == (3, 2, 1 if centered else 0)
            io = ios['backbone.conv2_block2_2_conv']
            assert io['in_shape'] == (64, 64, 64) and io['out_shape'] == (64, 64, 64) and io['residual']
            if stride < 32:
                assert table['backbone.conv4_block2_2_conv']['dil'] == 2 and ios['backbone.conv4_block2_2_conv']['residual']
        print(f'resnet{depth}@{side} s{stride}/{stride_train} centered={centered} [{precision}]: {len(seen)} ops, '
              f'worst |dev-ref|/tol {worst}')
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize('depth', [18, 34, 101, 152])
def test_resnet_family_16bit_end_to_end(H, depth):
    j, batch = 24, 4
    pcfg = port.PathConfig(proc_side=256, stride_test=8, stride_train=32, depth=32)
    spec = port_resnet.ResNetSpec(pcfg, depth)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=1)
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k)
    for precision in ('bf16', 'fp16'):
        m = device_model(H, depth, pcfg, j, sd, precision)
        out = m((crops.cuda(), k.cuda()))
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        print(f'resnet{depth} s8 [{precision}]: joints rel err vs fp32 restatement {H.rel_err(out, ref):.2e}, '
              f'{m.engine().last_launch_count} launches')
        del m
        torch.cuda.empty_cache()


@pytest.mark.parametrize('depth', [18, 101])
def test_resnet_family_host_pipelined_and_multiperson(H, depth):
    j = 8
    pcfg = port.PathConfig(proc_side=256, stride_test=32, depth=8)
    sd = tfb.make_state_dict(port_resnet.ResNetSpec(pcfg, depth), pcfg, j, seed=0, calib_batch=1)
    m = device_model(H, depth, pcfg, j, sd, 'bf16')
    eng = m.engine()
    crops, k = port.synthetic_inputs(3, 256, seed=2)
    out = m((crops.cuda(), k.cuda()))
    out_h = eng.forward_host(crops.pin_memory(), k.pin_memory())
    assert torch.equal(out_h, out.cpu())
    ch, kh = crops.float().contiguous().pin_memory(), k.float().contiguous().pin_memory()
    outs = [torch.empty(out_h.shape, dtype=torch.float32).pin_memory() for _ in range(2)]
    eng.forward_host_submit(ch, kh, outs[0], 0)
    eng.forward_host_submit(ch, kh, outs[1], 1)
    eng.forward_host_wait(0)
    eng.forward_host_wait(1)
    assert torch.equal(outs[0], out_h) and torch.equal(outs[1], out_h)
    from metrabs_b200.multiperson import Pose3dEstimator
    m.joint_names, m.joint_edges = [f'j{i}' for i in range(j)], [[0, 1]]
    est = Pose3dEstimator(m, {'': dict(indices=list(range(j)), names=m.joint_names, edges=[[0, 1]])}, None)
    frames = torch.randint(0, 256, (1, 3, 240, 320), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    res = est.estimate_poses_batched(frames.cuda(), [torch.tensor([[40., 20., 120., 180.], [150., 40., 100., 160.]])],
                                     num_aug=3)
    torch.cuda.synchronize()
    assert res['poses3d'][0].shape == (2, j, 3) and torch.isfinite(res['poses3d'][0]).all()
