"""GPU: ResNet-50, -101 and -152 V1.5 (metrabs_b200.backbones.resnet.resnet{50,101,152}v1_5) and the minimalistic
MobileNetV3-Small and -Large (mobilenet_v3_{small,large}(minimalistic=True)) against this build's torch restatement of the
Keras code (oracle/port_builder_variants.py; parity is "this build's restatement vs this build's kernels", the reference
has no test, golden or importable implementation of these backbones).

* fp32 and tf32x3: every layer within 1e-4 of the restatement on the restatement's own operands, features and joints within
  1e-3 (5e-3 for the joints of ResNet-101 and -152 V1.5, see below), V1.5 at output strides 32, 16 and 8 and once
  without the centered stride; the engine's FLOPs per crop equal the restatement's count; the kernel of every op.
* bf16 and fp16: every op of the forward against fp64 conv2d on the tensors the forward itself produced, at the benchmark
  batch (scripts/builder_variants_step.py), within the per-layer bound (port_builder_variants.layer_bound,
  port_ops.check_bound), with the kernel mtb_op_kernel reports asserted for each op.  ResNet-101 and -152 V1.5 have the
  distinct op shapes of ResNet-50 V1.5.
* per-crop batch invariance (test_gpu_batch_invariance.py's sub-batches) in bf16, fp16 and fp32;
* 16-bit end-to-end forwards of all five nets with calibrated weights: finite joints."""
import dataclasses

import pytest
import torch

from metrabs_b200 import _lib
from oracle import port, port_ops
from oracle import port_builder_variants as V
from oracle import port_tf_backbones as tfb
from tests.test_gpu_batch_invariance import first_differing_op, sub_batches
from tests.test_gpu_forward_ops16 import check_conv
from tests.test_gpu_ops16_vs_conv2d import dw_kernel

pytestmark = pytest.mark.gpu

NETS = ['resnet50v1_5', 'resnet101v1_5', 'resnet152v1_5', 'mobilenetv3-small-mini', 'mobilenetv3-large-mini']
DW = {'tma': _lib.DW_TMA, 'strip': _lib.DW_STRIP_16B, 'generic': _lib.DW_GENERIC}


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def spec_of(net, pcfg):
    if net.startswith('resnet'):
        return V.ResNetV15Spec(pcfg, int(net[len('resnet'):-len('v1_5')]))
    return V.MobileNetV3MiniSpec(pcfg, net.split('-')[1])


def device_model(H, net, pcfg, n_joints, sd, precision='fp32'):
    import metrabs_b200
    from metrabs_b200.backbones import mobilenet_v3, resnet
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    if net.startswith('resnet'):
        features = getattr(resnet, net)()
    else:
        features = getattr(mobilenet_v3, f'mobilenet_v3_{net.split("-")[1]}')(minimalistic=True)
    m = Metrabs(features, H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def expected_kernel(op, io, precision):
    """mtb_kernel of an op, restated from choose_kernels (csrc/engine.cu)"""
    if op['maxpool']:
        return _lib.MAXPOOL
    if op['stem']:  # 64 (ResNet) and 16 (MobileNetV3) channels
        return _lib.STEM_WIDE
    if op['depthwise']:
        if precision == 'tf32x3':  # the strip kernel in fp32 where the 16-bit modes have a TMA or strip plan
            return _lib.DW_STRIP_F32 if dw_kernel(op, io, 'bf16') != 'generic' else _lib.DW_GENERIC
        return DW[dw_kernel(op, io, precision)]
    cin, cout = io['in_shape'][2], io['out_shape'][2]
    if precision in ('bf16', 'fp16') and port_ops.tc_eligible(op, cin, cout):
        s1 = (op['kernel'] == 3 and op['stride'] == 1 and op['dil'] == 1 and cin <= 64 and cout <= 64 and op['act'] == 'relu')
        return _lib.TC_CONV3X3S1 if s1 else _lib.TC_CONV
    if precision == 'tf32x3' and port_ops.tc32_eligible(op, cin, cout):
        return _lib.TC32
    return _lib.IGEMM


def layer_operands(spec, tap, crops):
    """op name -> (input NCHW, residual NCHW or None), taken from the restatement's own tensors"""
    p = 'backbone.'
    if isinstance(spec, V.ResNetV15Spec):
        ops = {p + 'conv1_conv': (crops, None), p + 'pool1_pool': (tap[p + 'conv1_conv'], None)}
        x = tap[p + 'pool1_pool']
        for b in V.resnet_v1_5_blocks(spec.cfg, spec.depth):
            n = p + b['name']
            sc = x
            if b['conv_shortcut']:
                ops[n + '_0_conv'] = (x, None)
                sc = tap[n + '_0_conv']
            ops[n + '_1_conv'] = (x, None)
            ops[n + '_2_conv'] = (tap[n + '_1_conv'], None)
            ops[n + '_3_conv'] = (tap[n + '_2_conv'], sc)
            x = tap[n + '_3_conv']
        return ops
    ops = {p + 'Conv': (crops, None)}
    x = tap[p + 'Conv']
    for b in V.mini_blocks(spec.variant):
        n = p + b['name']
        if b['name'] != 'expanded_conv':
            ops[n + '.expand'] = (x, None)
        ops[n + '.depthwise'] = (tap[n + '.expand'] if b['name'] != 'expanded_conv' else x, None)
        ops[n + '.project'] = (tap[n + '.depthwise'], x if b['residual'] else None)
        x = tap[n + '.project']
    ops[p + 'Conv_1'] = (x, None)
    ops[p + 'Conv_2'] = (tap[p + 'Conv_1'], None)
    return ops


PARITY = [(n, dict(proc_side=256, stride_test=32, depth=8)) for n in NETS]
PARITY += [(n, dict(proc_side=256, stride_test=8, depth=32)) for n in NETS[:3]]
PARITY += [('resnet50v1_5', dict(proc_side=256, stride_test=16, depth=16)),
           ('resnet50v1_5', dict(proc_side=256, stride_test=8, depth=32, centered_stride=False))]


@pytest.mark.parametrize('net,cfgkw', PARITY)
def test_fp32_and_tf32x3(H, net, cfgkw):
    j, batch = 24, 2
    pcfg = port.PathConfig(**cfgkw)
    spec = spec_of(net, pcfg)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
    tap, stages = {}, {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    ops = layer_operands(spec, tap, crops)
    table = V.op_table(spec)
    for precision in ('fp32', 'tf32x3'):
        m = device_model(H, net, pcfg, j, sd, precision)
        eng = m.engine()
        names = eng.op_names()
        assert set(names) == set(tap) == set(ops) == set(table)
        if isinstance(spec, V.ResNetV15Spec):
            assert abs(eng.backbone_flops_per_crop / 1e9 - V.resnet_v1_5_gflop_per_crop(pcfg, spec.depth)) < 1e-9
        nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).cuda()  # noqa: E731
        bad = []
        for i, name in enumerate(names):
            assert eng.op_kernel(i) == expected_kernel(table[name], eng.op_io(i), precision), (name, precision)
            x, res = ops[name]
            out = eng.debug_run_op(i, x.cuda() if i == 0 else nhwc(x), nhwc(res)).permute(0, 3, 1, 2).cpu()
            err = port.relative_error(out, tap[name])
            if not err < 1e-4:
                bad.append((name, err))
        assert not bad, f'{precision}: first diverging layers: {bad[:5]}'
        out = m((crops.cuda(), k.cuda()))
        e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
        e_out = H.rel_err(out, ref)
        print(f'{net} {cfgkw} [{precision}]: features {e_feat:.2e}, joints {e_out:.2e}, '
              f'{eng.backbone_flops_per_crop / 1e9:.3f} GFLOP/crop, {eng.last_launch_count} launches')
        # ResNet-101 and -152 V1.5: as for ResNet-152 V1 (test_gpu_resnet_family.py), every layer is within 1e-4 on its own
        # and the features within 1e-3, but two fp32 evaluations drift apart over 100+ convs and the peaked soft-argmax of
        # the head amplifies that in the joints (1.6e-3 for ResNet-101 V1.5 at stride 8, 2.9e-3 for -152)
        assert e_feat < 1e-3 and e_out < (5e-3 if net in ('resnet101v1_5', 'resnet152v1_5') else 1e-3)
        del m, eng
        torch.cuda.empty_cache()


# (net, stride, D, crops): the benchmark script's configurations of the distinct op shapes
FORWARD = [('resnet50v1_5', 32, 8, 128), ('resnet50v1_5', 8, 32, 128), ('mobilenetv3-small-mini', 32, 8, 256),
           ('mobilenetv3-large-mini', 32, 8, 256)]


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
@pytest.mark.parametrize('net,stride,d,batch', FORWARD)
def test_forward_ops_vs_conv2d(H, net, stride, d, batch, precision):
    """each op k of the forward: its output is what debug_run_ops(crops, k + 1) stored, its input and residual the outputs
    of the latest earlier ops that wrote the buffers it reads (as test_gpu_forward_ops16.py)"""
    j = 8
    pcfg = port.PathConfig(proc_side=256, stride_test=stride, depth=d)
    spec = spec_of(net, pcfg)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=1)
    eng = device_model(H, net, pcfg, j, sd, precision).engine()
    table = V.op_table(spec)
    crops = port.synthetic_inputs(batch, pcfg.proc_side, seed=5)[0].cuda()
    names = eng.op_names()
    live, worst, reached = {}, {}, set()
    for k, nm in enumerate(names):
        op, io, bufs = table[nm], eng.op_io(k), eng.op_buffers(k)
        kern = eng.op_kernel(k)
        assert kern == expected_kernel(op, io, precision), (nm, kern)
        out = eng.debug_run_ops(crops, k + 1)
        assert torch.isfinite(out).all(), f'{nm} [{precision}]: {int((~torch.isfinite(out)).sum())} non-finite outputs'
        x = crops if k == 0 else live[bufs['input']]
        res = live[bufs['residual']] if bufs['residual'] != _lib.BUF_NONE else None
        assert (res is not None) == io['residual'] and bufs['scale'] == _lib.BUF_NONE, nm
        r = check_conv(lambda n, xx, rr, _sc: V.layer_bound(sd, spec, n, xx, rr, precision), nm, out, x, res, None, precision)
        worst[kern] = max(worst.get(kern, 0.0), r)
        reached |= {kern, ('dil', op['dil']), ('stride', op['stride'], op['kernel'], op['depthwise'])}
        live[bufs['output']] = out
    assert torch.equal(eng.backbone(crops).float(), live[_lib.BUF_FEATURES])
    if net.startswith('resnet'):
        # the strided 3x3 _2_convs and the 64-channel stride-1 3x3s on the tensor cores
        assert {_lib.TC_CONV, _lib.TC_CONV3X3S1, _lib.MAXPOOL, ('stride', 2, 3, False)} <= reached, reached
        if stride == 8:  # block1 of conv4 / conv5 at dil_in (1, 2), the other blocks at dil_out (2, 4)
            assert {('dil', 1), ('dil', 2), ('dil', 4)} <= reached, reached
            assert table['backbone.conv5_block1_2_conv']['dil'] == 2
    else:
        assert {_lib.TC_CONV, _lib.DW_TMA, _lib.DW_STRIP_16B, ('stride', 2, 3, True)} <= reached, reached
    del live, out
    torch.cuda.empty_cache()
    print(f'{net} s{stride} x{batch} [{precision}]: {len(names)} ops; worst |dev-ref|/tol by kernel '
          + ', '.join(f'{kk}: {v:.3f}' for kk, v in sorted(worst.items())))


@pytest.mark.parametrize('precision', ['bf16', 'fp16', 'fp32'])
@pytest.mark.parametrize('net,stride', [('resnet50v1_5', 8), ('mobilenetv3-small-mini', 32), ('mobilenetv3-large-mini', 32)])
def test_batch_invariance(H, net, stride, precision):
    n, side = 64, 224
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, depth=8)
    sd = tfb.make_state_dict(spec_of(net, pcfg), pcfg, 24, seed=0, calib_batch=1)
    eng = device_model(H, net, pcfg, 24, sd, precision).engine()
    crops = port.synthetic_inputs(n, side, seed=11)[0].cuda()
    feats = eng.backbone(crops)
    c2d, c3d = eng.head_decode(feats)
    assert all(torch.isfinite(t).all() for t in (feats, c2d, c3d))
    bad = []
    for s, e in sub_batches(n):
        f = eng.backbone(crops[s:e])
        a2, a3 = eng.head_decode(f)
        if not (torch.equal(f, feats[s:e]) and torch.equal(a2, c2d[s:e]) and torch.equal(a3, c3d[s:e])):
            bad.append(f'[{s}, {e}): {first_differing_op(eng, crops, s, e)}')
    assert not bad, bad[:4]


@pytest.mark.parametrize('net', NETS)
def test_16bit_end_to_end(H, net):
    j, batch = 24, 4
    stride, d = (8, 32) if net.startswith('resnet') else (32, 8)
    pcfg = port.PathConfig(proc_side=256, stride_test=stride, depth=d)
    spec = spec_of(net, pcfg)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=1)
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k)
    for precision in ('bf16', 'fp16'):
        m = device_model(H, net, pcfg, j, sd, precision)
        out = m((crops.cuda(), k.cuda()))
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        print(f'{net} s{stride} [{precision}]: joints rel err vs fp32 restatement {H.rel_err(out, ref):.2e}, '
              f'{m.engine().last_launch_count} launches')
        del m
        torch.cuda.empty_cache()
