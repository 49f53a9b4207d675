"""CPU: the pre-activation ResNet restatement (oracle/port_resnet_v2.py, ResNet-50/101/152 V2) against block tables
hand-derived from metrabs_tf/backbones/resnet.py:710-745, hand counts of its shapes and FLOPs, the key schema of
metrabs_b200.backbones.resnet's V2 factories (strict load into Metrabs), the C header's arch values, and the bound of the
BN-only pre-activation op.  Parity of these backbones is "this build's restatement vs this build's kernels"."""
import os
import re

import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import resnet
from oracle import port, port_ops, port_resnet_v2
from oracle import port_tf_backbones as tfb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTHS = [50, 101, 152]
COUNTS = {50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3]}


def _hand_table(depth, stride, centered):
    """(name, stride, shift, dilation, conv_shortcut, subsample) per block, from ResNetUnifiedV2 (:710-745) with
    get_strides_and_dilations written out for each output stride: strided stacks put stride 2 on their LAST block, the
    bottom-right shift on the last strided one; the later stacks have dilation 1, 2 (conv4 at stride 8), and conv5 has
    dil_out[-1] = 1 (stride 32), 2 (16) or 4 (8)."""
    plan = {32: ([2, 2, 2], [1, 1, 1], 1, 2), 16: ([2, 2, 1], [1, 1, 1], 2, 1), 8: ([2, 1, 1], [1, 1, 2], 4, 0)}
    strides, dils, d5, i_last = plan[stride]
    out = []
    for st, n in enumerate(COUNTS[depth]):
        for bi in range(n):
            last = st < 3 and bi == n - 1
            s = strides[st] if last else 1
            c = 1 if (last and centered and st == i_last) else 0
            d = dils[st] if st < 3 else d5
            out.append((f'conv{st + 2}_block{bi + 1}', s, c, d, bi == 0, bi > 0 and (s > 1 or c > 0)))
    return out


@pytest.mark.parametrize('depth', DEPTHS)
@pytest.mark.parametrize('stride', [32, 16, 8])
@pytest.mark.parametrize('centered', [True, False])
def test_block_tables(depth, stride, centered):
    blocks = port_resnet_v2.resnet_v2_blocks(port.PathConfig(stride_test=stride, centered_stride=centered), depth)
    got = [(b['name'], b['stride'], b['shift'], b['dil'], b['conv_shortcut'], b['subsample']) for b in blocks]
    assert got == _hand_table(depth, stride, centered)
    assert [b['filters'] for b in blocks] == sum(([f] * n for f, n in zip([64, 128, 256, 512], COUNTS[depth])), [])
    # stride_train plays no part
    assert blocks == port_resnet_v2.resnet_v2_blocks(port.PathConfig(stride_test=stride, stride_train=8, centered_stride=centered), depth)


def test_stride_8_plan_of_the_issue():
    b = {x['name']: x for x in port_resnet_v2.resnet_v2_blocks(port.PathConfig(stride_test=8), 50)}
    assert (b['conv2_block3']['stride'], b['conv2_block3']['shift'], b['conv2_block3']['subsample']) == (2, 1, True)
    assert all(b[f'conv3_block{i}']['dil'] == 1 and b[f'conv3_block{i}']['stride'] == 1 for i in range(1, 5))
    assert all(b[f'conv4_block{i}']['dil'] == 2 for i in range(1, 7))
    assert all(b[f'conv5_block{i}']['dil'] == 4 for i in range(1, 4))


def _meta_features(depth, side, stride):
    small = port.PathConfig(proc_side=32, stride_test=stride)
    sd = tfb.make_state_dict(port_resnet_v2.ResNetV2Spec(small, depth), small, 4, seed=0, calib_batch=1)
    meta = {k: v.to('meta') for k, v in sd.items()}
    spec = port_resnet_v2.ResNetV2Spec(port.PathConfig(proc_side=side, stride_test=stride), depth)
    tap = {}
    with torch.device('meta'):
        feats = spec.features(meta, torch.empty(1, 3, side, side), tap=tap)
    return sd, tap, feats


# GFLOP per crop at S = 256 (2 * MACs of every conv at its output size, plus one multiply-add per element of every
# pre-activation and of post_bn), by output stride (_stack_gflop)
HAND_GFLOP = {32: {50: 9.1033, 101: 18.8095, 152: 28.5177}, 8: {50: 49.3407, 101: 88.1653, 152: 120.1406}}


def _stack_gflop(side, stride, depth):
    """the closed form per stack: block1 = preact + _0 + _1 + _2 + _3, the others preact + _1 + _2 + _3, the stride of
    the last block applied to its _2 and _3"""
    h = side // 4
    strides = {32: [2, 2, 2], 8: [2, 1, 1]}[stride]
    total = 2.0 * (side // 2) ** 2 * 64 * 147
    c = 64
    for st, (f, n) in enumerate(zip([64, 128, 256, 512], COUNTS[depth])):
        for bi in range(n):
            s = strides[st] if (st < 3 and bi == n - 1) else 1
            total += 2.0 * h * h * (c + (c * 4 * f if bi == 0 else 0) + c * f)
            h //= s
            total += 2.0 * h * h * (9 * f * f + 4 * f * f)
            c = 4 * f
    return (total + 2.0 * h * h * c) / 1e9


@pytest.mark.parametrize('depth', DEPTHS)
@pytest.mark.parametrize('stride', [32, 8])
def test_shapes_and_flops(depth, stride):
    sd, tap, feats = _meta_features(depth, 256, stride)
    assert tuple(feats.shape) == (1, 2048, 256 // stride, 256 // stride)
    convs = [k for k in sd if k.endswith('_conv.weight')]
    assert len(convs) == 1 + 3 * sum(COUNTS[depth]) + 4
    total = 0.0
    for k, w in sd.items():
        name = k[:-len('.weight')]
        if k.endswith('_conv.weight'):
            _b, cout, h, w_ = tap[name].shape
            total += 2.0 * h * w_ * cout * w.shape[1] * w.shape[2] * w.shape[3]
        elif k.endswith(('_preact_bn.weight', 'post_bn.weight')):
            total += 2.0 * tap[name].numel()
    gflop = total / 1e9
    print(f'resnet{depth}v2 s{stride}: {gflop:.4f} GFLOP/crop')
    assert abs(gflop - HAND_GFLOP[stride][depth]) < 5e-4
    assert abs(_stack_gflop(256, stride, depth) - HAND_GFLOP[stride][depth]) < 5e-4
    assert abs(port_resnet_v2.gflop_per_crop(port.PathConfig(proc_side=256, stride_test=stride), depth) - gflop) < 1e-9


@pytest.mark.parametrize('depth', DEPTHS)
def test_key_schema_and_strict_load(depth):
    from metrabs_b200.models.metrabs import Metrabs
    from tests import helpers
    pcfg = port.PathConfig(proc_side=32, stride_test=32)
    sd = tfb.make_state_dict(port_resnet_v2.ResNetV2Spec(pcfg, depth), pcfg, 4, seed=0, calib_batch=1)
    feats = getattr(resnet, f'resnet{depth}v2')()
    assert {'backbone.' + k for k in feats.state_dict()} == {k for k in sd if k.startswith('backbone.')}
    assert feats.arch == getattr(_lib, f'ARCH_RESNET{depth}V2') and feats.last_channel == 2048
    keys = set(feats.state_dict())
    assert 'conv1_conv.bias' in keys and 'conv1_bn.weight' not in keys
    assert {k for k in keys if k.endswith('_0_conv.bias')} == {f'conv{s}_block1_0_conv.bias' for s in range(2, 6)}
    assert not any(k.endswith(('_1_conv.bias', '_2_conv.bias', '_3_bn.weight')) for k in keys)
    assert len([k for k in keys if k.endswith('_3_conv.bias')]) == sum(COUNTS[depth])
    m = Metrabs(feats, helpers.joint_info(4))
    m.load_state_dict(sd, strict=True)
    # every weight the engine reads is in the op table, and every op table key is a weight of the schema
    table = port_resnet_v2.op_table(port_resnet_v2.ResNetV2Spec(pcfg, depth))
    for op in table.values():
        for k in (op['weight'], op['bias']):
            assert k is None or k in sd
        if op['bn']:
            assert op['bn'] + '.running_var' in sd


def test_v1_features_unchanged():
    assert resnet.resnet50().arch == _lib.ARCH_RESNET50
    assert list(resnet.resnet50().state_dict())[:2] == ['conv1_conv.weight', 'conv1_conv.bias']


def test_header_arch_values():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    values = {m[0]: int(m[1]) for m in re.findall(r'MTB_ARCH_([A-Z0-9_]+) = (\d+)', src)}
    assert {d: values[f'RESNET{d}V2'] for d in DEPTHS} == {50: 10, 101: 11, 152: 12}
    assert {d: resnet.DEPTHS_V2[d][0] for d in DEPTHS} == {d: values[f'RESNET{d}V2'] for d in DEPTHS}


def test_op_table():
    spec = port_resnet_v2.ResNetV2Spec(port.PathConfig(stride_test=8, centered_stride=True), 50)
    t = port_resnet_v2.op_table(spec)
    stem = t['backbone.conv1_conv']
    assert (stem['bn'], stem['act'], stem['bias'], stem['pre']) == (None, None, 'backbone.conv1_conv.bias', ((2.0,) * 3, (-1.0,) * 3))
    sp = t['backbone.conv2_block3_shortcut_pool']
    assert (sp['maxpool'], sp['kernel'], sp['stride'], sp['pad']) == (True, 1, 2, (-1, 0))
    c2 = t['backbone.conv2_block3_2_conv']
    assert (c2['kernel'], c2['stride'], c2['sample'], c2['pad'], c2['dil']) == (3, 2, 1, (1, 1), 1)
    assert t['backbone.conv4_block2_2_conv']['dil'] == 2 and t['backbone.conv5_block3_2_conv']['pad'] == (4, 4)
    c3 = t['backbone.conv3_block1_3_conv']
    assert (c3['bn'], c3['act'], c3['bias']) == (None, None, 'backbone.conv3_block1_3_conv.bias')
    pre = t['backbone.conv3_block2_preact_bn']
    assert (pre['weight'], pre['depthwise'], pre['act'], pre['eps'], pre['kernel']) == (None, True, 'relu', 1e-5, 1)
    assert t['backbone.post_bn']['bn'] == 'backbone.post_bn'
    # the engine's op list minus the ops the reference has no layer for: the names follow the Keras layers
    assert len(t) == 2 + sum(4 for _ in range(16)) + 4 + 1 + 1  # stem, pool, 4 ops per block, 4 _0_convs, 1 subsample, post_bn


def _fp32_bn_op(sd, key, x, eps=1e-5, relu=True):
    """the BN-only op as the fp32 engine evaluates it: folded fp32 weight and bias, fmaf, then ReLU"""
    w = sd[key + '.weight'].double() / torch.sqrt(sd[key + '.running_var'].double() + eps)
    b = sd[key + '.bias'].double() - sd[key + '.running_mean'].double() * w
    w, b = w.float().double(), b.float().double()
    z = (x.double() * w + b).float()  # fmaf: one rounding of the exact product-sum
    return torch.relu(z) if relu else z


def test_bn_only_op_bound():
    pcfg = port.PathConfig(proc_side=64, stride_test=32)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, 50)
    sd = tfb.make_state_dict(spec, pcfg, 4, seed=0, calib_batch=2)
    g = torch.Generator().manual_seed(3)
    for key in ('backbone.conv3_block2_preact_bn', 'backbone.post_bn'):
        c = sd[key + '.weight'].numel()
        x = (sd[key + '.running_mean'] + sd[key + '.running_var'].sqrt() * torch.randn(2, 4, 4, c, generator=g)).float()
        ref, tol = port_resnet_v2.layer_bound(sd, spec, key, x.double(), precision='fp32')
        r, bad = port_ops.check_bound(_fp32_bn_op(sd, key, x), ref, tol, 'fp32')
        assert bad == 0, (key, r)
        assert port_ops.check_bound(_fp32_bn_op(sd, key, x, relu=False), ref, tol, 'fp32')[1] > 0  # a missing ReLU
        assert port_ops.check_bound(_fp32_bn_op(sd, key, x, eps=1e-3), ref, tol, 'fp32')[1] > 0  # a wrong eps
        ref16, tol16 = port_resnet_v2.layer_bound(sd, spec, key, x.bfloat16().double(), precision='bf16')
        dev16 = _fp32_bn_op(sd, key, x.bfloat16().float()).bfloat16()
        assert port_ops.check_bound(dev16, ref16, tol16, 'bf16')[1] == 0


def test_subsample_is_exact_and_equals_the_restatement():
    pcfg = port.PathConfig(proc_side=64, stride_test=8)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, 50)
    sd = tfb.make_state_dict(spec, pcfg, 4, seed=0, calib_batch=1)
    x = torch.randn(2, 16, 16, 256, dtype=torch.float64)
    ref, tol = port_resnet_v2.layer_bound(sd, spec, 'backbone.conv2_block3_shortcut_pool', x, precision='bf16')
    assert torch.equal(ref, x[:, 1::2, 1::2]) and not tol.any()


def test_features_finite_for_the_deepest_net():
    pcfg = port.PathConfig(proc_side=64, stride_test=32, depth=8)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, 152)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(2, 64, seed=0)
    with torch.no_grad():
        out = port.metrabs_forward(sd, spec, pcfg, 8, crops, k)
    assert torch.isfinite(out).all()
