"""CPU: the ResNet family restatement (oracle/port_resnet.py ResNetSpec, ResNet-18/34/50/101/152 V1) against hand
counts of its structure and, at depth 50, against the ResNet-50 restatement and op table the other tests use, the parameter holders of metrabs_b200.backbones.resnet against its key schema, the basic block's
stride_train-dependent dilations, and the C header's arch values against the ctypes constants.  Parity of these backbones
is "this build's restatement vs this build's kernels": the reference has them only as Keras code."""
import os
import re

import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import resnet
from oracle import port, port_ops, port_resnet
from oracle import port_tf_backbones as tfb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTHS = [18, 34, 50, 101, 152]
N_CONVS = {18: 20, 34: 36, 50: 53, 101: 104, 152: 155}
# conv GFLOP per crop at S=256 (2 * MACs of every conv, strided convs counted at their output size), by output stride
HAND_GFLOP = {32: {18: 4.74, 34: 9.57, 50: 10.07, 101: 19.77, 152: 29.47},
              8: {18: 24.06, 34: 45.20, 50: 49.63, 101: 88.42, 152: 120.37}}


def _meta_features(depth, side, stride_test, stride_train=32):
    """-> (state dict, tap) of ResNetSpec(depth) at side x side, shapes only: the weights are made at a small side, then
    everything runs on the meta device."""
    small = port.PathConfig(proc_side=32, stride_test=stride_test, stride_train=stride_train)
    spec = port_resnet.ResNetSpec(small, depth)
    sd = tfb.make_state_dict(spec, small, 4, seed=0, calib_batch=1)
    meta = {k: v.to('meta') for k, v in sd.items()}
    spec = port_resnet.ResNetSpec(port.PathConfig(proc_side=side, stride_test=stride_test, stride_train=stride_train), depth)
    tap = {}
    with torch.device('meta'):  # the restatement's own constants (the caffe mean) are made on the meta device too
        feats = spec.features(meta, torch.empty(1, 3, side, side), tap=tap)
    return sd, tap, feats


def _conv_gflop(sd, tap):
    total = 0.0
    for k, w in sd.items():
        if k.startswith('backbone.') and k.endswith('_conv.weight'):
            _b, cout, h, w_ = tap[k[:-len('.weight')]].shape
            total += 2.0 * h * w_ * cout * w.shape[1] * w.shape[2] * w.shape[3]
    return total / 1e9


@pytest.mark.parametrize('depth', DEPTHS)
@pytest.mark.parametrize('stride', [32, 8])
def test_structure_and_flops(depth, stride):
    sd, tap, feats = _meta_features(depth, 256, stride, stride_train=stride)
    convs = [k for k in sd if k.startswith('backbone.') and k.endswith('_conv.weight')]
    assert len(convs) == N_CONVS[depth]
    assert tuple(feats.shape) == (1, 512 if depth < 50 else 2048, 256 // stride, 256 // stride)
    gflop = _conv_gflop(sd, tap)
    print(f'resnet{depth} s{stride}: {gflop:.2f} GFLOP/crop')
    assert abs(gflop - HAND_GFLOP[stride][depth]) < 0.005 * HAND_GFLOP[stride][depth]


@pytest.mark.parametrize('depth', DEPTHS)
def test_parameter_names_match_the_restatement(depth):
    pcfg = port.PathConfig(proc_side=32)
    sd = tfb.make_state_dict(port_resnet.ResNetSpec(pcfg, depth), pcfg, 4, seed=0, calib_batch=1)
    ours = {'backbone.' + k for k in getattr(resnet, f'resnet{depth}')().state_dict()}
    assert ours == {k for k in sd if k.startswith('backbone.')}
    conv_biases = [k for k in ours if k.endswith('_conv.bias')]
    if depth < 50:
        assert not conv_biases
    else:
        assert len(conv_biases) == N_CONVS[depth]
    assert set(port_resnet.op_table(port_resnet.ResNetSpec(pcfg, depth))) >= {k[:-len('.weight')] for k in ours if k.endswith('_conv.weight')}


def test_resnet50_parameter_names_unchanged():
    names = list(resnet.resnet50().state_dict())
    assert names[:7] == ['conv1_conv.weight', 'conv1_conv.bias', 'conv1_bn.weight', 'conv1_bn.bias', 'conv1_bn.running_mean',
                         'conv1_bn.running_var', 'conv1_bn.num_batches_tracked']
    assert len(names) == 53 * 2 + 53 * 5
    assert resnet.resnet50().arch == _lib.ARCH_RESNET50 and resnet.resnet50().last_channel == 2048


def _dilations(stride_train, stride_test, depth=18):
    blocks = port_resnet.resnet_blocks(port.PathConfig(stride_train=stride_train, stride_test=stride_test), depth)
    return {b['name']: (b['dil'], b['dil2']) for b in blocks}


def test_basic_block_dilations():
    # train stride 32, test stride 8: block1 of conv4 / conv5 gets (2, 4) / (4, 8), the other blocks (2, 2) / (4, 4)
    d = _dilations(32, 8, 34)
    assert d['conv4_block1'] == (2, 4) and d['conv5_block1'] == (4, 8)
    assert all(d[f'conv4_block{i}'] == (2, 2) for i in range(2, 7))
    assert all(d[f'conv5_block{i}'] == (4, 4) for i in range(2, 4))
    assert all(v == (1, 1) for k, v in d.items() if k.startswith(('conv2', 'conv3')))
    # equal strides: both 3x3s of every block take dil_out of the stack
    d = _dilations(8, 8)
    assert d == {'conv2_block1': (1, 1), 'conv2_block2': (1, 1), 'conv3_block1': (1, 1), 'conv3_block2': (1, 1),
                 'conv4_block1': (2, 2), 'conv4_block2': (2, 2), 'conv5_block1': (4, 4), 'conv5_block2': (4, 4)}
    assert _dilations(32, 32) == {k: (1, 1) for k in d}
    # 16 / 8: only conv4's first block is strided in training and not at test time
    d = _dilations(16, 8)
    assert d['conv4_block1'] == (2, 4) and d['conv5_block1'] == (4, 4)
    # the bottleneck nets do not depend on stride_train
    assert port_resnet.resnet_blocks(port.PathConfig(stride_train=8, stride_test=8), 101) == \
        port_resnet.resnet_blocks(port.PathConfig(stride_train=32, stride_test=8), 101)


def test_stride_train_below_stride_test_is_refused():
    # the reference's int(1 * 1 / 2) gives a dilation of 0
    with pytest.raises(ValueError, match='dilation of 0'):
        port_resnet.resnet_blocks(port.PathConfig(stride_train=8, stride_test=32), 18)


def test_basic_op_table():
    t = port_resnet.op_table(port_resnet.ResNetSpec(port.PathConfig(stride_test=8, stride_train=32, centered_stride=True), 18))
    c3 = t['backbone.conv3_block1_1_conv']  # the centered stride: dense SAME 3x3 sampled at 1::2
    assert (c3['kernel'], c3['stride'], c3['sample'], c3['pad'], c3['act']) == (3, 2, 1, (1, 1), 'relu')
    assert t['backbone.conv3_block1_0_conv']['sample'] == 1
    assert 'backbone.conv2_block1_0_conv' not in t
    c4 = t['backbone.conv4_block1_2_conv']
    assert (c4['dil'], c4['pad'], c4['res_first'], c4['act'], c4['bias']) == (4, (4, 4), True, 'relu', None)
    assert t['backbone.conv1_conv']['bias'] is None


def test_header_arch_values_match_the_binding():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    values = {m[0]: int(m[1]) for m in re.findall(r'MTB_ARCH_([A-Z0-9_]+) = (\d+)', src)}
    for name, v in values.items():
        assert getattr(_lib, 'ARCH_' + name) == v
    assert {values[f'RESNET{d}'] for d in DEPTHS} == {1, 4, 5, 6, 7}
    assert {d: resnet.DEPTHS[d][0] for d in DEPTHS} == {d: values[f'RESNET{d}'] for d in DEPTHS}


@pytest.mark.parametrize('cfgkw', [dict(proc_side=64, stride_test=8), dict(proc_side=96, stride_test=16, centered_stride=False),
                                   dict(proc_side=64, stride_test=32)])
def test_depth50_equals_the_resnet50_restatement(cfgkw):
    """ResNetSpec(cfg, 50) draws the same random init, computes the same features and taps, and its op table and per-layer
    arithmetic equal port_tf_backbones.ResNet50Spec / port_ops.resnet50_op_table / port_ops.layer_bound."""
    pcfg = port.PathConfig(**cfgkw)
    old, new = tfb.ResNet50Spec(pcfg), port_resnet.ResNetSpec(pcfg, 50)
    sd_old = tfb.make_state_dict(old, pcfg, 4, seed=0, calib_batch=1)
    sd_new = tfb.make_state_dict(new, pcfg, 4, seed=0, calib_batch=1)
    assert list(sd_old) == list(sd_new) and all(torch.equal(sd_old[k], sd_new[k]) for k in sd_old)
    x, _ = port.synthetic_inputs(1, pcfg.proc_side)
    tap_old, tap_new = {}, {}
    with torch.no_grad():
        assert torch.equal(old.features(sd_old, x, tap=tap_old), new.features(sd_old, x, tap=tap_new))
    assert list(tap_old) == list(tap_new) and all(torch.equal(tap_old[k], tap_new[k]) for k in tap_old)
    assert port_resnet.op_table(new) == port_ops.resnet50_op_table(pcfg)
    assert [b[:5] + (b[5],) for b in tfb.resnet50_blocks(pcfg)] == \
        [(b['name'], b['filters'], b['stride'], b['shift'], b['dil'], b['conv_shortcut']) for b in port_resnet.resnet_blocks(pcfg, 50)]
    g = torch.Generator().manual_seed(1)
    nhwc = lambda key: tuple(tap_new[key].permute(0, 2, 3, 1).shape[1:])  # noqa: E731
    b2 = 'backbone.conv2_block3_3_conv'
    # op -> (input shape, residual shape or None)
    cases = {'backbone.conv1_conv': ((3, pcfg.proc_side, pcfg.proc_side), None),
             'backbone.pool1_pool': (nhwc('backbone.conv1_conv'), None),
             'backbone.conv3_block1_0_conv': (nhwc(b2), None), 'backbone.conv3_block1_1_conv': (nhwc(b2), None),
             'backbone.conv4_block2_2_conv': (nhwc('backbone.conv4_block2_1_conv'), None),
             'backbone.conv5_block3_3_conv': (nhwc('backbone.conv5_block3_2_conv'), nhwc('backbone.conv5_block3_3_conv'))}
    for name, (in_shape, res_shape) in cases.items():
        make = torch.rand if name == 'backbone.conv1_conv' else torch.randn  # the stem takes NCHW crops in [0, 1]
        xin = make((2,) + in_shape, generator=g, dtype=torch.float64)
        res = None if res_shape is None else torch.randn((2,) + res_shape, generator=g, dtype=torch.float64)
        for precision in ('exact', 'bf16', 'fp16_simt'):
            a = port_ops.conv_layer_reference(sd_old, old, name, xin, res, precision=precision)
            b = port_resnet.conv_layer_reference(sd_old, new, name, xin, res, precision=precision)
            assert torch.equal(a, b), (name, precision)
        for precision in ('bf16', 'fp16'):
            ra, ta = port_ops.layer_bound(sd_old, old, name, xin, res, precision=precision)
            rb, tb = port_resnet.layer_bound(sd_old, new, name, xin, res, precision=precision)
            assert torch.equal(ra, rb) and torch.equal(ta, tb), (name, precision)
