"""CPU: the ResNet V1.5 and minimalistic MobileNetV3 restatements (oracle/port_builder_variants.py) against readings of
the Keras code, the parameter holders of metrabs_b200.backbones against their key schema (strict loading), the C header's
arch values against the ctypes constants, and the stem bound of the torch_preproc stem.  Parity of these backbones is
"this build's restatement vs this build's kernels": the reference has them only as Keras code."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

from metrabs_b200 import _lib
from metrabs_b200.backbones import mobilenet_v3, resnet
from oracle import port, port_mobilenet, port_ops, port_resnet
from oracle import port_builder_variants as V
from oracle import port_tf_backbones as tfb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTHS = [50, 101, 152]


def keras_v1_5_convs(output_stride, centered, counts):
    """conv name -> (stride, shift, dilation), read off ResNetUnified(v1_5=True) (resnet.py:601-666) and block1_dense
    (:239-319) line by line, without the oracle's block table."""
    import math
    brs = [False] * 3
    i_last = int(round(math.log2(output_stride))) - 3
    if centered and i_last >= 0:
        brs[i_last] = True
    dil_in, dil_out, strides = [1, 1, 1], [1, 1, 1], [2, 2, 2]
    for i in range(max(0, i_last + 1), 3):
        strides[i], dil_in[i] = 1, 2 ** (i - i_last - 1)
        dil_out[i] = 2 * dil_in[i]
    # (strides, bottomright, dilation_rate) of the StridingInfos :629-645 (v1_5: dil_in on the way in)
    first = (1, False, dil_in[0])
    infos_in = [(strides[i], brs[i], dil_in[i]) for i in range(3)]
    infos_out = [(1, False, dil_out[i]) for i in range(3)]
    out = {}
    for st, n in enumerate(counts):
        for bi in range(n):
            s, br, d = (first if st == 0 else infos_in[st - 1]) if bi == 0 else (first if st == 0 else infos_out[st - 1])
            name = f'conv{st + 2}_block{bi + 1}'
            if bi == 0:  # conv_shortcut: Conv2DDenseSame 1x1 with the block's striding
                out[name + '_0_conv'] = (s, int(br), 1)
            out[name + '_1_conv'] = (1, 0, 1)  # layers.Conv2D(filters, 1, strides=1)
            out[name + '_2_conv'] = (s, int(br), d)  # Conv2DDenseSame 3x3 with strides, bottomright and dilation
            out[name + '_3_conv'] = (1, 0, 1)
    return out


@pytest.mark.parametrize('depth', DEPTHS)
@pytest.mark.parametrize('stride', [8, 16, 32])
@pytest.mark.parametrize('centered', [True, False])
def test_v1_5_table_matches_the_keras_reading(depth, stride, centered):
    pcfg = port.PathConfig(stride_test=stride, centered_stride=centered, stride_train=32)
    want = keras_v1_5_convs(stride, centered, port_resnet.DEPTHS[depth][0])
    t = V.resnet_v1_5_op_table(V.ResNetV15Spec(pcfg, depth))
    got = {}
    for name, op in t.items():
        if name.endswith(('conv1_conv', 'pool1_pool')):
            continue
        got[name[len('backbone.'):]] = (op['stride'], op['shift'], op['dil'])
        if op['kernel'] == 3:  # dense SAME sampled at shift::stride: symmetric pad dil, then the sample offset
            assert op['pad'] == (op['dil'], op['dil']) and op['sample'] == op['shift']
    assert got == want
    # V1.5 does not read stride_train, like the V1 bottleneck nets
    assert V.resnet_v1_5_blocks(pcfg, depth) == V.resnet_v1_5_blocks(port.PathConfig(stride_test=stride, centered_stride=centered,
                                                                                      stride_train=8), depth)


def test_v1_5_block1_takes_dil_in():
    """At output stride 8, conv4_block1's 3x3 has dilation 1 and conv5_block1's 2 (dil_in); V1 and the later blocks use
    dil_out (2 and 4).  At stride 16 only conv5 is dilated: 1 in block1, 2 after."""
    d = {b['name']: b['dil'] for b in V.resnet_v1_5_blocks(port.PathConfig(stride_test=8), 50)}
    assert d['conv4_block1'] == 1 and d['conv5_block1'] == 2
    assert all(d[f'conv4_block{i}'] == 2 for i in range(2, 7)) and all(d[f'conv5_block{i}'] == 4 for i in (2, 3))
    assert all(d[k] == 1 for k in d if k.startswith(('conv2', 'conv3')))
    v1 = {b['name']: b['dil'] for b in port_resnet.resnet_blocks(port.PathConfig(stride_test=8), 50)}
    assert v1['conv4_block1'] == 2 and v1['conv5_block1'] == 4  # what a dil_out block1 would give
    d16 = {b['name']: b['dil'] for b in V.resnet_v1_5_blocks(port.PathConfig(stride_test=16), 50)}
    assert d16['conv5_block1'] == 1 and d16['conv5_block2'] == 2 and d16['conv4_block1'] == 1
    t = V.resnet_v1_5_op_table(V.ResNetV15Spec(port.PathConfig(stride_test=8), 50))
    assert (t['backbone.conv4_block1_2_conv']['dil'], t['backbone.conv4_block1_2_conv']['stride']) == (1, 1)
    assert (t['backbone.conv5_block1_2_conv']['dil'], t['backbone.conv5_block1_2_conv']['stride']) == (2, 1)
    c3 = t['backbone.conv3_block1_2_conv']  # the centered stride of stride 8 sits on conv3
    assert (c3['stride'], c3['sample'], c3['pad'], c3['dil']) == (2, 1, (1, 1), 1)
    assert t['backbone.conv3_block1_1_conv']['stride'] == 1 and t['backbone.conv3_block1_1_conv']['sample'] is None


def test_basic_block_depths_have_no_v1_5():
    with pytest.raises(ValueError, match='no V1.5'):
        V.ResNetV15Spec(port.PathConfig(), 18)


@pytest.mark.parametrize('depth', DEPTHS)
@pytest.mark.parametrize('stride', [32, 8])
def test_v1_5_shapes_and_flops(depth, stride):
    small = port.PathConfig(proc_side=32, stride_test=stride)
    sd = tfb.make_state_dict(V.ResNetV15Spec(small, depth), small, 4, seed=0, calib_batch=1)
    pcfg = port.PathConfig(proc_side=256, stride_test=stride)
    tap = {}
    with torch.device('meta'):
        feats = V.ResNetV15Spec(pcfg, depth).features({k: v.to('meta') for k, v in sd.items()}, torch.empty(1, 3, 256, 256), tap=tap)
    assert tuple(feats.shape) == (1, 2048, 256 // stride, 256 // stride)
    total = sum(2.0 * tap[k[:-7]].shape[2] * tap[k[:-7]].shape[3] * v.shape[0] * v[0].numel()
                for k, v in sd.items() if k.startswith('backbone.') and k.endswith('_conv.weight') and k[:-7] in tap)
    # every _1_conv runs at the block's input resolution: V1.5 costs more than V1 at the strided blocks
    assert abs(total / 1e9 - V.resnet_v1_5_gflop_per_crop(pcfg, depth)) < 1e-3 * total / 1e9


@pytest.mark.parametrize('depth', DEPTHS)
def test_v1_5_state_dict_is_v1s_and_loads_strictly(depth):
    pcfg = port.PathConfig(proc_side=32)
    sd = tfb.make_state_dict(V.ResNetV15Spec(pcfg, depth), pcfg, 4, seed=0, calib_batch=1)
    sd_v1 = tfb.make_state_dict(port_resnet.ResNetSpec(pcfg, depth), pcfg, 4, seed=0, calib_batch=1)
    assert list(sd) == list(sd_v1) and all(sd[k].shape == sd_v1[k].shape for k in sd)
    m = getattr(resnet, f'resnet{depth}v1_5')()
    assert m.arch == resnet.DEPTHS_V1_5[depth] and m.last_channel == 2048
    assert list(m.state_dict()) == list(getattr(resnet, f'resnet{depth}')().state_dict())
    bb = {k[len('backbone.'):]: v for k, v in sd.items() if k.startswith('backbone.')}
    full = dict(bb, **{k: v for k, v in m.state_dict().items() if k.endswith('num_batches_tracked')})
    m.load_state_dict(full, strict=True)
    assert set(V.resnet_v1_5_op_table(V.ResNetV15Spec(pcfg, depth))) >= {k[:-7] for k in sd if k.endswith('_conv.weight')}
    missing = dict(full)
    del missing['conv3_block1_2_conv.bias']
    with pytest.raises(RuntimeError, match='Missing key'):
        m.load_state_dict(missing, strict=True)
    with pytest.raises(RuntimeError, match='Unexpected key'):
        m.load_state_dict(dict(full, **{'conv3_block1_2_bn.extra': torch.zeros(1)}), strict=True)


# MobileNetV3Small / Large stack_fn (mobilenet_v3.py:364-384 / :403-428) as written: the kernel, se_ratio and activation
# arguments are literal or the model's own (K, SE, ACT).  (expansion, filters, kernel, stride, se_ratio, activation)
K, SE, ACT = 'kernel', 'se_ratio', 'activation'
KERAS_SMALL = [(1, 16, 3, 2, SE, 'relu'), (72. / 16, 24, 3, 2, None, 'relu'), (88. / 24, 24, 3, 1, None, 'relu'),
               (4, 40, K, 2, SE, ACT), (6, 40, K, 1, SE, ACT), (6, 40, K, 1, SE, ACT), (3, 48, K, 1, SE, ACT),
               (3, 48, K, 1, SE, ACT), (6, 96, K, 2, SE, ACT), (6, 96, K, 1, SE, ACT), (6, 96, K, 1, SE, ACT)]
KERAS_LARGE = [(1, 16, 3, 1, None, 'relu'), (4, 24, 3, 2, None, 'relu'), (3, 24, 3, 1, None, 'relu'),
               (3, 40, K, 2, SE, 'relu'), (3, 40, K, 1, SE, 'relu'), (3, 40, K, 1, SE, 'relu'), (6, 80, 3, 2, None, ACT),
               (2.5, 80, 3, 1, None, ACT), (2.3, 80, 3, 1, None, ACT), (2.3, 80, 3, 1, None, ACT), (6, 112, 3, 1, SE, ACT),
               (6, 112, 3, 1, SE, ACT), (6, 160, K, 2, SE, ACT), (6, 160, K, 1, SE, ACT), (6, 160, K, 1, SE, ACT)]
KERAS = {'small': (KERAS_SMALL, 8), 'large': (KERAS_LARGE, 12)}  # rows, the bottom-right row


def _minimalistic(rows):
    """MobileNetV3(minimalistic=True) :250-253: kernel 3, activation relu, se_ratio None."""
    model = {K: 3, SE: None, ACT: 'relu'}
    return [(e, f, model.get(k, k), s, model.get(se, se) if se is not None else None, model.get(a, a)) for e, f, k, s, se, a in rows]


@pytest.mark.parametrize('variant', ['small', 'large'])
def test_mini_table_matches_the_keras_reading(variant):
    rows, br = KERAS[variant]
    want = _minimalistic(rows)
    blocks = V.mini_blocks(variant)
    assert [(b['kernel'], b['stride'], b['se'], b['act']) for b in blocks] == [(k, s, bool(se), a) for _e, _f, k, s, se, a in want]
    assert [i for i, b in enumerate(blocks) if b['br']] == [br]
    cin, exps = 16, []
    for e, f, *_ in want:
        exps.append(tfb._depth(cin * e))
        cin = f
    assert [b['exp'] for b in blocks] == exps
    full = port_mobilenet.mobilenet_blocks(variant)
    assert [(b['exp'], b['filters'], b['stride'], b['br'], b['residual']) for b in blocks] == \
        [(b['exp'], b['filters'], b['stride'], b['br'], b['residual']) for b in full]
    t = V.mini_op_table(V.MobileNetV3MiniSpec(port.PathConfig(proc_side=256), variant))
    assert {op['act'] for nm, op in t.items() if not nm.endswith('.project')} == {'relu'}
    assert all(op['kernel'] == 3 for nm, op in t.items() if op['depthwise'])


@pytest.mark.parametrize('variant', ['small', 'large'])
def test_mini_state_dict_loads_strictly(variant):
    pcfg = port.PathConfig(proc_side=64)
    spec = V.MobileNetV3MiniSpec(pcfg, variant)
    sd = tfb.make_state_dict(spec, pcfg, 4, seed=0, calib_batch=1)
    m = getattr(mobilenet_v3, f'mobilenet_v3_{variant}')(minimalistic=True)
    assert m.arch == {'small': _lib.ARCH_MOBILENETV3_SMALL_MINI, 'large': _lib.ARCH_MOBILENETV3_LARGE_MINI}[variant]
    assert not any('squeeze_excite' in k for k in m.state_dict())
    assert all(v.shape[-1] == 3 for k, v in m.state_dict().items() if k.endswith('depthwise.weight'))
    bb = {k[len('backbone.'):]: v for k, v in sd.items() if k.startswith('backbone.')}
    full = dict(bb, **{k: v for k, v in m.state_dict().items() if k.endswith('num_batches_tracked')})
    assert set(full) == set(m.state_dict()) and all(full[k].shape == v.shape for k, v in m.state_dict().items())
    m.load_state_dict(full, strict=True)
    assert {k + '.weight' for k in V.mini_op_table(spec)} == {'backbone.' + k for k in bb if k.endswith('.weight')
                                                             and not k.endswith('BatchNorm.weight')}
    # a full net's state dict has SE keys and 5x5 kernels: refused
    full_sd = getattr(mobilenet_v3, f'mobilenet_v3_{variant}')().state_dict()
    with pytest.raises(RuntimeError):
        m.load_state_dict(full_sd, strict=True)
    missing = dict(full)
    del missing['Conv_2.bias']
    with pytest.raises(RuntimeError, match='Missing key'):
        m.load_state_dict(missing, strict=True)
    with pytest.raises(RuntimeError, match='Unexpected key'):
        m.load_state_dict(dict(full, **{'expanded_conv_1.squeeze_excite.Conv.weight': torch.zeros(1)}), strict=True)


def test_header_arch_values():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    values = {m[0]: int(m[1]) for m in re.findall(r'MTB_ARCH_([A-Z0-9_]+) = (\d+)', src)}
    new = {'RESNET50V1_5': 13, 'RESNET101V1_5': 14, 'RESNET152V1_5': 15, 'MOBILENETV3_SMALL_MINI': 16,
           'MOBILENETV3_LARGE_MINI': 17}
    assert {k: values[k] for k in new} == new
    assert all(getattr(_lib, 'ARCH_' + k) == v for k, v in new.items())
    assert len(set(values.values())) == len(values) == 18
    assert _lib.MTB_ABI_VERSION == 2
    assert int(re.search(r'#define MTB_ABI_VERSION (\d+)', src)[1]) == 2


def _stem_case(seed):
    pcfg = port.PathConfig(proc_side=32)
    spec = V.ResNetV15Spec(pcfg, 50)
    sd = tfb.make_state_dict(spec, pcfg, 4, seed=0, calib_batch=1)
    x = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(seed))
    return spec, sd, x


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_stem_bound_holds_in_both_operation_orders(precision):
    """The torch_preproc stem evaluated in fp32 as the kernel orders it, x * fp32(1/std) + fp32(-mean/std), and as the
    reference does, (x - mean) / std, then the conv in fp32: both within layer_bound of the exact (x - mean) / std layer.
    The bound is port_ops' bound plus exactly the explicit constant term (stem_pre_error), and the two fp32 orders differ
    by more than port_ops' bound would allow for the constant rounding alone."""
    name = 'backbone.conv1_conv'
    for seed in range(3):
        spec, sd, x = _stem_case(seed)
        op = V.resnet_v1_5_op_table(spec)[name]
        ref, tol = V.layer_bound(sd, spec, name, x.double(), precision=precision)
        w, b = (t.float() for t in port_ops._fold(sd, op))
        mean, std, scale, shift = V.torch_preproc_constants()
        r = lambda t: t.reshape(1, 3, 1, 1)  # noqa: E731
        for pre in (x * r(scale) + r(shift), (x - r(mean)) / r(std)):
            dev = F.relu(F.conv2d(F.pad(pre, (3, 3, 3, 3)), w, b, stride=2)).permute(0, 2, 3, 1)
            worst, bad = port_ops.check_bound(dev, ref, tol, precision)
            assert bad == 0 and worst < 1.0, (seed, worst)
        # tol = port_ops' bound on the same layer + L_act * the constant term, nothing looser
        y, z, k = V._layer(sd, spec, op, x.double(), None, precision, torch.float64)
        zabs = V._layer(sd, spec, op, x.double(), None, precision, torch.float64, magnitude=True)[1]
        base = port_ops.bound_from_parts(z, y, zabs, k, 'relu', precision, False)
        e = V.stem_pre_error(op, port_ops._fold(sd, op)[0].float().double(), x.double(), torch.float64)
        assert torch.equal(tol, (base + e).permute(0, 2, 3, 1).contiguous())
        assert bool((e > 0).all()) and float((e / base).max()) < 0.1
    # the constants the stem kernel takes are not the reference's division: x * scale + shift != (x - mean) / std in fp32
    mean, std, scale, shift = V.torch_preproc_constants()
    xs = torch.rand(4096, 3, generator=torch.Generator().manual_seed(7))
    assert not torch.equal(xs * scale + shift, (xs - mean) / std)


def test_stem_bound_rejects_caffe_constants():
    """A stem fed 255 x - caffe mean (V1's preprocessing) instead of torch_preproc lies far outside the bound."""
    spec, sd, x = _stem_case(0)
    name = 'backbone.conv1_conv'
    op = V.resnet_v1_5_op_table(spec)[name]
    ref, tol = V.layer_bound(sd, spec, name, x.double(), precision='fp32')
    wrong = port_resnet.op_table(port_resnet.ResNetSpec(spec.cfg, 50))[name]
    dev = port_resnet._layer(sd, wrong, x, None, 'fp32', torch.float32)[0].permute(0, 2, 3, 1)
    assert port_ops.check_bound(dev, ref, tol, 'fp32')[1] > 0
    assert op['pre'] != wrong['pre']
