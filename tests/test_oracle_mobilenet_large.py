"""CPU: the MobileNetV3 restatement (oracle/port_mobilenet.py MobileNetV3Spec) for MobileNetV3-Large against hand counts
of its table and, at variant 'small', against the MobileNetV3-Small restatement and op table the other tests use; the
parameter holders of metrabs_b200.backbones.mobilenet_v3 against that key schema; and the C header's arch value.  Parity of
these backbones is "this build's restatement vs this build's kernels": the reference has them only as Keras code."""
import os
import re

import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import mobilenet_v3
from oracle import port, port_mobilenet, port_ops
from oracle import port_tf_backbones as tfb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# mobilenet_v3.py:403-428 with _depth applied: expanded widths and SE widths (0 = no SE) of the 15 blocks
LARGE_EXP = [16, 64, 72, 72, 120, 120, 240, 200, 184, 184, 480, 672, 672, 960, 960]
LARGE_SE = [0, 0, 0, 24, 32, 32, 0, 0, 0, 0, 120, 168, 168, 240, 240]
# stem + 2 (block 0: depthwise, project) + 14 * 3 + 8 SE blocks * 2 + Conv_1 + Conv_2
LARGE_CONVS = 63
# 2 * MACs of every conv (SE fcs included, at 1x1) per crop at S=256, counted by hand from the table: 712.58 MFLOP in the
# stem, blocks and Conv_1 / Conv_2, 3.01 MFLOP in the SE fcs
LARGE_GFLOP_256 = 0.71559552


def _meta_features(variant, side, centered=True):
    """-> (state dict, tap, features) of MobileNetV3Spec(variant) at side x side, shapes only: the weights are made at a
    small side, then everything runs on the meta device."""
    small = port.PathConfig(proc_side=64, stride_test=32)
    sd = tfb.make_state_dict(port_mobilenet.MobileNetV3Spec(small, variant), small, 4, seed=0, calib_batch=1)
    meta = {k: v.to('meta') for k, v in sd.items()}
    spec = port_mobilenet.MobileNetV3Spec(port.PathConfig(proc_side=side, stride_test=32, centered_stride=centered), variant)
    tap = {}
    with torch.device('meta'):
        feats = spec.features(meta, torch.empty(1, 3, side, side), tap=tap)
    return sd, tap, feats


def test_large_table():
    blocks = port_mobilenet.mobilenet_blocks('large')
    assert [b['exp'] for b in blocks] == LARGE_EXP
    assert [b['se_ch'] for b in blocks] == LARGE_SE
    assert [b['kernel'] for b in blocks] == [3, 3, 3, 5, 5, 5, 3, 3, 3, 3, 3, 3, 5, 5, 5]
    assert [b['stride'] for b in blocks] == [1, 2, 1, 2, 1, 1, 2, 1, 1, 1, 1, 1, 2, 1, 1]
    assert [i for i, b in enumerate(blocks) if b['br']] == [12]
    assert all(b['act'] == 'relu' for b in blocks[:6]) and all(b['act'] == 'hswish' for b in blocks[6:])
    assert blocks[0]['residual'] and blocks[0]['cin'] == 16  # block 0: no expand, 3x3 stride 1 on 16 channels + residual
    assert [i for i, b in enumerate(blocks) if b['residual']] == [0, 2, 4, 5, 7, 8, 9, 11, 13, 14]


@pytest.mark.parametrize('side', [256, 224])
def test_large_structure_and_flops(side):
    sd, tap, feats = _meta_features('large', side)
    convs = [k for k, v in sd.items() if k.startswith('backbone.') and k.endswith('.weight') and v.dim() == 4]
    assert len(convs) == LARGE_CONVS
    assert 'backbone.expanded_conv.expand.weight' not in sd
    assert tuple(feats.shape) == (1, 1280, -(-side // 32), -(-side // 32))
    assert tuple(tap['backbone.Conv_1'].shape)[1] == 960
    assert sd['backbone.Conv_2.bias'].shape == (1280,) and 'backbone.Conv_2.BatchNorm.weight' not in sd
    total = 0.0
    for k in convs:
        w = sd[k]
        name = k[:-len('.weight')]
        hw = 1 if '.squeeze_excite.' in name else tap[name].shape[2] * tap[name].shape[3]
        total += 2.0 * hw * w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3]
    print(f'mobilenetv3-large@{side}: {total / 1e9:.4f} GFLOP/crop')
    if side == 256:
        assert abs(total / 1e9 - LARGE_GFLOP_256) < 1e-9


def test_large_parameter_names_match_the_restatement():
    pcfg = port.PathConfig(proc_side=64)
    sd = tfb.make_state_dict(port_mobilenet.MobileNetV3Spec(pcfg, 'large'), pcfg, 4, seed=0, calib_batch=1)
    m = mobilenet_v3.mobilenet_v3_large()
    ours = {'backbone.' + k for k in m.state_dict()}
    assert ours == {k for k in sd if k.startswith('backbone.')}
    assert all(tuple(v.shape) == tuple(sd['backbone.' + k].shape) for k, v in m.state_dict().items())
    assert m.arch == _lib.ARCH_MOBILENETV3_LARGE and m.last_channel == 1280
    table = port_mobilenet.op_table(port_mobilenet.MobileNetV3Spec(pcfg, 'large'))
    assert {k + '.weight' for k in table} == {k for k in ours if k.endswith('.weight') and '.squeeze_excite.' not in k
                                              and not k.endswith('BatchNorm.weight')}


def test_small_parameter_names_unchanged():
    m = mobilenet_v3.mobilenet_v3_small()
    names = list(m.state_dict())
    assert names[:6] == ['Conv.weight', 'Conv.BatchNorm.weight', 'Conv.BatchNorm.bias', 'Conv.BatchNorm.running_mean',
                         'Conv.BatchNorm.running_var', 'Conv.BatchNorm.num_batches_tracked']
    assert m.arch == _lib.ARCH_MOBILENETV3_SMALL and m.last_channel == 1024
    pcfg = port.PathConfig(proc_side=64)
    sd = tfb.make_state_dict(tfb.MobileNetV3SmallSpec(pcfg), pcfg, 4, seed=0, calib_batch=1)
    assert {'backbone.' + k for k in names} == {k for k in sd if k.startswith('backbone.')}


def test_header_arch_value():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    assert int(re.search(r'MTB_ARCH_MOBILENETV3_LARGE = (\d+)', src)[1]) == _lib.ARCH_MOBILENETV3_LARGE == 8
    dw = {m[0]: int(m[1]) for m in re.findall(r'MTB_DW_([A-Z0-9_]+) = (\d+)', src)}
    assert dw == {'GENERIC': _lib.DW_GENERIC, 'TMA': _lib.DW_TMA, 'STRIP_16B': _lib.DW_STRIP_16B,
                  'STRIP_F32': _lib.DW_STRIP_F32, '5X5_16B': _lib.DW_5X5_16B}


@pytest.mark.parametrize('cfgkw', [dict(proc_side=64), dict(proc_side=96, centered_stride=False), dict(proc_side=70)])
def test_small_variant_equals_the_small_restatement(cfgkw):
    """MobileNetV3Spec(cfg, 'small') draws the same random init, computes the same features and taps, and its op table and
    per-layer arithmetic equal port_tf_backbones.MobileNetV3SmallSpec / port_ops.mobilenetv3_small_op_table /
    port_ops.conv_layer_reference / port_ops.layer_bound."""
    pcfg = port.PathConfig(stride_test=32, **cfgkw)
    old, new = tfb.MobileNetV3SmallSpec(pcfg), port_mobilenet.MobileNetV3Spec(pcfg, 'small')
    sd_old = tfb.make_state_dict(old, pcfg, 4, seed=0, calib_batch=1)
    sd_new = tfb.make_state_dict(new, pcfg, 4, seed=0, calib_batch=1)
    assert list(sd_old) == list(sd_new) and all(torch.equal(sd_old[k], sd_new[k]) for k in sd_old)
    x, _ = port.synthetic_inputs(2, pcfg.proc_side)
    tap_old, tap_new = {}, {}
    with torch.no_grad():
        assert torch.equal(old.features(sd_old, x, tap=tap_old), new.features(sd_old, x, tap=tap_new))
    assert list(tap_old) == list(tap_new) and all(torch.equal(tap_old[k], tap_new[k]) for k in tap_old)
    table = port_mobilenet.op_table(new)
    assert table == port_ops.mobilenetv3_small_op_table(pcfg)
    g = torch.Generator().manual_seed(1)
    nhwc = lambda key: tuple(tap_new[key].permute(0, 2, 3, 1).shape[1:])  # noqa: E731
    p = 'backbone.'
    # op -> (input shape, residual shape or None, SE scale)
    cases = {p + 'Conv': ((3, pcfg.proc_side, pcfg.proc_side), None, False),
             p + 'expanded_conv.depthwise': (nhwc(p + 'Conv'), None, False),
             p + 'expanded_conv.project': (nhwc(p + 'expanded_conv.depthwise'), None, True),
             p + 'expanded_conv_3.depthwise': (nhwc(p + 'expanded_conv_3.expand'), None, False),
             p + 'expanded_conv_8.depthwise': (nhwc(p + 'expanded_conv_8.expand'), None, False),
             p + 'expanded_conv_9.project': (nhwc(p + 'expanded_conv_9.depthwise'), nhwc(p + 'expanded_conv_9.project'), True),
             p + 'Conv_2': (nhwc(p + 'Conv_1'), None, False)}
    for name, (in_shape, res_shape, se) in cases.items():
        make = torch.rand if name == p + 'Conv' else torch.randn  # the stem takes NCHW crops in [0, 1]
        xin = make((2,) + in_shape, generator=g, dtype=torch.float64)
        res = None if res_shape is None else torch.randn((2,) + res_shape, generator=g, dtype=torch.float64)
        sc = torch.rand(2, in_shape[2], generator=g, dtype=torch.float64) if se else None
        for precision in ('exact', 'bf16', 'bf16_simt', 'fp16', 'fp16_simt'):
            a = port_ops.conv_layer_reference(sd_old, old, name, xin, res, sc, precision=precision)
            b = port_mobilenet.conv_layer_reference(sd_old, new, name, xin, res, sc, precision=precision)
            assert torch.equal(a, b), (name, precision)
        for precision in ('bf16', 'bf16_simt', 'fp16', 'fp16_simt'):
            ra, ta = port_ops.layer_bound(sd_old, old, name, xin, res, sc, precision=precision)
            rb, tb = port_mobilenet.layer_bound(sd_old, new, name, xin, res, sc, precision=precision)
            assert torch.equal(ra, rb) and torch.equal(ta, tb), (name, precision)


def test_large_bound_accepts_rounded_reference():
    """port_ops.check_bound applies to port_mobilenet.layer_bound unchanged: the 16-bit rounding of the exact layer
    passes, a result one dropped border tap away does not."""
    pcfg = port.PathConfig(proc_side=64, stride_test=32)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
    sd = tfb.make_state_dict(spec, pcfg, 4, seed=0, calib_batch=1)
    g = torch.Generator().manual_seed(3)
    name = 'backbone.expanded_conv_12.depthwise'  # 5x5 stride 2, hard-swish
    x = torch.randn(2, 4, 4, 672, generator=g, dtype=torch.float64).to(torch.bfloat16).double()
    ref, tol = port_mobilenet.layer_bound(sd, spec, name, x, precision='bf16')
    assert port_ops.check_bound(ref.to(torch.bfloat16).double(), ref, tol, 'bf16')[1] == 0
    x2 = x.clone()
    x2[:, 0, 0, :] = 0  # a corner input pixel lost
    bad = port_mobilenet.conv_layer_reference(sd, spec, name, x2, precision='bf16').to(torch.bfloat16).double()
    assert port_ops.check_bound(bad, ref, tol, 'bf16')[1] > 0
