"""EfficientNetV2 and EfficientNet-B0..B7 backbones for the H100 engine.

Mirrors the constructor surface of /root/reference/metrabs_pytorch/backbones/efficientnet.py
(``efficientnet_v2_{s,m,l}()`` and ``efficientnet_b0()`` .. ``efficientnet_b7()`` returning an object whose ``.features``
is used, plus ``efficientnet_v2_xl()`` and ``efficientnet_v2_b0()`` .. ``_b3()`` for the TF reference's
``efficientnetv2-xl`` / ``-b0`` .. ``-b3`` tables, and ``PreprocLayer``; model
assembly recipe scripts/demo_image.py:59-74).  The modules built here only HOLD parameters under the reference's
``state_dict`` key schema (``<stage>.<block>.block.<i>.{0.weight,1.weight,1.bias,1.running_mean,...}``); the
arithmetic runs in libmetrabs_b200.so (stem / FusedMBConv / MBConv / SE kernels), which receives the block table
(efficientnet.py:379-433) through ``mtb_config.stages``.
"""
import math

import torch
from torch import nn

from metrabs_b200 import _lib
from metrabs_b200.util import get_config

_TABLES = {
    # (block, expand, kernel, stride, cin, cout, layers[, bottomright on the last strided stage])
    's': ([('fused', 1, 3, 1, 24, 24, 2), ('fused', 4, 3, 2, 24, 48, 4), ('fused', 4, 3, 2, 48, 64, 4),
           ('mb', 4, 3, 2, 64, 128, 6), ('mb', 6, 3, 1, 128, 160, 9), ('mb', 6, 3, 2, 160, 256, 15, True)], 1280),
    'm': ([('fused', 1, 3, 1, 24, 24, 3), ('fused', 4, 3, 2, 24, 48, 5), ('fused', 4, 3, 2, 48, 80, 5),
           ('mb', 4, 3, 2, 80, 160, 7), ('mb', 6, 3, 1, 160, 176, 14), ('mb', 6, 3, 2, 176, 304, 18, True),
           ('mb', 6, 3, 1, 304, 512, 5)], 1280),
    'l': ([('fused', 1, 3, 1, 32, 32, 4), ('fused', 4, 3, 2, 32, 64, 7), ('fused', 4, 3, 2, 64, 96, 7),
           ('mb', 4, 3, 2, 96, 192, 10), ('mb', 6, 3, 1, 192, 224, 19), ('mb', 6, 3, 2, 224, 384, 25, True),
           ('mb', 6, 3, 1, 384, 640, 7)], 1280),
    'tiny': ([('fused', 1, 3, 1, 8, 8, 1), ('fused', 4, 3, 2, 8, 16, 2), ('fused', 4, 3, 2, 16, 24, 1),
              ('mb', 4, 3, 2, 24, 32, 2), ('mb', 6, 3, 1, 32, 40, 1), ('mb', 6, 3, 2, 40, 48, 2, True)], 64),
    # the TF reference's v2_xl_block (metrabs_tf effnetv2_configs.py:240-248), width and depth 1.0
    'xl': ([('fused', 1, 3, 1, 32, 32, 4), ('fused', 4, 3, 2, 32, 64, 8), ('fused', 4, 3, 2, 64, 96, 8),
            ('mb', 4, 3, 2, 96, 192, 16), ('mb', 6, 3, 1, 192, 256, 24), ('mb', 6, 3, 2, 256, 512, 32, True),
            ('mb', 6, 3, 1, 512, 640, 8)], 1280),
}

# The TF reference's v2_base_block (effnetv2_configs.py:145-152), scaled per EfficientNetV2-B variant by (width, depth)
# (:266-281) with TF's rules, not torchvision's: channels round_filters, layers round_repeats, head round_filters(1280)
_V2_BASE = [('fused', 1, 3, 1, 32, 16, 1), ('fused', 4, 3, 2, 16, 32, 2), ('fused', 4, 3, 2, 32, 48, 2),
            ('mb', 4, 3, 2, 48, 96, 3), ('mb', 6, 3, 1, 96, 112, 5), ('mb', 6, 3, 2, 112, 192, 8, True)]
_V2_SCALED = {'v2-b0': (1.0, 1.0), 'v2-b1': (1.0, 1.1), 'v2-b2': (1.1, 1.2), 'v2-b3': (1.2, 1.4)}


def round_filters(filters, width):
    """effnetv2_model.py:76-87 with depth_divisor 8: the nearest multiple of 8, at least 8 (no 0.9 rule)."""
    return max(8, int(filters * width + 4) // 8 * 8)


def round_repeats(repeats, depth):
    """effnetv2_model.py:90-94."""
    return int(math.ceil(depth * repeats))


for _v, (_w, _d) in _V2_SCALED.items():
    _TABLES[_v] = ([r[:4] + (round_filters(r[4], _w), round_filters(r[5], _w), round_repeats(r[6], _d)) + r[7:]
                    for r in _V2_BASE], round_filters(1280, _w))


# EfficientNet-B base table (efficientnet.py:388-396): (expand, kernel, stride, cin, cout, layers, bottomright on the last
# strided stage under centered_stride), scaled per variant by (width, depth) and built with BatchNorm eps (:753-1013;
# B0-B4 keep torchvision's default 1e-5, B5-B7 pass 1e-3)
_B_BASE = [(1, 3, 1, 32, 16, 1), (6, 3, 2, 16, 24, 2), (6, 5, 2, 24, 40, 2), (6, 3, 2, 40, 80, 3), (6, 5, 1, 80, 112, 3),
           (6, 5, 2, 112, 192, 4, True), (6, 3, 1, 192, 320, 1)]
_B_VARIANTS = {'b0': (1.0, 1.0, 1e-5), 'b1': (1.0, 1.1, 1e-5), 'b2': (1.1, 1.2, 1e-5), 'b3': (1.2, 1.4, 1e-5),
               'b4': (1.4, 1.8, 1e-5), 'b5': (1.6, 2.2, 1e-3), 'b6': (1.8, 2.6, 1e-3), 'b7': (2.0, 3.1, 1e-3)}
# BatchNorm eps -> mtb_arch of the block grammar
_ARCH_BY_EPS = {1e-3: _lib.ARCH_EFFNET, 1e-5: _lib.ARCH_EFFNET_EPS1E5}


def _make_divisible(v, divisor=8):
    """torchvision.models._utils._make_divisible with min_value = divisor (MBConvConfig.adjust_channels)."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def b_stage_table(variant, centered_stride=None):
    """-> (stages, last_channel, bn_eps) of EfficientNet-``variant`` ('b0'..'b7'): channels _make_divisible(c * width, 8),
    layers ceil(layers * depth) (MBConvConfig :62-93), last conv 4 * the last stage's cout (:320)."""
    if centered_stride is None:
        centered_stride = get_config().centered_stride
    width, depth, eps = _B_VARIANTS[variant]
    stages = [dict(block='mb', expand=r[0], kernel=r[1], stride=r[2], cin=_make_divisible(r[3] * width),
                   cout=_make_divisible(r[4] * width), layers=int(math.ceil(r[5] * depth)),
                   bottomright=bool(len(r) > 6 and r[6] and centered_stride), dilation_in=1, dilation_out=1)
               for r in _B_BASE]
    return stages, 4 * stages[-1]['cout'], eps


# output strides below 32 that the reference defines tables for (metrabs_tf effnetv2_configs.py:163-228); stride 4 would
# dilate FusedMBConv stages and is not built
_DILATED_SIZES = ('s', 'l', 'tiny')
_OUTPUT_STRIDES = (8, 16, 32)


def dilate_stages(stages, output_stride, centered_stride):
    """The stride-32 table ``stages`` re-strided to ``output_stride`` (the reference's ``efficientnetv2-{s,l}-stride{16,8}``
    tables, effnetv2_configs.py:163-228): with a running stride from 2 after the stem and a running dilation d = 1, a
    stride-2 row that would take the stride past ``output_stride`` becomes stride 1 with ``dilation_in`` d, then d doubles
    and is its ``dilation_out``; every other row gets d for both.  The bottom-right shift moves to the last row that still
    strides, under ``centered_stride`` only (:45)."""
    out, running, d = [], 2, 1
    for st in stages:
        st = dict(st, bottomright=False)
        if st['stride'] == 2 and running * 2 > output_stride:
            st.update(stride=1, dilation_in=d, dilation_out=2 * d)
            d *= 2
        else:
            running *= st['stride']
            st.update(dilation_in=d, dilation_out=d)
        out.append(st)
    last_strided = max(i for i, st in enumerate(out) if st['stride'] == 2)
    out[last_strided]['bottomright'] = bool(centered_stride)
    return out


def stage_table(size, centered_stride=None, output_stride=32):
    """-> (stages, last_channel) of EfficientNetV2-``size`` ('s', 'm', 'l', 'xl', 'v2-b0'..'v2-b3', 'tiny') at
    ``output_stride`` 32, or 16 / 8 for 's', 'l' and 'tiny'."""
    if centered_stride is None:
        centered_stride = get_config().centered_stride
    if output_stride not in _OUTPUT_STRIDES:
        raise ValueError(f'EfficientNetV2 output stride {output_stride} is not built: 32, 16 or 8')
    if output_stride != 32 and size not in _DILATED_SIZES:
        raise ValueError(f'EfficientNetV2-{size} has no table at output stride {output_stride}: only '
                         f'{", ".join(_DILATED_SIZES)} run at 16 or 8')
    rows, last = _TABLES[size]
    stages = [dict(block=r[0], expand=r[1], kernel=r[2], stride=r[3], cin=r[4], cout=r[5], layers=r[6],
                   bottomright=bool(len(r) > 7 and r[7] and centered_stride), dilation_in=1, dilation_out=1)
              for r in rows]
    if output_stride != 32:
        stages = dilate_stages(stages, output_stride, centered_stride)
    return stages, last


def _conv_bn(cin, cout, k, groups=1, eps=1e-3):
    """Parameter holder with the key layout of torchvision's Conv2dNormActivation: '0' conv (no bias), '1' BN."""
    return nn.Sequential(nn.Conv2d(cin, cout, k, groups=groups, bias=False), nn.BatchNorm2d(cout, eps=eps))


class _SE(nn.Module):
    def __init__(self, channels, squeeze):
        super().__init__()
        self.fc1 = nn.Conv2d(channels, squeeze, 1)
        self.fc2 = nn.Conv2d(squeeze, channels, 1)


class _Block(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.block = nn.Sequential()
        for i, m in enumerate(layers):
            self.block.add_module(str(i), m)


class Features(nn.Module):
    """Parameter tree of ``EfficientNet.features`` (children '0' stem, '1'..'n' stages, 'n+1' last conv), every BatchNorm
    with epsilon ``bn_eps``: 1e-3 (EfficientNetV2, B5-B7) runs as ``ARCH_EFFNET``, 1e-5 (B0-B4) as ``ARCH_EFFNET_EPS1E5``."""

    def __init__(self, stages, last_channel, bn_eps=1e-3):
        super().__init__()
        if bn_eps not in _ARCH_BY_EPS:
            raise ValueError(f'BatchNorm eps {bn_eps} is not built: 1e-3 or 1e-5')
        self.stages = stages
        self.last_channel = last_channel
        self.bn_eps = bn_eps
        self.arch = _ARCH_BY_EPS[bn_eps]
        self.output_stride = 2 * math.prod(st['stride'] for st in stages)
        bn = lambda cin, cout, k, groups=1: _conv_bn(cin, cout, k, groups, bn_eps)  # noqa: E731
        self.add_module('0', bn(3, stages[0]['cin'], 3))
        for si, st in enumerate(stages):
            blocks = []
            for bi in range(st['layers']):
                cin = st['cin'] if bi == 0 else st['cout']
                cexp = cin * st['expand']
                if st['block'] == 'fused':
                    if st['expand'] != 1:
                        layers = [bn(cin, cexp, st['kernel']), bn(cexp, st['cout'], 1)]
                    else:
                        layers = [bn(cin, st['cout'], st['kernel'])]
                else:
                    layers = [bn(cin, cexp, 1)] if st['expand'] != 1 else []
                    layers += [bn(cexp, cexp, st['kernel'], groups=cexp), _SE(cexp, max(1, cin // 4)),
                               bn(cexp, st['cout'], 1)]
                blocks.append(_Block(layers))
            self.add_module(str(si + 1), nn.Sequential(*blocks))
        self.add_module(str(len(stages) + 1), bn(stages[-1]['cout'], last_channel, 1))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so); wrap this in '
                           'metrabs_b200.models.metrabs.Metrabs')


class EfficientNet(nn.Module):
    """``size``: a V2 table ('s', 'm', 'l', 'xl', 'v2-b0'..'v2-b3', 'tiny') or a B variant ('b0'..'b7').  ``output_stride``
    16 or 8 builds the dilated V2-S / V2-L (and 'tiny') tables; the model's ``Config.stride_test`` must then equal it."""

    def __init__(self, size, output_stride=32):
        super().__init__()
        if size in _B_VARIANTS:
            if output_stride != 32:
                raise ValueError(f'EfficientNet-{size.upper()} has no table at output stride {output_stride}: only 32')
            stages, last, eps = b_stage_table(size)
        else:
            (stages, last), eps = stage_table(size, output_stride=output_stride), 1e-3
        self.size = size
        self.features = Features(stages, last, eps)


class PreprocLayer(nn.Module):
    """x*2-1 (efficientnet.py:1181-1186); folded into the stem kernel's input load."""

    def forward(self, inp):
        return inp


def efficientnet_v2_s(output_stride=32, **kwargs):
    return EfficientNet('s', output_stride)


def efficientnet_v2_m(**kwargs):
    return EfficientNet('m')


def efficientnet_v2_l(output_stride=32, **kwargs):
    return EfficientNet('l', output_stride)


def efficientnet_v2_xl(**kwargs):
    return EfficientNet('xl')


def efficientnet_v2_b0(**kwargs):
    return EfficientNet('v2-b0')


def efficientnet_v2_b1(**kwargs):
    return EfficientNet('v2-b1')


def efficientnet_v2_b2(**kwargs):
    return EfficientNet('v2-b2')


def efficientnet_v2_b3(**kwargs):
    return EfficientNet('v2-b3')


def efficientnet_v2_tiny(output_stride=32, **kwargs):
    return EfficientNet('tiny', output_stride)


def efficientnet_b0(**kwargs):
    return EfficientNet('b0')


def efficientnet_b1(**kwargs):
    return EfficientNet('b1')


def efficientnet_b2(**kwargs):
    return EfficientNet('b2')


def efficientnet_b3(**kwargs):
    return EfficientNet('b3')


def efficientnet_b4(**kwargs):
    return EfficientNet('b4')


def efficientnet_b5(**kwargs):
    return EfficientNet('b5')


def efficientnet_b6(**kwargs):
    return EfficientNet('b6')


def efficientnet_b7(**kwargs):
    return EfficientNet('b7')
