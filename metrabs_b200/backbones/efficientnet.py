"""EfficientNetV2 backbones for the H100 engine.

Mirrors the constructor surface of /root/reference/metrabs_pytorch/backbones/efficientnet.py
(``efficientnet_v2_{s,m,l}()`` returning an object whose ``.features`` is used, and ``PreprocLayer``; model
assembly recipe scripts/demo_image.py:59-74).  The modules built here only HOLD parameters under the reference's
``state_dict`` key schema (``<stage>.<block>.block.<i>.{0.weight,1.weight,1.bias,1.running_mean,...}``); the
arithmetic runs in libmetrabs_b200.so (stem / FusedMBConv / MBConv / SE kernels), which receives the block table
(efficientnet.py:379-433) through ``mtb_config.stages``.
"""
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
}


def stage_table(size, centered_stride=None):
    if centered_stride is None:
        centered_stride = get_config().centered_stride
    rows, last = _TABLES[size]
    stages = [dict(block=r[0], expand=r[1], kernel=r[2], stride=r[3], cin=r[4], cout=r[5], layers=r[6],
                   bottomright=bool(len(r) > 7 and r[7] and centered_stride)) for r in rows]
    return stages, last


def _conv_bn(cin, cout, k, groups=1):
    """Parameter holder with the key layout of torchvision's Conv2dNormActivation: '0' conv (no bias), '1' BN."""
    return nn.Sequential(nn.Conv2d(cin, cout, k, groups=groups, bias=False), nn.BatchNorm2d(cout, eps=1e-3))


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
    """Parameter tree of ``EfficientNet.features`` (children '0' stem, '1'..'n' stages, 'n+1' last conv)."""
    arch = _lib.ARCH_EFFNET

    def __init__(self, stages, last_channel):
        super().__init__()
        self.stages = stages
        self.last_channel = last_channel
        self.add_module('0', _conv_bn(3, stages[0]['cin'], 3))
        for si, st in enumerate(stages):
            blocks = []
            for bi in range(st['layers']):
                cin = st['cin'] if bi == 0 else st['cout']
                cexp = cin * st['expand']
                if st['block'] == 'fused':
                    if st['expand'] != 1:
                        layers = [_conv_bn(cin, cexp, st['kernel']), _conv_bn(cexp, st['cout'], 1)]
                    else:
                        layers = [_conv_bn(cin, st['cout'], st['kernel'])]
                else:
                    layers = [_conv_bn(cin, cexp, 1)] if st['expand'] != 1 else []
                    layers += [_conv_bn(cexp, cexp, st['kernel'], groups=cexp), _SE(cexp, max(1, cin // 4)),
                               _conv_bn(cexp, st['cout'], 1)]
                blocks.append(_Block(layers))
            self.add_module(str(si + 1), nn.Sequential(*blocks))
        self.add_module(str(len(stages) + 1), _conv_bn(stages[-1]['cout'], last_channel, 1))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so); wrap this in '
                           'metrabs_b200.models.metrabs.Metrabs')


class EfficientNet(nn.Module):
    def __init__(self, size):
        super().__init__()
        stages, last = stage_table(size)
        self.size = size
        self.features = Features(stages, last)


class PreprocLayer(nn.Module):
    """x*2-1 (efficientnet.py:1181-1186); folded into the stem kernel's input load."""

    def forward(self, inp):
        return inp


def efficientnet_v2_s(**kwargs):
    return EfficientNet('s')


def efficientnet_v2_m(**kwargs):
    return EfficientNet('m')


def efficientnet_v2_l(**kwargs):
    return EfficientNet('l')


def efficientnet_v2_tiny(**kwargs):
    return EfficientNet('tiny')
