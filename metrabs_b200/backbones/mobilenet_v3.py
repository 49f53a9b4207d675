"""MobileNetV3-Small and -Large parameter holders for the H100 engine.

Keras-only in the reference (/root/reference/metrabs_tf/backbones/mobilenet_v3.py:258-296, :348-428, :465-553); key schema
defined by this build from the Keras layer names with '/' -> '.': ``backbone.Conv.weight``,
``backbone.Conv.BatchNorm.*``, ``backbone.expanded_conv_<i>.{expand,depthwise,project}.weight`` (+ ``.BatchNorm.*``),
``backbone.expanded_conv_<i>.squeeze_excite.{Conv,Conv_1}.{weight,bias}``, ``backbone.Conv_1.*``, ``backbone.Conv_2.*``.
Block 0 (``expanded_conv``) has no expand conv.  Alpha 1.  ``minimalistic=True`` (Keras' keyword, the reference's
``mobilenetV3{Small,Large}mini``, :250-257) gives every block a 3x3 depthwise kernel and ReLU, and no squeeze-excitation
(no ``squeeze_excite`` keys); the stem, ``Conv_1`` and ``Conv_2`` use ReLU too."""
from torch import nn

from metrabs_b200 import _lib

_ROWS = [  # MobileNetV3-Small (:364-384): (expanded channels, filters, kernel, has SE)
    (16, 16, 3, True), (72, 24, 3, False), (88, 24, 3, False), (96, 40, 5, True), (240, 40, 5, True), (240, 40, 5, True),
    (120, 48, 5, True), (144, 48, 5, True), (288, 96, 5, True), (576, 96, 5, True), (576, 96, 5, True)]
_ROWS_LARGE = [  # MobileNetV3-Large (:403-428)
    (16, 16, 3, False), (64, 24, 3, False), (72, 24, 3, False), (72, 40, 5, True), (120, 40, 5, True), (120, 40, 5, True),
    (240, 80, 3, False), (200, 80, 3, False), (184, 80, 3, False), (184, 80, 3, False), (480, 112, 3, True),
    (672, 112, 3, True), (672, 160, 5, True), (960, 160, 5, True), (960, 160, 5, True)]
# variant -> (arch, rows, last point channels)
VARIANTS = {'small': (_lib.ARCH_MOBILENETV3_SMALL, _ROWS, 1024), 'large': (_lib.ARCH_MOBILENETV3_LARGE, _ROWS_LARGE, 1280)}
ARCH_MINI = {'small': _lib.ARCH_MOBILENETV3_SMALL_MINI, 'large': _lib.ARCH_MOBILENETV3_LARGE_MINI}


def _depth(v, divisor=8):
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


def _conv(cin, cout, k, groups=1, bn=True, bias=False):
    m = nn.Conv2d(cin, cout, k, groups=groups, bias=bias)
    if bn:
        m.add_module('BatchNorm', nn.BatchNorm2d(cout, eps=1e-3))
    return m


class Features(nn.Module):
    stages = []

    def __init__(self, variant='small', minimalistic=False):
        super().__init__()
        self.arch, rows, self.last_channel = VARIANTS[variant]
        if minimalistic:
            self.arch = ARCH_MINI[variant]
            rows = [(cexp, filters, 3, False) for cexp, filters, _k, _se in rows]
        self.variant = variant
        self.minimalistic = minimalistic
        self.add_module('Conv', _conv(3, 16, 3))
        cin = 16
        for i, (cexp, filters, k, se) in enumerate(rows):
            blk = nn.Module()
            if i != 0:
                blk.add_module('expand', _conv(cin, cexp, 1))
            blk.add_module('depthwise', _conv(cexp, cexp, k, groups=cexp))
            if se:
                sem = nn.Module()
                sem.add_module('Conv', _conv(cexp, _depth(cexp * 0.25), 1, bn=False, bias=True))
                sem.add_module('Conv_1', _conv(_depth(cexp * 0.25), cexp, 1, bn=False, bias=True))
                blk.add_module('squeeze_excite', sem)
            blk.add_module('project', _conv(cexp, filters, 1))
            self.add_module('expanded_conv' if i == 0 else f'expanded_conv_{i}', blk)
            cin = filters
        self.add_module('Conv_1', _conv(cin, _depth(cin * 6), 1))
        self.add_module('Conv_2', _conv(_depth(cin * 6), self.last_channel, 1, bn=False, bias=True))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so)')


def mobilenet_v3_small(minimalistic=False, **kwargs):
    """Use as ``Metrabs(mobilenet_v3_small(), joint_info)``; ``minimalistic=True`` for ``mobilenetV3Smallmini``."""
    return Features('small', minimalistic)


def mobilenet_v3_large(minimalistic=False, **kwargs):
    """Use as ``Metrabs(mobilenet_v3_large(), joint_info)`` (the backbone of metrabs_mob3l_y4 / _y4t);
    ``minimalistic=True`` for ``mobilenetV3Largemini``."""
    return Features('large', minimalistic)
