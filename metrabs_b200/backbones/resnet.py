"""ResNet (MeTRAbs stride/dilation switching) parameter holders for the H100 engine: ResNet-18 / 34 (V1 basic block),
ResNet-50 / 101 / 152 (V1 bottleneck), their V1.5 forms (``resnet50v1_5`` ...: the same parameters, block 1's stride on
the 3x3 conv, torch_preproc) and the pre-activation ResNet-50 / 101 / 152 V2 (``FeaturesV2``).

The reference has these backbones only as Keras code (metrabs_tf/backbones/resnet.py:239-319 bottleneck,
:322-388 basic block, :601-707 stride plan and stacks, :746-788 depths); there is no PyTorch key schema for them, so this
build defines one from the Keras layer names: ``backbone.conv1_conv.weight`` (+ ``.bias`` for 50/101/152),
``backbone.conv1_bn.{weight,bias,running_mean,running_var}``, ``backbone.conv<2-5>_block<i>_<0-3>_{conv,bn}.*`` (conv
weights in torch [Cout,Cin,kh,kw] layout).  No conv of ResNet-18/34 has a bias.  Arithmetic runs in libmetrabs_b200.so
(plan_resnet in csrc/engine.cu)."""
from torch import nn

from metrabs_b200 import _lib

# depth -> (arch, blocks in conv2..conv5, basic block)
DEPTHS = {18: (_lib.ARCH_RESNET18, [2, 2, 2, 2], True), 34: (_lib.ARCH_RESNET34, [3, 4, 6, 3], True),
          50: (_lib.ARCH_RESNET50, [3, 4, 6, 3], False), 101: (_lib.ARCH_RESNET101, [3, 4, 23, 3], False),
          152: (_lib.ARCH_RESNET152, [3, 8, 36, 3], False)}


# depth -> arch of the V1.5 bottleneck nets (ResNetUnified(v1_5=True), metrabs_tf/backbones/resnet.py:621-666, :791-800)
DEPTHS_V1_5 = {50: _lib.ARCH_RESNET50V1_5, 101: _lib.ARCH_RESNET101V1_5, 152: _lib.ARCH_RESNET152V1_5}


class Features(nn.Module):
    stages = []

    def __init__(self, depth=50, v1_5=False):
        super().__init__()
        self.arch, counts, basic = DEPTHS[depth]
        if v1_5:  # the same layers and keys as V1; only the plan (stride on _2_conv) and the preprocessing differ
            self.arch = DEPTHS_V1_5[depth]
        self.depth = depth
        bias = not basic
        self.last_channel = 512 if basic else 2048
        self._conv_bn('conv1', 3, 64, 7, bias)
        cin = 64
        for st, (f, n) in enumerate(zip([64, 128, 256, 512], counts)):
            for bi in range(n):
                name = f'conv{st + 2}_block{bi + 1}'
                if basic:
                    if bi == 0 and st > 0:  # conv2_block1 has an identity shortcut
                        self._conv_bn(name + '_0', cin, f, 1, bias)
                    self._conv_bn(name + '_1', cin, f, 3, bias)
                    self._conv_bn(name + '_2', f, f, 3, bias)
                    cin = f
                    continue
                if bi == 0:
                    self._conv_bn(name + '_0', cin, 4 * f, 1, bias)
                self._conv_bn(name + '_1', cin, f, 1, bias)
                self._conv_bn(name + '_2', f, f, 3, bias)
                self._conv_bn(name + '_3', f, 4 * f, 1, bias)
                cin = 4 * f

    def _conv_bn(self, name, cin, cout, k, bias):
        self.add_module(name + '_conv', nn.Conv2d(cin, cout, k, bias=bias))
        self.add_module(name + '_bn', nn.BatchNorm2d(cout, eps=1e-5))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so)')


def resnet18(**kwargs):
    """Use as ``Metrabs(resnet18(), joint_info)`` (keys ``backbone.<keras layer>...``, no conv biases)."""
    return Features(18)


def resnet34(**kwargs):
    """Use as ``Metrabs(resnet34(), joint_info)`` (keys ``backbone.<keras layer>...``, no conv biases)."""
    return Features(34)


def resnet50(**kwargs):
    """Use as ``Metrabs(resnet50(), joint_info)`` (keys ``backbone.<keras layer>...``)."""
    return Features(50)


def resnet101(**kwargs):
    """Use as ``Metrabs(resnet101(), joint_info)`` (keys ``backbone.<keras layer>...``)."""
    return Features(101)


def resnet152(**kwargs):
    """Use as ``Metrabs(resnet152(), joint_info)`` (keys ``backbone.<keras layer>...``)."""
    return Features(152)


def resnet50v1_5(**kwargs):
    """Use as ``Metrabs(resnet50v1_5(), joint_info)`` (the keys of ``resnet50()``)."""
    return Features(50, v1_5=True)


def resnet101v1_5(**kwargs):
    """Use as ``Metrabs(resnet101v1_5(), joint_info)`` (the keys of ``resnet101()``)."""
    return Features(101, v1_5=True)


def resnet152v1_5(**kwargs):
    """Use as ``Metrabs(resnet152v1_5(), joint_info)`` (the keys of ``resnet152()``)."""
    return Features(152, v1_5=True)


# depth -> (arch, blocks in conv2..conv5) of the pre-activation nets (metrabs_tf/backbones/resnet.py:803-831)
DEPTHS_V2 = {50: (_lib.ARCH_RESNET50V2, [3, 4, 6, 3]), 101: (_lib.ARCH_RESNET101V2, [3, 4, 23, 3]),
             152: (_lib.ARCH_RESNET152V2, [3, 8, 36, 3])}


class FeaturesV2(nn.Module):
    """ResNetUnifiedV2 (metrabs_tf/backbones/resnet.py:710-745, block2_dense :391-456) parameters under the Keras layer
    names: ``backbone.conv1_conv.{weight,bias}`` (no stem BN), per block ``_preact_bn``, ``_0_conv.{weight,bias}`` (block1
    of a stack only), ``_1_conv.weight`` + ``_1_bn``, ``_2_conv.weight`` + ``_2_bn``, ``_3_conv.{weight,bias}`` (no BN),
    and ``backbone.post_bn``.  The bias of ``_0_conv`` is Keras' default for a ``Conv2DDenseSame`` that does not pass
    ``use_bias`` (the class is from the un-vendored ``fleras``: a reading, as for V1)."""
    stages = []

    def __init__(self, depth=50):
        super().__init__()
        self.arch, counts = DEPTHS_V2[depth]
        self.depth = depth
        self.last_channel = 2048
        self.add_module('conv1_conv', nn.Conv2d(3, 64, 7, bias=True))
        cin = 64
        for st, (f, n) in enumerate(zip([64, 128, 256, 512], counts)):
            for bi in range(n):
                name = f'conv{st + 2}_block{bi + 1}'
                self.add_module(name + '_preact_bn', nn.BatchNorm2d(cin, eps=1e-5))
                if bi == 0:
                    self.add_module(name + '_0_conv', nn.Conv2d(cin, 4 * f, 1, bias=True))
                self.add_module(name + '_1_conv', nn.Conv2d(cin, f, 1, bias=False))
                self.add_module(name + '_1_bn', nn.BatchNorm2d(f, eps=1e-5))
                self.add_module(name + '_2_conv', nn.Conv2d(f, f, 3, bias=False))
                self.add_module(name + '_2_bn', nn.BatchNorm2d(f, eps=1e-5))
                self.add_module(name + '_3_conv', nn.Conv2d(f, 4 * f, 1, bias=True))
                cin = 4 * f
        self.add_module('post_bn', nn.BatchNorm2d(cin, eps=1e-5))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so)')


def resnet50v2(**kwargs):
    """Use as ``Metrabs(resnet50v2(), joint_info)`` (keys ``backbone.<keras layer>...``, see FeaturesV2)."""
    return FeaturesV2(50)


def resnet101v2(**kwargs):
    """Use as ``Metrabs(resnet101v2(), joint_info)`` (keys ``backbone.<keras layer>...``, see FeaturesV2)."""
    return FeaturesV2(101)


def resnet152v2(**kwargs):
    """Use as ``Metrabs(resnet152v2(), joint_info)`` (keys ``backbone.<keras layer>...``, see FeaturesV2)."""
    return FeaturesV2(152)
