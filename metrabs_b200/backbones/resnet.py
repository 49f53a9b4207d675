"""ResNet V1 (MeTRAbs stride/dilation switching) parameter holders for the H100 engine: ResNet-18 / 34 (basic block) and
ResNet-50 / 101 / 152 (bottleneck).

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


class Features(nn.Module):
    stages = []

    def __init__(self, depth=50):
        super().__init__()
        self.arch, counts, basic = DEPTHS[depth]
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
