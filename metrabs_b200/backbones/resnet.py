"""ResNet-50 (V1, MeTRAbs stride/dilation switching) parameter holder for the H100 engine.

The reference has this backbone only as Keras code (/root/reference/metrabs_tf/backbones/resnet.py:239-319, :601-666,
:764-770); there is no PyTorch key schema for it, so this build defines one from the Keras layer names:
``backbone.conv1_conv.{weight,bias}``, ``backbone.conv1_bn.{weight,bias,running_mean,running_var}``,
``backbone.conv<2-5>_block<i>_<0-3>_{conv,bn}.*`` (conv weights in torch [Cout,Cin,kh,kw] layout).  Arithmetic runs in
libmetrabs_b200.so (plan_resnet50 in csrc/engine.cu)."""
from torch import nn

from metrabs_b200 import _lib


class Features(nn.Module):
    arch = _lib.ARCH_RESNET50
    last_channel = 2048
    stages = []

    def __init__(self):
        super().__init__()
        self._conv_bn('conv1', 3, 64, 7, suffix=('_conv', '_bn'))
        cin = 64
        for st, (f, n) in enumerate(zip([64, 128, 256, 512], [3, 4, 6, 3])):
            for bi in range(n):
                name = f'conv{st + 2}_block{bi + 1}'
                if bi == 0:
                    self._conv_bn(name + '_0', cin, 4 * f, 1)
                self._conv_bn(name + '_1', cin, f, 1)
                self._conv_bn(name + '_2', f, f, 3)
                self._conv_bn(name + '_3', f, 4 * f, 1)
                cin = 4 * f

    def _conv_bn(self, name, cin, cout, k, suffix=('_conv', '_bn')):
        self.add_module(name + suffix[0], nn.Conv2d(cin, cout, k, bias=True))
        self.add_module(name + suffix[1], nn.BatchNorm2d(cout, eps=1e-5))

    def forward(self, x):
        raise RuntimeError('metrabs_b200 backbones run inside Metrabs.forward (libmetrabs_b200.so)')


def resnet50(**kwargs):
    """Use as ``Metrabs(resnet50(), joint_info)`` (keys ``backbone.<keras layer>...``)."""
    return Features()
