"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of EfficientNet-B0..B7 (the reference's
``/root/reference/metrabs_pytorch/backbones/efficientnet.py`` ``efficientnet_b0()`` .. ``efficientnet_b7()``, :753-1013),
and the per-layer reference arithmetic of their engine ops.

* Table: the base table of ``_efficientnet_conf`` :388-396 scaled by (width, depth): channels
  ``_make_divisible(c * width, 8)``, layers ``ceil(layers * depth)`` (MBConvConfig :62-93), the bottom-right shift on row 6
  under ``centered_stride`` (:394), last conv ``4 * last cout`` (:320).  Every row is an MBConv (:110-173); row 1 has
  expand 1 and so no expand conv.
* BatchNorm eps: torchvision's default 1e-5 for B0-B4, 1e-3 for B5-B7 (:973, :1011).  ``oracle/port.py`` fixes 1e-3 for
  the V2 tables; this module carries the eps on the spec instead (``EffNetBSpec.bn_eps``) and leaves port.py's V2 specs,
  their random init and their state-dict checksums as they are.

Parity pin: the reference runs these constructors unmodified on torch-cpu, so ``oracle/gen_golden_effnet_b.py`` builds
them through the public ``efficientnet_bN()`` and commits their outputs under ``tests/golden/effnetb*.npz``;
``tests/test_oracle_effnet_b.py`` checks this restatement against those files and, where the reference tree exists,
its tables and BN modules against the reference's.
"""
import dataclasses
import math
from typing import List

import torch
import torch.nn.functional as F

from oracle import port, port_mobilenet, port_ops

# _efficientnet_conf base table (:388-396): (expand, kernel, stride, cin, cout, layers, bottomright under centered_stride)
B_BASE = [(1, 3, 1, 32, 16, 1, False), (6, 3, 2, 16, 24, 2, False), (6, 5, 2, 24, 40, 2, False),
          (6, 3, 2, 40, 80, 3, False), (6, 5, 1, 80, 112, 3, False), (6, 5, 2, 112, 192, 4, True),
          (6, 3, 1, 192, 320, 1, False)]
# variant -> (width_mult, depth_mult, BatchNorm eps)  (:753-1013)
B_VARIANTS = {0: (1.0, 1.0, 1e-5), 1: (1.0, 1.1, 1e-5), 2: (1.1, 1.2, 1e-5), 3: (1.2, 1.4, 1e-5), 4: (1.4, 1.8, 1e-5),
              5: (1.6, 2.2, 1e-3), 6: (1.8, 2.6, 1e-3), 7: (2.0, 3.1, 1e-3)}


def make_divisible(v, divisor=8):
    """torchvision.models._utils._make_divisible with min_value = divisor."""
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


@dataclasses.dataclass
class EffNetBSpec:
    name: str
    stages: List[port.StageSpec]
    last_channel: int
    bn_eps: float

    @property
    def stem_channels(self):
        return self.stages[0].cin

    def features(self, sd, image, tap=None):
        """port.metrabs_forward calls this for a spec that is not a port.EffNetSpec."""
        return effnet_b_features(sd, self, image, tap=tap)


def effnet_b_spec(name, centered_stride=True):
    """'efficientnet-b0' .. 'efficientnet-b7'."""
    variant = int(name.rsplit('-b', 1)[1])
    width, depth, eps = B_VARIANTS[variant]
    rows = [port.StageSpec('mb', e, k, s, make_divisible(cin * width), make_divisible(cout * width),
                           int(math.ceil(n * depth)), bool(br and centered_stride))
            for e, k, s, cin, cout, n, br in B_BASE]
    return EffNetBSpec(name, rows, 4 * rows[-1].cout, eps)


def se_scale(sd, key, x):
    """torchvision SqueezeExcitation: avgpool -> fc1 -> SiLU -> fc2 -> sigmoid, [B,C,1,1]."""
    s = x.mean(dim=(2, 3), keepdim=True)
    s = F.silu(F.conv2d(s, sd[f'{key}.fc1.weight'], sd[f'{key}.fc1.bias']))
    return torch.sigmoid(F.conv2d(s, sd[f'{key}.fc2.weight'], sd[f'{key}.fc2.bias']))


def effnet_b_features(sd, spec: EffNetBSpec, image, prefix='backbone.1', tap=None):
    """[B,3,S,S] fp32 in [0,1] -> [B,last_channel,S/32,S/32]  (PreprocLayer + EfficientNet.features, MBConv rows)."""
    e = spec.bn_eps
    x = image * 2 - 1
    x = port._conv_bn(sd, f'{prefix}.0', port._fixed_pad(x, 3, 0), stride=2, eps=e, tap=tap)
    for b in port.effnet_block_list(spec):
        key = f'{prefix}.{b["key"]}.block'
        inp = x
        i = 0
        if b['expand'] != 1:
            x = port._conv_bn(sd, f'{key}.{i}', x, eps=e, tap=tap)
            i += 1
        x = port._fixed_pad(x, b['kernel'], b['shift'])
        x = port._conv_bn(sd, f'{key}.{i}', x, stride=b['stride'], groups=b['cin'] * b['expand'], eps=e, tap=tap)
        x = x * se_scale(sd, f'{key}.{i + 1}', x)
        x = port._conv_bn(sd, f'{key}.{i + 2}', x, act=False, eps=e, tap=tap)
        if b['residual']:
            x = x + inp
        if tap is not None:
            tap[f'{prefix}.{b["key"]}'] = x
    return port._conv_bn(sd, f'{prefix}.{len(spec.stages) + 1}', x, eps=e, tap=tap)


def make_state_dict(spec: EffNetBSpec, cfg: port.PathConfig, n_joints, seed=0, calib_batch=4, head_gain=10.0):
    """port.make_effnet_state_dict's conditioned random init (BN running stats calibrated layer by layer, residual-branch
    BNs damped, peaky head) for an MBConv-only table, with the spec's BN eps."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    prefix, e = 'backbone.1', spec.bn_eps
    calib, _ = port.synthetic_inputs(calib_batch, cfg.proc_side, seed=seed + 77)
    with torch.no_grad():
        x = port._init_conv_bn(sd, f'{prefix}.0', port._fixed_pad(calib * 2 - 1, 3, 0), g, spec.stem_channels, 3, stride=2,
                               eps=e)
        for b in port.effnet_block_list(spec):
            key = f'{prefix}.{b["key"]}.block'
            inp = x
            cexp = b['cin'] * b['expand']
            i = 0
            if b['expand'] != 1:
                x = port._init_conv_bn(sd, f'{key}.{i}', x, g, cexp, 1, eps=e)
                i += 1
            x = port._fixed_pad(x, b['kernel'], b['shift'])
            x = port._init_conv_bn(sd, f'{key}.{i}', x, g, cexp, b['kernel'], stride=b['stride'], groups=cexp, eps=e)
            se, csq = f'{key}.{i + 1}', max(1, b['cin'] // 4)
            sd[f'{se}.fc1.weight'] = torch.randn(csq, cexp, 1, 1, generator=g) * math.sqrt(2.0 / cexp)
            sd[f'{se}.fc1.bias'] = 0.2 * torch.randn(csq, generator=g)
            sd[f'{se}.fc2.weight'] = torch.randn(cexp, csq, 1, 1, generator=g) * math.sqrt(2.0 / csq)
            sd[f'{se}.fc2.bias'] = 0.5 * torch.randn(cexp, generator=g)
            x = x * se_scale(sd, se, x)
            x = port._init_conv_bn(sd, f'{key}.{i + 2}', x, g, b['cout'], 1, act=False, eps=e,
                                   gamma_scale=0.5 if b['residual'] else 1.0)
            if b['residual']:
                x = x + inp
        port._init_conv_bn(sd, f'{prefix}.{len(spec.stages) + 1}', x, g, spec.last_channel, 1, eps=e)
    port.init_head(sd, g, spec.last_channel, n_joints, cfg.depth, head_gain)
    return sd


# ---------------------------------------------------------------------------------------------- per-layer arithmetic
def op_table(spec: EffNetBSpec, prefix='backbone.1'):
    """engine op name -> op dict (port_ops._op): port_ops.effnet_op_table with the spec's BN eps."""
    return {k: dict(v, eps=spec.bn_eps) for k, v in port_ops.effnet_op_table(spec, prefix).items()}


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='exact', dtype=torch.float64):
    """port_ops.conv_layer_reference for the ops of ``spec``.  Returns NHWC in ``dtype``."""
    return port_mobilenet._layer(sd, op_table(spec)[name], x_nhwc, res_nhwc, scale, precision, dtype)[0].permute(
        0, 2, 3, 1).contiguous()


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='fp16'):
    """port_ops.layer_bound for the ops of ``spec``: -> (ref, tol), NHWC fp64, with the same bound
    tol = 2^-p (|ref| + e) + e + floor, e = L_act C_ACC (K + 4) 2^-24 refabs + e_act + 2^-23 |ref| (any engine mode:
    port_ops.bound_from_parts).  (port_mobilenet._layer is the op-dict form of port_ops._layer: no max pool or dilation, residual after the activation,
    which is also what an MBConv op needs.)"""
    op = op_table(spec)[name]
    y, z, k = port_mobilenet._layer(sd, op, x_nhwc, res_nhwc, scale, precision, torch.float64)
    zabs = port_mobilenet._layer(sd, op, x_nhwc, res_nhwc, scale, precision, torch.float64, magnitude=True)[1]
    tc32 = precision == 'tf32x3' and port_ops.tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
    tol = port_ops.bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)
