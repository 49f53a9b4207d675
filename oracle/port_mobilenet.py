"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of both MobileNetV3 variants of the reference's TF/Keras code
(metrabs_tf/backbones/mobilenet_v3.py), and the per-layer reference arithmetic of their engine ops.

* Shared: stem / ``Conv_1`` / ``Conv_2`` :258-296 (``Conv_1`` = ``_depth(6 * last filters)`` with BN and hard-swish,
  ``Conv_2`` = last point channels with a bias, no BN, hard-swish), ``_inverted_res_block`` :490-553 (block 0 has no expand
  conv; residual when stride 1 and the width is unchanged), ``_se_block`` :465-487 (width ``_depth(exp * 0.25)``, ReLU then
  hard-sigmoid), ``correct_pad`` :556-575 with the bottom-right shift, ``_depth`` :449-456, BN eps 1e-3, preprocessing
  builder.py:116-117 (x*255) followed by the in-model ``Rescaling(1/127.5, -1)`` :259.
* Small: table :364-384, last point 1024.  Large: table :403-428 (15 rows; the ReLU blocks 3-5 have 5x5 kernels and SE,
  block 12 takes the bottom-right shift under ``centered_stride``), last point 1280.  Alpha 1, not minimalistic.

PARITY UNPINNED: the reference has no test, golden or importable implementation of MobileNetV3 (Keras only), so
device-vs-oracle parity is "this build's restatement vs this build's kernels".  At ``variant='small'``
``MobileNetV3Spec`` equals ``port_tf_backbones.MobileNetV3SmallSpec`` (same random init stream, same features and taps)
and ``op_table`` equals ``port_ops.mobilenetv3_small_op_table``.

The per-layer part mirrors ``oracle/port_ops.py`` (``conv_layer_reference`` / ``layer_bound``: same rounding points and
the same bound) for the ops of either variant; ``port_ops.check_bound`` there applies to its results unchanged.
"""
import math

import torch
import torch.nn.functional as F

from oracle import port, port_ops
from oracle import port_tf_backbones as tfb

MOBILENETV3_LARGE_ROWS = [
    # (expansion, filters, kernel, stride, se, activation, bottomright)
    (1, 16, 3, 1, False, 'relu', False), (4, 24, 3, 2, False, 'relu', False), (3, 24, 3, 1, False, 'relu', False),
    (3, 40, 5, 2, True, 'relu', False), (3, 40, 5, 1, True, 'relu', False), (3, 40, 5, 1, True, 'relu', False),
    (6, 80, 3, 2, False, 'hswish', False), (2.5, 80, 3, 1, False, 'hswish', False), (2.3, 80, 3, 1, False, 'hswish', False),
    (2.3, 80, 3, 1, False, 'hswish', False), (6, 112, 3, 1, True, 'hswish', False), (6, 112, 3, 1, True, 'hswish', False),
    (6, 160, 5, 2, True, 'hswish', True), (6, 160, 5, 1, True, 'hswish', False), (6, 160, 5, 1, True, 'hswish', False)]
# variant -> (rows, last point channels)
VARIANTS = {'small': (tfb.MOBILENETV3_SMALL_ROWS, 1024), 'large': (MOBILENETV3_LARGE_ROWS, 1280)}


def mobilenet_blocks(variant):
    """[dict(name, cin, exp, filters, kernel, stride, se, se_ch, act, br, residual)] in execution order (widths after
    ``_depth``)."""
    rows, _ = VARIANTS[variant]
    out, cin = [], 16
    for bi, (exp, filters, k, stride, se, act, br) in enumerate(rows):
        cexp = tfb._depth(cin * exp)
        out.append(dict(name='expanded_conv' if bi == 0 else f'expanded_conv_{bi}', cin=cin, exp=cexp, filters=filters,
                        kernel=k, stride=stride, se=se, se_ch=tfb._depth(cexp * 0.25) if se else 0, act=act, br=br,
                        residual=stride == 1 and cin == filters))
        cin = filters
    return out


class MobileNetV3Spec:
    """MobileNetV3 ``variant`` 'small' or 'large'."""

    def __init__(self, cfg: port.PathConfig, variant='small'):
        self.cfg = cfg
        self.variant = variant
        self.name = f'mobilenetv3-{variant}'
        self.out_channels = VARIANTS[variant][1]

    def features(self, sd, image, tap=None, init=None):
        """[B,3,S,S] in [0,1] -> [B,C,S/32,S/32].  With ``init`` = (generator) the weights are created and BN-calibrated
        on the fly (conditioned random init, the draw order of MobileNetV3SmallSpec), otherwise read from ``sd``."""
        p = 'backbone.'
        g = init
        acts = {'relu': F.relu, 'hswish': tfb.hard_swish}

        def conv_bn(x, cname, cout, k, stride=1, groups=1, act=None, bn=True, bias=False, damp=1.0):
            if g is not None:
                cin = x.shape[1] // groups
                sd[p + cname + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))
                if bias:
                    sd[p + cname + '.bias'] = 0.1 * torch.randn(cout, generator=g)
            y = F.conv2d(x, sd[p + cname + '.weight'], sd[p + cname + '.bias'] if bias else None, stride=stride, groups=groups)
            if bn:
                if g is not None:
                    port._calibrate_bn(sd, p + cname + '.BatchNorm', y, g, tfb.MOBILENET_BN_EPS, damp)
                y = tfb._bn(sd, p + cname + '.BatchNorm', y, tfb.MOBILENET_BN_EPS)
            y = act(y) if act is not None else y
            if tap is not None:
                tap[p + cname] = y
            return y

        x = image * 2 - 1  # 255*x (builder.py:116-117) then Rescaling(1/127.5, -1) (mobilenet_v3.py:259)
        s = x.shape[-1]
        out = (s + 1) // 2
        pad_total = max((out - 1) * 2 + 3 - s, 0)  # TF 'same', stride 2
        pb = pad_total // 2
        x = conv_bn(F.pad(x, (pb, pad_total - pb, pb, pad_total - pb)), 'Conv', 16, 3, stride=2, act=tfb.hard_swish)
        for blk in mobilenet_blocks(self.variant):
            name, cexp, k, stride, a = blk['name'], blk['exp'], blk['kernel'], blk['stride'], acts[blk['act']]
            inp = x
            if name != 'expanded_conv':
                x = conv_bn(x, name + '.expand', cexp, 1, act=a)
            shift = 1 if (blk['br'] and self.cfg.centered_stride) else 0
            pbeg = (k - 1) // 2
            pend = k - 1 - pbeg
            if stride == 2:
                x = F.pad(x, (pbeg - shift, pend + shift, pbeg - shift, pend + shift))  # correct_pad, then VALID
            else:
                x = F.pad(x, (pbeg, pend, pbeg, pend))  # 'same', stride 1
            x = conv_bn(x, name + '.depthwise', cexp, k, stride=stride, groups=cexp, act=a)
            if blk['se']:
                csq = blk['se_ch']
                if g is not None:
                    sd[p + name + '.squeeze_excite.Conv.weight'] = torch.randn(csq, cexp, 1, 1, generator=g) * math.sqrt(2.0 / cexp)
                    sd[p + name + '.squeeze_excite.Conv.bias'] = 0.2 * torch.randn(csq, generator=g)
                    sd[p + name + '.squeeze_excite.Conv_1.weight'] = torch.randn(cexp, csq, 1, 1, generator=g) * math.sqrt(2.0 / csq)
                    sd[p + name + '.squeeze_excite.Conv_1.bias'] = 1.0 * torch.randn(cexp, generator=g)
                q = x.mean(dim=(2, 3), keepdim=True)
                q = F.relu(F.conv2d(q, sd[p + name + '.squeeze_excite.Conv.weight'], sd[p + name + '.squeeze_excite.Conv.bias']))
                q = tfb.hard_sigmoid(F.conv2d(q, sd[p + name + '.squeeze_excite.Conv_1.weight'],
                                              sd[p + name + '.squeeze_excite.Conv_1.bias']))
                x = x * q
            res = blk['residual']
            x = conv_bn(x, name + '.project', blk['filters'], 1, damp=0.5 if res else 1.0)
            if res:
                x = x + inp
                if tap is not None:
                    tap[p + name + '.project'] = x
        x = conv_bn(x, 'Conv_1', tfb._depth(x.shape[1] * 6), 1, act=tfb.hard_swish)
        x = conv_bn(x, 'Conv_2', self.out_channels, 1, act=tfb.hard_swish, bn=False, bias=True)
        return x


def op_table(spec: MobileNetV3Spec, prefix='backbone.'):
    """engine op name -> op dict (port_ops._op): TF-'same' stem on 2x-1, correct_pad before the stride-2 depthwise convs
    (bottom-right shift under centered_stride), ReLU / hard-swish, projection without activation (+ residual), Conv_2
    with bias and no BN."""
    e = tfb.MOBILENET_BN_EPS
    s = spec.cfg.proc_side
    pad_total = max(((s + 1) // 2 - 1) * 2 + 3 - s, 0)
    t = {prefix + 'Conv': port_ops._op(prefix + 'Conv.weight', 3, 2, (pad_total // 2, pad_total - pad_total // 2),
                                       act='hswish', bn=prefix + 'Conv.BatchNorm', eps=e, pre=((2.0,) * 3, (-1.0,) * 3))}
    for blk in mobilenet_blocks(spec.variant):
        b, k, stride, act = prefix + blk['name'], blk['kernel'], blk['stride'], blk['act']
        if blk['name'] != 'expanded_conv':
            t[b + '.expand'] = port_ops._op(b + '.expand.weight', act=act, bn=b + '.expand.BatchNorm', eps=e)
        shift = 1 if (blk['br'] and spec.cfg.centered_stride and stride == 2) else 0
        pb = (k - 1) // 2
        t[b + '.depthwise'] = port_ops._op(b + '.depthwise.weight', k, stride, (pb - shift, k - 1 - pb + shift), act=act,
                                           depthwise=True, bn=b + '.depthwise.BatchNorm', eps=e, shift=shift)
        t[b + '.project'] = port_ops._op(b + '.project.weight', bn=b + '.project.BatchNorm', eps=e)
    t[prefix + 'Conv_1'] = port_ops._op(prefix + 'Conv_1.weight', act='hswish', bn=prefix + 'Conv_1.BatchNorm', eps=e)
    t[prefix + 'Conv_2'] = port_ops._op(prefix + 'Conv_2.weight', act='hswish', bias=prefix + 'Conv_2.bias')
    return t


def _layer(sd, op, x_nhwc, res_nhwc, scale, precision, dtype, magnitude=False):
    """port_ops._layer for one op dict of a MobileNetV3 (no max pool, no dilation, residual after the activation):
    -> (output NCHW, pre-activation NCHW, products per output)."""
    dev = x_nhwc.device
    w, bias = port_ops._fold(sd, op)
    st = port_ops.MODES[precision][0] if precision in port_ops.MODES else None
    if st is not None or precision in port_ops.WIDE_MODES:  # folded in fp64, cast to fp32, GEMM weights rounded once to 16 bits
        w, bias = w.float().double(), bias.float().double()
        if st is not None and port_ops.tc_eligible(op, w.shape[1], w.shape[0]):
            w = w.float().to(st).double()
    w, bias = w.to(dev, dtype), bias.to(dev, dtype)
    if op['stem']:
        a, c = (torch.tensor(v, dtype=torch.float32).to(dev, dtype)[None, :, None, None] for v in op['pre'])
        x = x_nhwc.to(dtype)
        x = (x * a).abs() + c.abs() if magnitude else x * a + c
    else:
        x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    if scale is not None:
        s = scale.to(dev, dtype)[:, :, None, None]
        if st is not None and port_ops.MODES[precision][1] and not magnitude:  # se_scale_kernel: fp32 product, rounded
            x = (x.float() * s.float()).to(st).to(dtype)
        elif precision in port_ops.WIDE_MODES and not magnitude:  # fp32 product, no further rounding
            x = (x.float() * s.float()).to(dtype)
        else:
            x = x * s
    if magnitude:
        x, w, bias = x.abs(), w.abs(), bias.abs()
    x = F.pad(x, op['pad'] * 2)
    z = F.conv2d(x, w, bias, stride=op['stride'], groups=x.shape[1] if op['depthwise'] else 1)
    y = z if magnitude else port_ops._act(z, op['act'])
    if res_nhwc is not None:
        res = res_nhwc.permute(0, 3, 1, 2).to(dtype)
        y = y + (res.abs() if magnitude else res)
    return y, z, w.shape[1] * w.shape[2] * w.shape[3]


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='exact', dtype=torch.float64):
    """port_ops.conv_layer_reference for the ops of ``spec`` (either variant).  Returns NHWC in ``dtype``."""
    return _layer(sd, op_table(spec)[name], x_nhwc, res_nhwc, scale, precision, dtype)[0].permute(0, 2, 3, 1).contiguous()


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='fp16'):
    """port_ops.layer_bound for the ops of ``spec`` (either variant): -> (ref, tol), NHWC fp64, with the same bound
    tol = 2^-p (|ref| + e) + e + floor, e = L_act C_ACC (K + 4) 2^-24 refabs + e_act + 2^-23 |ref| (any engine mode:
    port_ops.bound_from_parts)."""
    op = op_table(spec)[name]
    y, z, k = _layer(sd, op, x_nhwc, res_nhwc, scale, precision, torch.float64)
    zabs = _layer(sd, op, x_nhwc, res_nhwc, scale, precision, torch.float64, magnitude=True)[1]
    tc32 = precision == 'tf32x3' and port_ops.tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
    tol = port_ops.bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)
