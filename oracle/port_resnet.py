"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of the whole ResNet V1 family of the reference's TF/Keras code
(metrabs_tf/backbones/resnet.py), and the per-layer reference arithmetic of its engine ops.

* ResNet-50 / 101 / 152: ``ResNetUnified`` :621-666 with the V1 bottleneck ``block1_dense`` :239-319 (stride on the first
  1x1 and on the shortcut 1x1, a bias on every conv :270), block counts [3,4,6,3] / [3,4,23,3] / [3,8,36,3] :764-788.
* ResNet-18 / 34: ``ResNetUnifiedBasic`` :669-707 with ``block1_basic_dense`` :322-388 and ``stack1_basic_dense``
  :540-555, block counts [2,2,2,2] / [3,4,6,3] :746-761.  No conv has a bias, the stem included (``ResNet(stack_fn,
  False, False, ...)`` :704-707); conv2_block1 has an identity shortcut (``conv1_shortcut=False``); the stride and the
  bottom-right shift sit on the first 3x3 and on the shortcut 1x1; the second 3x3 is dilated by
  ``dilation_rate_test * strides / strides_test`` (:377-383), with ``strides`` from the stride_train plan.
* Shared: stem + pool :170-198, BN eps 1e-5 :71, stride plan ``get_strides_and_dilations`` :601-618 (V1 uses ``dil_out``
  for the first block of a stack too, :636-644 / :680-684), ``caffe_preproc`` backbones/builder.py:106-108.

``Conv2DDenseSame`` (un-vendored ``fleras``) is read as in ``oracle/port_tf_backbones.py``: a SAME-padded conv evaluated
at pixels ``shift::stride``; for a 3x3 at stride 2 that is a begin pad of ``1 - shift``.  PARITY UNPINNED: the reference
has no test, golden or importable implementation of these backbones, so device-vs-oracle parity is "this build's
restatement vs this build's kernels".  At depth 50 ``ResNetSpec`` equals ``port_tf_backbones.ResNet50Spec`` (same random
init stream, same features) and ``op_table`` equals ``port_ops.resnet50_op_table``.

The per-layer part mirrors ``oracle/port_ops.py`` (``conv_layer_reference`` / ``layer_bound``, same rounding points and
the same bound) for the ops of any depth; ``check_bound`` there applies to its results unchanged.
"""
import math

import torch
import torch.nn.functional as F

from oracle import port, port_ops
from oracle import port_tf_backbones as tfb

# depth -> (blocks in conv2..conv5, basic block)
DEPTHS = {18: ([2, 2, 2, 2], True), 34: ([3, 4, 6, 3], True), 50: ([3, 4, 6, 3], False),
          101: ([3, 4, 23, 3], False), 152: ([3, 8, 36, 3], False)}


def resnet_blocks(cfg: port.PathConfig, depth):
    """[dict(name, filters, stride, shift, dil, dil2, conv_shortcut)] in execution order (inference: stride_test).

    ``stride`` / ``shift`` sit on the shortcut and on the first conv of block1 (V1); ``dil`` is the dilation of the
    bottleneck's 3x3 or of the basic block's first 3x3 (``dil_out`` of the stack in every block, ``dil_in[0]`` in conv2).
    ``dil2`` is the basic block's second 3x3, ``int(dil * strides / strides_test)`` as the reference's ``astype(int)``
    truncates it; it equals ``dil`` except in a block1 whose train and test strides differ."""
    counts, basic = DEPTHS[depth]
    strides, dil_in, dil_out, brs = tfb.resnet_stride_plan(cfg.stride_test, cfg.centered_stride)
    strides_train = tfb.resnet_stride_plan(cfg.stride_train, cfg.centered_stride)[0]
    out = []
    for st, (f, n) in enumerate(zip([64, 128, 256, 512], counts)):
        for bi in range(n):
            first = bi == 0
            stride = strides[st - 1] if (st > 0 and first) else 1
            shift = 1 if (st > 0 and first and brs[st - 1]) else 0
            dil = dil_in[0] if st == 0 else dil_out[st - 1]
            dil2 = dil
            if basic and st > 0 and first:
                dil2 = int(dil * strides_train[st - 1] / strides[st - 1])
                if dil2 < 1:
                    raise ValueError(f'stride_train {cfg.stride_train} < stride_test {cfg.stride_test}: the reference '
                                     f'gives conv{st + 2}_block1_2_conv a dilation of 0')
            out.append(dict(name=f'conv{st + 2}_block{bi + 1}', filters=f, stride=stride, shift=shift, dil=dil, dil2=dil2,
                            conv_shortcut=first and not (basic and st == 0)))
    return out


class ResNetSpec:
    """ResNet V1 of ``depth`` 18, 34, 50, 101 or 152."""

    def __init__(self, cfg: port.PathConfig, depth=50):
        self.cfg = cfg
        self.depth = depth
        self.basic = DEPTHS[depth][1]
        self.name = f'resnet{depth}'
        self.out_channels = 512 if self.basic else 2048

    def features(self, sd, image, tap=None, init=None):
        """[B,3,S,S] in [0,1] -> [B,C,S/s,S/s].  With ``init`` = (generator) the weights are created and BN-calibrated
        on the fly (conditioned random init, the draw order of ResNet50Spec), otherwise read from ``sd``."""
        p = 'backbone.'
        g = init
        bias = not self.basic

        def conv_bn(x, cname, bname, cout, k, stride=1, shift=0, dil=1, pad=0, relu=True, damp=1.0):
            if g is not None:
                cin = x.shape[1]
                sd[p + cname + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))
                if bias:
                    sd[p + cname + '.bias'] = 0.1 * torch.randn(cout, generator=g)
            y = F.conv2d(x, sd[p + cname + '.weight'], sd[p + cname + '.bias'] if bias else None, padding=pad, dilation=dil)
            if stride > 1 or shift:
                y = y[:, :, shift::stride, shift::stride]  # Conv2DDenseSame: dense SAME conv sampled at shift::stride
            if g is not None:
                port._calibrate_bn(sd, p + bname, y, g, tfb.RESNET_BN_EPS, damp)
            y = tfb._bn(sd, p + bname, y, tfb.RESNET_BN_EPS)
            y = F.relu(y) if relu else y
            if tap is not None:
                tap[p + cname] = y
            return y

        mean = torch.tensor([103.939, 116.779, 123.68]).reshape(1, 3, 1, 1)
        x = 255.0 * image - mean  # caffe_preproc, no channel swap
        x = conv_bn(F.pad(x, (3, 3, 3, 3)), 'conv1_conv', 'conv1_bn', 64, 7, stride=2)
        x = F.max_pool2d(F.pad(x, (1, 1, 1, 1)), 3, stride=2)  # zero pad (post-ReLU values are >= 0), then VALID
        if tap is not None:
            tap[p + 'pool1_pool'] = x
        for b in resnet_blocks(self.cfg, self.depth):
            name, f, stride, shift, dil = b['name'], b['filters'], b['stride'], b['shift'], b['dil']
            inp = x
            cout = f if self.basic else 4 * f
            sc = conv_bn(inp, name + '_0_conv', name + '_0_bn', cout, 1, stride, shift, relu=False) if b['conv_shortcut'] else inp
            if self.basic:
                y = conv_bn(inp, name + '_1_conv', name + '_1_bn', f, 3, stride, shift, dil=dil, pad=dil)
                y = conv_bn(y, name + '_2_conv', name + '_2_bn', f, 3, dil=b['dil2'], pad=b['dil2'], relu=False, damp=0.5)
                last = name + '_2_conv'
            else:
                y = conv_bn(inp, name + '_1_conv', name + '_1_bn', f, 1, stride, shift)
                y = conv_bn(y, name + '_2_conv', name + '_2_bn', f, 3, dil=dil, pad=dil)
                y = conv_bn(y, name + '_3_conv', name + '_3_bn', 4 * f, 1, relu=False, damp=0.5)
                last = name + '_3_conv'
            x = F.relu(sc + y)
            if tap is not None:
                tap[p + last] = x
        return x


def op_table(spec: ResNetSpec, prefix='backbone.'):
    """engine op name -> op dict (port_ops._op): conv bias (50/101/152 only) folded by BN (eps 1e-5), caffe stem,
    zero-padded max pool, dense-SAME convs sampled at shift::stride (the strided 1x1s; the basic block's strided 3x3),
    dilated 3x3, relu(shortcut + last conv)."""
    e = tfb.RESNET_BN_EPS
    basic = spec.basic
    mean = torch.tensor([103.939, 116.779, 123.68])  # fp32 constants, as in the restatement and the stem kernel
    t = {prefix + 'conv1_conv': port_ops._op(prefix + 'conv1_conv.weight', 7, 2, (3, 3), act='relu', bn=prefix + 'conv1_bn',
                                             eps=e, bias=None if basic else prefix + 'conv1_conv.bias',
                                             pre=((255.0,) * 3, tuple((-mean).double().tolist())))}
    t[prefix + 'pool1_pool'] = dict(port_ops._op(None, 3, 2, (1, 1)), maxpool=True)
    for blk in resnet_blocks(spec.cfg, spec.depth):
        b, stride, shift, dil = prefix + blk['name'], blk['stride'], blk['shift'], blk['dil']

        def cb(j, k=1, **kw):
            return port_ops._op(f'{b}_{j}_conv.weight', k, bn=f'{b}_{j}_bn', eps=e,
                                bias=None if basic else f'{b}_{j}_conv.bias', **kw)
        if blk['conv_shortcut']:
            t[f'{b}_0_conv'] = cb(0, stride=stride, sample=shift, shift=shift)
        if basic:
            t[f'{b}_1_conv'] = cb(1, 3, stride=stride, sample=shift, shift=shift, pad=(dil, dil), dil=dil, act='relu')
            d2 = blk['dil2']
            t[f'{b}_2_conv'] = cb(2, 3, pad=(d2, d2), dil=d2, act='relu', res_first=True)
        else:
            t[f'{b}_1_conv'] = cb(1, stride=stride, sample=shift, shift=shift, act='relu')
            t[f'{b}_2_conv'] = cb(2, 3, pad=(dil, dil), dil=dil, act='relu')
            t[f'{b}_3_conv'] = cb(3, act='relu', res_first=True)
    return t


def _layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude=False):
    """port_ops._layer for one op dict of a ResNet (no depthwise convs, no squeeze-excitation scale):
    -> (output NCHW, pre-activation NCHW, products per output)."""
    if op['maxpool']:  # zero pad (the pad value takes part in the max), then VALID
        x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
        x = x.abs() if magnitude else x
        y = F.max_pool2d(F.pad(x, op['pad'] * 2), op['kernel'], op['stride'])
        return y, y, 1
    dev = x_nhwc.device
    w, bias = port_ops._fold(sd, op)
    if precision in port_ops.MODES or precision in port_ops.WIDE_MODES:  # folded in fp64, cast to fp32, GEMM weights
        w, bias = w.float().double(), bias.float().double()                 # rounded once to 16 bits
        if precision in port_ops.MODES and port_ops.tc_eligible(op, w.shape[1], w.shape[0]):
            w = w.float().to(port_ops.MODES[precision][0]).double()
    w, bias = w.to(dev, dtype), bias.to(dev, dtype)
    if op['stem']:
        a, c = (torch.tensor(v, dtype=torch.float32).to(dev, dtype)[None, :, None, None] for v in op['pre'])
        x = x_nhwc.to(dtype)
        x = (x * a).abs() + c.abs() if magnitude else x * a + c
    else:
        x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    if magnitude:
        x, w, bias = x.abs(), w.abs(), bias.abs()
    x = F.pad(x, op['pad'] * 2)
    if op['sample'] is not None:
        z = F.conv2d(x, w, bias, dilation=op['dil'])[:, :, op['sample']::op['stride'], op['sample']::op['stride']]
    else:
        z = F.conv2d(x, w, bias, stride=op['stride'], dilation=op['dil'])
    if res_nhwc is not None:  # every ResNet residual is added before the ReLU
        res = res_nhwc.permute(0, 3, 1, 2).to(dtype)
        z = z + (res.abs() if magnitude else res)
    y = z if magnitude else port_ops._act(z, op['act'])
    return y, z, w.shape[1] * w.shape[2] * w.shape[3]


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, precision='exact', dtype=torch.float64):
    """port_ops.conv_layer_reference for the ops of ``spec`` (any depth).  Returns NHWC in ``dtype``."""
    return _layer(sd, op_table(spec)[name], x_nhwc, res_nhwc, precision, dtype)[0].permute(0, 2, 3, 1).contiguous()


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, precision='fp16'):
    """port_ops.layer_bound for the ops of ``spec`` (any depth): -> (ref, tol), NHWC fp64, with the same bound
    tol = 2^-p (|ref| + e) + e + floor, e = L_act C_ACC (K + 4) 2^-24 refabs + e_act + 2^-23 |ref|."""
    op = op_table(spec)[name]
    y, z, k = _layer(sd, op, x_nhwc, res_nhwc, precision, torch.float64)
    zabs = _layer(sd, op, x_nhwc, res_nhwc, precision, torch.float64, magnitude=True)[1]
    if op['maxpool']:  # a max of stored values is exact
        tol = torch.zeros_like(y)
    else:
        tc32 = precision == 'tf32x3' and port_ops.tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
        tol = port_ops.bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)
