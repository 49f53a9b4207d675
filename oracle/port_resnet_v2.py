"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of the pre-activation ResNets of the reference's TF/Keras code
(metrabs_tf/backbones/resnet.py), and the per-layer reference arithmetic of their engine ops.

* ``ResNetUnifiedV2`` :710-745 over ``ResNet(stack_fn, preact=True, use_bias=True)`` :160-193, ``block2_dense`` :391-456 and
  ``stack2_dense`` :558-580; block counts [3,4,6,3] / [3,4,23,3] / [3,8,36,3] (ResNet50V2 / 101V2 / 152V2, :803-831); BN eps
  1e-5 :52; preprocessing ``tf_preproc`` 2x - 1 (backbones/builder.py:111-113).
* Stem: 7x7 stride-2 ``conv1_conv`` with bias after a zero pad of 3, no BN and no ReLU (skipped under ``preact``), then a
  zero pad of 1 and a 3x3 stride-2 VALID max pool: the stem output is signed, so the zero pad takes part in the max.
* Block: preact = relu(_preact_bn(x)); shortcut = _0_conv(preact) (1x1 with bias, block1 of a stack, never strided),
  x[c::2, c::2] (``Cropping2D`` c + ``MaxPooling2D(1, 2)``, the strided last block of conv2..conv4) or x; _1_conv 1x1 + BN
  + ReLU and _2_conv 3x3 + BN + ReLU without biases (the 3x3 dense SAME, dilated, evaluated at ``c::s``); out = shortcut +
  _3_conv (1x1 with bias, no BN, no activation).  After conv5: relu(post_bn(x)).
* Stride plan: ``get_strides_and_dilations`` :601-618 for stride_test; the stride sits on the LAST block of conv2..conv4
  (``striding_info_out``: stride, ``dil_in`` of its stack, bottom-right shift), the other blocks of those stacks have
  stride 1 and ``dil_in``; conv5 uses ``dil_out[-1]`` in every block.  ``stride_train`` plays no part.

``Conv2DDenseSame`` and the default bias of ``_0_conv`` are read as in ``oracle/port_resnet.py`` (the un-vendored ``fleras``).
PARITY UNPINNED: the reference has no test, golden or importable implementation of these backbones, so device-vs-oracle
parity is "this build's restatement vs this build's kernels".

The engine runs each BatchNorm + ReLU of a block input (``_preact_bn``, ``post_bn``) as a 1x1 depthwise op with the folded
weight gamma / sqrt(var + eps) and bias beta - mean * weight, and the shortcut subsample as a 1x1 max pool with stride 2 and
begin pad -c (op ``<block>_shortcut_pool``).  ``layer_bound`` covers both: the BN-only op with the bound of
``port_ops.bound_from_parts`` for one product per output, the subsample exactly (tolerance 0).
"""
import math

import torch
import torch.nn.functional as F

from oracle import port, port_ops, port_resnet
from oracle import port_tf_backbones as tfb

# depth -> blocks in conv2..conv5
DEPTHS = {50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3]}
EPS = tfb.RESNET_BN_EPS
# the conditioned init scales every _3_conv (no BN behind it) by this, so that the residual stream of the 50 blocks of
# ResNet-152 V2 grows slowly and the features and joints stay finite
CONV3_GAIN = 0.5


def resnet_v2_blocks(cfg: port.PathConfig, depth):
    """[dict(name, filters, stride, shift, dil, conv_shortcut, subsample)] in execution order (inference: stride_test).
    ``stride`` / ``shift`` sit on the 3x3 of the last block of conv2..conv4; ``subsample``: the shortcut is x[c::2, c::2]."""
    strides, dil_in, dil_out, brs = tfb.resnet_stride_plan(cfg.stride_test, cfg.centered_stride)
    out = []
    for st, (f, n) in enumerate(zip([64, 128, 256, 512], DEPTHS[depth])):
        for bi in range(n):
            last = bi == n - 1
            stride = strides[st] if (st < 3 and last) else 1
            shift = 1 if (st < 3 and last and brs[st]) else 0
            dil = dil_in[st] if st < 3 else dil_out[2]
            out.append(dict(name=f'conv{st + 2}_block{bi + 1}', filters=f, stride=stride, shift=shift, dil=dil,
                            conv_shortcut=bi == 0, subsample=bi > 0 and (stride > 1 or shift > 0)))
    return out


class ResNetV2Spec:
    """Pre-activation ResNet of ``depth`` 50, 101 or 152."""

    out_channels = 2048

    def __init__(self, cfg: port.PathConfig, depth=50):
        self.cfg = cfg
        self.depth = depth
        self.name = f'resnet{depth}v2'

    def features(self, sd, image, tap=None, init=None):
        """[B,3,S,S] in [0,1] -> [B,2048,S/s,S/s].  With ``init`` = (generator) the weights are created and the BNs
        calibrated on the fly (each _preact_bn normalises its block input over the calibration batch), otherwise read
        from ``sd``."""
        p = 'backbone.'
        g = init

        def conv(x, name, cout, k, bias, stride=1, shift=0, dil=1, pad=0, gain=1.0):
            if g is not None:
                cin = x.shape[1]
                sd[p + name + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * (gain * math.sqrt(2.0 / (cin * k * k)))
                if bias:
                    sd[p + name + '.bias'] = 0.1 * torch.randn(cout, generator=g)
            y = F.conv2d(x, sd[p + name + '.weight'], sd[p + name + '.bias'] if bias else None, padding=pad, dilation=dil)
            if stride > 1 or shift:
                y = y[:, :, shift::stride, shift::stride]  # Conv2DDenseSame: dense SAME conv sampled at shift::stride
            return y

        def bn_relu(y, name):
            if g is not None:
                port._calibrate_bn(sd, p + name, y, g, EPS)
            return F.relu(tfb._bn(sd, p + name, y, EPS))

        def put(name, y):
            if tap is not None:
                tap[p + name] = y
            return y

        x = put('conv1_conv', conv(F.pad(2.0 * image - 1.0, (3, 3, 3, 3)), 'conv1_conv', 64, 7, True, stride=2))
        x = put('pool1_pool', F.max_pool2d(F.pad(x, (1, 1, 1, 1)), 3, stride=2))  # zero pad of a signed map, then VALID
        for b in resnet_v2_blocks(self.cfg, self.depth):
            n, f, stride, shift, dil = b['name'], b['filters'], b['stride'], b['shift'], b['dil']
            pre = put(n + '_preact_bn', bn_relu(x, n + '_preact_bn'))
            if b['conv_shortcut']:
                sc = put(n + '_0_conv', conv(pre, n + '_0_conv', 4 * f, 1, True))
            elif b['subsample']:
                sc = put(n + '_shortcut_pool', x[:, :, shift::stride, shift::stride])
            else:
                sc = x
            y = put(n + '_1_conv', bn_relu(conv(pre, n + '_1_conv', f, 1, False), n + '_1_bn'))
            y = put(n + '_2_conv', bn_relu(conv(y, n + '_2_conv', f, 3, False, stride, shift, dil, dil), n + '_2_bn'))
            x = put(n + '_3_conv', sc + conv(y, n + '_3_conv', 4 * f, 1, True, gain=CONV3_GAIN))
        return put('post_bn', bn_relu(x, 'post_bn'))


def _bn_op(key):
    """BatchNorm + ReLU alone: a 1x1 depthwise op with no conv weight"""
    return port_ops._op(None, 1, act='relu', depthwise=True, bn=key, eps=EPS)


def op_table(spec: ResNetV2Spec, prefix='backbone.'):
    """engine op name -> op dict (port_ops._op): the tf_preproc stem with bias and no BN, the zero-padded max pool of a
    signed map, BN-only pre-activations, dense-SAME 3x3s sampled at shift::stride, the shortcut subsample as a 1x1 max
    pool with begin pad -c, _3_conv + shortcut without activation."""
    t = {prefix + 'conv1_conv': port_ops._op(prefix + 'conv1_conv.weight', 7, 2, (3, 3), bias=prefix + 'conv1_conv.bias',
                                             eps=EPS, pre=((2.0,) * 3, (-1.0,) * 3)),
         prefix + 'pool1_pool': dict(port_ops._op(None, 3, 2, (1, 1)), maxpool=True)}
    for blk in resnet_v2_blocks(spec.cfg, spec.depth):
        b, stride, shift, dil = prefix + blk['name'], blk['stride'], blk['shift'], blk['dil']
        t[b + '_preact_bn'] = _bn_op(b + '_preact_bn')
        if blk['conv_shortcut']:
            t[b + '_0_conv'] = port_ops._op(b + '_0_conv.weight', bias=b + '_0_conv.bias', eps=EPS)
        if blk['subsample']:
            t[b + '_shortcut_pool'] = dict(port_ops._op(None, 1, stride, (-shift, 0)), maxpool=True)
        t[b + '_1_conv'] = port_ops._op(b + '_1_conv.weight', bn=b + '_1_bn', eps=EPS, act='relu')
        sampled = stride > 1 or shift > 0
        t[b + '_2_conv'] = port_ops._op(b + '_2_conv.weight', 3, stride, (dil, dil), dil, act='relu', bn=b + '_2_bn', eps=EPS,
                                        sample=shift if sampled else None, shift=shift)
        t[b + '_3_conv'] = port_ops._op(b + '_3_conv.weight', bias=b + '_3_conv.bias', eps=EPS)
    t[prefix + 'post_bn'] = _bn_op(prefix + 'post_bn')
    return t


def _bn_layer(sd, op, x_nhwc, precision, dtype, magnitude=False, eps=None):
    """The BN-only op: y = relu(x * w + b) per channel with the folded w = gamma / sqrt(var + eps), b = beta - mean * w
    (fp64, cast to fp32 in every mode: a depthwise weight is never rounded to 16 bits) -> (y, z, 1) NCHW."""
    k = op['bn']
    e = op['eps'] if eps is None else eps
    w = sd[k + '.weight'].double() / torch.sqrt(sd[k + '.running_var'].double() + e)
    b = sd[k + '.bias'].double() - sd[k + '.running_mean'].double() * w
    if precision in port_ops.MODES or precision in port_ops.WIDE_MODES:
        w, b = w.float().double(), b.float().double()
    x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    w, b = w.to(x.device, dtype)[None, :, None, None], b.to(x.device, dtype)[None, :, None, None]
    if magnitude:
        x, w, b = x.abs(), w.abs(), b.abs()
    z = x * w + b
    y = z if magnitude else port_ops._act(z, op['act'])
    return y, z, 1


def _layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude=False):
    if op['weight'] is None and not op['maxpool']:
        return _bn_layer(sd, op, x_nhwc, precision, dtype, magnitude)
    return port_resnet._layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude)


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, precision='exact', dtype=torch.float64):
    """port_ops.conv_layer_reference for the ops of ``spec``.  Returns NHWC in ``dtype``."""
    return _layer(sd, op_table(spec)[name], x_nhwc, res_nhwc, precision, dtype)[0].permute(0, 2, 3, 1).contiguous()


def bound_for_op(sd, op, x_nhwc, res_nhwc=None, precision='fp16'):
    """(ref, tol) NHWC fp64 of one op dict: port_ops.layer_bound's bound (bound_from_parts), 0 for a max pool."""
    y, z, k = _layer(sd, op, x_nhwc, res_nhwc, precision, torch.float64)
    zabs = _layer(sd, op, x_nhwc, res_nhwc, precision, torch.float64, magnitude=True)[1]
    if op['maxpool']:  # a max of stored values is exact
        tol = torch.zeros_like(y)
    else:
        tc32 = precision == 'tf32x3' and port_ops.tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
        tol = port_ops.bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, precision='fp16'):
    """port_ops.layer_bound for the ops of ``spec``: -> (ref, tol), NHWC fp64."""
    return bound_for_op(sd, op_table(spec)[name], x_nhwc, res_nhwc, precision)


def gflop_per_crop(cfg: port.PathConfig, depth):
    """2 * MACs per crop of the convs and the BN-only ops (the engine's mtb_backbone_flops_per_crop), from the shapes"""
    s = (cfg.proc_side + 6 - 7) // 2 + 1
    total = 2.0 * s * s * 64 * 147
    h = (s + 2 - 3) // 2 + 1
    c = 64
    for b in resnet_v2_blocks(cfg, depth):
        f = b['filters']
        total += 2.0 * h * h * c  # pre-activation
        if b['conv_shortcut']:
            total += 2.0 * h * h * c * 4 * f
        total += 2.0 * h * h * c * f
        h //= b['stride']
        total += 2.0 * h * h * f * f * 9 + 2.0 * h * h * f * 4 * f
        c = 4 * f
    return (total + 2.0 * h * h * c) / 1e9
