"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of the last backbone names the reference's builder accepts
(metrabs_tf/backbones/builder.py:22-82) and this build did not: the ResNet V1.5 bottleneck nets and the minimalistic
MobileNetV3s, with the per-layer reference arithmetic of their engine ops.

* ``resnet{50,101,152}V1_5`` (also ``V1-5``): ``ResNetUnified(v1_5=True)`` (metrabs_tf/backbones/resnet.py:621-666,
  :791-800) with ``block1_dense`` :239-319.  The layers and keys are ResNet V1's (oracle/port_resnet.py); in every block
  ``_1_conv`` is a plain 1x1 at stride 1 (:282-283) and the 3x3 ``_2_conv`` carries the stride and the bottom-right shift
  of the stack (:295-303).  Its dilation is ``dil_in`` of the stack in block1 (``striding_infos_in`` :629-634; V1 uses
  ``dil_out`` there) and ``dil_out`` in the other blocks.  Preprocessing ``torch_preproc`` (builder.py:45-46, :99-103):
  ``(x - mean) / std`` with fp32 constants.
* ``mobilenetV3{Small,Large}mini``: ``MobileNetV3{Small,Large}(minimalistic=True)`` (builder.py:75-81,
  mobilenet_v3.py:250-257): kernel 3, ReLU and no squeeze-excitation in every row that takes ``kernel`` / ``activation`` /
  ``se_ratio`` from the model (the other rows already have kernel 3, ReLU and no SE in the minimalistic form); the stem,
  ``Conv_1`` and ``Conv_2`` use ReLU.  Expanded widths, strides and the bottom-right row are those of the full nets.

PARITY UNPINNED: the reference has these nets only as Keras code (no test, golden or importable implementation), so
device-vs-oracle parity is "this build's restatement vs this build's kernels".

The stem of V1.5 computes ``x * fp32(1/std) + fp32(-mean/std)``, not the reference's ``(x - mean) / std``.  The per-layer
reference here is the exact layer on ``(x - mean) / std`` (fp32 ``mean`` and ``std``, as the reference holds them), and
the stem's bound carries one explicit term for the two rounded constants, ``PRE_CONST_REL * conv(|x - mean| / std + ...)``
(``stem_pre_error``); the fp32 roundings of either operation order are the preprocessing terms port_ops.C_ACC's K + 4
already counts.  The other ops reuse the V1 / MobileNetV3 arithmetic of port_resnet / port_mobilenet and the bound of
port_ops.bound_from_parts unchanged.
"""
import math

import torch
import torch.nn.functional as F

from oracle import port, port_mobilenet, port_ops, port_resnet
from oracle import port_tf_backbones as tfb

TORCH_MEAN = (0.485, 0.456, 0.406)
TORCH_STD = (0.229, 0.224, 0.225)
# |fp32(1/std) - 1/std| <= 2^-24 / std and |fp32(-mean/std) + mean/std| <= 2^-24 mean / std (each one correctly rounded
# fp32 division of the fp32 constants, as the planner computes them)
PRE_CONST_REL = 2.0 ** -24


def torch_preproc_constants():
    """-> (mean, std, scale, shift) fp32 [3]: the reference's constants and the stem kernel's x * scale + shift."""
    mean, std = torch.tensor(TORCH_MEAN, dtype=torch.float32), torch.tensor(TORCH_STD, dtype=torch.float32)
    return mean, std, 1.0 / std, -mean / std


# ------------------------------------------------------------------------------------------------------- ResNet V1.5
def resnet_v1_5_blocks(cfg: port.PathConfig, depth):
    """[dict(name, filters, stride, shift, dil, conv_shortcut)] in execution order (inference: stride_test).  ``stride`` /
    ``shift`` sit on the shortcut and on the 3x3 ``_2_conv`` of block1; ``dil`` is the dilation of the 3x3: ``dil_in`` of
    the stack in block1 (``dil_in[0]`` throughout conv2), ``dil_out`` in the other blocks."""
    counts, basic = port_resnet.DEPTHS[depth]
    if basic:
        raise ValueError(f'ResNet-{depth} has no V1.5 form (resnet.py:669-671: the basic-block nets have no V1 / V1.5 split)')
    strides, dil_in, dil_out, brs = tfb.resnet_stride_plan(cfg.stride_test, cfg.centered_stride)
    out = []
    for st, (f, n) in enumerate(zip([64, 128, 256, 512], counts)):
        for bi in range(n):
            first = bi == 0
            stride = strides[st - 1] if (st > 0 and first) else 1
            shift = 1 if (st > 0 and first and brs[st - 1]) else 0
            if st == 0:
                dil = dil_in[0]
            else:
                dil = dil_in[st - 1] if first else dil_out[st - 1]
            out.append(dict(name=f'conv{st + 2}_block{bi + 1}', filters=f, stride=stride, shift=shift, dil=dil,
                            conv_shortcut=first))
    return out


class ResNetV15Spec:
    """ResNet V1.5 of ``depth`` 50, 101 or 152 (the keys and the random-init draw order of port_resnet.ResNetSpec)."""

    def __init__(self, cfg: port.PathConfig, depth=50):
        resnet_v1_5_blocks(cfg, depth)  # refuses the basic-block depths
        self.cfg = cfg
        self.depth = depth
        self.name = f'resnet{depth}v1_5'
        self.out_channels = 2048

    def features(self, sd, image, tap=None, init=None):
        """[B,3,S,S] in [0,1] -> [B,2048,S/s,S/s].  With ``init`` = (generator) the weights are created and BN-calibrated
        on the fly, otherwise read from ``sd``."""
        p = 'backbone.'
        g = init

        def conv_bn(x, cname, bname, cout, k, stride=1, shift=0, dil=1, pad=0, relu=True, damp=1.0):
            if g is not None:
                cin = x.shape[1]
                sd[p + cname + '.weight'] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))
                sd[p + cname + '.bias'] = 0.1 * torch.randn(cout, generator=g)
            y = F.conv2d(x, sd[p + cname + '.weight'], sd[p + cname + '.bias'], padding=pad, dilation=dil)
            if stride > 1 or shift:
                y = y[:, :, shift::stride, shift::stride]  # Conv2DDenseSame: dense SAME conv sampled at shift::stride
            if g is not None:
                port._calibrate_bn(sd, p + bname, y, g, tfb.RESNET_BN_EPS, damp)
            y = tfb._bn(sd, p + bname, y, tfb.RESNET_BN_EPS)
            y = F.relu(y) if relu else y
            if tap is not None:
                tap[p + cname] = y
            return y

        mean, std, _, _ = torch_preproc_constants()
        x = (image - mean.to(image).reshape(1, 3, 1, 1)) / std.to(image).reshape(1, 3, 1, 1)  # torch_preproc
        x = conv_bn(F.pad(x, (3, 3, 3, 3)), 'conv1_conv', 'conv1_bn', 64, 7, stride=2)
        x = F.max_pool2d(F.pad(x, (1, 1, 1, 1)), 3, stride=2)  # zero pad (post-ReLU values are >= 0), then VALID
        if tap is not None:
            tap[p + 'pool1_pool'] = x
        for b in resnet_v1_5_blocks(self.cfg, self.depth):
            name, f, stride, shift, dil = b['name'], b['filters'], b['stride'], b['shift'], b['dil']
            inp = x
            sc = conv_bn(inp, name + '_0_conv', name + '_0_bn', 4 * f, 1, stride, shift, relu=False) if b['conv_shortcut'] else inp
            y = conv_bn(inp, name + '_1_conv', name + '_1_bn', f, 1)
            y = conv_bn(y, name + '_2_conv', name + '_2_bn', f, 3, stride, shift, dil=dil, pad=dil)
            y = conv_bn(y, name + '_3_conv', name + '_3_bn', 4 * f, 1, relu=False, damp=0.5)
            x = F.relu(sc + y)
            if tap is not None:
                tap[p + name + '_3_conv'] = x
        return x


def resnet_v1_5_op_table(spec: ResNetV15Spec, prefix='backbone.'):
    """engine op name -> op dict (port_ops._op): the V1 ops of port_resnet.op_table with the stride on the 3x3 (dense SAME
    sampled at shift::stride, begin pad dil - shift) and the torch_preproc stem; ``torch_pre`` = (mean, std) marks the stem
    whose reference is (x - mean) / std."""
    e = tfb.RESNET_BN_EPS
    mean, std, scale, shift = torch_preproc_constants()
    dbl = lambda t: tuple(t.double().tolist())  # noqa: E731
    t = {prefix + 'conv1_conv': dict(port_ops._op(prefix + 'conv1_conv.weight', 7, 2, (3, 3), act='relu', bn=prefix + 'conv1_bn',
                                                  eps=e, bias=prefix + 'conv1_conv.bias', pre=(dbl(scale), dbl(shift))),
                                     torch_pre=(dbl(mean), dbl(std)))}
    t[prefix + 'pool1_pool'] = dict(port_ops._op(None, 3, 2, (1, 1)), maxpool=True)
    for blk in resnet_v1_5_blocks(spec.cfg, spec.depth):
        b, stride, sh, dil = prefix + blk['name'], blk['stride'], blk['shift'], blk['dil']

        def cb(j, k=1, **kw):
            return port_ops._op(f'{b}_{j}_conv.weight', k, bn=f'{b}_{j}_bn', eps=e, bias=f'{b}_{j}_conv.bias', **kw)
        if blk['conv_shortcut']:
            t[f'{b}_0_conv'] = cb(0, stride=stride, sample=sh, shift=sh)
        t[f'{b}_1_conv'] = cb(1, act='relu')
        t[f'{b}_2_conv'] = cb(2, 3, stride=stride, sample=sh, shift=sh, pad=(dil, dil), dil=dil, act='relu')
        t[f'{b}_3_conv'] = cb(3, act='relu', res_first=True)
    return t


def resnet_v1_5_gflop_per_crop(cfg: port.PathConfig, depth):
    """2 * MACs of every conv per crop (strided convs at their output size), from the block table."""
    s = cfg.proc_side // 2  # stem output
    total = 2.0 * s * s * 64 * 3 * 49
    h, cin = s // 2, 64
    for b in resnet_v1_5_blocks(cfg, depth):
        f, st = b['filters'], b['stride']
        ho = h // st
        if b['conv_shortcut']:
            total += 2.0 * ho * ho * 4 * f * cin
        total += 2.0 * h * h * f * cin + 2.0 * ho * ho * f * f * 9 + 2.0 * ho * ho * 4 * f * f
        h, cin = ho, 4 * f
    return total / 1e9


def stem_pre_error(op, w, x_nchw, dtype):
    """The stem's bound term for the rounded preprocessing constants: PRE_CONST_REL * conv(|x| / std + mean / std, |w|),
    NCHW, before the activation's Lipschitz factor (ReLU: 1)."""
    mean, std = (torch.tensor(v, dtype=torch.float32).to(x_nchw.device, dtype)[None, :, None, None] for v in op['torch_pre'])
    m = x_nchw.to(dtype).abs() / std + mean / std
    return PRE_CONST_REL * F.conv2d(F.pad(m, op['pad'] * 2), w.abs(), stride=op['stride'])


def _resnet_layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude=False):
    """port_resnet._layer, except for the torch_preproc stem: its value is the exact layer on (x - mean) / std, its
    magnitude the layer on |x * scale| + |shift| as the kernel evaluates it (port_ops._layer)."""
    if not op.get('torch_pre') or magnitude:
        return port_resnet._layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude)
    w, bias = port_ops._fold(sd, op)
    if precision in port_ops.MODES or precision in port_ops.WIDE_MODES:  # stem weights: folded in fp64, cast to fp32
        w, bias = w.float().double(), bias.float().double()
    dev = x_nhwc.device
    w, bias = w.to(dev, dtype), bias.to(dev, dtype)
    mean, std = (torch.tensor(v, dtype=torch.float32).to(dev, dtype)[None, :, None, None] for v in op['torch_pre'])
    x = F.pad((x_nhwc.to(dtype) - mean) / std, op['pad'] * 2)
    z = F.conv2d(x, w, bias, stride=op['stride'])
    return port_ops._act(z, op['act']), z, w.shape[1] * w.shape[2] * w.shape[3]


# -------------------------------------------------------------------------------------------- MobileNetV3 minimalistic
# MobileNetV3Small / Large stack_fn (mobilenet_v3.py:364-384 / :403-428), read with minimalistic=True: kernel 3, ReLU,
# se_ratio None.  (expansion, filters, kernel, stride, se, activation, bottomright)
MINI_ROWS = {v: [(exp, filters, 3, stride, False, 'relu', br) for exp, filters, _k, stride, _se, _act, br in rows]
             for v, (rows, _) in port_mobilenet.VARIANTS.items()}


def mini_blocks(variant):
    """port_mobilenet.mobilenet_blocks of the minimalistic form: [dict(name, cin, exp, filters, kernel, stride, se, se_ch,
    act, br, residual)]."""
    out, cin = [], 16
    for bi, (exp, filters, k, stride, se, act, br) in enumerate(MINI_ROWS[variant]):
        out.append(dict(name='expanded_conv' if bi == 0 else f'expanded_conv_{bi}', cin=cin, exp=tfb._depth(cin * exp),
                        filters=filters, kernel=k, stride=stride, se=se, se_ch=0, act=act, br=br,
                        residual=stride == 1 and cin == filters))
        cin = filters
    return out


class MobileNetV3MiniSpec:
    """MobileNetV3 ``variant`` 'small' or 'large' with minimalistic=True."""

    def __init__(self, cfg: port.PathConfig, variant='small'):
        self.cfg = cfg
        self.variant = variant
        self.name = f'mobilenetv3-{variant}-mini'
        self.out_channels = port_mobilenet.VARIANTS[variant][1]

    def features(self, sd, image, tap=None, init=None):
        """[B,3,S,S] in [0,1] -> [B,C,S/32,S/32] (conditioned random init with ``init``, the draw order of
        port_mobilenet.MobileNetV3Spec without the SE weights)."""
        p = 'backbone.'
        g = init

        def conv_bn(x, cname, cout, k, stride=1, groups=1, bn=True, bias=False, damp=1.0):
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
            return y

        def tapped(name, y):
            if tap is not None:
                tap[p + name] = y
            return y

        x = image * 2 - 1  # 255*x (builder.py:116-117) then Rescaling(1/127.5, -1) (mobilenet_v3.py:259)
        s = x.shape[-1]
        pad_total = max(((s + 1) // 2 - 1) * 2 + 3 - s, 0)  # TF 'same', stride 2
        pb = pad_total // 2
        x = tapped('Conv', F.relu(conv_bn(F.pad(x, (pb, pad_total - pb, pb, pad_total - pb)), 'Conv', 16, 3, stride=2)))
        for blk in mini_blocks(self.variant):
            name, cexp, k, stride = blk['name'], blk['exp'], blk['kernel'], blk['stride']
            inp = x
            if name != 'expanded_conv':
                x = tapped(name + '.expand', F.relu(conv_bn(x, name + '.expand', cexp, 1)))
            shift = 1 if (blk['br'] and self.cfg.centered_stride) else 0
            pbeg, pend = (k - 1) // 2, k - 1 - (k - 1) // 2
            if stride == 2:
                x = F.pad(x, (pbeg - shift, pend + shift, pbeg - shift, pend + shift))  # correct_pad, then VALID
            else:
                x = F.pad(x, (pbeg, pend, pbeg, pend))
            x = tapped(name + '.depthwise', F.relu(conv_bn(x, name + '.depthwise', cexp, k, stride=stride, groups=cexp)))
            res = blk['residual']
            x = conv_bn(x, name + '.project', blk['filters'], 1, damp=0.5 if res else 1.0)
            x = tapped(name + '.project', x + inp if res else x)
        x = tapped('Conv_1', F.relu(conv_bn(x, 'Conv_1', tfb._depth(x.shape[1] * 6), 1)))
        return tapped('Conv_2', F.relu(conv_bn(x, 'Conv_2', self.out_channels, 1, bn=False, bias=True)))


def mini_op_table(spec: MobileNetV3MiniSpec, prefix='backbone.'):
    """engine op name -> op dict (port_ops._op): port_mobilenet.op_table's ops with ReLU everywhere, 3x3 depthwise convs and
    no SE scale on the projections."""
    e = tfb.MOBILENET_BN_EPS
    s = spec.cfg.proc_side
    pad_total = max(((s + 1) // 2 - 1) * 2 + 3 - s, 0)
    t = {prefix + 'Conv': port_ops._op(prefix + 'Conv.weight', 3, 2, (pad_total // 2, pad_total - pad_total // 2),
                                       act='relu', bn=prefix + 'Conv.BatchNorm', eps=e, pre=((2.0,) * 3, (-1.0,) * 3))}
    for blk in mini_blocks(spec.variant):
        b, k, stride = prefix + blk['name'], blk['kernel'], blk['stride']
        if blk['name'] != 'expanded_conv':
            t[b + '.expand'] = port_ops._op(b + '.expand.weight', act='relu', bn=b + '.expand.BatchNorm', eps=e)
        shift = 1 if (blk['br'] and spec.cfg.centered_stride and stride == 2) else 0
        pb = (k - 1) // 2
        t[b + '.depthwise'] = port_ops._op(b + '.depthwise.weight', k, stride, (pb - shift, k - 1 - pb + shift), act='relu',
                                           depthwise=True, bn=b + '.depthwise.BatchNorm', eps=e, shift=shift)
        t[b + '.project'] = port_ops._op(b + '.project.weight', bn=b + '.project.BatchNorm', eps=e)
    t[prefix + 'Conv_1'] = port_ops._op(prefix + 'Conv_1.weight', act='relu', bn=prefix + 'Conv_1.BatchNorm', eps=e)
    t[prefix + 'Conv_2'] = port_ops._op(prefix + 'Conv_2.weight', act='relu', bias=prefix + 'Conv_2.bias')
    return t


# ---------------------------------------------------------------------------------------------------- both families
def op_table(spec):
    return resnet_v1_5_op_table(spec) if isinstance(spec, ResNetV15Spec) else mini_op_table(spec)


def _layer(sd, spec, op, x_nhwc, res_nhwc, precision, dtype, magnitude=False):
    if isinstance(spec, ResNetV15Spec):
        return _resnet_layer(sd, op, x_nhwc, res_nhwc, precision, dtype, magnitude)
    return port_mobilenet._layer(sd, op, x_nhwc, res_nhwc, None, precision, dtype, magnitude)


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, precision='exact', dtype=torch.float64):
    """port_ops.conv_layer_reference for the ops of ``spec``.  Returns NHWC in ``dtype``."""
    return _layer(sd, spec, op_table(spec)[name], x_nhwc, res_nhwc, precision, dtype)[0].permute(0, 2, 3, 1).contiguous()


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, precision='fp16'):
    """port_ops.layer_bound for the ops of ``spec``: -> (ref, tol), NHWC fp64, tol = port_ops.bound_from_parts, plus
    L_act * stem_pre_error on the torch_preproc stem (after the output rounding term, so every mode carries it)."""
    op = op_table(spec)[name]
    y, z, k = _layer(sd, spec, op, x_nhwc, res_nhwc, precision, torch.float64)
    zabs = _layer(sd, spec, op, x_nhwc, res_nhwc, precision, torch.float64, magnitude=True)[1]
    if op['maxpool']:  # a max of stored values is exact
        tol = torch.zeros_like(y)
    else:
        tc32 = precision == 'tf32x3' and port_ops.tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
        tol = port_ops.bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
        if op.get('torch_pre'):
            w = port_ops._fold(sd, op)[0].float().double().to(x_nhwc.device)
            e = port_ops.LIPSCHITZ[op['act']] * stem_pre_error(op, w, x_nhwc, torch.float64)
            st = port_ops.storage(precision)
            tol = tol + (e if st == torch.float32 else (1.0 + 2.0 ** -(8 if st == torch.bfloat16 else 11)) * e)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)
