"""TEST INFRASTRUCTURE ONLY - per-layer reference arithmetic for the device kernels' unit tests.

``oracle/port.py`` restates the whole path; this file exposes ONE conv layer of it at a time (same reference lines:
``/root/reference/metrabs_pytorch/backbones/efficientnet.py`` :110-173 MBConv, :176-234 FusedMBConv, :290-293 stem,
:319-324 last conv, :1127-1161 fixed padding; eval-mode BatchNorm eps 1e-3 :1051) so that a single device launch
(``mtb_debug_run_op``) can be compared with plain ``torch.nn.functional.conv2d`` arithmetic on identical operands instead
of with another kernel of this repository.  The ResNet-50 and MobileNetV3-small layers are those of
``oracle/port_tf_backbones.py`` (stride / dilation plan, ``_depth``, BN eps, preprocessing, correct_pad).

``precision``:
* ``'exact'``  conv -> BN (eval) -> act -> (+res) evaluated in the requested dtype (fp64 on the CPU, fp32 on the GPU with
               TF32 disabled): the bar for the fp32 / 3xTF32 kernels.
* ``'bf16'``, ``'bf16_simt'``, ``'fp16'``, ``'fp16_simt'``: the SAME arithmetic at the rounding points of that engine mode
  (csrc/engine.cu ``mtb_finalize_weights`` op loop and ``run_op_t``):
  - BN is folded in fp64 and the folded weight / bias cast to fp32 (engine.cu:615-624);
  - the weights of ops that pass ``tc_eligible`` (csrc/tc_gemm.cuh:471-475) are then rounded ONCE to the 16-bit storage
    type, in the tensor-core AND the CUDA-core mode of that type (engine.cu:625-630); depthwise and stem weights stay fp32;
  - the squeeze-excitation scaled input ``x*s`` is formed in fp32 and rounded to 16 bits in the tensor-core modes
    (``se_scale_kernel`` in place ahead of the GEMM, engine.cu:794-801); the CUDA-core modes keep the fp32 product
    (``conv_igemm_kernel`` a_scale, csrc/conv_simt.cuh:97-99);
  - everything else is wide; the device rounds the result once to 16 bits.
  ``layer_bound`` gives the per-element tolerance of that device result; ``'bf16'`` alone keeps its old meaning.
* ``'fp32'``, ``'tf32x3'``: the fp32-storage modes.  The folded weights are cast to fp32 and not rounded further (the
  3xTF32 kernel splits them into hi / lo planes whose sum is the fp32 weight, tc_tf32.cuh tc32_prepare_weights); the SE
  product ``x*s`` is formed in fp32 (``t32_split_a`` and ``conv_igemm_kernel`` a_scale) and not rounded further.
"""
import math

import torch
import torch.nn.functional as F

from oracle import port
from oracle import port_tf_backbones as tfb

# engine mode -> (16-bit storage dtype, tensor-core kernels)
MODES = {'bf16': (torch.bfloat16, True), 'bf16_simt': (torch.bfloat16, False),
         'fp16': (torch.float16, True), 'fp16_simt': (torch.float16, False)}
# the fp32-storage modes: 'fp32' (CUDA-core FMA) and 'tf32x3' (tc32_conv_kernel on its eligible convs, CUDA cores elsewhere)
WIDE_MODES = {'fp32': (torch.float32, False), 'tf32x3': (torch.float32, True)}


def storage(precision):
    """activation storage dtype of an engine mode (16-bit or fp32)"""
    return (MODES.get(precision) or WIDE_MODES[precision])[0]


def _op(weight, kernel=1, stride=1, pad=(0, 0), dil=1, act=None, depthwise=False, bn=None, eps=port.BN_EPS_EFFNETV2,
        bias=None, sample=None, res_first=False, pre=None, shift=0):
    """One engine op.  pad: explicit zero pad (begin, end) on both spatial axes, then VALID; sample: dense conv evaluated
    at pixels ``shift::stride`` instead (Conv2DDenseSame); pre: per-channel (scale, shift) of the stem input."""
    return dict(weight=weight, kernel=kernel, stride=stride, pad=pad, dil=dil, act=act, depthwise=depthwise, bn=bn, eps=eps,
                bias=bias, sample=sample, res_first=res_first, pre=pre, stem=pre is not None, shift=shift, maxpool=False)


def _effnet_conv(key, k, stride, shift, act, depthwise=False, stem=False):
    pb = (k - 1) // 2
    return _op(key + '.0.weight', k, stride, (pb - shift, k - 1 - pb + shift), act='silu' if act else None,
               depthwise=depthwise, bn=key + '.1', pre=((2.0,) * 3, (-1.0,) * 3) if stem else None, shift=shift)


def effnet_op_table(spec: port.EffNetSpec, prefix='backbone.1'):
    """engine op name (= reference key prefix of the layer) -> op dict (see _op)."""
    t = {f'{prefix}.0': _effnet_conv(f'{prefix}.0', 3, 2, 0, True, stem=True)}
    for b in port.effnet_block_list(spec):
        key = f'{prefix}.{b["key"]}.block'
        if b['block'] == 'fused':
            t[f'{key}.0'] = _effnet_conv(f'{key}.0', b['kernel'], b['stride'], b['shift'], True)
            if b['expand'] != 1:
                t[f'{key}.1'] = _effnet_conv(f'{key}.1', 1, 1, 0, False)
        else:
            i = 0
            if b['expand'] != 1:
                t[f'{key}.{i}'] = _effnet_conv(f'{key}.{i}', 1, 1, 0, True)
                i += 1
            t[f'{key}.{i}'] = _effnet_conv(f'{key}.{i}', b['kernel'], b['stride'], b['shift'], True, depthwise=True)
            i += 2  # squeeze-excitation sits between the depthwise conv and the projection
            t[f'{key}.{i}'] = _effnet_conv(f'{key}.{i}', 1, 1, 0, False)
    t[f'{prefix}.{len(spec.stages) + 1}'] = _effnet_conv(f'{prefix}.{len(spec.stages) + 1}', 1, 1, 0, True)
    return t


def resnet50_op_table(cfg: port.PathConfig, prefix='backbone.'):
    """ResNet50Spec.features (oracle/port_tf_backbones.py): conv bias folded by BN (eps 1e-5), caffe stem, zero-padded
    max pool, dense-SAME 1x1 convs sampled at shift::stride, dilated 3x3, relu(shortcut + _3_conv)."""
    e = tfb.RESNET_BN_EPS
    mean = torch.tensor([103.939, 116.779, 123.68])  # fp32 constants, as in port_tf_backbones and the stem kernel
    t = {prefix + 'conv1_conv': _op(prefix + 'conv1_conv.weight', 7, 2, (3, 3), act='relu', bn=prefix + 'conv1_bn', eps=e,
                                    bias=prefix + 'conv1_conv.bias', pre=((255.0,) * 3, tuple((-mean).double().tolist())))}
    t[prefix + 'pool1_pool'] = dict(_op(None, 3, 2, (1, 1)), maxpool=True)
    for name, _f, stride, shift, dil, conv_shortcut in tfb.resnet50_blocks(cfg):
        b = prefix + name

        def cb(j, k=1, **kw):
            return _op(f'{b}_{j}_conv.weight', k, bn=f'{b}_{j}_bn', eps=e, bias=f'{b}_{j}_conv.bias', **kw)
        if conv_shortcut:
            t[f'{b}_0_conv'] = cb(0, stride=stride, sample=shift, shift=shift)
        t[f'{b}_1_conv'] = cb(1, stride=stride, sample=shift, shift=shift, act='relu')
        t[f'{b}_2_conv'] = cb(2, 3, pad=(dil, dil), dil=dil, act='relu')
        t[f'{b}_3_conv'] = cb(3, act='relu', res_first=True)
    return t


def mobilenetv3_small_op_table(cfg: port.PathConfig, prefix='backbone.'):
    """MobileNetV3SmallSpec.features (oracle/port_tf_backbones.py): TF-'same' stem on 2x-1, correct_pad before the
    stride-2 depthwise convs, ReLU / hard-swish, projection without activation (+ residual), Conv_2 with bias and no BN."""
    e = tfb.MOBILENET_BN_EPS
    s = cfg.proc_side
    pad_total = max(((s + 1) // 2 - 1) * 2 + 3 - s, 0)
    t = {prefix + 'Conv': _op(prefix + 'Conv.weight', 3, 2, (pad_total // 2, pad_total - pad_total // 2), act='hswish',
                              bn=prefix + 'Conv.BatchNorm', eps=e, pre=((2.0,) * 3, (-1.0,) * 3))}
    for bi, (_exp, _filters, k, stride, _se, act, br) in enumerate(tfb.MOBILENETV3_SMALL_ROWS):
        b = prefix + ('expanded_conv' if bi == 0 else f'expanded_conv_{bi}')
        act = 'hswish' if act == 'hswish' else 'relu'
        if bi != 0:
            t[b + '.expand'] = _op(b + '.expand.weight', act=act, bn=b + '.expand.BatchNorm', eps=e)
        shift = 1 if (br and cfg.centered_stride and stride == 2) else 0
        pb = (k - 1) // 2
        t[b + '.depthwise'] = _op(b + '.depthwise.weight', k, stride, (pb - shift, k - 1 - pb + shift), act=act, depthwise=True,
                                  bn=b + '.depthwise.BatchNorm', eps=e, shift=shift)
        t[b + '.project'] = _op(b + '.project.weight', bn=b + '.project.BatchNorm', eps=e)
    t[prefix + 'Conv_1'] = _op(prefix + 'Conv_1.weight', act='hswish', bn=prefix + 'Conv_1.BatchNorm', eps=e)
    t[prefix + 'Conv_2'] = _op(prefix + 'Conv_2.weight', act='hswish', bias=prefix + 'Conv_2.bias')
    return t


def op_table(spec):
    if isinstance(spec, tfb.ResNet50Spec):
        return resnet50_op_table(spec.cfg)
    if isinstance(spec, tfb.MobileNetV3SmallSpec):
        return mobilenetv3_small_op_table(spec.cfg)
    return effnet_op_table(spec)


def _fold(sd, op):
    """(w, b) of an op with the conv bias folded through BN as (b - mean) * s + beta (engine.cu:609-613), in fp64."""
    w = sd[op['weight']].double()
    b = sd[op['bias']].double() if op['bias'] else torch.zeros(w.shape[0], dtype=torch.float64)
    if op['bn']:
        k = op['bn']
        s = sd[k + '.weight'].double() / torch.sqrt(sd[k + '.running_var'].double() + op['eps'])
        w = w * s[:, None, None, None]
        b = (b - sd[k + '.running_mean'].double()) * s + sd[k + '.bias'].double()
    return w, b


def tc_eligible(op, cin, cout):
    """tc_eligible (csrc/tc_gemm.cuh:471-475): the convs whose weights the 16-bit modes round to 16 bits."""
    return (not op['stem'] and not op['depthwise'] and not op['maxpool'] and cin % 8 == 0 and cout % 8 == 0
            and op['stride'] in (1, 2) and op['kernel'] in (1, 3))


def tc32_eligible(op, cin, cout):
    """tc32_eligible (csrc/tc_tf32.cuh:282) for the ops of an op table: the convs that 'tf32x3' runs on tc32_conv_kernel
    (the others on CUDA cores).  The engine's rule also excludes its small_io ops, the squeeze-excitation fcs; those are
    not in the op tables (se_fc_bound covers them), so stem / depthwise / max pool stand in for is_conv / depthwise here."""
    return (not op['stem'] and not op['depthwise'] and not op['maxpool'] and cin % 4 == 0 and cout % 4 == 0
            and op['stride'] in (1, 2) and op['kernel'] in (1, 3))


def _act(y, act):
    if act == 'silu':
        return F.silu(y)
    if act == 'relu':
        return F.relu(y)
    if act == 'hswish':
        return tfb.hard_swish(y)
    if act == 'sigmoid':
        return torch.sigmoid(y)
    if act == 'hsigmoid':
        return tfb.hard_sigmoid(y)
    return y


def _layer(sd, spec, name, x_nhwc, res_nhwc, scale, precision, dtype, magnitude=False):
    """-> (output NCHW, pre-activation NCHW, products per output).  magnitude: the same layer on |x|, |w|, |b|, |res| with
    no activation (the pre-activation magnitude that bounds the accumulation error)."""
    op = op_table(spec)[name]
    dev = x_nhwc.device
    if op['maxpool']:  # zero pad (the pad value takes part in the max), then VALID
        x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
        x = x.abs() if magnitude else x
        y = F.max_pool2d(F.pad(x, op['pad'] * 2), op['kernel'], op['stride'])
        return y, y, 1
    w, bias = _fold(sd, op)
    st = MODES[precision][0] if precision in MODES else None
    if st is not None or precision in WIDE_MODES:
        w, bias = w.float().double(), bias.float().double()
        if st is not None and tc_eligible(op, w.shape[1], w.shape[0]):
            w = w.float().to(st).double()
    w, bias = w.to(dev, dtype), bias.to(dev, dtype)
    if op['stem']:
        a, c = (torch.tensor(v, dtype=torch.float32).to(dev, dtype)[None, :, None, None] for v in op['pre'])
        x = x_nhwc.to(dtype)
        x = (x * a).abs() + c.abs() if magnitude else x * a + c  # magnitude also bounds the fp32 rounding of x*a + c
    else:
        x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    if scale is not None:
        s = scale.to(dev, dtype)[:, :, None, None]
        if st is not None and MODES[precision][1] and not magnitude:  # se_scale_kernel: fp32 product, rounded to 16 bits
            x = (x.float() * s.float()).to(st).to(dtype)
        elif precision in WIDE_MODES and not magnitude:  # fp32 product, no further rounding
            x = (x.float() * s.float()).to(dtype)
        else:
            x = x * s
    if magnitude:
        x, w, bias = x.abs(), w.abs(), bias.abs()
    x = F.pad(x, op['pad'] * 2)
    groups = x.shape[1] if op['depthwise'] else 1
    if op['sample'] is not None:
        z = F.conv2d(x, w, bias, dilation=op['dil'])[:, :, op['sample']::op['stride'], op['sample']::op['stride']]
    else:
        z = F.conv2d(x, w, bias, stride=op['stride'], dilation=op['dil'], groups=groups)
    k = w.shape[1] * w.shape[2] * w.shape[3]
    res = None
    if res_nhwc is not None:
        res = res_nhwc.permute(0, 3, 1, 2).to(dtype)
        res = res.abs() if magnitude else res
    if res is not None and op['res_first']:
        z = z + res
    y = z if magnitude else _act(z, op['act'])
    if res is not None and not op['res_first']:
        y = y + res
    return y, z, k


def conv_layer_reference(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='exact', dtype=torch.float64):
    """One conv layer (or the max pool) of the backbone on ``x_nhwc`` [B,H,W,C] (the stem takes NCHW crops in [0,1] and
    applies the model's preprocessing).  Returns NHWC in ``dtype``."""
    return _layer(sd, spec, name, x_nhwc, res_nhwc, scale, precision, dtype)[0].permute(0, 2, 3, 1).contiguous()


# ---------------------------------------------------------------------------------------------- per-element bound
# Accumulation: any fp32 summation order of n terms errs by at most gamma_n = n*u/(1-n*u) times the sum of |terms|
# (u = 2^-24 for round-to-nearest).  C_ACC = 2 allows u = 2^-23 (the tensor cores' fp32 accumulate aligns and truncates
# rather than rounding to nearest) and the 1/(1-n*u) factor; n = products + bias + residual + the fp32 x*s / stem
# preprocessing products, so K + 4.
C_ACC = 2.0
# 3xTF32 products (tc_tf32.cuh): x = hi + lo with hi = RN_tf32(x), so |lo| <= 2^-11 |x|; the tensor core reads the lo
# operands (the split activations and the host lo weight plane) as tf32, truncating: |lo - tf32(lo)| < 2^-10 |lo| <= 2^-21 |x|;
# the lo*lo product is dropped: <= 2^-22 |x w|.  Per product |x*w - (hi_x hi_w + lo_x' hi_w + hi_x lo_w')|
# <= (2^-22 + 2 * 2^-21 (1 + 2^-11)) |x| |w| <= 5 * 2^-22 * (1 + 2^-10) |x| |w|.
TC32_SPLIT = 5.0 * 2.0 ** -22 * (1.0 + 2.0 ** -10)
# smallest normal fp32: the MUFU approximations (ex2 / rcp .ftz) flush subnormal results to zero
FP32_FLOOR = 2.0 ** -126
# tanh.approx.f32: maximum relative error 2^-10.987 (PTX ISA, tanh instruction)
TANH_APPROX_REL = 2.0 ** -10.987
# sup |act'|: SiLU 1.0998 (x = 2.40), hard-swish 1.5 (x = 3), ReLU / none 1, sigmoid 1/4, hard-sigmoid 1/6
LIPSCHITZ = {'silu': 1.1, 'hswish': 1.5, 'relu': 1.0, None: 1.0, 'sigmoid': 0.25, 'hsigmoid': 1.0 / 6.0}


def _act_error(z, y, act, precision):
    """|device activation - exact activation| at pre-activation z (y = act(z))."""
    az, ay = z.abs(), y.abs()
    if act == 'silu' and precision == 'bf16':
        # tc_act / fast_act for bf16 outputs: h + h*tanh.approx(h), h = x/2 (csrc/tc_gemm.cuh:169-183, conv_simt.cuh:272-287)
        h = 0.5 * az
        return h * torch.tanh(h) * TANH_APPROX_REL + 2.0 ** -22 * (az + ay)
    if act in ('silu', 'sigmoid'):
        # silu_f16out and t32_act<ACT_SILU> (ex2.approx.ftz + rcp.approx.ftz, csrc/common.cuh:156-166, tc_tf32.cuh:74-83) and
        # act_t (x / (1 + __expf(-x)), IEEE divide): the fp32 rounding of x*log2(e) gives |x|*2^-24 relative error in e^-x,
        # ex2 2 ulp, 1 + e 1/2 ulp, rcp 1 ulp (or the divide 1/2 ulp), the product 1/2 ulp: (8 + |x|) * 2^-24 relative, as
        # |dsig/sig| <= |de/e|
        return (8.0 + 2.0 * az) * 2.0 ** -24 * ay
    if act == 'hswish':  # x * sat(x/6 + 0.5): the rounded 1/6, the fma and the product
        return 2.0 ** -22 * (az + ay)
    if act == 'hsigmoid':  # min(max(x + 3, 0), 6) * (1/6): the sum, the rounded 1/6 and the product
        return 2.0 ** -22 * (az + 3.0)
    return torch.zeros_like(z)


def bound_from_parts(z, y, zabs, k, act, precision, tc32=False):
    """The per-element tolerance of a device result from the exact layer: pre-activation z, output y (after the
    residual), pre-activation magnitude zabs and k products per output; tc32 adds the 3xTF32 split term per product.

        16-bit modes: tol = 2^-p * (|y| + e) + e + floor16,  fp32 modes: tol = e + 2^-126,
        e = L_act * (C_ACC * (K + 4) * 2^-24 + [TC32_SPLIT]) * zabs + e_act + 2^-23 * |y|"""
    rate = C_ACC * (k + 4) * 2.0 ** -24 + (TC32_SPLIT if tc32 else 0.0)
    e = LIPSCHITZ[act] * rate * zabs + _act_error(z, _act(z, act), act, precision) + 2.0 ** -23 * y.abs()
    st = storage(precision)
    if st == torch.float32:
        return e + FP32_FLOOR
    p = 8 if st == torch.bfloat16 else 11
    return 2.0 ** -p * (y.abs() + e) + e + (2.0 ** -25 if st == torch.float16 else 0.0)


def layer_bound(sd, spec, name, x_nhwc, res_nhwc=None, scale=None, precision='fp16'):
    """-> (ref, tol), NHWC fp64: the exact layer on this mode's rounded operands and the per-element bound on
    |device - ref| (bound_from_parts),

        tol = 2^-p * (|ref| + e) + e + floor,   e = L_act * C_ACC * (K + 4) * 2^-24 * refabs + e_act + 2^-23 * |ref|

    with p = 8 (bf16) / 11 (fp16) (half an ulp of the output, rounded to nearest even), floor = half the fp16 subnormal
    spacing (2^-25), refabs the pre-activation magnitude (the layer on |x|, |w|, |b|, |res|), e_act the activation's own
    error (_act_error) and 2^-23 * |ref| the fp32 residual add / epilogue roundings.  In the fp32-storage modes there is
    no output rounding (tol = e + 2^-126), and a 'tf32x3' op that reaches tc32_conv_kernel adds TC32_SPLIT * refabs."""
    op = op_table(spec)[name]
    y, z, k = _layer(sd, spec, name, x_nhwc, res_nhwc, scale, precision, torch.float64)
    zabs = _layer(sd, spec, name, x_nhwc, res_nhwc, scale, precision, torch.float64, magnitude=True)[1]
    if op['maxpool']:  # a max of stored values is exact
        tol = torch.zeros_like(y)
    else:
        tc32 = precision == 'tf32x3' and tc32_eligible(op, x_nhwc.shape[-1], y.shape[1])
        tol = bound_from_parts(z, y, zabs, k, op['act'], precision, tc32)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
    return nhwc(y), nhwc(tol)


def overflow_threshold(dtype):
    """Smallest magnitude that rounds to inf in ``dtype`` (max + half an ulp of max): 65520 for fp16."""
    fi = torch.finfo(dtype)
    return fi.max + fi.eps * 2.0 ** math.floor(math.log2(fi.max)) / 2


def check_bound(dev, ref, tol, precision):
    """-> (worst |dev - ref| / tol over the finite device elements, number of violating elements).  Violations: a NaN;
    an inf where |ref| - tol still overflows the storage type (or a finite value there); an inf of the wrong sign or
    where |ref| + tol does not reach the overflow threshold; a finite value farther than tol from ref."""
    dev, ref, tol = dev.double(), ref.double().to(dev.device), tol.double().to(dev.device)
    top = overflow_threshold(storage(precision))
    must_inf = ref.abs() - tol >= top
    may_inf = ref.abs() + tol >= top
    fin = torch.isfinite(dev)
    inf_ok = torch.isinf(dev) & may_inf & (torch.sign(dev) == torch.sign(ref))
    err = torch.where(fin, (dev - ref).abs(), torch.zeros_like(dev))
    bad = torch.isnan(dev) | (fin & (must_inf | (err > tol))) | (torch.isinf(dev) & ~inf_ok)
    ratio = torch.where(fin & ~must_inf, err / tol.clamp_min(1e-300), torch.zeros_like(dev))
    return float(ratio.max()) if ratio.numel() else 0.0, int(bad.sum())


def se_fc_bound(x, xabs, n_in, w, b, act, x_err=None):
    """One squeeze-excitation fc (1x1 conv on [B, Cin], fp32 weights and output: small_io ops are never tc_eligible) on
    an input ``x`` [B, Cin] whose fp32 evaluation summed ``n_in`` terms of magnitude ``xabs`` per element (the pooled
    mean of an HxW map: H*W pixels, the partial slices and the 1/(H*W) product; 0 for an exact input), and which may
    also differ from ``x`` by ``x_err`` (absolute, per element).
    -> (ref, tol) [B, Cout] fp64: act(x @ w.T + b) and the bound on the device's fp32 result,
    tol = L_act * (C_ACC * (Cin + n_in + 4) * 2^-24 * (|w| @ xabs + |b|) + |w| @ x_err) + e_act + 2^-23 * |ref|."""
    w = w.reshape(w.shape[0], -1).float().double().to(x.device)
    b = b.float().double().to(x.device)
    z = x.double() @ w.T + b
    y = _act(z, act)
    e = C_ACC * (w.shape[1] + n_in + 4) * 2.0 ** -24 * (xabs.double() @ w.abs().T + b.abs())
    if x_err is not None:
        e = e + x_err.double() @ w.abs().T
    return y, LIPSCHITZ[act] * e + _act_error(z, y, act, 'fp32') + 2.0 ** -23 * y.abs()


def pool_mean_bound(x_nhwc):
    """pool_mean_kernel (csrc/conv_simt.cuh:821): the mean over H*W of x [B,H,W,C], summed in fp32 (a strided per-thread sum,
    then an 8-way tree) and multiplied by the rounded 1/(H*W).  -> (mean, tol) [B, C] fp64, tol = C_ACC (P + 2) 2^-24 mean|x|."""
    x = x_nhwc.double()
    n = x.shape[1] * x.shape[2]
    return x.mean(dim=(1, 2)), C_ACC * (n + 2) * 2.0 ** -24 * x.abs().mean(dim=(1, 2)) + FP32_FLOOR


# ------------------------------------------------------------------------------------------ soft-argmax decode bound
def head_logit_delta(feats_nchw, w, b, tc32=False):
    """Per-logit bound on |device logit - exact logit| of the head's 1x1 conv on features [B,C,H,W] with weight w
    [N,C,1,1] and bias b [N] (the operands the device multiplies: 16-bit features and weights for the fused 16-bit head,
    fp32 otherwise): C_ACC (C + 2) 2^-24 (|w| |f| + |b|), the fp32 accumulation of exact products (tc_head_kernel,
    conv_igemm_kernel), plus TC32_SPLIT |w| |f| for the 3xTF32 head GEMM."""
    mag = F.conv2d(feats_nchw.abs(), w.abs())
    c = feats_nchw.shape[1]
    return C_ACC * (c + 2) * 2.0 ** -24 * (mag + b.abs()[None, :, None, None]) + (TC32_SPLIT * mag if tc32 else 0.0)


def _soft_argmax_bound(logits, delta, dims):
    """-> (coords [..., len(dims)] in [0,1] heatmap units, tol of the same shape) of port.soft_argmax over ``dims`` for
    device logits within ``delta`` (absolute, per logit) of ``logits``, decoded by softargmax_bhwn_kernel or the fused
    head's epilogue (online softmax in fp32, exp2 on the MUFU):

        |c' - c| <= e^Dmax * sum_i p_i (e^D_i - 1) |x_i - c|  +  (2 gamma_n + 3 * 2^-24) |c|  +  n * 2^-120

    p the exact softmax, x_i the linspace coordinate of element i on that axis, and D_i = delta_i + the decode's own
    error in the weight of element i: the rounding of its exponent argument, in either form ((v - m) * log2e, or
    v * log2e - m * log2e with the bias folded in) 8 * 2^-24 (|v_i| + |m|) as a natural-log error, and one ex2 (2 ulp) and
    one product (1/2 ulp) per running-max rescale or merge it passes through (at most n_exp = P + D + 4).  gamma_n =
    C_ACC (n + n_exp + 4) 2^-24 covers the fp32 sums s, sx, sy, sz (n = P in 2D, P * D in 3D), and 3 * 2^-24 the two
    divisions; n * 2^-120 the weights ex2.approx.ftz flushes to zero."""
    dims = tuple(d if d >= 0 else logits.ndim + d for d in dims)
    n = 1
    for d in dims:
        n *= logits.shape[d]
    spatial = logits.shape[dims[0]] * logits.shape[dims[1]]
    depth = logits.shape[dims[2]] if len(dims) > 2 else 0
    n_exp = spatial + depth + 4
    mx = torch.amax(logits, dim=dims, keepdim=True)
    e = torch.exp(logits - mx)
    p = e / e.sum(dim=dims, keepdim=True)
    dmax_all = torch.amax(delta, dim=dims, keepdim=True)
    big = 8.0 * 2.0 ** -24 * (logits.abs() + mx.abs() + 2 * dmax_all) + n_exp * (2.0 ** -22 + 2.0 ** -24)
    dtot = delta + big
    dmax = torch.amax(dtot, dim=dims, keepdim=True)
    gamma = C_ACC * (n + n_exp + 4) * 2.0 ** -24
    coords, tols = [], []
    for d in dims:
        shape = [1] * logits.ndim
        shape[d] = logits.shape[d]
        x = port.linspace01(logits.shape[d], torch.float64).reshape(shape)
        c = (p * x).sum(dim=dims, keepdim=True)
        t = torch.exp(dmax) * (p * torch.expm1(dtot) * (x - c).abs()).sum(dim=dims, keepdim=True)
        t = t + (2 * gamma + 3 * 2.0 ** -24) * c.abs() + n * 2.0 ** -120
        for hd in sorted(dims, reverse=True):
            c, t = c.squeeze(hd), t.squeeze(hd)
        coords.append(c)
        tols.append(t)
    return torch.stack(coords, dim=-1), torch.stack(tols, dim=-1)


def decode_bound(logits, delta, cfg, n_joints):
    """The head's decode on exact fp64 logits [B, J + D*J, H, W] (CPU) with per-logit device tolerance ``delta`` (same
    shape) -> (coords2d px [B,J,2], tol2d, coords3d_rel mm [B,J,3], tol3d): port.heads' soft-argmax and
    heatmap_to_image / heatmap_to_metric, each coordinate with the bound of _soft_argmax_bound carried through the
    device's fmaf scale (c * mul + add with mul, add rounded to fp32: 4 * 2^-24 (|c mul| + |add|))."""
    l2, l3 = port.split_logits(logits, n_joints, cfg.depth)
    d2, d3 = port.split_logits(delta, n_joints, cfg.depth)
    c2, t2 = _soft_argmax_bound(l2, d2, dims=(3, 2))
    c3, t3 = _soft_argmax_bound(l3, d3, dims=(4, 3, 1))
    last = cfg.proc_side - 1
    mul = float(last - last % cfg.stride_test)
    add = float(cfg.stride_test // 2) * (int(cfg.centered_stride) + int(cfg.legacy_centered_stride_bug))
    mm = cfg.box_size_mm / cfg.proc_side
    px2 = port.heatmap_to_image(c2, cfg)
    tol2 = mul * t2 + 4 * 2.0 ** -24 * (mul * c2.abs() + abs(add))
    mm3 = port.heatmap_to_metric(c3, cfg)
    scale3 = torch.tensor([mul * mm, mul * mm, cfg.box_size_mm], dtype=torch.float64)
    add3 = torch.tensor([add * mm, add * mm, 0.0], dtype=torch.float64)
    tol3 = scale3 * t3 + 4 * 2.0 ** -24 * (scale3 * c3.abs() + add3.abs())
    return px2, tol2, mm3, tol3
