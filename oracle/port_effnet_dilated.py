"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of EfficientNetV2 at output stride 16 and 8: the TF reference's
``efficientnetv2-{s,l}-stride{16,8}`` backbones (the reference's ``metrabs_tf/backbones/efficientnet/effnetv2_configs.py``
:163-228, built by ``effnetv2_model.py`` :574-600), and the per-layer reference arithmetic of their engine ops.

* Table: the stride-32 table of ``port.effnet_spec`` re-strided in one pass (``dilate``): with a running stride from 2 after
  the stem and a running dilation d = 1, a stride-2 row that would take the stride past the output stride becomes stride 1
  with ``dilation_in`` d, then d doubles and is its ``dilation_out``; every other row gets d for both.  The bottom-right
  shift moves to the last row that still strides, under ``centered_stride`` only (effnetv2_configs.py:45).
* Block: the first block of a stage dilates its depthwise conv by ``dilation_in``, the later ones by ``dilation_out``, each
  with ``fixed_padding_layer(k, rate=d)`` (``metrabs_pytorch/backbones/efficientnet.py`` :1127-1161).

``oracle/port.py`` keeps its stride-32 specs, random init and state-dict checksums as they are; at output stride 32 the
spec here has the same rows with dilations 1 and gives the same state dict.

Parity pin: the TF model cannot run without TensorFlow, so ``oracle/gen_golden_effnet_dilated.py`` builds the reference's
PyTorch ``EfficientNet`` from the derived rows, dilates its depthwise convs and swaps in the reference's own
``fixed_padding_layer(k, rate=d)``, and commits its outputs under ``tests/golden/effnet*_os{16,8}*.npz``;
``tests/test_oracle_effnet_dilated.py`` checks this restatement against those files and the tables against the TF ones.
"""
import dataclasses
import math
from typing import List

import torch
import torch.nn.functional as F

from oracle import port, port_ops

OUTPUT_STRIDES = (8, 16, 32)
DILATED_NAMES = ('efficientnetv2-s', 'efficientnetv2-l', 'efficientnetv2-tiny')


@dataclasses.dataclass
class DilatedStageSpec(port.StageSpec):
    dilation_in: int = 1
    dilation_out: int = 1


@dataclasses.dataclass
class EffNetDilatedSpec:
    """port.EffNetSpec with dilated rows; not a subclass, so port.metrabs_forward runs ``features`` below."""
    name: str
    stages: List[DilatedStageSpec]
    last_channel: int
    output_stride: int = 32

    @property
    def stem_channels(self):
        return self.stages[0].cin

    def features(self, sd, image, tap=None):
        """port.metrabs_forward calls this for a spec that is not a port.EffNetSpec."""
        return effnet_features(sd, self, image, tap=tap)


def dilate(stages, output_stride, centered_stride):
    """The stride-32 rows ``stages`` (port.StageSpec) at ``output_stride`` (module docstring) -> [DilatedStageSpec]."""
    out, running, d = [], 2, 1
    for st in stages:
        row = DilatedStageSpec(**dict(dataclasses.asdict(st), bottomright=False))
        if st.stride == 2 and running * 2 > output_stride:
            row.stride, row.dilation_in, row.dilation_out = 1, d, 2 * d
            d *= 2
        else:
            running *= st.stride
            row.dilation_in = row.dilation_out = d
        out.append(row)
    last_strided = max(i for i, r in enumerate(out) if r.stride == 2)
    out[last_strided].bottomright = bool(centered_stride)
    return out


def effnet_spec(name, centered_stride=True, output_stride=32):
    """port.effnet_spec(name, centered_stride) at ``output_stride`` 32, 16 or 8 (16 and 8: V2-S, V2-L and 'tiny' only)."""
    if output_stride not in OUTPUT_STRIDES:
        raise ValueError(f'output stride {output_stride}')
    if output_stride != 32 and name not in DILATED_NAMES:
        raise ValueError(f'{name} has no table at output stride {output_stride}')
    base = port.effnet_spec(name, centered_stride)
    if output_stride == 32:
        rows = [DilatedStageSpec(**dataclasses.asdict(st)) for st in base.stages]
    else:
        rows = dilate(base.stages, output_stride, centered_stride)
    return EffNetDilatedSpec(name, rows, base.last_channel, output_stride)


def fixed_pad(x, kernel, shift, rate=1):
    """efficientnet.py:1127-1161: explicit zero pad (pb - shift, pe + shift) of the dilated kernel, then VALID."""
    total = kernel + (kernel - 1) * (rate - 1) - 1
    pb = total // 2
    return F.pad(x, (pb - shift, total - pb + shift, pb - shift, total - pb + shift))


def block_list(spec):
    """port.effnet_block_list with each block's depthwise dilation ``dil``."""
    blocks = port.effnet_block_list(spec)
    i = 0
    for st in spec.stages:
        for bi in range(st.layers):
            blocks[i]['dil'] = st.dilation_in if bi == 0 else st.dilation_out
            i += 1
    return blocks


def _conv_bn(sd, key, x, stride=1, groups=1, act=True, dil=1, tap=None):
    x = F.conv2d(x, sd[key + '.0.weight'], None, stride=stride, dilation=dil, groups=groups)
    x = port._bn(sd, key + '.1', x, port.BN_EPS_EFFNETV2)
    x = F.silu(x) if act else x
    if tap is not None:
        tap[key] = x
    return x


def effnet_features(sd, spec, image, prefix='backbone.1', tap=None):
    """port.effnet_features with dilated MBConv depthwise convs: [B,3,S,S] -> [B,last_channel,S/os,S/os]."""
    x = image * 2 - 1
    x = _conv_bn(sd, f'{prefix}.0', fixed_pad(x, 3, 0), stride=2, tap=tap)
    for b in block_list(spec):
        key = f'{prefix}.{b["key"]}.block'
        inp = x
        if b['block'] == 'fused':
            assert b['dil'] == 1, b
            x = fixed_pad(x, b['kernel'], b['shift'])
            x = _conv_bn(sd, f'{key}.0', x, stride=b['stride'], tap=tap)
            if b['expand'] != 1:
                x = _conv_bn(sd, f'{key}.1', x, act=False, tap=tap)
        else:
            i = 0
            if b['expand'] != 1:
                x = _conv_bn(sd, f'{key}.{i}', x, tap=tap)
                i += 1
            x = fixed_pad(x, b['kernel'], b['shift'], b['dil'])
            x = _conv_bn(sd, f'{key}.{i}', x, stride=b['stride'], groups=b['cin'] * b['expand'], dil=b['dil'], tap=tap)
            s = x.mean(dim=(2, 3), keepdim=True)
            s = F.silu(F.conv2d(s, sd[f'{key}.{i + 1}.fc1.weight'], sd[f'{key}.{i + 1}.fc1.bias']))
            x = x * torch.sigmoid(F.conv2d(s, sd[f'{key}.{i + 1}.fc2.weight'], sd[f'{key}.{i + 1}.fc2.bias']))
            x = _conv_bn(sd, f'{key}.{i + 2}', x, act=False, tap=tap)
        if b['residual']:
            x = x + inp
        if tap is not None:
            tap[f'{prefix}.{b["key"]}'] = x
    return _conv_bn(sd, f'{prefix}.{len(spec.stages) + 1}', x, tap=tap)


def make_state_dict(spec, cfg: port.PathConfig, n_joints, seed=0, calib_batch=4, head_gain=10.0):
    """port.make_effnet_state_dict's conditioned random init (same generator draws in the same order, so the same state
    dict at output stride 32), with the BN statistics calibrated on the dilated network."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    prefix = 'backbone.1'
    calib, _ = port.synthetic_inputs(calib_batch, cfg.proc_side, seed=seed + 77)
    with torch.no_grad():
        x = port._init_conv_bn(sd, f'{prefix}.0', fixed_pad(calib * 2 - 1, 3, 0), g, spec.stem_channels, 3, stride=2)
        for b in block_list(spec):
            key = f'{prefix}.{b["key"]}.block'
            inp = x
            cexp = b['cin'] * b['expand']
            damp = 0.5 if b['residual'] else 1.0
            if b['block'] == 'fused':
                x = fixed_pad(x, b['kernel'], b['shift'])
                if b['expand'] != 1:
                    x = port._init_conv_bn(sd, f'{key}.0', x, g, cexp, b['kernel'], stride=b['stride'])
                    x = port._init_conv_bn(sd, f'{key}.1', x, g, b['cout'], 1, act=False, gamma_scale=damp)
                else:
                    x = port._init_conv_bn(sd, f'{key}.0', x, g, b['cout'], b['kernel'], stride=b['stride'], gamma_scale=damp)
            else:
                i = 0
                if b['expand'] != 1:
                    x = port._init_conv_bn(sd, f'{key}.{i}', x, g, cexp, 1)
                    i += 1
                x = fixed_pad(x, b['kernel'], b['shift'], b['dil'])
                w = torch.randn(cexp, 1, b['kernel'], b['kernel'], generator=g) * math.sqrt(2.0 / (b['kernel'] ** 2))
                sd[f'{key}.{i}.0.weight'] = w
                x = F.conv2d(x, w, None, stride=b['stride'], dilation=b['dil'], groups=cexp)
                x = F.silu(port._calibrate_bn(sd, f'{key}.{i}.1', x, g, port.BN_EPS_EFFNETV2))
                i += 1
                csq = max(1, b['cin'] // 4)
                sd[f'{key}.{i}.fc1.weight'] = torch.randn(csq, cexp, 1, 1, generator=g) * math.sqrt(2.0 / cexp)
                sd[f'{key}.{i}.fc1.bias'] = 0.2 * torch.randn(csq, generator=g)
                sd[f'{key}.{i}.fc2.weight'] = torch.randn(cexp, csq, 1, 1, generator=g) * math.sqrt(2.0 / csq)
                sd[f'{key}.{i}.fc2.bias'] = 0.5 * torch.randn(cexp, generator=g)
                s = x.mean(dim=(2, 3), keepdim=True)
                s = F.silu(F.conv2d(s, sd[f'{key}.{i}.fc1.weight'], sd[f'{key}.{i}.fc1.bias']))
                x = x * torch.sigmoid(F.conv2d(s, sd[f'{key}.{i}.fc2.weight'], sd[f'{key}.{i}.fc2.bias']))
                i += 1
                x = port._init_conv_bn(sd, f'{key}.{i}', x, g, b['cout'], 1, act=False, gamma_scale=damp)
            if b['residual']:
                x = x + inp
        port._init_conv_bn(sd, f'{prefix}.{len(spec.stages) + 1}', x, g, spec.last_channel, 1)
    port.init_head(sd, g, spec.last_channel, n_joints, cfg.depth, head_gain)
    return sd


# ---------------------------------------------------------------------------------------------- per-layer arithmetic
def op_table(spec, prefix='backbone.1'):
    """engine op name -> op dict (port_ops._op): port_ops.effnet_op_table with each depthwise op's dilation and padding."""
    t = port_ops.effnet_op_table(spec, prefix)
    for b in block_list(spec):
        if b['block'] == 'mb':
            nm = f'{prefix}.{b["key"]}.block.{1 if b["expand"] != 1 else 0}'
            d, k = b['dil'], b['kernel']
            total = (k - 1) * d
            t[nm] = dict(t[nm], dil=d, pad=(total // 2 - b['shift'], total - total // 2 + b['shift']))
    return t


def dw_layer_bound(sd, spec, name, x_nhwc, precision='fp16'):
    """port_ops.layer_bound for a (dilated) depthwise op of ``spec``: the exact layer on this mode's rounded operands and
    the same per-element bound, tol = 2^-p (|ref| + e) + e + floor.  -> (ref, tol), NHWC fp64."""
    op = op_table(spec)[name]
    assert op['depthwise'] and op['act'] == 'silu', name
    w, bias = (t.float().double().to(x_nhwc.device) for t in port_ops._fold(sd, op))
    x = F.pad(x_nhwc.permute(0, 3, 1, 2).double(), op['pad'] * 2)
    conv = lambda x_, w_, b_: F.conv2d(x_, w_, b_, stride=op['stride'], dilation=op['dil'], groups=x_.shape[1])  # noqa: E731
    z = conv(x, w, bias)
    zabs = conv(x.abs(), w.abs(), bias.abs())
    y = port_ops._act(z, 'silu')
    k = w.shape[2] * w.shape[3]
    tol = port_ops.bound_from_parts(z, y, zabs, k, 'silu', precision)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()  # noqa: E731
    return nhwc(y), nhwc(tol)
