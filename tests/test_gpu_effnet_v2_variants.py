"""GPU: EfficientNetV2-B0..B3 and -XL (metrabs_b200.backbones.efficientnet.efficientnet_v2_b0() .. _b3(), _xl()), and
fmb_kernel on identity-shaped FusedMBConv blocks whose width is a multiple of 8 but not of 16 (40 and 56 in V2-B2 / -B3).

* fp32 and tf32x3: V2-B0@224, V2-B3@256 and XL@256 against the goldens the reference's PyTorch module produced
  (tests/golden/effnetv2{b0,b3,xl}_*.npz) and against the restatement: features and joints within 1e-3.
* bf16 and fp16: every op of the V2-B0, V2-B3 and XL forwards element by element against fp64 conv2d on the tensors the
  forward itself produced (test_gpu_forward_ops16.py's walk and bars), the fused blocks included.
* V2-B2 and V2-B3 in bf16 and fp16: every identity-shaped FusedMBConv block, the 40- and 56-channel ones among them, runs as
  one fmb_kernel launch, and its output on the forward's own input is bit-equal to the two launches it replaces.  A forward
  with those blocks unfused runs every other op unchanged on the same buffers, so its poses are bit-identical too.  Each
  crop's features and decoded joints are bit-identical whatever batch it runs in, and from run to run.
* fmb_kernel against the two-launch path at every width it admits that is not a multiple of 16 (24, 40, 56, 72, 88), on a
  small table built for it."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib
from oracle import port, port_ops
from oracle import port_effnet_v2_variants as V
from tests.test_gpu_forward_ops16 import (DW_NAMES, POOLS_FP32, check_conv, check_head_per_coordinate, check_se_fc,
                                          heads_reference)
from tests.test_gpu_ops16_vs_conv2d import H, POOL_SLICES, expected_class  # noqa: F401  (H: the fixture)

pytestmark = pytest.mark.gpu

SIZES = {'efficientnetv2-b0': 'v2-b0', 'efficientnetv2-b1': 'v2-b1', 'efficientnetv2-b2': 'v2-b2',
         'efficientnetv2-b3': 'v2-b3', 'efficientnetv2-xl': 'xl'}
GOLDENS = ['effnetv2b0_s224_j24.npz', 'effnetv2b3_s256_j24.npz', 'effnetv2xl_s256_j24.npz']
MODES16 = ['bf16', 'fp16']


def device_model(H, stages, last, pcfg, n_joints, sd, precision):
    """Metrabs(Sequential(PreprocLayer(), Features(stages, last)), ji): efficientnet_v2_*().features for a named table."""
    import metrabs_b200
    from metrabs_b200.backbones import efficientnet as E
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    m = Metrabs(torch.nn.Sequential(E.PreprocLayer(), E.Features(stages, last)), H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def named_model(H, name, side, n_joints, precision, calib_batch=1):
    from metrabs_b200.backbones import efficientnet as E
    pcfg = port.PathConfig(proc_side=side)
    spec = V.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, n_joints, seed=0, calib_batch=calib_batch)
    bb = getattr(E, 'efficientnet_v2_' + name.split('-')[1])()
    m = device_model(H, bb.features.stages, bb.features.last_channel, pcfg, n_joints, sd, precision)
    return pcfg, spec, sd, m


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('fname', GOLDENS)
def test_goldens_and_oracle(H, golden_dir, fname, precision):
    g = np.load(os.path.join(golden_dir, fname), allow_pickle=False)
    name, side, j, batch = str(g['name']), int(g['proc_side']), int(g['n_joints']), int(g['batch'])
    pcfg, spec, sd, m = named_model(H, name, side, j, precision, calib_batch=int(g['calib_batch']))
    crops, k = port.synthetic_inputs(batch, side, seed=int(g['seed']))
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    eng = m.engine()
    feats = eng.backbone(crops.cuda()).permute(0, 3, 1, 2)
    out = m((crops.cuda(), k.cuda()))
    e_feat, e_out = H.rel_err(feats, stages['features']), H.rel_err(out, ref)
    e_gfeat = H.rel_err(feats.reshape(batch, -1)[:, ::int(g['feature_stride'])], g['features'])
    e_gold = H.rel_err(out, g['coords3d_abs'])
    print(f'{name}@{side} [{precision}]: vs oracle features {e_feat:.2e} joints {e_out:.2e}; vs reference goldens features '
          f'{e_gfeat:.2e} joints {e_gold:.2e}; {eng.last_launch_count} launches, '
          f'{eng.backbone_flops_per_crop / 1e9:.2f} GFLOP/crop')
    assert e_feat < 1e-3 and e_out < 1e-3 and e_gfeat < 1e-3 and e_gold < 1e-3


@pytest.mark.parametrize('precision', MODES16)
@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-b0', 224, 64), ('efficientnetv2-b3', 256, 32),
                                             ('efficientnetv2-xl', 256, 8)])
def test_forward_ops_vs_conv2d(H, name, side, batch, precision):
    """test_gpu_forward_ops16.py's walk: op k's output is what debug_run_ops(crops, k + 1) stored, its operands the outputs
    of the latest ops that wrote the buffers it reads; each conv within port_ops.layer_bound, each SE fc within
    se_fc_bound, the head within the decode bound, backbone() bit-equal to the full prefix."""
    j = 8
    pcfg, spec, sd, m = named_model(H, name, side, j, precision)
    eng = m.engine()
    table = port_ops.effnet_op_table(spec)
    st = port_ops.MODES[precision][0]
    p = 8 if st == torch.bfloat16 else 11
    crops, intr = (t.cuda() for t in port.synthetic_inputs(batch, side, seed=5))
    names = eng.op_names()
    eng.profile_begin()
    eng.backbone(crops)
    eng.profile_end()
    classes = {nm: cls for nm, cls, *_ in eng.profile_op_times()}
    live, worst, fmb = {}, {}, set()
    for k, nm in enumerate(names):
        bufs, io = eng.op_buffers(k), eng.op_io(k)
        out = eng.debug_run_ops(crops, k + 1)
        assert torch.isfinite(out).all(), f'{nm} [{precision}]: {int((~torch.isfinite(out)).sum())} non-finite outputs'
        if nm.endswith('.avgpool'):  # fused pooling leaves partial slices here; fc1 is checked on their sum below
            live[bufs['output']] = out
            continue
        if nm.endswith('.fc1'):
            d = live[eng.op_buffers(k - 1)['input']]
            dk = eng.op_kernel(k - 2)
            xabs = d.abs().mean(dim=(1, 2), dtype=torch.float64)
            x_err = 2.0 ** -p * (1 + 2.0 ** -p) * xabs if dk in POOLS_FP32 else None
            kind = f'se fc1 after {DW_NAMES[dk]}'
            r = check_se_fc(sd, nm, out, d.mean(dim=(1, 2), dtype=torch.float64), xabs,
                            d.shape[1] * d.shape[2] + POOL_SLICES + 2, x_err, 'silu', precision)
        elif nm.endswith('.fc2'):
            f1 = live[bufs['input']][:, 0, 0].double()
            kind = 'se fc2'
            r = check_se_fc(sd, nm, out, f1, f1.abs(), 0, None, 'sigmoid', precision)
        else:
            op = table[nm]
            assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
            x = crops if k == 0 else live[bufs['input']]
            res = live[bufs['residual']] if bufs['residual'] != _lib.BUF_NONE else None
            sc = live[bufs['scale']][:, 0, 0] if bufs['scale'] != _lib.BUF_NONE else None
            assert (res is not None) == io['residual'] and (sc is not None) == io['scale'], nm
            if k > 0 and eng.op_is_fused_block(k - 1):
                kind = 'fmb_kernel'
                fmb.add(io['out_shape'][2])
            elif op['depthwise']:
                kind = f'dwconv_kernel/{DW_NAMES[eng.op_kernel(k)]}'
            else:
                kind = classes[nm]
            r = check_conv(lambda nm_, x_, res_, sc_: port_ops.layer_bound(sd, spec, nm_, x_, res_, sc_, precision),
                           nm, out, x, res, sc, precision)
        worst[kind] = max(worst.get(kind, 0.0), r)
        live[bufs['output']] = out
    feats = eng.backbone(crops)
    assert torch.equal(feats.float(), live[_lib.BUF_FEATURES])
    c2d, c3d = eng.head_decode(feats)
    head = {'heatmap_heads.conv_final.weight': sd['heatmap_heads.conv_final.weight'].to(st).double().cuda(),
            'heatmap_heads.conv_final.bias': sd['heatmap_heads.conv_final.bias'].float().double().cuda()}
    ref2d, ref3d = heads_reference(head, feats, pcfg, j)
    assert H.rel_err(c2d, ref2d) < 2e-4 and H.rel_err(c3d, ref3d) < 2e-4
    worst['head 2D'], worst['head 3D'] = check_head_per_coordinate(head, feats, pcfg, c2d, c3d, tc32=False, n_joints=j)
    assert fmb == {cin for cin, _ in V.identity_fused_blocks(spec)}, fmb
    del live, out, feats
    torch.cuda.empty_cache()
    ratios = ', '.join(f'{kd}: {v:.3f}' for kd, v in sorted(worst.items()))
    print(f'{name}@{side} x{batch} [{precision}]: {len(names)} ops, fused block widths {sorted(fmb)}; '
          f'worst |dev-ref|/tol {{{ratios}}}')


def fused_blocks_bit_equal(eng, crops):
    """-> {Cin: count} of the fused blocks; each one's output on the forward (fmb_kernel) is bit-equal to the expand and
    the projection launched one after the other on the forward's own block input, and to debug_run_fused_block."""
    widths = {}
    names = eng.op_names()
    for i in range(len(names) - 1):
        if not eng.op_is_fused_block(i):
            continue
        x = eng.debug_run_ops(crops, i)  # the previous block's output: this block's input and residual
        assert tuple(x.shape[1:]) == eng.op_io(i)['in_shape'], names[i]
        fused = eng.debug_run_ops(crops, i + 2)
        res = x if eng.op_io(i + 1)['residual'] else None
        two = eng.debug_run_op(i + 1, eng.debug_run_op(i, x), res)
        assert torch.equal(fused, two), (names[i], int((fused != two).sum()))
        assert torch.equal(eng.debug_run_fused_block(i, x), two), names[i]
        cin = eng.op_io(i)['in_shape'][2]
        widths[cin] = widths.get(cin, 0) + 1
    return widths


@pytest.mark.parametrize('precision', MODES16)
@pytest.mark.parametrize('name,widths', [('efficientnetv2-b2', {32: 2, 56: 2}), ('efficientnetv2-b3', {40: 2, 56: 2})])
def test_fused_40_and_56_channel_blocks(H, name, widths, precision):
    side, j, batch = 256, 8, 24
    _pcfg, spec, _sd, m = named_model(H, name, side, j, precision)
    eng = m.engine()
    names = eng.op_names()
    # every identity-shaped FusedMBConv block with an expand conv is fused, and only those
    expect = {f'backbone.1.{b["key"]}.block.0' for b in port.effnet_block_list(spec)
              if b['block'] == 'fused' and b['expand'] != 1 and b['stride'] == 1 and b['cin'] == b['cout']}
    assert {names[i] for i in range(len(names)) if eng.op_is_fused_block(i)} == expect
    crops, intr = (t.cuda() for t in port.synthetic_inputs(batch, side, seed=9))
    assert fused_blocks_bit_equal(eng, crops) == widths
    # one fmb_kernel launch per fused block on the forward
    eng.profile_begin()
    eng.backbone(crops)
    prof = eng.profile_end()
    assert prof['fmb_kernel']['launches'] == sum(widths.values()), prof.get('fmb_kernel')
    # run to run, and each crop whatever batch it runs in: features and decoded joints bit-identical
    o1, o2 = m((crops, intr)).clone(), m((crops, intr)).clone()
    assert torch.equal(o1, o2) and torch.isfinite(o1).all()
    full = eng.backbone(crops).clone()
    c2d, c3d = (t.clone() for t in eng.head_decode(full))
    for sub in [slice(0, 1), slice(7, 8), slice(0, 5), slice(5, 24), slice(3, 20), slice(23, 24)]:
        f = eng.backbone(crops[sub].contiguous())
        assert torch.equal(f, full[sub]), (name, precision, sub)
        a2, a3 = eng.head_decode(f)
        assert torch.equal(a2, c2d[sub]) and torch.equal(a3, c3d[sub]), (name, precision, sub)
    print(f'{name} [{precision}]: fused blocks {widths} bit-equal to the two-launch path on the forward; '
          f'batch invariance over 6 sub-batches of {batch} crops')


@pytest.mark.parametrize('precision', MODES16)
def test_fused_block_at_every_width_off_16(H, precision):
    """Identity-shaped FusedMBConv blocks of 24, 40, 56, 72 and 88 channels (one and two 64-channel k-chunks, BN2 32, 64 and
    128, partial last expand chunks at Cexp 96, 160, 224, 288 and 352), on 64x64, 32x32 and 16x16 maps with three crops."""
    f, mb = 'fused', 'mb'
    rows = [(f, 1, 3, 1, 24, 24, 1), (f, 4, 3, 1, 24, 24, 1), (f, 4, 3, 2, 24, 40, 2), (f, 4, 3, 1, 40, 56, 2),
            (f, 4, 3, 2, 56, 72, 2), (f, 4, 3, 1, 72, 88, 2), (mb, 4, 3, 2, 88, 96, 1), (mb, 6, 3, 2, 96, 128, 1, True)]
    spec = port.EffNetSpec('fmb-widths', [port.StageSpec(*r) for r in rows], last_channel=64)
    pcfg = port.PathConfig(proc_side=128)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    stages = [dict(block=s.block, expand=s.expand, kernel=s.kernel, stride=s.stride, cin=s.cin, cout=s.cout,
                   layers=s.layers, bottomright=s.bottomright, dilation_in=1, dilation_out=1) for s in spec.stages]
    eng = device_model(H, stages, 64, pcfg, 8, sd, precision).engine()
    crops = port.synthetic_inputs(3, 128, seed=2)[0].cuda()
    widths = fused_blocks_bit_equal(eng, crops)
    assert widths == {24: 1, 40: 1, 56: 1, 72: 1, 88: 1}, widths
    g = torch.Generator().manual_seed(4)
    st = port_ops.MODES[precision][0]
    for i in range(len(eng.op_names()) - 1):  # and on random 16-bit inputs in isolation, batch 1 and 5
        if eng.op_is_fused_block(i):
            for b in (1, 5):
                x = torch.randn((b,) + eng.op_io(i)['in_shape'], generator=g).to(st).float().cuda()
                two = eng.debug_run_op(i + 1, eng.debug_run_op(i, x), x)
                assert torch.equal(eng.debug_run_fused_block(i, x), two), (eng.op_names()[i], b)
    print(f'[{precision}] fused blocks {widths} bit-equal to the two-launch path')
