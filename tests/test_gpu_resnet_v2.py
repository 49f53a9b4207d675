"""GPU: the pre-activation ResNet-50, -101 and -152 (V2, metrabs_b200.backbones.resnet.resnet{50,101,152}v2) against this
build's torch restatement of the Keras code (oracle/port_resnet_v2.py; parity is "this build's restatement vs this build's
kernels", the reference has no test, golden or importable implementation of these backbones).

* fp32 and tf32x3: every layer within 1e-4 of the restatement on the restatement's own operands, features and joints within
  1e-3 (5e-3 for the joints of ResNet-152 V2, see below), at output strides 32 and 8 and once without the centered stride;
  the engine's FLOPs per crop equal the restatement's count.
* bf16, bf16_simt, fp16, fp16_simt: every distinct op element by element against fp64 conv2d at the mode's rounding
  points (port_resnet_v2.layer_bound, port_ops.check_bound), its kernel asserted: the _3_convs that run fused with the
  pre-activation behind them on tc_conv_preact_kernel, the other GEMMs on tc_conv_kernel in the tensor-core modes, the
  pre-activations on dwconv_kernel, the shortcut subsample on maxpool_kernel, exactly.  ResNet-101 and -152 V2 have the
  same distinct op shapes as ResNet-50 V2, so ResNet-50 V2 covers them.
* every fused _3_conv + pre-activation pair torch.equal to its two separate launches, at batches whose GEMM has an M tail;
* per-crop batch invariance of ResNet-50 V2 (test_gpu_batch_invariance.py's sub-batches);
* a 16-bit end-to-end forward of each depth with finite joints."""
import dataclasses

import pytest
import torch

from metrabs_b200 import _lib
from oracle import port, port_ops, port_resnet_v2
from oracle import port_tf_backbones as tfb
from tests.test_gpu_batch_invariance import first_differing_op, sub_batches
from tests.test_gpu_ops16_vs_conv2d import MODES, expected_class, op_classes, operands

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def device_model(H, depth, pcfg, n_joints, sd, precision='fp32'):
    import metrabs_b200
    from metrabs_b200.backbones import resnet
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    m = Metrabs(getattr(resnet, f'resnet{depth}v2')(), H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def layer_operands(spec, tap, crops):
    """op name -> (input NCHW, residual NCHW or None), taken from the restatement's own tensors"""
    p = 'backbone.'
    ops = {p + 'conv1_conv': (crops, None), p + 'pool1_pool': (tap[p + 'conv1_conv'], None)}
    x = tap[p + 'pool1_pool']
    for b in port_resnet_v2.resnet_v2_blocks(spec.cfg, spec.depth):
        n = p + b['name']
        pre = tap[n + '_preact_bn']
        ops[n + '_preact_bn'] = (x, None)
        if b['conv_shortcut']:
            ops[n + '_0_conv'] = (pre, None)
            sc = tap[n + '_0_conv']
        elif b['subsample']:
            ops[n + '_shortcut_pool'] = (x, None)
            sc = tap[n + '_shortcut_pool']
        else:
            sc = x
        ops[n + '_1_conv'] = (pre, None)
        ops[n + '_2_conv'] = (tap[n + '_1_conv'], None)
        ops[n + '_3_conv'] = (tap[n + '_2_conv'], sc)
        x = tap[n + '_3_conv']
    ops[p + 'post_bn'] = (x, None)
    return ops


PARITY = [(d, dict(proc_side=256, stride_test=32, depth=8)) for d in (50, 101, 152)]
PARITY += [(d, dict(proc_side=256, stride_test=8, depth=32)) for d in (50, 101, 152)]
PARITY += [(50, dict(proc_side=256, stride_test=32, depth=8, centered_stride=False))]


@pytest.mark.parametrize('depth,cfgkw', PARITY)
def test_resnet_v2_fp32_and_tf32x3(H, depth, cfgkw):
    j, batch = 24, 2
    pcfg = port.PathConfig(**cfgkw)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, depth)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
    tap, stages = {}, {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    for precision in ('fp32', 'tf32x3'):
        m = device_model(H, depth, pcfg, j, sd, precision)
        eng = m.engine()
        names = eng.op_names()
        assert set(names) == set(tap)
        assert abs(eng.backbone_flops_per_crop / 1e9 - port_resnet_v2.gflop_per_crop(pcfg, depth)) < 1e-9
        ops = layer_operands(spec, tap, crops)
        nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).cuda()  # noqa: E731
        bad = []
        for i, name in enumerate(names):
            x, res = ops[name]
            out = eng.debug_run_op(i, x.cuda() if i == 0 else nhwc(x), nhwc(res)).permute(0, 3, 1, 2).cpu()
            err = port.relative_error(out, tap[name])
            if not err < 1e-4:
                bad.append((name, err))
        assert not bad, f'{precision}: first diverging layers: {bad[:5]}'
        out = m((crops.cuda(), k.cuda()))
        e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
        e_out = H.rel_err(out, ref)
        print(f'resnet{depth}v2 {cfgkw} [{precision}]: features {e_feat:.2e}, joints {e_out:.2e}, '
              f'{eng.backbone_flops_per_crop / 1e9:.2f} GFLOP/crop, {eng.last_launch_count} launches')
        # ResNet-152 V2: as for ResNet-152 V1 (test_gpu_resnet_family.py), every layer is within 1e-4 on its own and the
        # features within 1e-3, but two fp32 evaluations drift apart over its 155 convs and the peaked soft-argmax of the
        # head amplifies that in the joints
        assert e_feat < 1e-3 and e_out < (5e-3 if depth == 152 else 1e-3)
        del m, eng
        torch.cuda.empty_cache()


def pair_ops(eng):
    return {i for i in range(len(eng.op_names()) - 1) if eng.op_is_preact_pair(i)}


@pytest.mark.parametrize('side,stride,centered,batch', [(256, 8, True, 2), (256, 32, False, 3), (224, 32, True, 3)])
def test_resnet_v2_ops16_vs_conv2d(H, side, stride, centered, batch):
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, centered_stride=centered, depth=8)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, 50)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    table = port_resnet_v2.op_table(spec)
    for precision in MODES:
        eng = device_model(H, 50, pcfg, 8, sd, precision).engine()
        classes = op_classes(eng, side)
        pairs = pair_ops(eng)
        names = eng.op_names()
        tc = precision in ('bf16', 'fp16')
        # the fused pairs: every _3_conv and the pre-activation behind it, in the tensor-core modes only
        assert {names[i] for i in pairs} == ({n for n in names if n.endswith('_3_conv')} if tc else set())
        st = port_ops.MODES[precision][0]
        g = torch.Generator().manual_seed(stride)
        seen, feats = set(), set()
        for i, nm in enumerate(names):
            op, io = table[nm], eng.op_io(i)
            sig = (io['in_shape'], io['out_shape'], io['residual'], op['stride'], op['shift'], op['dil'], op['act'],
                   op['kernel'], op['maxpool'], op['stem'], op['depthwise'], i in pairs)
            if sig in seen:
                continue
            seen.add(sig)
            want = {'tc_conv_preact_kernel'} if i in pairs else expected_class(op, io, precision)
            assert classes[nm] in want, (nm, classes[nm], want)
            if nm.endswith(('_preact_bn', 'post_bn')):
                assert eng.op_kernel(i) == _lib.DW_GENERIC
            if nm.endswith('_shortcut_pool'):
                assert eng.op_kernel(i) == _lib.MAXPOOL
            feats |= {classes[nm], ('dil', op['dil']), ('shift', op['shift'])}
            x, res, _ = operands(io, batch, st, g, i == 0)
            out = eng.debug_run_op(i, x, res)
            ref, tol = port_resnet_v2.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), precision)
            assert out.shape == ref.shape, (nm, tuple(out.shape), tuple(ref.shape))
            if op['maxpool']:
                assert torch.equal(out.double().cpu(), ref.cpu()), nm
            r, bad = port_ops.check_bound(out, ref, tol, precision)
            assert bad == 0, f'{nm} [{precision}]: {bad} elements outside the bound (worst |dev-ref|/tol {r:.2f})'
        assert {'dwconv_kernel', 'other', 'stem_conv_kernel'} <= feats
        assert ('tc_conv_preact_kernel' in feats) == tc and ('tc_conv_kernel' in feats) == tc
        if stride == 8:
            assert ('dil', 2) in feats and ('dil', 4) in feats
        assert (('shift', 1) in feats) == centered
        print(f'resnet50v2@{side} s{stride} centered={centered} [{precision}]: {len(seen)} distinct ops')
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize('side,stride,batch', [(224, 32, 3), (224, 32, 5), (256, 8, 3)])
def test_fused_pair_equals_two_launches(H, side, stride, batch):
    """tc_conv_preact_kernel's two outputs are bit-identical to tc_conv_kernel then dwconv_kernel; at side 224 the 7x7 and
    14x14 maps give GEMMs with a partial last row tile (batch * 49 or * 196 rows)"""
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, depth=8)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, 50)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    tails = 0
    for precision in ('bf16', 'fp16'):
        eng = device_model(H, 50, pcfg, 8, sd, precision).engine()
        st = port_ops.MODES[precision][0]
        g = torch.Generator().manual_seed(batch)
        pairs = sorted(pair_ops(eng))
        assert len(pairs) == 16
        for i in pairs:
            # the pre-activation is stored while later tiles of the GEMM still read its input and residual
            a, b = eng.op_buffers(i), eng.op_buffers(i + 1)
            assert b['input'] == a['output'] and b['output'] not in (a['input'], a['residual'], a['output']), (a, b)
            io = eng.op_io(i)
            x, res, _ = operands(io, batch, st, g, False)
            y, z = eng.debug_run_preact_pair(i, x, res)
            y_sep = eng.debug_run_op(i, x, res)
            z_sep = eng.debug_run_op(i + 1, y_sep)
            assert torch.equal(y, y_sep) and torch.equal(z, z_sep), (eng.op_names()[i], precision)
            tails += batch * io['out_shape'][0] * io['out_shape'][1] % 128 != 0
        del eng
        torch.cuda.empty_cache()
    assert (tails > 0) == (side == 224)


@pytest.mark.parametrize('precision', ['bf16', 'fp16', 'fp32'])
def test_resnet50v2_batch_invariance(H, precision):
    n, side = 64, 224
    pcfg = port.PathConfig(proc_side=side, stride_test=32, depth=8)
    sd = tfb.make_state_dict(port_resnet_v2.ResNetV2Spec(pcfg, 50), pcfg, 24, seed=0, calib_batch=1)
    eng = device_model(H, 50, pcfg, 24, sd, precision).engine()
    crops = port.synthetic_inputs(n, side, seed=11)[0].cuda()
    feats = eng.backbone(crops)
    c2d, c3d = eng.head_decode(feats)
    assert all(torch.isfinite(t).all() for t in (feats, c2d, c3d))
    bad = []
    for s, e in sub_batches(n):
        f = eng.backbone(crops[s:e])
        a2, a3 = eng.head_decode(f)
        if not (torch.equal(f, feats[s:e]) and torch.equal(a2, c2d[s:e]) and torch.equal(a3, c3d[s:e])):
            bad.append(f'[{s}, {e}): {first_differing_op(eng, crops, s, e)}')
    assert not bad, bad[:4]


@pytest.mark.parametrize('depth', [50, 101, 152])
def test_resnet_v2_16bit_end_to_end(H, depth):
    j, batch = 24, 4
    pcfg = port.PathConfig(proc_side=256, stride_test=8, depth=32)
    spec = port_resnet_v2.ResNetV2Spec(pcfg, depth)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=1)
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k)
    for precision in ('bf16', 'fp16'):
        m = device_model(H, depth, pcfg, j, sd, precision)
        out = m((crops.cuda(), k.cuda()))
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        print(f'resnet{depth}v2 s8 [{precision}]: joints rel err vs fp32 restatement {H.rel_err(out, ref):.2e}, '
              f'{m.engine().last_launch_count} launches')
        del m
        torch.cuda.empty_cache()
