"""GPU: every distinct op of ResNet-50 and MobileNetV3-small in the four 16-bit modes ('bf16', 'fp16' on the tensor cores,
'bf16_simt', 'fp16_simt' on CUDA cores), the depthwise kernels at batch sizes around their crop group, and fp16 overflow,
element by element against fp64 conv2d at the mode's rounding points (oracle/port_ops.py: layer_bound / check_bound).

Each test asserts what it reached: the kernel class of every checked op (Engine.profile_op_times over one forward), the
depthwise kernel (TMA-staged / strip / generic, restated from choose_dw_kernel in csrc/engine.cu with mtb_debug_dw_plan),
and the epilogues only these backbones have: residual before ReLU, hard-swish, dilation > 1, the bottom-right shift.

The squeeze-excitation fc ops are checked on the device's own forward (debug_run_ops), where the TMA and strip depthwise
kernels also write the partial pooling slices that fc1 sums: fc1 against act(W1 mean(D) + b1) in fp64 on the depthwise
output D the device stored, fc2 against act(W2 F1 + b2) on the fc1 output F1 it produced.  The fused pooling sums the
fp32 activations before they are rounded to 16 bits (dw_tma.cuh, dwconv3x3_pool_16b_kernel), so its mean may differ from
mean(D) by half an output ulp per element on top of the fp32 summation; the separate pool kernel averages D itself."""
import ctypes as C

import pytest
import torch

from oracle import port, port_ops
from oracle import port_tf_backbones as tfb

pytestmark = pytest.mark.gpu

MODES = ['bf16', 'bf16_simt', 'fp16', 'fp16_simt']
POOL_SLICES = 8  # kPoolSlices (csrc/engine.cu)


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def dw_plan(h, w):
    """mtb_debug_dw_plan -> (crops per item G, rows per item, row bands); G = 0 when no TMA plan fits."""
    from metrabs_b200 import _lib
    g, bh, nrb, sb = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    assert _lib.lib().mtb_debug_dw_plan(h, w, C.byref(g), C.byref(bh), C.byref(nrb), C.byref(sb)) == 0
    return g.value, bh.value, nrb.value


def dw_kernel(op, io, precision):
    """choose_dw_kernel (csrc/engine.cu): 'tma' | 'strip' | 'generic'."""
    (hin, win, c), (hout, wout, _) = io['in_shape'], io['out_shape']
    strip = op['kernel'] == 3 and op['dil'] == 1 and c % 8 == 0 and op['stride'] in (1, 2) and op['act'] is not None
    if not strip or precision not in ('bf16', 'fp16'):
        return 'generic'
    if op['stride'] == 1 and (hin, win) == (hout, wout):
        g, _bh, nrb = dw_plan(hout, wout)
        if g and nrb <= POOL_SLICES:
            return 'tma'
    return 'strip'


def expected_class(op, io, precision):
    if op['maxpool']:
        return {'other'}
    if op['stem']:
        return {'stem_conv_kernel'}
    if op['depthwise']:
        return {'dwconv_kernel'}
    if precision in ('bf16', 'fp16') and port_ops.tc_eligible(op, io['in_shape'][2], io['out_shape'][2]):
        return {'tc_conv_kernel', 'fmb_kernel'}
    return {'conv_igemm_kernel'}


def op_classes(eng, side, batch=2):
    """op name -> kernel class, from a profiled forward."""
    eng.profile_begin()
    eng.backbone(port.synthetic_inputs(batch, side, seed=9)[0].cuda())
    eng.profile_end()
    return {nm: cls for nm, cls, *_ in eng.profile_op_times()}


def operands(io, batch, st, g, first):
    if first:  # the stem takes NCHW crops in [0, 1]
        x = torch.rand((batch, 3) + io['in_shape'][:2], generator=g)
    else:
        x = torch.randn((batch,) + io['in_shape'], generator=g).to(st).float()
    res = torch.randn((batch,) + io['out_shape'], generator=g).to(st).float() if io['residual'] else None
    sc = torch.rand(batch, io['in_shape'][2], generator=g) if io['scale'] else None
    return tuple(t.cuda() if t is not None else None for t in (x, res, sc))


def check_op(eng, sd, spec, i, nm, x, res, sc, precision):
    out = eng.debug_run_op(i, x, res, sc)
    ref, tol = port_ops.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), sc, precision)
    assert out.shape == ref.shape, (nm, tuple(out.shape), tuple(ref.shape))
    worst, bad = port_ops.check_bound(out, ref, tol, precision)
    assert bad == 0, f'{nm} [{precision}] batch {x.shape[0]}: {bad} elements outside the bound (worst |dev-ref|/tol {worst:.2f})'
    return worst, out, ref


def check_all_ops(H, eng, sd, spec, side, precision, batch, seed):
    """every distinct op (stems and max pool included) -> (ops checked, features seen, worst ratio per kernel)"""
    table = port_ops.op_table(spec)
    classes = op_classes(eng, side)
    st = port_ops.MODES[precision][0]
    g = torch.Generator().manual_seed(seed)
    seen, feats, worst = set(), set(), {}
    for i, nm in enumerate(eng.op_names()):
        if nm not in table:  # squeeze-excitation pool / fc ops
            continue
        op, io = table[nm], eng.op_io(i)
        sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], op['stride'], op['shift'], op['dil'], op['act'],
               op['kernel'], op['depthwise'], op['maxpool'], op['stem'], op.get('res_first'))
        if sig in seen:
            continue
        seen.add(sig)
        assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
        kind = classes[nm] + ('/' + dw_kernel(op, io, precision) if op['depthwise'] else '')
        feats |= {kind, ('act', op['act']), ('dil', op['dil']), ('shift', op['shift']), ('res_first', op.get('res_first'))}
        r, _out, _ref = check_op(eng, sd, spec, i, nm, *operands(io, batch, st, g, i == 0), precision)
        worst[kind] = max(worst.get(kind, 0.0), r)
    return seen, feats, worst


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('side,stride,centered,batch', [(256, 8, True, 2), (256, 16, False, 3), (224, 32, True, 2)])
def test_resnet50_ops_vs_conv2d(H, precision, side, stride, centered, batch):
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, centered_stride=centered, depth=8)
    spec = tfb.ResNet50Spec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model_tf('resnet50', pcfg, 8, sd, precision=precision).engine()
    seen, feats, worst = check_all_ops(H, eng, sd, spec, side, precision, batch, seed=stride)
    assert ('res_first', True) in feats and 'other' in feats and 'stem_conv_kernel' in feats
    if stride < 32:
        assert ('dil', 2) in feats
    if centered:
        assert ('shift', 1) in feats
    print(f'resnet50@{side} s{stride} centered={centered} [{precision}]: {len(seen)} ops, worst |dev-ref|/tol {worst}')


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('side,batch', [(256, 4), (224, 3)])
def test_mobilenetv3_small_ops_vs_conv2d(H, precision, side, batch):
    pcfg = port.PathConfig(proc_side=side, stride_test=32, depth=8)
    spec = tfb.MobileNetV3SmallSpec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model_tf('mobilenetv3-small', pcfg, 8, sd, precision=precision).engine()
    seen, feats, worst = check_all_ops(H, eng, sd, spec, side, precision, batch, seed=side)
    assert ('act', 'hswish') in feats and ('act', 'relu') in feats and ('shift', 1) in feats
    assert 'dwconv_kernel/generic' in feats  # the 5x5 depthwise convs
    if precision in ('bf16', 'fp16'):
        assert 'dwconv_kernel/strip' in feats and 'tc_conv_kernel' in feats
    print(f'mobilenetv3-small@{side} [{precision}]: {len(seen)} ops, worst |dev-ref|/tol {worst}')


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_depthwise_around_the_crop_group(H, precision):
    """The TMA-staged depthwise kernel groups G crops per work item (dw_tma_plan); batches 1, G-1, G+1 and 2G+1 leave a
    ragged last group.  EfficientNetV2-S@224 has 28x28 / 14x14 / 7x7 depthwise maps (odd sizes, not multiples of the
    4-wide strips), stride-2 ones on the strip kernel, bottom-right shift included."""
    side = 224
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec('efficientnetv2-s')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model('efficientnetv2-s', pcfg, 8, sd, precision=precision).engine()
    table = port_ops.effnet_op_table(spec)
    st = port_ops.MODES[precision][0]
    g = torch.Generator().manual_seed(12)
    seen, kinds, worst = set(), set(), {}
    for i, nm in enumerate(eng.op_names()):
        if nm not in table or not table[nm]['depthwise']:
            continue
        op, io = table[nm], eng.op_io(i)
        sig = (io['in_shape'], io['out_shape'], op['stride'], op['shift'])
        if sig in seen:
            continue
        seen.add(sig)
        kind = dw_kernel(op, io, precision)
        kinds.add(kind)
        G = dw_plan(*io['out_shape'][:2])[0] if kind == 'tma' else 4
        for batch in sorted({1, max(G - 1, 1), G + 1, 2 * G + 1}):
            r = check_op(eng, sd, spec, i, nm, *operands(io, batch, st, g, False), precision)[0]
            worst[kind] = max(worst.get(kind, 0.0), r)
    assert kinds == {'tma', 'strip'}, kinds
    assert any(s[3] == 1 for s in seen) and any(s[0][0] % 2 for s in seen)  # bottom-right shift; an odd map
    print(f'efficientnetv2-s@{side} depthwise [{precision}]: {len(seen)} ops, worst |dev-ref|/tol {worst}')


def se_fc_key(sd, nm):
    """weight key prefix of an SE fc op: EfficientNet '<se>.fc1|fc2', MobileNetV3 '<se>.Conv|Conv_1'."""
    if nm + '.weight' in sd:
        return nm
    return nm[:-len('.fc1')] + ('.Conv' if nm.endswith('.fc1') else '.Conv_1')


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('model,side,batch', [
    ('efficientnetv2-tiny', 320, 2),   # 20x20 depthwise: TMA row bands of 12 + 8 rows (two pooling slices)
    ('efficientnetv2-tiny', 224, 5),   # 7x7 depthwise: TMA crop groups of 4, the last holding 1 crop
    ('mobilenetv3-small', 224, 3)])    # ReLU / hard-sigmoid SE; strip (3x3) and generic (5x5) depthwise + separate pool
def test_fused_se_squeeze_on_the_forward(H, precision, model, side, batch):
    if model == 'mobilenetv3-small':
        pcfg = port.PathConfig(proc_side=side, stride_test=32, depth=8)
        spec = tfb.MobileNetV3SmallSpec(pcfg)
        sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
        eng = H.device_model_tf(model, pcfg, 8, sd, precision=precision).engine()
        acts = ('relu', 'hsigmoid')
    else:
        pcfg = port.PathConfig(proc_side=side)
        spec = port.effnet_spec(model)
        sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
        eng = H.device_model(model, pcfg, 8, sd, precision=precision).engine()
        acts = ('silu', 'sigmoid')
    table = port_ops.op_table(spec)
    names = eng.op_names()
    crops = port.synthetic_inputs(batch, side, seed=14)[0].cuda()
    reached, worst = set(), {}
    for i, nm in enumerate(names):
        if not nm.endswith('.avgpool'):
            continue
        dw = names[i - 1]
        io = eng.op_io(i - 1)
        hh, ww, c = io['out_shape']
        kind = dw_kernel(table[dw], io, precision)
        if kind == 'tma':
            G, BH, nrb = dw_plan(hh, ww)
            if nrb > 1 and hh % BH:
                reached.add('ragged row band')
            if G > 1 and batch % G:
                reached.add('ragged crop group')
        reached.add(kind)
        d = eng.debug_run_ops(crops, i).double()                     # the depthwise output the device stored
        f1 = eng.debug_run_ops(crops, i + 2)[:, 0, 0].double()       # fc1 on the fused (or separate) pooling
        f2 = eng.debug_run_ops(crops, i + 3)[:, 0, 0].double()       # fc2 on that fc1 output
        p = 8 if port_ops.MODES[precision][0] == torch.bfloat16 else 11
        fused = kind != 'generic'  # choose_dw_kernel: the TMA and strip kernels pool; fc1 then sums their slices
        pool_err = 2.0 ** -p * (1 + 2.0 ** -p) * d.abs().mean(dim=(1, 2)) if fused else None
        for j, (x, xabs, n_in, x_err, dev, act) in enumerate([
                (d.mean(dim=(1, 2)), d.abs().mean(dim=(1, 2)), hh * ww + POOL_SLICES + 2, pool_err, f1, acts[0]),
                (f1, f1.abs(), 0, None, f2, acts[1])]):
            key = se_fc_key(sd, names[i + 1 + j])
            w, b = sd[key + '.weight'], sd[key + '.bias']
            n_real = w.shape[0]
            ref, tol = port_ops.se_fc_bound(x[:, :w.shape[1]], xabs[:, :w.shape[1]], n_in, w, b, act,
                                            None if x_err is None else x_err[:, :w.shape[1]])
            err = (dev[:, :n_real] - ref).abs()
            r = float((err / tol).max())
            assert bool((err <= tol).all()), f'{names[i + 1 + j]} [{precision}] after {kind} depthwise: |dev-ref|/tol {r:.2f}'
            assert not dev[:, n_real:].any()  # hidden channels zero-padded to a multiple of 4
            worst[f'{kind}/fc{j + 1}'] = max(worst.get(f'{kind}/fc{j + 1}', 0.0), r)
    if model == 'mobilenetv3-small':
        assert 'generic' in reached and (precision.endswith('simt') or 'strip' in reached), reached
    elif precision in ('bf16', 'fp16'):
        assert {'tma', 'strip', 'ragged row band' if side == 320 else 'ragged crop group'} <= reached, reached
    print(f'{model}@{side} x{batch} SE [{precision}]: worst |dev-ref|/tol {worst}')


@pytest.mark.parametrize('precision', ['fp16', 'fp16_simt'])
def test_fp16_overflow_gives_inf(H, precision):
    """Outputs past 65504 round to +-inf (no saturation) and nothing becomes NaN: tc_conv_kernel and the TMA / strip
    depthwise kernels in 'fp16', conv_igemm_kernel and the generic depthwise kernel in 'fp16_simt'; fmb_kernel below."""
    side = 224
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec('efficientnetv2-s')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model('efficientnetv2-s', pcfg, 8, sd, precision=precision).engine()
    names = eng.op_names()
    table = port_ops.effnet_op_table(spec)
    classes = op_classes(eng, side)
    g = torch.Generator().manual_seed(13)
    tc = precision == 'fp16'
    picked = [('backbone.1.4.1.block.0', 'tc_conv_kernel' if tc else 'conv_igemm_kernel', None),  # 1x1 expand + SiLU, 14x14
              ('backbone.1.4.1.block.1', 'dwconv_kernel', 'tma' if tc else 'generic'),             # depthwise 3x3, 14x14
              ('backbone.1.4.0.block.1', 'dwconv_kernel', 'strip' if tc else 'generic')]           # depthwise 3x3 s2, 28 -> 14
    for nm, cls, dwk in picked:
        i = names.index(nm)
        io = eng.op_io(i)
        assert classes[nm] == cls, (nm, classes[nm])
        assert dwk is None or dw_kernel(table[nm], io, precision) == dwk
        x, res, sc = operands(io, 3, torch.float16, g, False)
        ref = port_ops.conv_layer_reference(sd, spec, nm, x.double(), None if res is None else res.double(), sc, precision)
        k = 4 * 65520 / float(ref.abs().max())  # the largest outputs land at ~4x the overflow threshold
        x = (x * k).clamp(-60000, 60000).half().float()
        r, out, ref = check_op(eng, sd, spec, i, nm, x, res, sc, precision)
        n_inf = int(torch.isinf(out).sum())
        assert 0 < n_inf < out.numel() and not torch.isnan(out).any(), (nm, n_inf)
        print(f'{nm} [{precision}] {cls} {dwk or ""}: {n_inf} of {out.numel()} outputs inf, worst |dev-ref|/tol {r:.3g}')


def test_fp16_overflow_in_the_fused_block(H):
    """fmb_kernel: the projection of a FusedMBConv block overflows while its expanded intermediate stays finite (the
    projection's BN gain is raised so that its largest outputs land at ~4x the overflow threshold).  The fused output is
    checked against the projection's bound on the unfused path's fp16 intermediate, which the fused kernel reproduces bit
    for bit (same MMA order and rounding: test_gpu_f16.py::test_f16_fused_block_is_bit_equal_to_two_launches)."""
    side, batch = 224, 3
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec('efficientnetv2-s')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    nm, proj = 'backbone.1.2.1.block.0', 'backbone.1.2.1.block.1'
    eng = H.device_model('efficientnetv2-s', pcfg, 8, sd, precision='fp16').engine()
    i = eng.op_names().index(nm)
    assert eng.op_is_fused_block(i)
    x = operands(eng.op_io(i), batch, torch.float16, torch.Generator().manual_seed(15), False)[0]
    mid = eng.debug_run_op(i, x)
    gain = 4 * 65520 / float(port_ops.conv_layer_reference(sd, spec, proj, mid.double(), precision='fp16').abs().max())
    sd[proj + '.1.weight'] = sd[proj + '.1.weight'] * gain
    sd[proj + '.1.bias'] = sd[proj + '.1.bias'] * gain
    eng = H.device_model('efficientnetv2-s', pcfg, 8, sd, precision='fp16').engine()
    assert eng.op_is_fused_block(i)
    out = eng.debug_run_fused_block(i, x)
    assert torch.equal(eng.debug_run_op(i, x), mid) and torch.isfinite(mid).all()
    ref, tol = port_ops.layer_bound(sd, spec, proj, mid.double(), x.double(), None, 'fp16')
    r, bad = port_ops.check_bound(out, ref, tol, 'fp16')
    n_inf = int(torch.isinf(out).sum())
    assert bad == 0, (bad, r)
    assert 0 < n_inf < out.numel() and not torch.isnan(out).any(), n_inf
    print(f'{nm} fmb_kernel [fp16]: {n_inf} of {out.numel()} outputs inf, worst |dev-ref|/tol {r:.3g}')
