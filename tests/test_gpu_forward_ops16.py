"""GPU: every op of the benchmarked 16-bit forwards ('bf16', 'fp16') against fp64 conv2d, at the benchmark batch, on the
tensors the forward itself produced.

The per-op tests elsewhere run one op in isolation (mtb_debug_run_op: its own buffers, no fused SE pooling, a few crops).
Here each backbone op k of the forward is checked on the forward's own code path: its output is what
``debug_run_ops(crops, k + 1)`` stored (the real prefix: the planner's buffers, the depthwise kernels that pool for
squeeze-excitation (SE), the fused FusedMBConv blocks, the SE scale that fc2 computed applied in the projection GEMM or by
se_scale_kernel), and its input, residual and SE scale are the outputs of the latest earlier ops that wrote the buffers it
reads (Engine.op_buffers).  Those stay cached while they are live, so every prefix runs once.

* conv ops, stem and max pool: element by element within the family's per-layer bound on those exact 16-bit operands,
  over all crops (port_ops.layer_bound, port_effnet_dilated.dw_layer_bound, port_effnet_b.layer_bound,
  port_mobilenet.layer_bound; port_ops.check_bound), the fp64 reference on the device in crop chunks.
* fused FusedMBConv blocks: a prefix that stops after the expand runs it unfused; the block output, from fmb_kernel, is
  checked against the projection's bound on that unfused intermediate (as test_gpu_ops16_vs_conv2d.py's overflow test).
* SE fc1 / fc2: port_ops.se_fc_bound on the depthwise output and fc1 output the forward stored, as
  test_gpu_ops16_vs_conv2d.py::test_fused_se_squeeze_on_the_forward.
* every stored tensor finite; head_decode on the forward's features against port.heads with the head weight rounded to
  the mode's type (2e-4, the bar of test_gpu_tc.py::test_fused_head_vs_oracle) and every coordinate within
  port_ops.decode_bound; backbone() bit-equal to the full prefix;
  three forward() calls on the same buffers (eager run, graph capture, graph replay) give identical joints.
* what each configuration reached is asserted (kernel classes, depthwise and tensor-core kernels, SE projection widths),
  and the worst |dev-ref|/tol per kernel kind and the wall time are printed."""
import time

import pytest
import torch

from metrabs_b200 import _lib
from oracle import port, port_effnet_b, port_mobilenet, port_ops
from oracle import port_effnet_dilated as D
from oracle import port_tf_backbones as tfb
from tests.test_gpu_ops16_vs_conv2d import H, POOL_SLICES, dw_plan, expected_class, se_fc_key  # noqa: F401  (H: the fixture)

pytestmark = pytest.mark.gpu

J = 8  # joints of the head, except where JOINTS says otherwise
JOINTS = {'efficientnetv2-s-j122': 122}  # c4: 122 joints, 1098 head channels = 9 M tiles of 128, the last one ragged
CHUNK = 1 << 25  # elements per crop chunk of the fp64 reference (input or output, whichever is larger)
DW_NAMES = {_lib.DW_GENERIC: 'generic', _lib.DW_TMA: 'tma', _lib.DW_STRIP_16B: 'strip16',
            _lib.DW_STRIP_F32: 'strip32', _lib.DW_5X5_16B: '5x5', _lib.DW_5X5_POOL_16B: '5x5_pool',
            _lib.DW_TMA_DIL: 'tma_dil'}
# depthwise kernels that pool their fp32 activations before rounding them to 16 bits (fc1 sums their slices)
POOLS_FP32 = {_lib.DW_TMA, _lib.DW_TMA_DIL, _lib.DW_STRIP_16B, _lib.DW_STRIP_F32}

# (configuration, crops): the benchmark scripts' models and batches (bench.py / f16_step.py, effnet_stride_step.py,
# effnet_b_step.py, mobilenet_step.py, resnet_step.py), and BASELINE.md's c3 (EfficientNetV2-L@384, one GPU's 32 crops
# of the strong-scaling batch) and c4 (EfficientNetV2-S@256 with 122 joints, 64 crops)
CONFIGS = [('efficientnetv2-l', 256), ('efficientnetv2-s-os8', 256), ('efficientnet-b0', 256), ('efficientnet-b4', 256),
           ('mobilenetv3-large', 256), ('resnet50-s8', 128), ('efficientnetv2-l@384', 32), ('efficientnetv2-s-j122', 64)]
# EfficientNetV2 configurations of the reference's own block grammar: configuration -> (model, crop side)
EFFNETV2 = {'efficientnetv2-l': ('efficientnetv2-l', 256), 'efficientnetv2-l@384': ('efficientnetv2-l', 384),
            'efficientnetv2-s-j122': ('efficientnetv2-s', 256)}


def n_joints(config):
    return JOINTS.get(config, J)


def build(H, config, precision):
    """-> (pcfg, spec, state dict, engine, op table, bound(name, x, res, scale) -> (ref, tol), SE activations (fc1, fc2))."""
    if config in EFFNETV2:
        name, side = EFFNETV2[config]
        pcfg = port.PathConfig(proc_side=side)
        spec = port.effnet_spec(name)
        sd = port.make_effnet_state_dict(spec, pcfg, n_joints(config), seed=0, calib_batch=1)
        eng = H.device_model(name, pcfg, n_joints(config), sd, precision=precision).engine()
        return (pcfg, spec, sd, eng, port_ops.effnet_op_table(spec),
                lambda nm, x, res, sc: port_ops.layer_bound(sd, spec, nm, x, res, sc, precision), ('silu', 'sigmoid'))
    if config == 'efficientnetv2-s-os8':
        from tests.test_gpu_effnet_dilated import device_model, model_and_weights
        pcfg, spec, sd = model_and_weights('efficientnetv2-s', 8, 256, n_joints=J)
        eng = device_model('efficientnetv2-s', 8, pcfg, J, sd, precision).engine()
        table = D.op_table(spec)

        def bound(nm, x, res, sc):
            if table[nm]['depthwise']:
                return D.dw_layer_bound(sd, spec, nm, x, precision)
            return port_ops.layer_bound(sd, spec, nm, x, res, sc, precision)
        return pcfg, spec, sd, eng, table, bound, ('silu', 'sigmoid')
    if config.startswith('efficientnet-b'):
        from tests.test_gpu_effnet_b import device_model, model
        pcfg, spec, sd = model(config, 256, j=J)
        eng = device_model(H, config, pcfg, J, sd, precision).engine()
        return (pcfg, spec, sd, eng, port_effnet_b.op_table(spec),
                lambda nm, x, res, sc: port_effnet_b.layer_bound(sd, spec, nm, x, res, sc, precision), ('silu', 'sigmoid'))
    if config == 'mobilenetv3-large':
        from tests.test_gpu_mobilenet_large import device_model
        pcfg = port.PathConfig(proc_side=256, stride_test=32, depth=8)
        spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
        sd = tfb.make_state_dict(spec, pcfg, J, seed=0, calib_batch=1)
        eng = device_model(H, 'large', pcfg, J, sd, precision).engine()
        return (pcfg, spec, sd, eng, port_mobilenet.op_table(spec),
                lambda nm, x, res, sc: port_mobilenet.layer_bound(sd, spec, nm, x, res, sc, precision), ('relu', 'hsigmoid'))
    assert config == 'resnet50-s8'  # resnet_step.py's stride-8 configuration: D = 32
    pcfg = port.PathConfig(proc_side=256, stride_test=8, depth=32)
    spec = tfb.ResNet50Spec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, J, seed=0, calib_batch=1)
    eng = H.device_model_tf('resnet50', pcfg, J, sd, precision=precision).engine()
    return (pcfg, spec, sd, eng, port_ops.op_table(spec),
            lambda nm, x, res, sc: port_ops.layer_bound(sd, spec, nm, x, res, sc, precision), None)


def check_conv(bound, nm, out, x, res, sc, precision):
    """out within bound(nm, ...) over all crops, the fp64 reference in crop chunks -> worst |dev-ref|/tol"""
    step = max(1, CHUNK // max(x[0].numel(), out[0].numel()))
    worst, bad = 0.0, 0
    for c0 in range(0, out.shape[0], step):
        s = slice(c0, c0 + step)
        ref, tol = bound(nm, x[s].double(), None if res is None else res[s].double(), None if sc is None else sc[s])
        assert ref.shape == out[s].shape, (nm, tuple(ref.shape), tuple(out[s].shape))
        r, b = port_ops.check_bound(out[s], ref, tol, precision)
        worst, bad = max(worst, r), bad + b
        del ref, tol
    assert bad == 0, f'{nm} [{precision}]: {bad} elements outside the bound (worst |dev-ref|/tol {worst:.2f})'
    return worst


def check_se_fc(sd, nm, out, x, xabs, n_in, x_err, act, precision):
    """fc1 / fc2 output [B,1,1,C] of the forward within port_ops.se_fc_bound -> worst |dev-ref|/tol"""
    key = se_fc_key(sd, nm)
    w, b = sd[key + '.weight'], sd[key + '.bias']
    n_real, cin = w.shape[0], w.shape[1]
    ref, tol = port_ops.se_fc_bound(x[:, :cin], xabs[:, :cin], n_in, w, b, act, None if x_err is None else x_err[:, :cin])
    dev = out[:, 0, 0].double()
    err = (dev[:, :n_real] - ref).abs()
    r = float((err / tol).max())
    assert bool((err <= tol).all()), f'{nm} [{precision}]: |dev-ref|/tol {r:.2f}'
    assert not dev[:, n_real:].any()  # hidden channels zero-padded to a multiple of 4
    return r


def check_head_per_coordinate(sd, feats, pcfg, c2d, c3d, tc32, n_joints=J):
    """head_decode's coordinates within port_ops.decode_bound, each one: the exact fp64 logits of the head's 1x1 conv on
    the features the device decoded (on the device), their per-logit bound port_ops.head_logit_delta, the decode on the
    host.  sd holds the head weight and bias as the device multiplies them (on the device), feats is NHWC.  -> (worst 2D, worst 3D |dev-ref|/tol)"""
    w, b = sd['heatmap_heads.conv_final.weight'], sd['heatmap_heads.conv_final.bias']
    f = feats.double().permute(0, 3, 1, 2)
    logits = torch.nn.functional.conv2d(f, w, b).cpu()
    delta = port_ops.head_logit_delta(f, w, b, tc32).cpu()
    r2, t2, r3, t3 = port_ops.decode_bound(logits, delta, pcfg, n_joints)
    e2, e3 = (c2d.double().cpu() - r2).abs(), (c3d.double().cpu() - r3).abs()
    w2, w3 = float((e2 / t2).max()), float((e3 / t3).max())
    assert bool((e2 <= t2).all()) and bool((e3 <= t3).all()), (
        f'head decode outside the per-coordinate bound: 2D {w2:.2f} (max {float(e2.max()):.2e} px), 3D {w3:.2f} '
        f'(max {float(e3.max()):.2e} mm)')
    return w2, w3


def heads_reference(sd, feats, pcfg, n_joints=J):
    """port.heads with the head's 1x1 conv evaluated in fp64 on the device (ResNet-50 at stride 8: 2048 channels on 32x32
    maps) and the soft-argmax decode on the host, where port.heads keeps its coordinate grids."""
    logits = port.head_logits(sd, feats.double().permute(0, 3, 1, 2)).cpu()
    logits2d, logits3d = port.split_logits(logits, n_joints, pcfg.depth)
    coords3d = port.heatmap_to_metric(port.soft_argmax(logits3d.float(), dims=(4, 3, 1)), pcfg)
    return port.heatmap_to_image(port.soft_argmax(logits2d.float(), dims=(3, 2)), pcfg), coords3d


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
@pytest.mark.parametrize('config,batch', CONFIGS)
def test_forward_ops_vs_conv2d(H, config, batch, precision):
    t0 = time.perf_counter()
    pcfg, _spec, sd, eng, table, bound, se_acts = build(H, config, precision)
    st = port_ops.MODES[precision][0]
    p = 8 if st == torch.bfloat16 else 11
    crops, intr = (t.cuda() for t in port.synthetic_inputs(batch, pcfg.proc_side, seed=5))
    names = eng.op_names()
    eng.profile_begin()
    eng.backbone(crops)
    prof = eng.profile_end()
    classes = {nm: cls for nm, cls, *_ in eng.profile_op_times()}

    live = {}  # buffer id -> fp32 copy of what the latest op that wrote it stored there
    worst, reached, se_proj = {}, set(), []
    n_checked = n_fc = 0
    for k, nm in enumerate(names):
        bufs = eng.op_buffers(k)
        io = eng.op_io(k)
        out = eng.debug_run_ops(crops, k + 1)
        assert torch.isfinite(out).all(), f'{nm} [{precision}]: {int((~torch.isfinite(out)).sum())} non-finite outputs'
        if nm.endswith('.avgpool'):  # fused pooling leaves partial slices here; fc1 is checked on their sum below
            reached.add(('se after', table[names[k - 1]]['act']))
        elif nm.endswith('.fc1'):
            assert names[k - 1].endswith('.avgpool')
            d = live[eng.op_buffers(k - 1)['input']]  # the depthwise output the forward stored
            dk = eng.op_kernel(k - 2)
            xabs = d.abs().mean(dim=(1, 2), dtype=torch.float64)
            x_err = 2.0 ** -p * (1 + 2.0 ** -p) * xabs if dk in POOLS_FP32 else None
            kind = f'se fc1 after {DW_NAMES[dk]}'
            r = check_se_fc(sd, nm, out, d.mean(dim=(1, 2), dtype=torch.float64), xabs, d.shape[1] * d.shape[2] + POOL_SLICES + 2,
                            x_err, se_acts[0], precision)
        elif nm.endswith('.fc2'):
            f1 = live[bufs['input']][:, 0, 0].double()
            kind = 'se fc2'
            r = check_se_fc(sd, nm, out, f1, f1.abs(), 0, None, se_acts[1], precision)
        else:
            op = table[nm]
            assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
            x = crops if k == 0 else live[bufs['input']]
            res = live[bufs['residual']] if bufs['residual'] != _lib.BUF_NONE else None
            sc = live[bufs['scale']][:, 0, 0] if bufs['scale'] != _lib.BUF_NONE else None
            assert (res is not None) == io['residual'] and (sc is not None) == io['scale'], nm
            if op['maxpool']:
                kind = 'maxpool'
                reached.add(kind)
            elif op['stem']:
                kind = classes[nm]
                if op['kernel'] == 3 and op['stride'] == 2 and io['out_shape'][2] in (24, 32):
                    reached.add('stem3x3s2')
            elif op['depthwise']:
                dk = eng.op_kernel(k)
                kind = f'dwconv_kernel/{DW_NAMES[dk]}' + ('+pool' if names[k + 1].endswith('.avgpool') else '')
                reached |= {('dw', dk), ('dw dil', dk, op['dil'])}
                if dk in (_lib.DW_TMA, _lib.DW_TMA_DIL):
                    hh, ww = (-(-n // op['dil']) for n in io['out_shape'][:2])
                    assert dw_plan(hh, ww)[0] > 0, nm
                    reached.add(('dw tma', hh))
            elif k > 0 and eng.op_is_fused_block(k - 1):
                kind = 'fmb_kernel'  # the block output; its input is the unfused expand's output, checked one op before
                reached |= {'fmb', ('fmb', io['out_shape'][0])}
            elif classes[nm] in ('tc_conv_kernel', 'fmb_kernel'):
                tk = eng.op_kernel(k)
                kind = 'tc_conv3x3s1_kernel' if tk == _lib.TC_CONV3X3S1 else 'tc_conv_kernel'
                reached.add(('tc', tk))
                if eng.op_is_fused_block(k):
                    kind += ' (fmb expand, unfused)'
                if sc is not None:
                    cin, cout = io['in_shape'][2], io['out_shape'][2]
                    se_proj.append((cin, cout))
                    kind += ' + SE in GEMM' if tk == _lib.TC_CONV_SE else ' behind se_scale_kernel'
            else:
                kind = classes[nm]
            reached |= {('act', op['act']), ('dil', op['dil'])}
            if op.get('res_first') and res is not None:
                reached.add('residual before act')
            if nm.endswith('_0_conv') and op['stride'] == 2:
                reached.add('strided 1x1 shortcut')
            r = check_conv(bound, nm, out, x, res, sc, precision)
            n_checked += 1
        if not nm.endswith('.avgpool'):
            worst[kind] = max(worst.get(kind, 0.0), r)
            n_fc += nm.endswith(('.fc1', '.fc2'))
        live[bufs['output']] = out

    # the backbone's features are the full prefix's, bit for bit; the fused head decodes them like the reference
    feats = eng.backbone(crops)
    assert torch.equal(feats.float(), live[_lib.BUF_FEATURES])
    eng.profile_begin()
    c2d, c3d = eng.head_decode(feats)
    head_prof = eng.profile_end()
    head = {'heatmap_heads.conv_final.weight': sd['heatmap_heads.conv_final.weight'].to(st).double().cuda(),
            'heatmap_heads.conv_final.bias': sd['heatmap_heads.conv_final.bias'].float().double().cuda()}
    nj = n_joints(config)
    ref2d, ref3d = heads_reference(head, feats, pcfg, nj)
    e2, e3 = H.rel_err(c2d, ref2d), H.rel_err(c3d, ref3d)
    assert e2 < 2e-4 and e3 < 2e-4, (e2, e3)
    worst['head 2D'], worst['head 3D'] = check_head_per_coordinate(head, feats, pcfg, c2d, c3d, tc32=False, n_joints=nj)
    # eager run, graph capture, graph replay (mtb_forward keys its graphs on buffers, batch and stream)
    o = torch.empty(batch, eng.n_out, 3, device=crops.device)
    joints = []
    for _ in range(3):
        eng.forward(crops, intr, out=o)
        joints.append(o.clone())
    assert torch.isfinite(joints[0]).all()
    assert all(torch.equal(joints[0], j) for j in joints[1:])

    n_conv = sum(not nm.endswith(('.avgpool', '.fc1', '.fc2')) for nm in names)
    assert n_checked == n_conv and n_fc == 2 * sum(nm.endswith('.avgpool') for nm in names), (n_checked, n_conv, n_fc)
    se_wide = sum(c > 256 for _, c in se_proj)
    assert prof.get('se_scale_kernel', {}).get('launches', 0) == se_wide, (prof.get('se_scale_kernel'), se_wide)
    if config == 'efficientnetv2-l':
        assert {('dw', _lib.DW_TMA), ('dw', _lib.DW_STRIP_16B), ('tc', _lib.TC_CONV3X3S1), 'fmb', 'stem3x3s2'} <= reached, reached
        assert {c for _, c in se_proj} == {192, 224, 384, 640} and se_wide == 32, se_proj
    elif config == 'efficientnetv2-l@384':
        # the fused head with one crop per tile (tc_head_plan: P = 144, 256 // 144 = 1 crop), the TMA depthwise plans of
        # the 24x24 and 12x12 maps, fmb_kernel on the 96x96 and 48x48 stages
        assert eng.feature_side == 12 and set(head_prof) == {'tc_head_softargmax_kernel'}, set(head_prof)
        assert {('dw tma', 24), ('dw tma', 12), ('fmb', 96), ('fmb', 48)} <= reached, reached
    elif config == 'efficientnetv2-s-j122':
        # nine M tiles of the fused head, the last one 74 of 128 channels
        n_out = sd['heatmap_heads.conv_final.weight'].shape[0]
        assert n_out == 122 * 9 and -(-n_out // 128) == 9 and n_out % 128 == 74, n_out
        assert set(head_prof) == {'tc_head_softargmax_kernel'}, set(head_prof)
    elif config == 'efficientnetv2-s-os8':
        assert {('dw dil', _lib.DW_TMA_DIL, 2), ('dw dil', _lib.DW_TMA_DIL, 4)} <= reached, reached
    elif config.startswith('efficientnet-b'):
        assert ('dw', _lib.DW_5X5_POOL_16B) in reached, reached
        assert any(c % 64 for c, _ in se_proj), se_proj  # partial 64-channel k-blocks in the SE projections
    elif config == 'mobilenetv3-large':
        assert {('act', 'hswish'), ('se after', 'relu'), ('se after', 'hswish')} <= reached, reached
    else:
        assert {'maxpool', ('dil', 2), ('dil', 4), 'residual before act', 'strided 1x1 shortcut'} <= reached, reached
    del live, out, feats
    torch.cuda.empty_cache()
    ratios = ', '.join(f'{kd}: {v:.3f}' for kd, v in sorted(worst.items()))
    print(f'{config} x{batch} [{precision}]: {len(names)} ops ({n_conv} conv), head rel err {e2:.1e} / {e3:.1e}, '
          f'{time.perf_counter() - t0:.1f} s; worst |dev-ref|/tol {{{ratios}}}')
