"""GPU: every op of the fp32-storage forwards ('tf32x3', the parity mode bench.py measures, and 'fp32') against fp64
conv2d element by element, at the benchmark batch, on the tensors the forward itself produced; the head per coordinate;
the joints against the oracle forward on the same crops.

The walk is test_gpu_forward_ops16.py's (its build / check_conv / check_se_fc): op k's output is what
``debug_run_ops(crops, k + 1)`` stored, its input, residual and SE scale what the latest earlier ops stored in the buffers
it reads.  In these modes that path runs tc32_conv_kernel (3xTF32 wgmma) on every tc32_eligible conv, with the SE scale
applied in its A-tile split and dilated spatial (mode 1) tiles; conv_igemm_kernel on the others and on every conv in
'fp32'; dwconv3x3_pool_f32_kernel (fused SE pooling slices) in 'tf32x3', the generic depthwise kernel and
pool_mean_kernel elsewhere; the tc32 or CUDA-core head GEMM and softargmax_bhwn_kernel.

* conv, depthwise, stem and max-pool ops: within the per-element bound (port_ops.layer_bound and the family bounds in
  their fp32 form) over all crops, and within the aggregate ||dev-ref||inf / ||ref||inf bar (AGG), which catches a bias
  that the worst-case accumulation term of a long-K GEMM would still admit.
* SE: the unfused pool against port_ops.pool_mean_bound, fc1 on that stored mean (or on the depthwise output the fused
  slices pooled), fc2 on fc1's output (port_ops.se_fc_bound); the projection on the scale fc2 stored, as a conv op.
* head: every decoded coordinate within port_ops.decode_bound.
* joints (port.relative_error), stage by stage: the forward's against the host reconstruction of its own decode (2e-5);
  the features against the fp64 oracle's (1e-3); the joints against the oracle head and reconstruction applied to the
  device's features (1e-3); end to end against the fp64 oracle forward (1e-3, JOINT_CAP on EfficientNetV2-L@256).
* backbone() bit-equal to the full prefix; eager, capture and replay give identical joints.
* what each configuration reached is asserted, and the worst |dev-ref|/tol per kernel kind and the wall time printed."""
import time

import pytest
import torch

from metrabs_b200 import _lib
from oracle import port, port_ops
from tests.test_gpu_forward_ops16 import (CONFIGS, DW_NAMES, build, check_conv, check_head_per_coordinate, check_se_fc,
                                          heads_reference, n_joints)
from tests.test_gpu_ops16_vs_conv2d import H, POOL_SLICES  # noqa: F401  (H: the fixture)

pytestmark = pytest.mark.gpu

# aggregate bar per op: test_gpu_tf32.py's for 'tf32x3'; the parity tests' per-layer 1e-4 for 'fp32'
AGG = {'tf32x3': 5e-5, 'fp32': 1e-4}
ORACLE_CHUNK = 32  # crops per chunk of the oracle backbone on the device


def expected_class(op, io, precision):
    if op['maxpool']:
        return 'other'
    if op['stem']:
        return 'stem_conv_kernel'
    if op['depthwise']:
        return 'dwconv_kernel'
    if precision == 'tf32x3' and port_ops.tc32_eligible(op, io['in_shape'][2], io['out_shape'][2]):
        return 'tc32_conv_kernel'
    return 'conv_igemm_kernel'


# Joint bar of the end-to-end comparison with the fp64 oracle: bench's 1e-3, except on EfficientNetV2-L@256.  There the
# untrained head amplifies feature differences about 17x into the joints, so no fp32 evaluation meets 1e-3 at 256 crops.
# Measured on an H100 SXM (700 W) at 256 crops:
# - tf32x3: features 4.8e-4 from the fp64 oracle's, joints 8.0e-3;
# - fp32: features 8.4e-5, joints 1.8e-3;
# - the oracle port itself in fp32 (bench's reference): 2.4e-3 on the CPU and 1.1e-3 on the device with TF32 off.
# The fp64 oracle head and reconstruction on the device's own features reproduce those joint errors (8.0e-3 / 1.8e-3).
# The device's decode of those features is within 2e-5 of that, and its reconstruction within 3e-7.  Those stages are
# asserted separately below at their own bars; the cap of 1e-2 bounds the amplified remainder.
JOINT_CAP = {'efficientnetv2-l': 1e-2}
FEATURE_BAR = 1e-3  # the parity tests' feature bar (test_gpu_parity.py)


def oracle_features(spec, sd, crops):
    """the oracle backbone (as port.metrabs_forward) in fp64 on the device in crop chunks -> NHWC fp64"""
    sd_dev = {k: v.cuda().double() if torch.is_tensor(v) and v.is_floating_point() else v for k, v in sd.items()}
    if isinstance(spec, port.EffNetSpec):
        features = lambda sd_, im: port.effnet_features(sd_, spec, im)  # noqa: E731
    else:
        features = spec.features
    feats = []
    with torch.device('cuda'), torch.inference_mode():  # constants the backbones create land on the device too
        for c0 in range(0, crops.shape[0], ORACLE_CHUNK):
            feats.append(features(sd_dev, crops[c0:c0 + ORACLE_CHUNK].double()).permute(0, 2, 3, 1).contiguous())
    return torch.cat(feats)


def oracle_tail(sd, feats, pcfg, intr, nj):
    """port.heads + port.reconstruct_absolute on NHWC features: the head's 1x1 conv in fp64 on the device, the soft-argmax
    (in fp32, as port.heads) and the reconstruction on the host."""
    head = {k: sd[k].double().cuda() for k in ('heatmap_heads.conv_final.weight', 'heatmap_heads.conv_final.bias')}
    with torch.inference_mode():
        c2d, c3d = heads_reference(head, feats, pcfg, nj)
    return port.reconstruct_absolute(c2d, c3d, intr.cpu(), pcfg)


@pytest.mark.parametrize('precision', ['tf32x3', 'fp32'])
@pytest.mark.parametrize('config,batch', CONFIGS)
def test_forward_ops_vs_conv2d(H, config, batch, precision):
    t0 = time.perf_counter()
    pcfg, spec, sd, eng, table, bound, se_acts = build(H, config, precision)
    crops, intr = (t.cuda() for t in port.synthetic_inputs(batch, pcfg.proc_side, seed=5))
    names = eng.op_names()
    eng.profile_begin()
    eng.backbone(crops)
    prof = eng.profile_end()
    classes = {nm: cls for nm, cls, *_ in eng.profile_op_times()}

    live = {}  # buffer id -> what the latest op that wrote it stored there
    worst, agg, reached = {}, {}, set()
    n_checked = n_fc = 0
    for k, nm in enumerate(names):
        bufs = eng.op_buffers(k)
        io = eng.op_io(k)
        out = eng.debug_run_ops(crops, k + 1)
        assert torch.isfinite(out).all(), f'{nm} [{precision}]: {int((~torch.isfinite(out)).sum())} non-finite outputs'
        r = None
        if nm.endswith('.avgpool'):
            dk = eng.op_kernel(k - 1)
            reached.add(('se after', table[names[k - 1]]['act'], DW_NAMES[dk]))
            if dk == _lib.DW_GENERIC:  # pool_mean_kernel; the fused kernels leave partial slices here (fc1 sums them)
                assert classes[nm] == 'pool_mean_kernel', (nm, classes[nm])
                ref, tol = port_ops.pool_mean_bound(live[bufs['input']])
                err = (out[:, 0, 0].double() - ref).abs()
                r, kind = float((err / tol).max()), 'pool_mean_kernel'
                assert bool((err <= tol).all()), f'{nm} [{precision}]: |dev-ref|/tol {r:.2f}'
        elif nm.endswith('.fc1'):
            assert names[k - 1].endswith('.avgpool')
            dk = eng.op_kernel(k - 2)
            if dk == _lib.DW_GENERIC:  # on the mean pool_mean_kernel stored
                x = live[eng.op_buffers(k - 1)['output']][:, 0, 0].double()
                r = check_se_fc(sd, nm, out, x, x.abs(), 0, None, se_acts[0], precision)
            else:  # on the sum of the slices the depthwise kernel pooled from the fp32 values it stored
                assert dk == _lib.DW_STRIP_F32, (nm, dk)
                d = live[eng.op_buffers(k - 1)['input']]
                r = check_se_fc(sd, nm, out, d.mean(dim=(1, 2), dtype=torch.float64), d.abs().mean(dim=(1, 2), dtype=torch.float64),
                                d.shape[1] * d.shape[2] + POOL_SLICES + 2, None, se_acts[0], precision)
            kind = f'se fc1 after {DW_NAMES[dk]}'
        elif nm.endswith('.fc2'):
            f1 = live[bufs['input']][:, 0, 0].double()
            kind = 'se fc2'
            r = check_se_fc(sd, nm, out, f1, f1.abs(), 0, None, se_acts[1], precision)
        else:
            op = table[nm]
            cls = classes[nm]
            assert cls == expected_class(op, io, precision), (nm, cls)
            x = crops if k == 0 else live[bufs['input']]
            res = live[bufs['residual']] if bufs['residual'] != _lib.BUF_NONE else None
            sc = live[bufs['scale']][:, 0, 0] if bufs['scale'] != _lib.BUF_NONE else None
            assert (res is not None) == io['residual'] and (sc is not None) == io['scale'], nm
            kind = cls
            if op['maxpool']:
                kind = 'maxpool'
                reached.add(kind)
            elif op['depthwise']:
                dk = eng.op_kernel(k)
                kind += f'/{DW_NAMES[dk]}' + ('+pool' if names[k + 1].endswith('.avgpool') else '')
                reached.add(('dw', dk))
            elif cls == 'tc32_conv_kernel':
                mode1 = not (op['kernel'] == 1 and op['stride'] == 1)
                reached.add(('tc32', 'spatial' if mode1 else 'flat', op['dil']))
                if sc is not None:
                    kind += ' + SE in split'
                    reached.add('se in split')
            elif sc is not None:
                kind += ' + SE'
            reached |= {('act', op['act']), ('dil', op['dil'])}
            if op.get('res_first') and res is not None:
                reached.add('residual before act')
            # aggregate bar: track max |dev - ref| and max |ref| over the crop chunks check_conv evaluates
            seen = {'c0': 0, 'err': 0.0, 'ref': 0.0}

            def tracked(nm_, xs, rs, ss):
                ref, tol = bound(nm_, xs, rs, ss)
                n = ref.shape[0]
                dev = out[seen['c0']:seen['c0'] + n].double()
                seen['err'] = max(seen['err'], float((dev - ref).abs().max()))
                seen['ref'] = max(seen['ref'], float(ref.abs().max()))
                seen['c0'] += n
                return ref, tol
            r = check_conv(tracked, nm, out, x, res, sc, precision)
            assert seen['c0'] == out.shape[0]
            a = seen['err'] / max(seen['ref'], 1e-30)
            agg[kind] = max(agg.get(kind, 0.0), a)
            assert a < AGG[precision], f'{nm} [{precision}]: ||dev-ref||inf/||ref||inf {a:.2e} >= {AGG[precision]}'
            n_checked += 1
        if r is not None:
            worst[kind] = max(worst.get(kind, 0.0), r)
            n_fc += nm.endswith(('.fc1', '.fc2'))
        live[bufs['output']] = out

    # the backbone's features are the full prefix's, bit for bit
    feats = eng.backbone(crops)
    assert torch.equal(feats, live[_lib.BUF_FEATURES])
    del live, out
    # head: every coordinate within the decode bound on the weights the device multiplies (fp32)
    eng.profile_begin()
    c2d, c3d = eng.head_decode(feats)
    head_prof = eng.profile_end()
    tc32_head = 'tc32_conv_kernel' in head_prof
    head = {'heatmap_heads.conv_final.weight': sd['heatmap_heads.conv_final.weight'].float().double().cuda(),
            'heatmap_heads.conv_final.bias': sd['heatmap_heads.conv_final.bias'].float().double().cuda()}
    nj = n_joints(config)
    worst['head 2D'], worst['head 3D'] = check_head_per_coordinate(head, feats, pcfg, c2d, c3d, tc32_head, nj)
    # joints: eager run, graph capture, graph replay identical
    o = torch.empty(batch, eng.n_out, 3, device=crops.device)
    joints = []
    for _ in range(3):
        eng.forward(crops, intr, out=o)
        joints.append(o.clone())
    assert all(torch.equal(joints[0], j) for j in joints[1:])
    torch.cuda.empty_cache()
    # the forward's tail is the host reconstruction of the device's own decode
    tail = port.reconstruct_absolute(c2d.double().cpu(), c3d.double().cpu(), intr.double().cpu(), pcfg)
    e_tail = port.relative_error(joints[0].cpu(), tail)
    assert e_tail < 2e-5, f'{config} x{batch} [{precision}]: forward vs the reconstruction of its decode {e_tail:.2e}'
    # the device's features against the fp64 oracle's; the device's joints against the oracle head and reconstruction on
    # the device's own features (head, decode and reconstruction alone), and end to end against the fp64 oracle forward
    f64 = oracle_features(spec, sd, crops)
    e_feat = float((feats.double() - f64).abs().max() / f64.abs().max())
    assert e_feat < FEATURE_BAR, f'{config} x{batch} [{precision}]: features vs the fp64 oracle {e_feat:.2e}'
    e_head = port.relative_error(joints[0].cpu(), oracle_tail(sd, feats.double(), pcfg, intr, nj))
    assert e_head < 1e-3, f'{config} x{batch} [{precision}]: joints vs the oracle head on the device features {e_head:.2e}'
    e_joints = port.relative_error(joints[0].cpu(), oracle_tail(sd, f64, pcfg, intr, nj))
    del feats, f64
    torch.cuda.empty_cache()

    # what this configuration reached
    n_conv = sum(not nm.endswith(('.avgpool', '.fc1', '.fc2')) for nm in names)
    n_pool = sum(nm.endswith('.avgpool') for nm in names)
    assert n_checked == n_conv and n_fc == 2 * n_pool, (n_checked, n_conv, n_fc)
    assert set(head_prof) == ({'tc32_conv_kernel', 'softargmax_bhwn_kernel'} if precision == 'tf32x3'
                              else {'head_conv(conv_igemm_kernel)', 'softargmax_bhwn_kernel'}), set(head_prof)
    assert 'se_scale_kernel' not in prof and 'tc_conv_kernel' not in prof and 'fmb_kernel' not in prof, set(prof)
    n_generic_pools = sum(eng.op_kernel(i - 1) == _lib.DW_GENERIC for i, nm in enumerate(names) if nm.endswith('.avgpool'))
    assert prof.get('pool_mean_kernel', {}).get('launches', 0) == n_generic_pools
    if precision == 'fp32':
        assert 'tc32_conv_kernel' not in prof and n_generic_pools == n_pool, set(prof)
        assert all(eng.op_kernel(i) == _lib.DW_GENERIC for i, nm in enumerate(names) if table.get(nm, {}).get('depthwise'))
    else:
        assert any(t[0] == 'tc32' for t in reached if isinstance(t, tuple)), reached
        if config.startswith('efficientnet'):
            assert {('dw', _lib.DW_STRIP_F32), 'se in split'} <= reached, reached
            assert ('se after', 'silu', 'strip32') in reached, reached
        if config == 'efficientnetv2-l':
            assert ('tc32', 'spatial', 1) in reached, reached  # the 3x3 FusedMBConv expands
    if config == 'mobilenetv3-large':
        assert {('act', 'hswish'), ('se after', 'relu', DW_NAMES[_lib.DW_GENERIC])} <= reached, reached
        if precision == 'tf32x3':
            assert 'se in split' in reached and ('se after', 'hswish', 'strip32') in reached, reached
    elif config == 'efficientnetv2-s-os8':
        assert {('dil', 2), ('dil', 4)} <= reached, reached
    elif config == 'resnet50-s8':
        assert {'maxpool', ('dil', 2), ('dil', 4), 'residual before act'} <= reached, reached
        if precision == 'tf32x3':
            assert {('tc32', 'spatial', 2), ('tc32', 'spatial', 4)} <= reached, reached  # dilated mode-1 tiles
    ratios = ', '.join(f'{kd}: {v:.3f}' for kd, v in sorted(worst.items()))
    aggs = ', '.join(f'{kd}: {v:.1e}' for kd, v in sorted(agg.items()))
    print(f'{config} x{batch} [{precision}]: {len(names)} ops ({n_conv} conv), features vs oracle {e_feat:.1e}, joints vs '
          f'oracle {e_joints:.1e} (oracle head on the device features {e_head:.1e}, tail {e_tail:.1e}), '
          f'{time.perf_counter() - t0:.1f} s; worst |dev-ref|/tol {{{ratios}}}; worst ||dev-ref||/||ref|| {{{aggs}}}')
    cap = JOINT_CAP.get(config, 1e-3)
    assert e_joints < cap, f'{config} x{batch} [{precision}]: joints vs the fp64 oracle forward {e_joints:.2e} >= {cap}'
