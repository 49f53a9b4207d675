"""GPU: MobileNetV3-Large (metrabs_b200.backbones.mobilenet_v3) against this build's torch restatement of the Keras code
(oracle/port_mobilenet.py MobileNetV3Spec; the reference has no test, golden or importable MobileNetV3, so parity is
"this build's restatement vs this build's kernels"), and the 16-bit 5x5 depthwise kernel of both variants.

* fp32 and tf32x3: every layer within 1e-4 of the restatement on the restatement's own operands (the SE-scaled
  projections take the restatement's own SE scale), features and joints within 1e-3, at S=256 and S=224, with and without
  the centered stride.
* bf16, bf16_simt, fp16, fp16_simt: every distinct op element by element against fp64 conv2d at the mode's rounding points
  (port_mobilenet.layer_bound, port_ops.check_bound), with its kernel class and depthwise kernel (mtb_op_kernel)
  asserted: every GEMM on tc_conv_kernel and every 5x5 depthwise op on dwconv5x5_16b_kernel in the tensor-core modes.
  The SE fc1 / fc2 ops are checked on the device's own forward: fc1 reads a separately pooled mean behind the 5x5 kernel.
* dwconv5x5_16b_kernel against dwconv_kernel: every distinct 5x5 op shape of Small and Large (stride 1 and 2, the
  bottom-right shift, ReLU and hard-swish, the odd 7x7 / 14x14 maps of S=224) at batch sizes 1, 3 and 5, run in 'bf16' and
  in 'bf16_simt' (and 'fp16' / 'fp16_simt') on the same inputs: the outputs must be equal (torch.equal).
* 16-bit end-to-end forwards (finite joints, deviation from the fp32 restatement printed) and the host-buffer, pipelined
  and Pose3dEstimator entry points."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from oracle import port, port_mobilenet, port_ops
from oracle import port_tf_backbones as tfb
from tests.test_gpu_ops16_vs_conv2d import MODES, POOL_SLICES, expected_class, op_classes, operands

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def device_model(H, variant, pcfg, n_joints, sd, precision='fp32'):
    import metrabs_b200
    from metrabs_b200.backbones import mobilenet_v3
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    m = Metrabs(mobilenet_v3.Features(variant), H.joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def se_scale(sd, name, d):
    """The restatement's SE scale of block `name` on its depthwise output d (NCHW), the same ops in the same order."""
    p = f'backbone.{name}.squeeze_excite.'
    q = d.mean(dim=(2, 3), keepdim=True)
    q = F.relu(F.conv2d(q, sd[p + 'Conv.weight'], sd[p + 'Conv.bias']))
    return tfb.hard_sigmoid(F.conv2d(q, sd[p + 'Conv_1.weight'], sd[p + 'Conv_1.bias']))[:, :, 0, 0]


def layer_operands(sd, spec, tap, crops):
    """op name -> (input NCHW, residual NCHW or None, SE scale [B,C] or None), from the restatement's own tensors."""
    p = 'backbone.'
    ops = {p + 'Conv': (crops, None, None)}
    x = tap[p + 'Conv']
    for b in port_mobilenet.mobilenet_blocks(spec.variant):
        n = p + b['name']
        if b['name'] != 'expanded_conv':
            ops[n + '.expand'] = (x, None, None)
        ops[n + '.depthwise'] = (tap[n + '.expand'] if b['name'] != 'expanded_conv' else x, None, None)
        d = tap[n + '.depthwise']
        ops[n + '.project'] = (d, x if b['residual'] else None, se_scale(sd, b['name'], d) if b['se'] else None)
        x = tap[n + '.project']
    ops[p + 'Conv_1'] = (x, None, None)
    ops[p + 'Conv_2'] = (tap[p + 'Conv_1'], None, None)
    return ops


def is_se(name):
    return name.endswith(('.avgpool', '.fc1', '.fc2'))


PARITY = [dict(proc_side=256, stride_test=32, depth=8), dict(proc_side=256, stride_test=32, depth=8, centered_stride=False),
          dict(proc_side=224, stride_test=32, depth=8), dict(proc_side=224, stride_test=32, depth=8, centered_stride=False)]


@pytest.mark.parametrize('cfgkw', PARITY)
def test_large_fp32_and_tf32x3(H, cfgkw):
    j, batch = 24, 2
    pcfg = port.PathConfig(**cfgkw)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
    tap, stages = {}, {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
        operands_ = layer_operands(sd, spec, tap, crops)
    for precision in ('fp32', 'tf32x3'):
        m = device_model(H, 'large', pcfg, j, sd, precision)
        eng = m.engine()
        names = eng.op_names()
        assert {n for n in names if not is_se(n)} == set(tap) == set(operands_)
        nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).cuda()  # noqa: E731
        bad = []
        for i, name in enumerate(names):
            if is_se(name):
                continue
            x, res, sc = operands_[name]
            out = eng.debug_run_op(i, x.cuda() if i == 0 else nhwc(x), nhwc(res),
                                   None if sc is None else sc.cuda()).permute(0, 3, 1, 2).cpu()
            err = port.relative_error(out, tap[name])
            if not err < 1e-4:
                bad.append((name, err))
        assert not bad, f'{precision}: first diverging layers: {bad[:5]}'
        out = m((crops.cuda(), k.cuda()))
        e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
        e_out = H.rel_err(out, ref)
        print(f'mobilenetv3-large {cfgkw} [{precision}]: features {e_feat:.2e}, joints {e_out:.2e}, '
              f'{eng.backbone_flops_per_crop / 1e9:.3f} GFLOP/crop, {eng.last_launch_count} launches')
        assert e_feat < 1e-3 and e_out < 1e-3
        del m, eng
        torch.cuda.empty_cache()


def dw_expected(op, precision):
    """the depthwise kernel mtb_finalize_weights must choose (apart from TMA vs strip for 3x3 stride-1 ops)"""
    from metrabs_b200 import _lib
    if precision not in ('bf16', 'fp16'):
        return {_lib.DW_GENERIC}
    if op['kernel'] == 5:
        return {_lib.DW_5X5_16B}
    return {_lib.DW_STRIP_16B} if op['stride'] == 2 else {_lib.DW_TMA, _lib.DW_STRIP_16B}


@pytest.mark.parametrize('side,centered,batch', [(256, True, 4), (224, True, 3), (224, False, 2)])
def test_large_ops16_vs_conv2d(H, side, centered, batch):
    from metrabs_b200 import _lib
    pcfg = port.PathConfig(proc_side=side, stride_test=32, centered_stride=centered, depth=8)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    table = port_mobilenet.op_table(spec)
    for precision in MODES:
        eng = device_model(H, 'large', pcfg, 8, sd, precision).engine()
        classes = op_classes(eng, side)
        st = port_ops.MODES[precision][0]
        g = torch.Generator().manual_seed(side)
        seen, feats, worst = set(), set(), {}
        for i, nm in enumerate(eng.op_names()):
            if is_se(nm):
                continue
            op, io = table[nm], eng.op_io(i)
            sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], op['stride'], op['shift'], op['act'],
                   op['kernel'], op['depthwise'], op['stem'])
            if sig in seen:
                continue
            seen.add(sig)
            assert classes[nm] in expected_class(op, io, precision), (nm, classes[nm])
            kind = classes[nm]
            if op['depthwise']:
                dk = eng.op_kernel(i)
                assert dk in dw_expected(op, precision), (nm, precision, dk)
                kind += f'/{dk}'
            elif not op['stem'] and precision in ('bf16', 'fp16'):
                assert classes[nm] == 'tc_conv_kernel', (nm, classes[nm])
            feats |= {kind, ('act', op['act']), ('shift', op['shift']), ('k', op['kernel'])}
            x, res, sc = operands(io, batch, st, g, i == 0)
            out = eng.debug_run_op(i, x, res, sc)
            ref, tol = port_mobilenet.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), sc,
                                                  precision)
            assert out.shape == ref.shape, (nm, tuple(out.shape), tuple(ref.shape))
            r, bad = port_ops.check_bound(out, ref, tol, precision)
            assert bad == 0, f'{nm} [{precision}] batch {batch}: {bad} elements outside the bound (worst |dev-ref|/tol {r:.2f})'
            worst[kind] = max(worst.get(kind, 0.0), r)
        assert ('act', 'hswish') in feats and ('act', 'relu') in feats and ('k', 5) in feats
        assert (('shift', 1) in feats) == centered
        if precision in ('bf16', 'fp16'):
            assert f'dwconv_kernel/{_lib.DW_5X5_16B}' in feats and 'tc_conv_kernel' in feats
            assert 'conv_igemm_kernel' not in feats and 'fmb_kernel' not in feats
        else:
            assert f'dwconv_kernel/{_lib.DW_GENERIC}' in feats and 'conv_igemm_kernel' in feats
        print(f'mobilenetv3-large@{side} centered={centered} [{precision}]: {len(seen)} ops, worst |dev-ref|/tol {worst}')
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('side,batch', [(256, 2), (224, 3)])
def test_large_se_squeeze_on_the_forward(H, precision, side, batch):
    """fc1 against act(W1 mean(D) + b1) in fp64 on the depthwise output D the device stored, fc2 against act(W2 F1 + b2) on
    the fc1 output F1 it produced (the premise of test_gpu_ops16_vs_conv2d.py::test_fused_se_squeeze_on_the_forward).
    Behind dwconv5x5_16b_kernel and dwconv_kernel fc1 reads the separate pool kernel's mean of D; behind the TMA and strip
    3x3 kernels it sums their fused pooling slices."""
    from metrabs_b200 import _lib
    from tests.test_gpu_ops16_vs_conv2d import se_fc_key
    pcfg = port.PathConfig(proc_side=side, stride_test=32, depth=8)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = device_model(H, 'large', pcfg, 8, sd, precision).engine()
    names = eng.op_names()
    crops = port.synthetic_inputs(batch, side, seed=14)[0].cuda()
    reached, worst = set(), {}
    for i, nm in enumerate(names):
        if not nm.endswith('.avgpool'):
            continue
        hh, ww, _c = eng.op_io(i - 1)['out_shape']
        dk = eng.op_kernel(i - 1)
        reached.add(dk)
        d = eng.debug_run_ops(crops, i).double()                     # the depthwise output the device stored
        f1 = eng.debug_run_ops(crops, i + 2)[:, 0, 0].double()       # fc1 on the fused (or separate) pooling
        f2 = eng.debug_run_ops(crops, i + 3)[:, 0, 0].double()       # fc2 on that fc1 output
        p = 8 if port_ops.MODES[precision][0] == torch.bfloat16 else 11
        fused = dk in (_lib.DW_TMA, _lib.DW_STRIP_16B, _lib.DW_STRIP_F32)
        pool_err = 2.0 ** -p * (1 + 2.0 ** -p) * d.abs().mean(dim=(1, 2)) if fused else None
        for j, (x, xabs, n_in, x_err, dev, act) in enumerate([
                (d.mean(dim=(1, 2)), d.abs().mean(dim=(1, 2)), hh * ww + POOL_SLICES + 2, pool_err, f1, 'relu'),
                (f1, f1.abs(), 0, None, f2, 'hsigmoid')]):
            key = se_fc_key(sd, names[i + 1 + j])
            w, b = sd[key + '.weight'], sd[key + '.bias']
            n_real = w.shape[0]
            ref, tol = port_ops.se_fc_bound(x[:, :w.shape[1]], xabs[:, :w.shape[1]], n_in, w, b, act,
                                            None if x_err is None else x_err[:, :w.shape[1]])
            err = (dev[:, :n_real] - ref).abs()
            r = float((err / tol).max())
            assert bool((err <= tol).all()), f'{names[i + 1 + j]} [{precision}] after depthwise kernel {dk}: |dev-ref|/tol {r:.2f}'
            assert not dev[:, n_real:].any()  # hidden channels zero-padded to a multiple of 4
            worst[f'{dk}/fc{j + 1}'] = max(worst.get(f'{dk}/fc{j + 1}', 0.0), r)
    if precision in ('bf16', 'fp16'):
        assert _lib.DW_5X5_16B in reached and reached & {_lib.DW_TMA, _lib.DW_STRIP_16B}, reached
    else:
        assert reached == {_lib.DW_GENERIC}, reached
    print(f'mobilenetv3-large@{side} x{batch} SE [{precision}]: worst |dev-ref|/tol {worst}')


@pytest.mark.parametrize('variant', ['small', 'large'])
@pytest.mark.parametrize('side', [256, 224])
def test_dw5x5_bit_equal_to_the_generic_kernel(H, variant, side):
    from metrabs_b200 import _lib
    pcfg = port.PathConfig(proc_side=side, stride_test=32, centered_stride=True, depth=8)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, variant)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    table = port_mobilenet.op_table(spec)
    g = torch.Generator().manual_seed(21)
    reached = set()
    for tc_mode, simt_mode in (('bf16', 'bf16_simt'), ('fp16', 'fp16_simt')):
        tc = device_model(H, variant, pcfg, 8, sd, tc_mode).engine()
        simt = device_model(H, variant, pcfg, 8, sd, simt_mode).engine()
        st = port_ops.MODES[tc_mode][0]
        seen = set()
        for i, nm in enumerate(tc.op_names()):
            if nm not in table or not table[nm]['depthwise'] or table[nm]['kernel'] != 5:
                continue
            op, io = table[nm], tc.op_io(i)
            sig = (io['in_shape'], io['out_shape'], op['stride'], op['shift'], op['act'])
            if sig in seen:
                continue
            seen.add(sig)
            assert tc.op_kernel(i) == _lib.DW_5X5_16B and simt.op_kernel(i) == _lib.DW_GENERIC, nm
            for batch in (1, 3, 5):
                x = (3 * torch.randn((batch,) + io['in_shape'], generator=g)).to(st).float().cuda()
                a, b = tc.debug_run_op(i, x), simt.debug_run_op(i, x)
                assert torch.isfinite(a).all()
                assert torch.equal(a, b), (nm, tc_mode, batch, int((a != b).sum()))
            reached |= {('stride', op['stride']), ('shift', op['shift']), ('act', op['act']), ('odd', io['out_shape'][0] % 2)}
        print(f'mobilenetv3-{variant}@{side} [{tc_mode} vs {simt_mode}]: {len(seen)} distinct 5x5 ops bit-equal at batch 1, 3, 5')
        del tc, simt
        torch.cuda.empty_cache()
    assert {('stride', 1), ('stride', 2), ('shift', 1), ('act', 'hswish')} <= reached, reached
    if variant == 'large':
        assert ('act', 'relu') in reached
    if side == 224:
        assert ('odd', 1) in reached  # the 7x7 maps


def test_large_16bit_end_to_end(H):
    j, batch = 24, 4
    pcfg = port.PathConfig(proc_side=256, stride_test=32, depth=8)
    spec = port_mobilenet.MobileNetV3Spec(pcfg, 'large')
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=1)
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k)
    for precision in ('bf16', 'fp16'):
        m = device_model(H, 'large', pcfg, j, sd, precision)
        out = m((crops.cuda(), k.cuda()))
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        print(f'mobilenetv3-large [{precision}]: joints rel err vs fp32 restatement {H.rel_err(out, ref):.2e}, '
              f'{m.engine().last_launch_count} launches')
        del m
        torch.cuda.empty_cache()


def test_large_host_pipelined_and_multiperson(H):
    j = 8
    pcfg = port.PathConfig(proc_side=256, stride_test=32, depth=8)
    sd = tfb.make_state_dict(port_mobilenet.MobileNetV3Spec(pcfg, 'large'), pcfg, j, seed=0, calib_batch=1)
    m = device_model(H, 'large', pcfg, j, sd, 'bf16')
    eng = m.engine()
    crops, k = port.synthetic_inputs(3, 256, seed=2)
    out = m((crops.cuda(), k.cuda()))
    out_h = eng.forward_host(crops.pin_memory(), k.pin_memory())
    assert torch.equal(out_h, out.cpu())
    ch, kh = crops.float().contiguous().pin_memory(), k.float().contiguous().pin_memory()
    outs = [torch.empty(out_h.shape, dtype=torch.float32).pin_memory() for _ in range(2)]
    eng.forward_host_submit(ch, kh, outs[0], 0)
    eng.forward_host_submit(ch, kh, outs[1], 1)
    eng.forward_host_wait(0)
    eng.forward_host_wait(1)
    assert torch.equal(outs[0], out_h) and torch.equal(outs[1], out_h)
    from metrabs_b200.multiperson import Pose3dEstimator
    m.joint_names, m.joint_edges = [f'j{i}' for i in range(j)], [[0, 1]]
    est = Pose3dEstimator(m, {'': dict(indices=list(range(j)), names=m.joint_names, edges=[[0, 1]])}, None)
    frames = torch.randint(0, 256, (1, 3, 240, 320), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    res = est.estimate_poses_batched(frames.cuda(), [torch.tensor([[40., 20., 120., 180.], [150., 40., 100., 160.]])],
                                     num_aug=3)
    torch.cuda.synchronize()
    assert res['poses3d'][0].shape == (2, j, 3) and torch.isfinite(res['poses3d'][0]).all()
