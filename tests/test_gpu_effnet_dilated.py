"""GPU: EfficientNetV2 at output stride 16 and 8 (dilated MBConv stages).

* Parity: joints within 1e-3 of the reference's dilated modules (tests/golden/*_os{16,8}.npz) in 'fp32' and 'tf32x3'; the
  'bf16' and 'fp16' deviations are printed.
* Every distinct dilated depthwise op runs dw3x3s1_dil_tma_kernel in bf16 and fp16 and meets fp64 conv2d on the same 16-bit
  operands within the bound of test_gpu_ops16_vs_conv2d.py, at batches around the kernel's crop group; fc1 on the forward's
  fused pooling meets that file's SE bound.
* Polyphase: each phase of a dilated op's output is bit-identical to dw3x3s1_tma_kernel's output on that phase's sub-grid.
"""
import dataclasses
import os

import numpy as np
import pytest
import torch

import metrabs_b200
from metrabs_b200 import _lib
from metrabs_b200.backbones import efficientnet as E
from metrabs_b200.models.metrabs import Metrabs
from oracle import port, port_ops
from oracle import port_effnet_dilated as D
from tests.helpers import joint_info
from tests.test_gpu_ops16_vs_conv2d import H, POOL_SLICES, dw_plan, operands  # noqa: F401  (H: the GPU fixture)

pytestmark = pytest.mark.gpu

SIZES = {'efficientnetv2-tiny': 'tiny', 'efficientnetv2-s': 's', 'efficientnetv2-l': 'l'}


def device_model(name, output_stride, pcfg, n_joints, sd, precision):
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision))
    bb = E.EfficientNet(SIZES[name], output_stride)
    m = Metrabs(torch.nn.Sequential(E.PreprocLayer(), bb.features), joint_info(n_joints)).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def model_and_weights(name, output_stride, side, n_joints=8, calib_batch=1):
    pcfg = port.PathConfig(proc_side=side, stride_test=output_stride)
    spec = D.effnet_spec(name, output_stride=output_stride)
    return pcfg, spec, D.make_state_dict(spec, pcfg, n_joints, seed=0, calib_batch=calib_batch)


@pytest.mark.parametrize('fname', ['tiny_s64_j8_os16.npz', 'tiny_s64_j8_os8.npz', 'effnetv2s_s256_j24_os16.npz',
                                   'effnetv2l_s256_j24_os8.npz'])
def test_parity_with_the_reference(H, golden_dir, fname):
    g = np.load(os.path.join(golden_dir, fname))
    name, os_, s, j, b = str(g['name']), int(g['output_stride']), int(g['proc_side']), int(g['n_joints']), int(g['batch'])
    pcfg = port.PathConfig(proc_side=s, stride_test=os_)
    if 'sd/backbone.1.0.0.weight' in g.files:
        sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith('sd/')}
        crops, k = torch.from_numpy(g['crops']), torch.from_numpy(g['intrinsics'])
    else:
        sd = D.make_state_dict(D.effnet_spec(name, output_stride=os_), pcfg, j, seed=0, calib_batch=2 if b < 3 else 4)
        crops, k = port.synthetic_inputs(b, s, seed=0)
    errs = {}
    for precision in ('fp32', 'tf32x3', 'bf16', 'fp16'):
        m = device_model(name, os_, pcfg, j, sd, precision)
        eng = m.engine()
        assert eng.feature_side == s // os_
        out = m((crops.cuda(), k.cuda()))
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        errs[precision] = H.rel_err(out, g['coords3d_abs'])
    print(f'{fname}: joints rel err vs reference {errs}')
    assert errs['fp32'] < 1e-3 and errs['tf32x3'] < 1e-3, errs


def dilated_ops(eng, spec):
    """-> [(op index, name, op dict, io)] of the distinct dilated depthwise ops."""
    table = D.op_table(spec)
    seen, out = set(), []
    for i, nm in enumerate(eng.op_names()):
        op = table.get(nm)
        if op is None or not op['depthwise'] or op['dil'] == 1:
            continue
        io = eng.op_io(i)
        sig = (io['in_shape'], op['dil'])
        if sig not in seen:
            seen.add(sig)
            out.append((i, nm, op, io))
    return out


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
@pytest.mark.parametrize('name,side,output_stride', [
    ('efficientnetv2-s', 256, 16), ('efficientnetv2-s', 256, 8), ('efficientnetv2-s', 224, 16),
    ('efficientnetv2-s', 224, 8), ('efficientnetv2-l', 256, 8),
    ('efficientnetv2-tiny', 72, 8)])  # 9x9 maps: phases of 5 and 4 rows / columns at d = 2, 3 and 2 at d = 4
def test_dilated_ops_vs_conv2d(H, precision, name, side, output_stride):
    pcfg, spec, sd = model_and_weights(name, output_stride, side)
    eng = device_model(name, output_stride, pcfg, 8, sd, precision).engine()
    st = port_ops.MODES[precision][0]
    g = torch.Generator().manual_seed(side + output_stride)
    ops = dilated_ops(eng, spec)
    assert ops and {op['dil'] for _, _, op, _ in ops} == ({2} if output_stride == 16 else {2, 4})
    worst = 0.0
    for i, nm, op, io in ops:
        assert eng.op_kernel(i) == _lib.DW_TMA_DIL, nm
        hh, ww, _c = io['out_shape']
        G = dw_plan(-(-hh // op['dil']), -(-ww // op['dil']))[0]
        assert G > 0, (nm, hh, ww)
        for batch in sorted({1, max(G - 1, 1), G + 1, 2 * G + 1}):
            x, _res, _sc = operands(io, batch, st, g, False)
            out = eng.debug_run_op(i, x)
            ref, tol = D.dw_layer_bound(sd, spec, nm, x.double(), precision)
            assert out.shape == ref.shape
            r, bad = port_ops.check_bound(out, ref, tol, precision)
            assert bad == 0, f'{nm} [{precision}] batch {batch}: {bad} elements outside the bound ({r:.2f})'
            worst = max(worst, r)
    # fc1 on the fused pooling of the device's own forward (test_gpu_ops16_vs_conv2d.test_fused_se_squeeze_on_the_forward)
    names = eng.op_names()
    crops = port.synthetic_inputs(2, side, seed=14)[0].cuda()
    p = 8 if st == torch.bfloat16 else 11
    for i, nm, op, io in ops:
        hh, ww, _c = io['out_shape']
        assert names[i + 1].endswith('.avgpool')
        d = eng.debug_run_ops(crops, i + 1).double()
        f1 = eng.debug_run_ops(crops, i + 3)[:, 0, 0].double()
        key = names[i + 2]
        w, b = sd[key + '.weight'], sd[key + '.bias']
        xm, xabs = d.mean(dim=(1, 2))[:, :w.shape[1]], d.abs().mean(dim=(1, 2))[:, :w.shape[1]]
        ref, tol = port_ops.se_fc_bound(xm, xabs, hh * ww + POOL_SLICES + 2, w, b, 'silu', 2.0 ** -p * (1 + 2.0 ** -p) * xabs)
        err = (f1[:, :w.shape[0]] - ref).abs()
        assert bool((err <= tol).all()), f'{key} [{precision}] after the dilated depthwise: {float((err / tol).max()):.2f}'
    print(f'{name}@{side} os{output_stride} [{precision}]: {len(ops)} dilated ops, worst |dev-ref|/tol {worst:.3f}')


def test_no_pool_kernel_at_output_stride_8(H):
    pcfg, spec, sd = model_and_weights('efficientnetv2-s', 8, 256)
    eng = device_model('efficientnetv2-s', 8, pcfg, 8, sd, 'bf16').engine()
    eng.profile_begin()
    eng.backbone(port.synthetic_inputs(2, 256, seed=3)[0].cuda())
    classes = eng.profile_end()
    assert 'pool_mean_kernel' not in classes, classes
    assert classes['dwconv_kernel']['launches'] > 0


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_phases_equal_the_undilated_kernel(H, precision):
    """tiny@64: backbone.1.5.0.block.1 is a d = 2 op on an 8x8 map at output stride 8 and a d = 1 op on a 4x4 map at output
    stride 32, with the same parameter keys and shapes.  Each phase X[:, py::2, px::2] of the dilated op must give, bit for
    bit, what dw3x3s1_tma_kernel gives on that sub-grid."""
    nm = 'backbone.1.5.0.block.1'
    pcfg8, spec8, sd8 = model_and_weights('efficientnetv2-tiny', 8, 64)
    pcfg32, _spec32, sd32 = model_and_weights('efficientnetv2-tiny', 32, 64)
    sd32 = {k: (sd8[k] if k.startswith(nm + '.') else v) for k, v in sd32.items()}
    e8 = device_model('efficientnetv2-tiny', 8, pcfg8, 8, sd8, precision).engine()
    e32 = device_model('efficientnetv2-tiny', 32, pcfg32, 8, sd32, precision).engine()
    i8, i32 = e8.op_names().index(nm), e32.op_names().index(nm)
    assert e8.op_kernel(i8) == _lib.DW_TMA_DIL and e32.op_kernel(i32) == _lib.DW_TMA
    assert e8.op_io(i8)['in_shape'] == (8, 8, 192) and e32.op_io(i32)['in_shape'] == (4, 4, 192)
    g = torch.Generator().manual_seed(5)
    for batch in (1, 3, 9):
        x = torch.randn(batch, 8, 8, 192, generator=g).to(port_ops.MODES[precision][0]).float().cuda()
        out8 = e8.debug_run_op(i8, x)
        for py in range(2):
            for px in range(2):
                out32 = e32.debug_run_op(i32, x[:, py::2, px::2].contiguous())
                assert torch.equal(out8[:, py::2, px::2], out32), (batch, py, px)


def test_create_rejects_l8_at_stride_test_32(H):
    stages, last = E.stage_table('l', True, output_stride=8)
    from metrabs_b200.engine import Engine, make_config
    with pytest.raises(_lib.MetrabsB200Error, match='output stride 8 but stride_test is 32'):
        Engine(make_config(metrabs_b200.Config(proc_side=256, stride_test=32), 24, stages=stages, last_channel=last))
