"""GPU: tc_conv3x3s1_kernel, the tensor-core kernel of the 3x3 stride-1 convs with Cin, Cout <= 64 (stage 1 of
EfficientNetV2, conv2_x of the ResNets), in bf16 and fp16.

* Selection: Engine.op_kernel reports tc_conv3x3s1_kernel for exactly the ops it takes (3x3, stride 1, dilation 1,
  Cin and Cout <= 64, SiLU or ReLU) and tc_conv_kernel for every other tensor-core op: 1x1, stride 2, dilated (ResNets at
  output stride 8), Cin or Cout > 64.  Both report the profiler class tc_conv_kernel.
* Values: every distinct op it takes, against the CUDA-core twin on identical 16-bit inputs (bf16 1e-2, fp16 1.5e-3 of
  ||.||inf/||ref||inf, the bounds of test_gpu_tc_persistent.py) and element by element against fp64 conv2d at the mode's
  rounding points (port_ops.layer_bound / port_resnet.layer_bound), for both engines.  Residual after SiLU
  (EfficientNetV2-S / -L, Cin 24 / 32), before ReLU (ResNet-18 basic blocks, Cin 64) and none (ResNet-18 / -50).
* Launch shapes: side 200 and 72 leave partial 16 x 8 tiles (stage 1 / conv2_x maps of 100 x 100, 50 x 50, 36 x 36,
  18 x 18); 1 crop runs fewer tiles than the grid, 97 crops a tile count that is not a multiple of twice the grid.

EfficientNetV2 runs at output stride 32 only; the ResNets at 32 and 8, where the later stages are dilated and must stay on
tc_conv_kernel."""
import pytest
import torch

from oracle import port, port_ops, port_resnet
from oracle import port_tf_backbones as tfb

pytestmark = pytest.mark.gpu

PRECISIONS = [('bf16', 'bf16_simt', torch.bfloat16, 1e-2), ('fp16', 'fp16_simt', torch.float16, 1.5e-3)]
SHAPES = [(200, 97), (72, 1)]


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def takes(op, io):
    """tc3x3s1_eligible (csrc/tc_gemm.cuh) on an op of the oracle's table"""
    cin, cout = io['in_shape'][2], io['out_shape'][2]
    return (op['kernel'] == 3 and op['stride'] == 1 and op['dil'] == 1 and cin <= 64 and cout <= 64
            and op['act'] in ('silu', 'relu'))


def check(e_tc, e_ref, table, bound_of, batch, dtype, bound, seed, prec, twin, side):
    """-> (names of the distinct ops checked, kinds of rejected tensor-core ops seen)"""
    from metrabs_b200 import _lib
    from tests.test_gpu_ops16_vs_conv2d import op_classes
    classes = op_classes(e_tc, side)
    g = torch.Generator().manual_seed(seed)
    seen, checked, rejected = set(), [], set()
    for i, nm in enumerate(e_tc.op_names()):
        if nm not in table:
            continue
        op, io = table[nm], e_tc.op_io(i)
        if not port_ops.tc_eligible(op, io['in_shape'][2], io['out_shape'][2]):
            continue
        k = e_tc.op_kernel(i)
        if not takes(op, io):
            # tc_conv_kernel, with or without the squeeze-excitation scale of a projection
            tc_conv = (_lib.TC_CONV_SE, _lib.SE_SCALE_TC_CONV) if io['scale'] else (_lib.TC_CONV,)
            assert k in tc_conv, (nm, io, k)
            if op['kernel'] == 3:
                rejected.add('stride 2' if op['stride'] == 2 else 'dilated' if op['dil'] > 1 else
                             'wide' if max(io['in_shape'][2], io['out_shape'][2]) > 64 else 'other')
            continue
        assert k == _lib.TC_CONV3X3S1, (nm, io, k)
        assert classes.get(nm, 'tc_conv_kernel') == 'tc_conv_kernel', (nm, classes[nm])
        sig = str((io['in_shape'], io['out_shape'], io['residual'], op['act'], op.get('res_first')))
        if sig in seen:
            continue
        seen.add(sig)
        x = torch.randn((batch,) + io['in_shape'], generator=g).to(dtype).float().cuda()
        res = torch.randn((batch,) + io['out_shape'], generator=g).to(dtype).float().cuda() if io['residual'] else None
        a = e_tc.debug_run_op(i, x, res)
        b = e_ref.debug_run_op(i, x, res)
        assert torch.isfinite(a).all(), nm
        err = port.relative_error(a.cpu(), b.cpu())
        assert err < bound, f'{nm} {io}: tc_conv3x3s1_kernel vs CUDA-core rel err {err:.3e}'
        ratio = {}
        for mode, dev in [(prec, a), (twin, b)]:
            ref, tol = bound_of(nm, x.double(), None if res is None else res.double(), mode)
            r, bad = port_ops.check_bound(dev, ref, tol, mode)
            assert bad == 0, f'{nm} {io} [{mode}]: {bad} elements outside the conv2d bound (worst ratio {r:.2f})'
            ratio[mode] = r
        print(f'{nm} {io} x{batch}: rel err vs twin {err:.2e}, worst |dev-ref|/tol {ratio}')
        checked.append((nm, io['residual'], op.get('res_first', False)))
        del a, b
    return checked, rejected


@pytest.mark.parametrize('prec,twin,dtype,bound', PRECISIONS)
@pytest.mark.parametrize('side,batch', SHAPES)
@pytest.mark.parametrize('name,cin', [('efficientnetv2-s', 24), ('efficientnetv2-l', 32)])
def test_conv3x3s1_effnetv2_stage1(H, name, cin, side, batch, prec, twin, dtype, bound):
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision=prec).engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision=twin).engine()

    def bound_of(nm, x, res, mode):
        return port_ops.layer_bound(sd, spec, nm, x, res, None, mode)

    checked, rejected = check(e_tc, e_ref, port_ops.effnet_op_table(spec), bound_of, batch, dtype, bound, 21, prec, twin,
                              side)
    # stage 1: FusedMBConv without expansion, Cin = Cout, residual added after SiLU
    assert [c[0] for c in checked] == ['backbone.1.1.0.block.0'] and checked[0][1], checked
    assert e_tc.op_io(e_tc.op_names().index('backbone.1.1.0.block.0'))['in_shape'] == (side // 2, side // 2, cin)
    assert 'stride 2' in rejected and 'wide' in rejected, rejected


@pytest.mark.parametrize('prec,twin,dtype,bound', PRECISIONS)
@pytest.mark.parametrize('side,batch', SHAPES)
@pytest.mark.parametrize('stride', [32, 8])
@pytest.mark.parametrize('depth', [18, 50])
def test_conv3x3s1_resnet_conv2(H, depth, stride, side, batch, prec, twin, dtype, bound):
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, depth=8)
    if depth == 50:
        spec = tfb.ResNet50Spec(pcfg)
        sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
        e_tc = H.device_model_tf('resnet50', pcfg, 8, sd, precision=prec).engine()
        e_ref = H.device_model_tf('resnet50', pcfg, 8, sd, precision=twin).engine()
        table = port_ops.op_table(spec)

        def bound_of(nm, x, res, mode):
            return port_ops.layer_bound(sd, spec, nm, x, res, None, mode)
    else:
        from tests.test_gpu_resnet_family import device_model
        spec = port_resnet.ResNetSpec(pcfg, depth)
        sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
        e_tc = device_model(H, depth, pcfg, 8, sd, prec).engine()
        e_ref = device_model(H, depth, pcfg, 8, sd, twin).engine()
        table = port_resnet.op_table(spec)

        def bound_of(nm, x, res, mode):
            return port_resnet.layer_bound(sd, spec, nm, x, res, mode)

    checked, rejected = check(e_tc, e_ref, table, bound_of, batch, dtype, bound, 22 + stride, prec, twin, side)
    names = {c[0] for c in checked}
    assert checked and all(nm.startswith('backbone.conv2_') for nm in names), checked
    if depth == 18:  # basic blocks: a 3x3 + ReLU, and a 3x3 with the identity residual before ReLU
        assert ('backbone.conv2_block1_1_conv', False, False) in checked, checked
        assert any(c[1] and c[2] for c in checked), checked
        assert 'stride 2' in rejected, rejected
    else:  # bottleneck: the 3x3 between two 1x1s, no residual
        assert [c[0] for c in checked] == ['backbone.conv2_block1_2_conv'], checked
    if stride == 8:
        assert 'dilated' in rejected, rejected
