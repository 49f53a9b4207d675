"""GPU: the persistent tc_conv_kernel (one CTA per SM walking tiles N-fastest, two consumer warpgroups on alternate tiles)
against the CUDA-core twins on identical 16-bit inputs, on launches the small-batch per-op tests never reach:

* many tiles per CTA, with tile counts that are not a multiple of the grid or of 2 (one consumer warpgroup ends with one
  tile fewer): EfficientNetV2-L@256 stages 4-7 at 97 crops;
* Cout tails whose last N tile is partly filled: 192, 224 and 1344 (= 10.5 x 128) in the same network;
* mode-1 tiles whose 16 x 8 pixel box exceeds an 8 x 8 map, and ResNet-50 at stride 8 (dilated 3x3, residual before
  ReLU), at 37 and 9 crops.

Bounds: those of test_gpu_tc.py (bf16, 1e-2) and test_gpu_f16.py (fp16, 1.5e-3) on ||.||inf/||ref||inf against the twin,
and element by element against fp64 conv2d at the mode's rounding points (port_ops.layer_bound) for both engines."""
import pytest
import torch

from oracle import port, port_ops

pytestmark = pytest.mark.gpu

PRECISIONS = [('bf16', 'bf16_simt', torch.bfloat16, 1e-2), ('fp16', 'fp16_simt', torch.float16, 1.5e-3)]


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def _compare(e_tc, e_ref, dtype, bound, batch, seed, sig_of, keep, sd, spec, prec, twin):
    g = torch.Generator().manual_seed(seed)
    seen, worst = set(), (0.0, None)
    ratio = {prec: 0.0, twin: 0.0}
    for i, nm in enumerate(e_tc.op_names()):
        if nm.endswith(('.avgpool', '.fc1', '.fc2')) or i == 0:
            continue
        io = e_tc.op_io(i)
        if not keep(io):
            continue
        sig = str((io['in_shape'], io['out_shape'], io['residual'], io['scale'], sig_of(nm)))
        if sig in seen:
            continue
        seen.add(sig)
        x = torch.randn((batch,) + io['in_shape'], generator=g).to(dtype).float().cuda()
        res = torch.randn((batch,) + io['out_shape'], generator=g).to(dtype).float().cuda() if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g).cuda() if io['scale'] else None
        a = e_tc.debug_run_op(i, x, res, sc)
        b = e_ref.debug_run_op(i, x, res, sc)
        assert torch.isfinite(a).all(), (i, nm)
        err = port.relative_error(a.cpu(), b.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        assert err < bound, f'op {i} {nm} {io}: tensor-core vs CUDA-core rel err {err:.3e}'
        for mode, dev in [(prec, a), (twin, b)]:
            ref, tol = port_ops.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), sc, mode)
            r, bad = port_ops.check_bound(dev, ref, tol, mode)
            assert bad == 0, f'op {i} {nm} {io} [{mode}]: {bad} elements outside the conv2d bound (worst ratio {r:.2f})'
            ratio[mode] = max(ratio[mode], r)
        del a, b
    assert seen
    print(f'worst |dev-ref|/tol vs conv2d: {ratio}')
    return seen, worst


@pytest.mark.parametrize('prec,twin,dtype,bound', PRECISIONS)
def test_persistent_tc_effnetv2l_late_stages(H, prec, twin, dtype, bound):
    name, side, batch = 'efficientnetv2-l', 256, 97
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision=prec).engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision=twin).engine()
    couts = set()

    def keep(io):  # stages 4-7: 16 x 16 and 8 x 8 maps
        if io['out_shape'][0] > 16:
            return False
        couts.add(io['out_shape'][2])
        return True

    seen, worst = _compare(e_tc, e_ref, dtype, bound, batch, 6, lambda nm: nm.rsplit('.', 1)[-1], keep, sd, spec, prec, twin)
    assert {192, 224, 1344} <= couts, couts
    print(f'{name}@{side} x{batch} {prec}: {len(seen)} op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')


@pytest.mark.parametrize('prec,twin,dtype,bound', PRECISIONS)
@pytest.mark.parametrize('side,batch', [(64, 37), (256, 9)])
def test_persistent_tc_resnet50_stride8(H, prec, twin, dtype, bound, side, batch):
    from oracle import port_tf_backbones as tfb
    pcfg = port.PathConfig(proc_side=side, stride_test=8, depth=8)
    spec = tfb.ResNet50Spec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model_tf('resnet50', pcfg, 8, sd, precision=prec).engine()
    e_ref = H.device_model_tf('resnet50', pcfg, 8, sd, precision=twin).engine()
    seen, worst = _compare(e_tc, e_ref, dtype, bound, batch, 7, lambda nm: nm.rsplit('_', 2)[-2:], lambda io: True, sd, spec,
                           prec, twin)
    print(f'resnet50 s8 @{side} x{batch} {prec}: {len(seen)} op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')
