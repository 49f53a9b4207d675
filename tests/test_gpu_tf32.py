"""GPU: every conv/GEMM kernel shape of the tensor-core modes against plain ``torch.nn.functional.conv2d`` arithmetic on
identical operands (oracle/port_ops.py restates one reference layer at a time) - NOT against other kernels of this repo.

* 'tf32x3' (tc32_conv_kernel: wgmma tf32, hi/lo split operands, three products, fp32 accumulate): vs fp64 conv2d,
  bar 5e-5 on ||.||inf/||ref||inf (fp32-chain quality; the 1e-3 joint bar of BASELINE.json is checked end to end in
  test_gpu_parity.py::test_full_models_parity_modes).
* 'bf16' (tc_conv_kernel: kind::f16 bf16 operands, fp32 accumulate, bf16 store): vs conv2d on the same bf16-rounded input
  and the same bf16-rounded BN-folded weights, wide accumulation; bar = one bf16 ulp per element (the device rounds once
  after bias + activation + residual; tanh.approx SiLU error 2^-11 sits below it).
Large-batch cases (64 / 256 crops: different N-tile widths, multi-wave persistent tile walks) run the heaviest EffNetV2-L
shapes against conv2d on the GPU (fp32, TF32 disabled)."""
import pytest
import torch

from oracle import port, port_ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def _gemm_ops(eng):
    """indices of the conv ops that run on the tensor-core kernels (not stem, depthwise, squeeze-excitation)."""
    out = []
    for i, nm in enumerate(eng.op_names()):
        if i == 0 or nm.endswith(('.avgpool', '.fc1', '.fc2')):
            continue
        out.append((i, nm))
    return out


def _ulp_bf16_ok(dev, ref):
    """|dev - bf16(ref)| <= one bf16 ulp of the reference magnitude (plus a floor for values near zero)."""
    ref = ref.float()
    tol = ref.abs() * 2.0 ** -7 + 2.0 ** -9
    return bool(((dev.float() - ref).abs() <= tol).all())


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-tiny', 64, 5), ('efficientnetv2-s', 256, 3),
                                             ('efficientnetv2-l', 384, 2)])
@pytest.mark.parametrize('precision', ['tf32x3', 'bf16'])
def test_tensor_core_ops_vs_conv2d(H, name, side, batch, precision):
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    eng = H.device_model(name, pcfg, 8, sd, precision=precision).engine()
    table = port_ops.effnet_op_table(spec)
    g = torch.Generator().manual_seed(3)
    seen, worst = set(), (0.0, None)
    for i, nm in _gemm_ops(eng):
        io = eng.op_io(i)
        if table[nm]['depthwise']:
            continue
        sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], table[nm]['stride'], table[nm]['shift'])
        if sig in seen:
            continue
        seen.add(sig)
        x = torch.randn((batch,) + io['in_shape'], generator=g)
        res = torch.randn((batch,) + io['out_shape'], generator=g) if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g) if io['scale'] else None
        if precision == 'bf16':
            x = x.bfloat16().float()
            res = res.bfloat16().float() if res is not None else None
        out = eng.debug_run_op(i, x.cuda(), res.cuda() if res is not None else None, sc.cuda() if sc is not None else None)
        ref = port_ops.conv_layer_reference(sd, spec, nm, x.cuda(), res.cuda() if res is not None else None,
                                            sc.cuda() if sc is not None else None,
                                            precision='bf16' if precision == 'bf16' else 'exact', dtype=torch.float64)
        err = port.relative_error(out.cpu(), ref.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        if precision == 'bf16':
            assert _ulp_bf16_ok(out, ref), f'op {i} {nm} {io}: more than one bf16 ulp from conv2d (rel err {err:.3e})'
        else:
            assert err < 5e-5, f'op {i} {nm} {io}: 3xTF32 vs fp64 conv2d rel err {err:.3e}'
    print(f'{name}@{side} [{precision}]: {len(seen)} distinct op shapes, worst rel err vs conv2d {worst[0]:.2e} at {worst[1]}')


@pytest.mark.parametrize('precision', ['tf32x3', 'bf16'])
@pytest.mark.parametrize('batch', [64, 256])
def test_heaviest_shapes_at_bench_batch(H, batch, precision):
    """The five heaviest EfficientNetV2-L@256 GEMM shapes (FLOP share) at 64 and 256 crops: the tile plan (N-tile width,
    persistent multi-wave tile walk, ring depth) differs from the batch-2 plan the other tests see."""
    name, side = 'efficientnetv2-l', 256
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model(name, pcfg, 8, sd, precision=precision).engine()
    table = port_ops.effnet_op_table(spec)
    want = ['backbone.1.2.1.block.0',   # 64->256 3x3 @64^2   (FusedMBConv expand)
            'backbone.1.2.1.block.1',   # 256->64 1x1 @64^2   (FusedMBConv project, residual)
            'backbone.1.3.1.block.0',   # 96->384 3x3 @32^2
            'backbone.1.5.1.block.0',   # 224->1344 1x1 @16^2 (MBConv expand)
            'backbone.1.5.1.block.3',   # 1344->224 1x1 @16^2 (MBConv project, SE scale, residual)
            'backbone.1.1.1.block.0']   # 32->32 3x3 @128^2   (the latency-bound stage-1 conv)
    names = eng.op_names()
    g = torch.Generator().manual_seed(11)
    for nm in want:
        i = names.index(nm)
        io = eng.op_io(i)
        x = torch.randn((batch,) + io['in_shape'], generator=g)
        res = torch.randn((batch,) + io['out_shape'], generator=g) if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g) if io['scale'] else None
        if precision == 'bf16':
            x = x.bfloat16().float()
            res = res.bfloat16().float() if res is not None else None
        xc = x.cuda()
        rc = res.cuda() if res is not None else None
        scc = sc.cuda() if sc is not None else None
        out = eng.debug_run_op(i, xc, rc, scc)
        ref = port_ops.conv_layer_reference(sd, spec, nm, xc, rc, scc, precision='bf16' if precision == 'bf16' else 'exact',
                                            dtype=torch.float32)
        err = port.relative_error(out.cpu(), ref.cpu())
        print(f'{nm} batch {batch} [{precision}]: rel err vs conv2d {err:.2e}')
        if precision == 'bf16':
            assert _ulp_bf16_ok(out, ref), (nm, err)
        else:
            assert err < 5e-5, (nm, err)
        del out, ref, xc, rc
        torch.cuda.empty_cache()


def test_tf32x3_head_and_tf_backbones(H):
    """3xTF32 on the other BASELINE configs: the head GEMM + NHWC soft-argmax (J=122: N=1098 padded to 1100) and the
    TF-only backbones (ResNet-50 dilated 3x3 / strided 1x1 / residual-before-ReLU; MobileNetV3 hard-swish)."""
    from oracle import port_tf_backbones as tfb
    for kind, cfgkw, j, batch in [('resnet50', dict(proc_side=256, stride_test=8, depth=32), 24, 2),
                                  ('mobilenetv3-small', dict(proc_side=256, stride_test=32, depth=8), 8, 4)]:
        pcfg = port.PathConfig(**cfgkw)
        spec = tfb.ResNet50Spec(pcfg) if kind == 'resnet50' else tfb.MobileNetV3SmallSpec(pcfg)
        sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
        crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
        stages = {}
        with torch.inference_mode():
            ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
        m = H.device_model_tf(kind, pcfg, j, sd, precision='tf32x3')
        out = m((crops.cuda(), k.cuda()))
        e_feat = H.rel_err(m.engine().backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
        e_out = H.rel_err(out, ref)
        print(f'{kind} [tf32x3]: features {e_feat:.2e}, joints {e_out:.2e}')
        assert e_feat < 1e-3 and e_out < 1e-3
