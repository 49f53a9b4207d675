"""GPU: every conv/GEMM kernel shape of the tensor-core modes against plain ``torch.nn.functional.conv2d`` arithmetic on
identical operands (oracle/port_ops.py restates one reference layer at a time) - NOT against other kernels of this repo.

* 'tf32x3' (tc32_conv_kernel: wgmma tf32, hi/lo split operands, three products, fp32 accumulate): vs fp64 conv2d,
  bar 5e-5 on ||.||inf/||ref||inf (fp32-chain quality; the 1e-3 joint bar of BASELINE.json is checked end to end in
  test_gpu_parity.py::test_full_models_parity_modes).
* 16-bit modes 'bf16' / 'fp16' (tensor cores: tc_conv_kernel, the TMA / strip / generic depthwise kernels, the stem kernel)
  and their CUDA-core twins 'bf16_simt' / 'fp16_simt' (conv_igemm_kernel, dwconv_kernel): vs fp64 conv2d at that mode's
  rounding points, element by element within port_ops.layer_bound (half an output ulp + the fp32 accumulation bound + the
  activation's own error), which a one-ulp defect such as the bf16 SiLU form in an fp16 kernel exceeds.
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


def _conv_ops(eng):
    """indices of the conv ops: stem, dense and depthwise (not the squeeze-excitation pool / fc ops)."""
    return [(i, nm) for i, nm in enumerate(eng.op_names()) if not nm.endswith(('.avgpool', '.fc1', '.fc2'))]


def _within_bound(sd, spec, nm, out, x, res, sc, precision):
    """-> worst |out - ref| / tol; asserts every element of the 16-bit device result is within port_ops.layer_bound."""
    ref, tol = port_ops.layer_bound(sd, spec, nm, x.double(), None if res is None else res.double(), sc, precision)
    worst, bad = port_ops.check_bound(out, ref, tol, precision)
    assert bad == 0, f'{nm} [{precision}]: {bad} elements outside the bound, worst |dev-ref|/tol {worst:.2f}'
    return worst


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-tiny', 64, 5), ('efficientnetv2-s', 256, 3),
                                             ('efficientnetv2-l', 384, 2),
                                             ('efficientnetv2-s', 224, 3),   # 7x7 last maps, 14x14 / 28x28 depthwise
                                             ('efficientnetv2-s', 160, 2)])  # 5x5 last maps, 10x10 / 20x20 depthwise
@pytest.mark.parametrize('precision', ['tf32x3', 'bf16', 'bf16_simt', 'fp16', 'fp16_simt'])
def test_tensor_core_ops_vs_conv2d(H, name, side, batch, precision):
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    eng = H.device_model(name, pcfg, 8, sd, precision=precision).engine()
    table = port_ops.effnet_op_table(spec)
    g = torch.Generator().manual_seed(3)
    st = port_ops.MODES[precision][0] if precision in port_ops.MODES else torch.float32
    seen, worst = set(), (0.0, None)
    for i, nm in _conv_ops(eng):
        io = eng.op_io(i)
        op = table[nm]
        sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], op['stride'], op['shift'], op['depthwise'], i == 0)
        if sig in seen:
            continue
        seen.add(sig)
        if i == 0:  # the stem takes NCHW crops in [0, 1]
            x = port.synthetic_inputs(batch, side, seed=len(seen))[0]
        else:
            x = torch.randn((batch,) + io['in_shape'], generator=g).to(st).float()
        res = torch.randn((batch,) + io['out_shape'], generator=g).to(st).float() if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g) if io['scale'] else None
        x, res, sc = (t.cuda() if t is not None else None for t in (x, res, sc))
        out = eng.debug_run_op(i, x, res, sc)
        if st != torch.float32:
            ratio = _within_bound(sd, spec, nm, out, x, res, sc, precision)
            if ratio > worst[0]:
                worst = (ratio, (nm, io))
            continue
        ref = port_ops.conv_layer_reference(sd, spec, nm, x, res, sc, precision='exact', dtype=torch.float64)
        err = port.relative_error(out.cpu(), ref.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        assert err < 5e-5, f'op {i} {nm} {io}: 3xTF32 vs fp64 conv2d rel err {err:.3e}'
    assert any(table[nm]['depthwise'] for i, nm in _conv_ops(eng))
    what = 'rel err' if st == torch.float32 else '|dev-ref|/tol'
    print(f'{name}@{side} [{precision}]: {len(seen)} distinct ops, worst {what} vs conv2d {worst[0]:.3g} at {worst[1]}')


@pytest.mark.parametrize('precision', ['tf32x3', 'bf16', 'bf16_simt', 'fp16', 'fp16_simt'])
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
            'backbone.1.1.1.block.0',   # 32->32 3x3 @128^2   (the latency-bound stage-1 conv)
            'backbone.1.4.1.block.1',   # 768 depthwise 3x3 @16^2 (TMA-staged in the tensor-core modes)
            'backbone.1.4.0.block.1']   # 768 depthwise 3x3 stride 2 @32^2 -> 16^2 (strip kernel)
    names = eng.op_names()
    st = port_ops.MODES[precision][0] if precision in port_ops.MODES else torch.float32
    g = torch.Generator().manual_seed(11)
    for nm in want:
        i = names.index(nm)
        io = eng.op_io(i)
        x = torch.randn((batch,) + io['in_shape'], generator=g).to(st).float()
        res = torch.randn((batch,) + io['out_shape'], generator=g).to(st).float() if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g) if io['scale'] else None
        xc = x.cuda()
        rc = res.cuda() if res is not None else None
        scc = sc.cuda() if sc is not None else None
        out = eng.debug_run_op(i, xc, rc, scc)
        if st != torch.float32:
            ratio = _within_bound(sd, spec, nm, out, xc, rc, scc, precision)
            print(f'{nm} batch {batch} [{precision}]: worst |dev-ref|/tol {ratio:.3g}')
            del out, xc, rc
            torch.cuda.empty_cache()
            continue
        ref = port_ops.conv_layer_reference(sd, spec, nm, xc, rc, scc, precision='exact', dtype=torch.float32)
        err = port.relative_error(out.cpu(), ref.cpu())
        print(f'{nm} batch {batch} [{precision}]: rel err vs conv2d {err:.2e}')
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
