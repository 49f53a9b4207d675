"""GPU: the wgmma tensor-core kernels (MTB_PRECISION_BF16_TC) against the CUDA-core kernels on IDENTICAL bf16 inputs
and bf16-rounded weights (MTB_PRECISION_BF16_SIMT; those kernels are themselves pinned to the oracle in fp32 mode by
test_gpu_parity.py), and the fused head against the oracle on bf16-rounded operands.

Tolerances: both paths accumulate in fp32 and round the output once to bf16, so they may differ by one bf16 ulp
(2^-8 relative) per element -> 1e-2 on ||.||inf/||ref||inf; a descriptor / swizzle / tiling bug gives O(1) errors."""
import pytest
import torch

from oracle import port
from tests.test_gpu_forward_ops16 import check_head_per_coordinate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-tiny', 64, 5), ('efficientnetv2-s', 256, 3),
                                             ('efficientnetv2-l', 384, 2)])
def test_tc_ops_match_cuda_core_ops(H, name, side, batch):
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision='bf16').engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision='bf16_simt').engine()
    names = e_tc.op_names()
    g = torch.Generator().manual_seed(3)
    seen, worst = set(), (0.0, None)
    for i, nm in enumerate(names):
        if nm.endswith(('.avgpool', '.fc1', '.fc2')) or i == 0:
            continue
        io = e_tc.op_io(i)
        sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], nm.rsplit('.', 1)[-1])
        if sig in seen:
            continue
        seen.add(sig)
        x = torch.randn((batch,) + io['in_shape'], generator=g).bfloat16().float().cuda()
        res = torch.randn((batch,) + io['out_shape'], generator=g).bfloat16().float().cuda() if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g).cuda() if io['scale'] else None
        a = e_tc.debug_run_op(i, x, res, sc)
        b = e_ref.debug_run_op(i, x, res, sc)
        err = port.relative_error(a.cpu(), b.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        assert err < 1e-2, f'op {i} {nm} {io}: tensor-core vs CUDA-core rel err {err:.3e}'
    print(f'{name}@{side}: {len(seen)} distinct op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')


@pytest.mark.parametrize('kind,cfgkw,batch', [
    ('resnet50', dict(proc_side=256, stride_test=8, depth=8), 2),     # dilated 3x3, strided 1x1, residual BEFORE ReLU
    ('resnet50', dict(proc_side=128, stride_test=32, depth=8), 3),
    ('mobilenetv3-small', dict(proc_side=256, stride_test=32, depth=8), 3),  # hard-swish epilogues, 5x5 depthwise (CUDA cores)
])
def test_tc_ops_match_cuda_core_ops_tf_backbones(H, kind, cfgkw, batch):
    from oracle import port_tf_backbones as tfb
    pcfg = port.PathConfig(**cfgkw)
    spec = tfb.ResNet50Spec(pcfg) if kind == 'resnet50' else tfb.MobileNetV3SmallSpec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model_tf(kind, pcfg, 8, sd, precision='bf16').engine()
    e_ref = H.device_model_tf(kind, pcfg, 8, sd, precision='bf16_simt').engine()
    g = torch.Generator().manual_seed(4)
    seen, worst = set(), (0.0, None)
    for i, nm in enumerate(e_tc.op_names()):
        if nm.endswith(('.avgpool', '.fc1', '.fc2')) or i == 0:
            continue
        io = e_tc.op_io(i)
        sig = (io['in_shape'], io['out_shape'], io['residual'], io['scale'], nm.rsplit('_', 2)[-2:] if kind == 'resnet50' else nm.rsplit('.', 1)[-1])
        sig = str(sig)
        if sig in seen:
            continue
        seen.add(sig)
        x = torch.randn((batch,) + io['in_shape'], generator=g).bfloat16().float().cuda()
        res = torch.randn((batch,) + io['out_shape'], generator=g).bfloat16().float().cuda() if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g).cuda() if io['scale'] else None
        a = e_tc.debug_run_op(i, x, res, sc)
        b = e_ref.debug_run_op(i, x, res, sc)
        err = port.relative_error(a.cpu(), b.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        assert err < 1e-2, f'op {i} {nm} {io}: tensor-core vs CUDA-core rel err {err:.3e}'
    print(f'{kind} {cfgkw}: {len(seen)} distinct op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')


def test_fused_depthwise_pooling_matches_separate_pool(H):
    """BF16_TC fuses the SE squeeze into the depthwise kernel (block reduction -> partial slices summed by fc1 in a
    fixed order); BF16_SIMT runs the plain depthwise kernel and a separate pooling pass.  Compared at the output of the
    squeeze-excitation (the per-channel scale after fc2) through the op chain of the first MBConv blocks (short prefix,
    so upstream bf16 drift stays small)."""
    name, side, batch = 'efficientnetv2-s', 256, 3
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision='bf16').engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision='bf16_simt').engine()
    crops, _ = port.synthetic_inputs(batch, side, seed=0)
    pools = [i for i, n in enumerate(e_tc.op_names()) if n.endswith('.avgpool')][:3]
    for i in pools:
        a = e_tc.debug_run_ops(crops.cuda(), i + 3)   # avgpool, fc1, fc2 -> scale [B,1,1,C]
        b = e_ref.debug_run_ops(crops.cuda(), i + 3)
        err = port.relative_error(a.cpu(), b.cpu())
        assert err < 3e-2, (i, err)


@pytest.mark.parametrize('channels,hw,j,depth,batch', [
    (1280, 8, 24, 8, 9),      # EffNetV2 @256: P=64, 4 crops per MMA, ragged last group
    (1280, 8, 122, 8, 5),     # c4: N=1098 -> 9 channel tiles, last one ragged
    (1280, 12, 24, 8, 3),     # c3: P=144, one crop per MMA (N=144)
    (256, 32, 24, 8, 2),      # P=1024: 4 pixel tiles per crop, state carried across tiles
    (2048, 32, 24, 32, 2),    # c2/c5b geometry: N=792, D=32
    (64, 6, 8, 8, 7),         # P=36: crop boundaries inside a 16-column chunk (element-wise path)
    (1024, 8, 8, 8, 4),       # c1 geometry
    (1280, 6, 24, 8, 256),    # P=36 at the benchmark batch: crop-straddling chunks over 256 crops
    (1280, 7, 24, 8, 5),      # P=49: no fused plan (tc_head_plan), the 16-bit unfused fallback
])
def test_fused_head_vs_oracle(H, channels, hw, j, depth, batch):
    """bf16 head against port.heads (2e-4 of the largest coordinate) and, coordinate by coordinate, against
    port_ops.decode_bound on the operands the device multiplies (bf16 features and weight, fp32 bias)."""
    import metrabs_b200
    from metrabs_b200 import _lib
    from metrabs_b200.engine import Engine, make_config
    stride = 256 // hw if 256 % hw == 0 else 32
    side = hw * stride
    cfg = metrabs_b200.Config(proc_side=side, stride_test=stride, depth=depth, precision='bf16')
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, depth=depth)
    feats, sd = port.head_only_inputs(batch, channels, hw, j, depth, seed=1)
    eng = Engine(make_config(cfg, j, arch=_lib.ARCH_HEAD_ONLY, feature_channels=channels))
    eng.load_state_dict(sd)
    f16 = feats.permute(0, 2, 3, 1).contiguous().bfloat16().cuda()
    eng.profile_begin()
    c2d, c3d = eng.head_decode(f16)
    head_cls = set(eng.profile_end())
    fused = tc_head_plan_fits(hw * hw)
    assert head_cls == ({'tc_head_softargmax_kernel'} if fused
                        else {'head_conv(conv_igemm_kernel)', 'softargmax_bhwn_kernel'}), head_cls
    ref2d, ref3d = port.heads(sd, feats, pcfg, j)
    e2, e3 = H.rel_err(c2d, ref2d), H.rel_err(c3d, ref3d)
    w2, w3 = check_head_per_coordinate(head_operands(sd, torch.bfloat16), f16, pcfg, c2d, c3d, False, j)
    print(f'C={channels} hw={hw} J={j} D={depth} x{batch} ({"fused" if fused else "unfused"}): coords2d {e2:.2e} '
          f'coords3d {e3:.2e}, worst |dev-ref|/tol {w2:.3f} / {w3:.3f}, launches {eng.last_launch_count}')
    assert e2 < 2e-4 and e3 < 2e-4
    # the CUDA-core head on the same bf16 operands agrees too
    cfg_s = metrabs_b200.Config(proc_side=side, stride_test=stride, depth=depth, precision='bf16_simt')
    eng_s = Engine(make_config(cfg_s, j, arch=_lib.ARCH_HEAD_ONLY, feature_channels=channels))
    eng_s.load_state_dict(sd)
    s2d, s3d = eng_s.head_decode(f16)
    assert H.rel_err(s2d, ref2d) < 2e-4 and H.rel_err(s3d, ref3d) < 2e-4
    check_head_per_coordinate(head_operands(sd, torch.bfloat16), f16, pcfg, s2d, s3d, False, j)


def tc_head_plan_fits(P):
    """tc_head_plan (csrc/tc_gemm.cuh): a fused head tile of c whole crops with c*P % 16 == 0 (P <= 256), or whole
    256-pixel tiles of one crop."""
    if P <= 256:
        return any(c * P % 16 == 0 for c in range(1, 256 // P + 1))
    return P % 256 == 0


def head_operands(sd, st):
    """the head weight rounded to the 16-bit type and the fp32 bias, fp64 on the device"""
    return {'heatmap_heads.conv_final.weight': sd['heatmap_heads.conv_final.weight'].float().to(st).double().cuda(),
            'heatmap_heads.conv_final.bias': sd['heatmap_heads.conv_final.bias'].float().double().cuda()}


def test_bf16_forward_deviation_is_reported(H):
    """Throughput mode end to end.  An untrained 170-conv net amplifies bf16 rounding (SURVEY.md 7.2-1), so the
    deviation from the fp32 oracle is REPORTED, not held to 1e-3; what is asserted is that the tensor-core chain stays
    as close to fp32 as the CUDA-core bf16 chain does (same storage precision, same weights)."""
    name, side, j, batch = 'efficientnetv2-s', 256, 24, 4
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, j, seed=0)
    crops, k = port.synthetic_inputs(batch, side, seed=0)
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    errs = {}
    for prec in ('bf16', 'bf16_simt'):
        m = H.device_model(name, pcfg, j, sd, precision=prec)
        feats = m.engine().backbone(crops.cuda()).float().permute(0, 3, 1, 2)
        out = m((crops.cuda(), k.cuda()))
        assert torch.isfinite(out).all()
        errs[prec] = (H.rel_err(feats, stages['features']), H.rel_err(out, ref))
    print('bf16 deviation from the fp32 oracle (features, joints):', errs)
    assert errs['bf16'][0] < max(3 * errs['bf16_simt'][0], 0.05)
    # the same scale from the CPU: the reference arithmetic with bf16 STORAGE emulated (oracle/port_bf16.py) deviates from
    # the fp32 oracle as much as the device does - reported, not asserted (two bf16 evaluations of a chaotic map agree with
    # each other no better than either agrees with fp32)
    from oracle import port_bf16
    st16 = {}
    with torch.inference_mode():
        out16 = port_bf16.metrabs_forward_bf16(sd, spec, pcfg, j, crops, k, stages=st16)
    print('CPU bf16-storage restatement vs the fp32 oracle (features, joints):',
          (port.relative_error(st16['features'], stages['features']), port.relative_error(out16, ref)))

