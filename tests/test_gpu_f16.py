"""GPU: the fp16 tensor-core mode (MTB_PRECISION_F16_TC, Config(precision='fp16')) - the arithmetic the reference deploys
under fp16 autocast - against its CUDA-core twin (MTB_PRECISION_F16_SIMT: the same fp16 storage and fp16-rounded weights,
every conv on fp32 FMA) on IDENTICAL fp16 inputs, the fused head against the oracle on fp16-rounded operands, and the
whole forward against the fp32 oracle and the bf16 mode.

Tolerances: both paths accumulate in fp32 and round the output once to fp16, so they may differ by one fp16 ulp (up to
2^-10 relative) per element; 1.5e-3 on ||.||inf/||ref||inf is about 3 fp16 ulps, the ulp multiple of the bf16 tests'
1e-2 (tests/test_gpu_tc.py).  A descriptor / swizzle / element-type bug gives O(1) errors."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import port
from tests.test_gpu_forward_ops16 import check_head_per_coordinate
from tests.test_gpu_tc import head_operands, tc_head_plan_fits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OP_TOL = 1.5e-3


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def _h(shape, g):
    return torch.randn(shape, generator=g).half().float().cuda()


def _compare_ops(e_tc, e_ref, g, batch, sig_of):
    seen, worst = set(), (0.0, None)
    for i, nm in enumerate(e_tc.op_names()):
        if nm.endswith(('.avgpool', '.fc1', '.fc2')) or i == 0:
            continue
        io = e_tc.op_io(i)
        sig = str((io['in_shape'], io['out_shape'], io['residual'], io['scale'], sig_of(nm)))
        if sig in seen:
            continue
        seen.add(sig)
        x = _h((batch,) + io['in_shape'], g)
        res = _h((batch,) + io['out_shape'], g) if io['residual'] else None
        sc = torch.rand(batch, io['in_shape'][2], generator=g).cuda() if io['scale'] else None
        a = e_tc.debug_run_op(i, x, res, sc)
        b = e_ref.debug_run_op(i, x, res, sc)
        assert torch.isfinite(a).all(), (i, nm)
        err = port.relative_error(a.cpu(), b.cpu())
        if err > worst[0]:
            worst = (err, (nm, io))
        assert err < OP_TOL, f'op {i} {nm} {io}: fp16 tensor-core vs CUDA-core rel err {err:.3e}'
    return seen, worst


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-tiny', 64, 5), ('efficientnetv2-s', 256, 3),
                                             ('efficientnetv2-l', 384, 2)])
def test_f16_tc_ops_match_cuda_core_ops(H, name, side, batch):
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision='fp16').engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision='fp16_simt').engine()
    assert e_tc.feature_dtype == torch.float16 and e_ref.feature_dtype == torch.float16
    seen, worst = _compare_ops(e_tc, e_ref, torch.Generator().manual_seed(3), batch, lambda nm: nm.rsplit('.', 1)[-1])
    print(f'{name}@{side}: {len(seen)} distinct op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')


@pytest.mark.parametrize('kind,cfgkw,batch', [
    ('resnet50', dict(proc_side=256, stride_test=8, depth=8), 2),     # dilated 3x3, strided 1x1, residual BEFORE ReLU
    ('resnet50', dict(proc_side=128, stride_test=32, depth=8), 3),
    ('mobilenetv3-small', dict(proc_side=256, stride_test=32, depth=8), 3),  # hard-swish epilogues, 5x5 depthwise (CUDA cores)
])
def test_f16_tc_ops_match_cuda_core_ops_tf_backbones(H, kind, cfgkw, batch):
    from oracle import port_tf_backbones as tfb
    pcfg = port.PathConfig(**cfgkw)
    spec = tfb.ResNet50Spec(pcfg) if kind == 'resnet50' else tfb.MobileNetV3SmallSpec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model_tf(kind, pcfg, 8, sd, precision='fp16').engine()
    e_ref = H.device_model_tf(kind, pcfg, 8, sd, precision='fp16_simt').engine()
    sig_of = (lambda nm: nm.rsplit('_', 2)[-2:]) if kind == 'resnet50' else (lambda nm: nm.rsplit('.', 1)[-1])
    seen, worst = _compare_ops(e_tc, e_ref, torch.Generator().manual_seed(4), batch, sig_of)
    print(f'{kind} {cfgkw}: {len(seen)} distinct op shapes, worst rel err {worst[0]:.2e} at {worst[1]}')


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-s', 256, 3), ('efficientnetv2-l', 256, 2),
                                             ('efficientnetv2-tiny', 64, 5), ('efficientnetv2-l', 32, 3)])
def test_f16_fused_block_is_bit_equal_to_two_launches(H, name, side, batch):
    """fmb_kernel in fp16: the same MMA order and the same roundings as its two tc_conv_kernel launches."""
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model(name, pcfg, 8, sd, precision='fp16').engine()
    g = torch.Generator().manual_seed(5)
    seen = set()
    for i in range(len(eng.op_names())):
        if not eng.op_is_fused_block(i):
            continue
        io = eng.op_io(i)
        if io['in_shape'] in seen:
            continue
        seen.add(io['in_shape'])
        x = _h((batch,) + io['in_shape'], g)
        out = eng.debug_run_fused_block(i, x)
        mid = eng.debug_run_op(i, x)
        two = eng.debug_run_op(i + 1, mid, x if eng.op_io(i + 1)['residual'] else None)
        assert torch.isfinite(out).all()
        d = (out - two).abs()
        print(f'{name}@{side} op {i} {io["in_shape"]}: {float((d == 0).float().mean()) * 100:.2f} % bit-equal, '
              f'max diff {float(d.max()):.3e}')
        assert torch.equal(out, two), (i, float(d.max()))
    assert seen, 'no fused FusedMBConv block in this model'


def test_f16_fused_depthwise_pooling_matches_separate_pool(H):
    """F16_TC fuses the SE squeeze into the depthwise kernel; F16_SIMT runs the plain depthwise kernel and a separate pooling
    pass.  Compared at the SE output (the per-channel scale after fc2) through the op chain of the first MBConv blocks: the
    bf16 test's 3e-2 scaled by the 3 extra significand bits of fp16."""
    name, side, batch = 'efficientnetv2-s', 256, 3
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=2)
    e_tc = H.device_model(name, pcfg, 8, sd, precision='fp16').engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision='fp16_simt').engine()
    crops, _ = port.synthetic_inputs(batch, side, seed=0)
    pools = [i for i, n in enumerate(e_tc.op_names()) if n.endswith('.avgpool')][:3]
    assert pools
    for i in pools:
        a = e_tc.debug_run_ops(crops.cuda(), i + 3)   # avgpool, fc1, fc2 -> scale [B,1,1,C]
        b = e_ref.debug_run_ops(crops.cuda(), i + 3)
        err = port.relative_error(a.cpu(), b.cpu())
        print(f'SE scale after op {i}: fused vs separate pool {err:.2e}')
        assert err < 3e-2 / 8, (i, err)


@pytest.mark.parametrize('channels,hw,j,depth,batch', [
    (1280, 8, 24, 8, 9),
    (1280, 8, 122, 8, 5),
    (1280, 12, 24, 8, 3),
    (256, 32, 24, 8, 2),
    (2048, 32, 24, 32, 2),
    (64, 6, 8, 8, 7),
    (1024, 8, 8, 8, 4),
    (1280, 6, 24, 8, 256),
    (1280, 7, 24, 8, 5),
])
def test_f16_fused_head_vs_oracle(H, channels, hw, j, depth, batch):
    """The geometries of test_gpu_tc.test_fused_head_vs_oracle, with features and head weights rounded to fp16: 2e-4 of
    the largest coordinate, and every coordinate within port_ops.decode_bound."""
    import metrabs_b200
    from metrabs_b200 import _lib
    from metrabs_b200.engine import Engine, make_config
    stride = 256 // hw if 256 % hw == 0 else 32
    side = hw * stride
    pcfg = port.PathConfig(proc_side=side, stride_test=stride, depth=depth)
    feats, sd = port.head_only_inputs(batch, channels, hw, j, depth, seed=1)
    feats = feats.half().float()
    sd = dict(sd)
    sd['heatmap_heads.conv_final.weight'] = sd['heatmap_heads.conv_final.weight'].half().float()
    ref2d, ref3d = port.heads(sd, feats, pcfg, j)
    for prec in ('fp16', 'fp16_simt'):
        cfg = metrabs_b200.Config(proc_side=side, stride_test=stride, depth=depth, precision=prec)
        eng = Engine(make_config(cfg, j, arch=_lib.ARCH_HEAD_ONLY, feature_channels=channels))
        eng.load_state_dict(sd)
        f16 = feats.permute(0, 2, 3, 1).contiguous().half().cuda()
        eng.profile_begin()
        c2d, c3d = eng.head_decode(f16)
        head_cls = set(eng.profile_end())
        fused = prec == 'fp16' and tc_head_plan_fits(hw * hw)
        assert head_cls == ({'tc_head_softargmax_kernel'} if fused
                            else {'head_conv(conv_igemm_kernel)', 'softargmax_bhwn_kernel'}), (prec, head_cls)
        e2, e3 = H.rel_err(c2d, ref2d), H.rel_err(c3d, ref3d)
        w2, w3 = check_head_per_coordinate(head_operands(sd, torch.float16), f16, pcfg, c2d, c3d, False, j)
        print(f'[{prec}] C={channels} hw={hw} J={j} D={depth} x{batch}: coords2d {e2:.2e} coords3d {e3:.2e}, '
              f'worst |dev-ref|/tol {w2:.3f} / {w3:.3f}, launches {eng.last_launch_count}')
        assert e2 < 2e-4 and e3 < 2e-4, (prec, e2, e3)


def test_f16_forward_vs_oracle_and_bf16(H):
    """End to end on EfficientNetV2-S@256: the fp16 features are as close to the fp32 oracle as the CUDA-core fp16 chain's
    and several times closer than the bf16 mode's.  Joint errors on untrained weights are chaotic: printed, not asserted."""
    name, side, j, batch = 'efficientnetv2-s', 256, 24, 4
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, j, seed=0)
    crops, k = port.synthetic_inputs(batch, side, seed=0)
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    errs = {}
    for prec in ('fp16', 'fp16_simt', 'bf16'):
        m = H.device_model(name, pcfg, j, sd, precision=prec)
        eng = m.engine()
        feats = eng.backbone(crops.cuda())
        assert feats.dtype == (torch.bfloat16 if prec == 'bf16' else torch.float16)
        out = m((crops.cuda(), k.cuda()))
        assert torch.isfinite(out).all()
        errs[prec] = (H.rel_err(feats.float().permute(0, 3, 1, 2), stages['features']), H.rel_err(out, ref))
        if prec == 'fp16':
            # the reference's head entry point on the device features, and the host / pipelined forwards
            c2d, c3d = m.heatmap_heads(feats.float().permute(0, 3, 1, 2))
            assert torch.isfinite(c2d).all() and torch.isfinite(c3d).all()
            host = eng.forward_host(crops, k)
            assert torch.equal(host, out.cpu())
            out_host = torch.empty(batch, j, 3).pin_memory()
            eng.forward_host_submit(crops.pin_memory(), k.pin_memory(), out_host, 0)
            eng.forward_host_wait(0)
            assert torch.equal(out_host, out.cpu())
    print('deviation from the fp32 oracle (features, joints):', errs)
    assert errs['fp16'][0] < max(3 * errs['fp16_simt'][0], 0.01)
    assert errs['fp16'][0] < 0.25 * errs['bf16'][0]


def test_f16_latent_point_model_runs(H, tmp_path):
    """transform_coords with an affine-combining autoencoder head, in fp16"""
    import numpy as np
    from oracle import port_latents
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'latents_tiny_s64.npz'))
    J, L, B, S = int(g['n_joints']), int(g['n_latents']), int(g['batch']), int(g['proc_side'])
    path = str(tmp_path / 'affine_tiny.npz')
    np.savez(path, w1=g['w1'], w2=g['w2'])
    spec = port.effnet_spec('efficientnetv2-tiny')
    sd = port.make_effnet_state_dict(spec, port.PathConfig(proc_side=S), L, seed=0)
    m = H.device_model('efficientnetv2-tiny', port.PathConfig(proc_side=S, affine_weights=path, transform_coords=True), J, sd,
                       precision='fp16')
    crops, k = port.synthetic_inputs(B, S, seed=0)
    out = m((crops.cuda(), k.cuda()))
    torch.cuda.synchronize()
    with torch.inference_mode():
        ref = port_latents.metrabs_forward(sd, spec, port.PathConfig(proc_side=S), L, crops, k, g['w2'], L)
    assert out.shape == (B, J, 3) and torch.isfinite(out).all()
    assert m.engine().n_points == L and m.engine().n_out == J
    print(f'latent-point model in fp16: joints rel err vs the fp32 oracle {port.relative_error(out.cpu(), ref):.2e}')


def _sharded_worker(rank, world, port_no, out_dir):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port_no)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from metrabs_b200 import parallel
    from tests import helpers
    pcfg = port.PathConfig(proc_side=64)
    sd = port.make_effnet_state_dict(port.effnet_spec('efficientnetv2-tiny'), pcfg, 8, seed=0)
    m = helpers.device_model('efficientnetv2-tiny', pcfg, 8, sd, precision='fp16').to(dev)
    eng = m.engine(dev)

    def bcast(raw):
        t = torch.tensor(list(raw) if raw is not None else [0] * 128, dtype=torch.uint8, device=dev)
        dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())
    eng.comm_init(rank, world, bcast)
    sh = parallel.ShardedMetrabs(m, rank, world)
    res = {}
    for n_total in (8, 5):  # equal shards (library path), ragged
        crops, k = port.synthetic_inputs(n_total, 64, seed=3)
        crops, k = crops.to(dev), k.to(dev)
        out = sh.forward(crops, k)
        ref = eng.forward(crops, k)
        torch.cuda.synchronize()
        res[n_total] = (out.cpu(), ref.cpu())
    torch.save(res, os.path.join(out_dir, f'r{rank}.pt'))
    dist.destroy_process_group()


def test_f16_sharded_equals_unsharded_nccl(tmp_path):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 CUDA devices')
    world = 2
    mp.spawn(_sharded_worker, args=(world, 35600 + os.getpid() % 2000, str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f'r{r}.pt') for r in range(world)]
    for n_total in (8, 5):
        for r in range(world):
            out, ref = outs[r][n_total]
            assert out.shape == (n_total, 8, 3)
            err = float((out - ref).abs().max() / ref.abs().max())
            assert err <= 2e-2, (n_total, r, err)
        assert torch.equal(outs[0][n_total][0], outs[1][n_total][0])
