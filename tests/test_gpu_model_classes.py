"""GPU: the reference's Metro and Model25D classes (metrabs_b200.models.metro / twofive) against their restatement
(oracle/port_model_classes.py) on four backbones in the four arithmetic modes, the fused against the non-fused head, batch
invariance of the decoded coordinates, the host / graph / sharded entry points, the C argument checks and the multi-person
estimator on a 2.5D model.

Tolerances: fp32 and tf32x3 joints within the project's 1e-3; bf16 and fp16 decoded coordinates within 2e-4 of the
restated head run on the same 16-bit features and 16-bit-rounded head weights (the bound of test_gpu_f16's fused-head test),
and the absolute joints within 1e-3 of the restated solve on the device's own coords25d."""
import ctypes as C
import dataclasses
import functools

import numpy as np
import pytest
import torch

import metrabs_b200
from metrabs_b200 import _lib
from metrabs_b200.models.metro import Metro
from metrabs_b200.models.twofive import Model25D
from oracle import port, port_tf_backbones
from oracle import port_model_classes as pm

pytestmark = pytest.mark.gpu

J, BATCH = 8, 4
EDGES = pm.tree_edges(J)
LENGTHS = pm.seeded_bone_lengths(len(EDGES))
BACKBONES = {
    'efficientnetv2-tiny@64': dict(proc_side=64),
    'efficientnetv2-s@256': dict(proc_side=256),
    'resnet50@256/8': dict(proc_side=256, stride_test=8, stride_train=32),
    'mobilenetv3-small@256': dict(proc_side=256),
}


def _joint_info():
    import types
    return types.SimpleNamespace(names=[f'j{i}' for i in range(J)], stick_figure_edges=EDGES, n_joints=J)


@functools.lru_cache(maxsize=None)
def oracle_setup(name):
    """-> (PathConfig, class state dict, features_fn, oracle features of the test crops, crops, intrinsics)"""
    pcfg = port.PathConfig(**BACKBONES[name])
    kind = name.split('@')[0]
    if kind.startswith('efficientnet'):
        spec = port.effnet_spec(kind)
        sd = port.make_effnet_state_dict(spec, pcfg, J, seed=0)
        features_fn = functools.partial(lambda spec, sd, img: port.effnet_features(sd, spec, img), spec)
    else:
        spec = (port_tf_backbones.ResNet50Spec if kind == 'resnet50' else port_tf_backbones.MobileNetV3SmallSpec)(pcfg)
        sd = port_tf_backbones.make_state_dict(spec, pcfg, J, seed=0)
        features_fn = spec.features
    crops, k = port.synthetic_inputs(BATCH, pcfg.proc_side, seed=0)
    with torch.inference_mode():
        feats = features_fn(sd, crops)
    return pcfg, pm.to_volumetric_state_dict(sd, J), features_fn, feats, crops, k


def backbone_module(name):
    from metrabs_b200.backbones import efficientnet as E
    from metrabs_b200.backbones import mobilenet_v3, resnet
    kind = name.split('@')[0]
    if kind.startswith('efficientnet'):
        return torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet({'efficientnetv2-tiny': 'tiny',
                                                                     'efficientnetv2-s': 's'}[kind]).features)
    return resnet.resnet50() if kind == 'resnet50' else mobilenet_v3.mobilenet_v3_small()


def device_model(cls, name, precision, **cfg_extra):
    pcfg, sd, *_ = oracle_setup(name)
    metrabs_b200.set_config(metrabs_b200.Config(**dataclasses.asdict(pcfg), precision=precision, **cfg_extra))
    bb = backbone_module(name)
    m = Metro(bb, _joint_info()) if cls == 'metro' else Model25D(bb, _joint_info(), LENGTHS)
    m.eval().load_state_dict(sd, strict=True)
    return m.cuda()


def rel(a, b):
    return port.relative_error(a.detach().float().cpu(), torch.as_tensor(b).float().cpu())


def head16(sd, dtype):
    return {k: (v.to(dtype).float() if k.endswith('weight') else v) for k, v in sd.items()}


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'bf16', 'fp16'])
@pytest.mark.parametrize('name', list(BACKBONES))
def test_parity_vs_restatement(name, precision):
    pcfg, sd, features_fn, feats, crops, k = oracle_setup(name)
    metro, m25 = device_model('metro', name, precision), device_model('25d', name, precision)
    out_metro = metro(crops.cuda())
    out_25d = m25((crops.cuda(), k.cuda()))
    eng = m25.engine()
    dev_feats = eng.backbone(crops.cuda())
    c2d, c25 = eng.head_decode(dev_feats)
    torch.cuda.synchronize()
    assert torch.isfinite(out_metro).all() and torch.isfinite(out_25d).all()
    assert torch.equal(c2d, c25[..., :2])
    if precision in ('fp32', 'tf32x3'):
        ref_metro = pm.metro_head(sd, feats, pcfg, J)
        ref_25d = pm.reconstruct_by_bone_lengths(pm.head_25d(sd, feats, pcfg, J), k, LENGTHS, EDGES, pcfg)
        errs = rel(out_metro, ref_metro), rel(out_25d, ref_25d)
        print(f'{name} [{precision}] Metro {errs[0]:.2e}, Model25D {errs[1]:.2e}')
        assert max(errs) < 1e-3, errs
    else:
        f = dev_feats.float().permute(0, 3, 1, 2).cpu()
        w = head16(sd, torch.bfloat16 if precision == 'bf16' else torch.float16)
        ref_metro, ref_25d = pm.metro_head(w, f, pcfg, J), pm.head_25d(w, f, pcfg, J)
        ref_abs = pm.reconstruct_by_bone_lengths(c25.cpu(), k, LENGTHS, EDGES, pcfg)
        errs = rel(out_metro, ref_metro), rel(c25, ref_25d), rel(out_25d, ref_abs)
        print(f'{name} [{precision}] Metro {errs[0]:.2e}, coords25d {errs[1]:.2e}, Model25D absolute {errs[2]:.2e}')
        assert errs[0] < 2e-4 and errs[1] < 2e-4 and errs[2] < 1e-3, errs


def test_fused_and_unfused_heads_agree():
    """bf16: tc_head_kernel + head_finalize_kernel<true>; bf16_simt: the CUDA-core logits GEMM +
    softargmax_bhwn_kernel<float, true>, on the same bf16 features."""
    name = 'efficientnetv2-s@256'
    f = None
    outs = {}
    for prec, head_classes in (('bf16', {'tc_head_softargmax_kernel'}),
                               ('bf16_simt', {'head_conv(conv_igemm_kernel)', 'softargmax_bhwn_kernel'})):
        for cls in ('metro', '25d'):
            eng = device_model(cls, name, prec).engine()
            if f is None:
                f = eng.backbone(oracle_setup(name)[4].cuda())
            eng.profile_begin()
            outs[prec, cls] = eng.head_decode(f)[1]
            assert set(eng.profile_end()) == head_classes, (prec, cls)
    for cls in ('metro', '25d'):
        err = rel(outs['bf16', cls], outs['bf16_simt', cls])
        print(f'{cls}: fused vs non-fused head {err:.2e}')
        assert err < 2e-4, (cls, err)


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_decoded_coordinates_are_batch_invariant(precision):
    name = 'efficientnetv2-tiny@64'
    crops, k = port.synthetic_inputs(7, 64, seed=5)
    for cls in ('metro', '25d'):
        eng = device_model(cls, name, precision).engine()
        full = eng.head_decode(eng.backbone(crops.cuda()))[1]
        for lo, hi in ((0, 1), (2, 5), (3, 7)):
            part = eng.head_decode(eng.backbone(crops[lo:hi].cuda()))[1]
            assert torch.equal(part, full[lo:hi]), (cls, lo, hi)


def test_entry_points_bit_identical():
    """forward == head_decode + the standalone solve, CUDA-graph replay, forward_host, forward_host_submit and a one-rank
    forward_sharded give the forward's joints bit for bit; a Metro forward takes no intrinsics."""
    name = 'efficientnetv2-tiny@64'
    crops, k = port.synthetic_inputs(6, 64, seed=7)
    for cls in ('metro', '25d'):
        m = device_model(cls, name, 'bf16')
        eng = m.engine()
        kk = None if cls == 'metro' else k.cuda()
        ref = eng.forward(crops.cuda(), kk)
        if cls == '25d':
            c25 = eng.head_decode(eng.backbone(crops.cuda()))[1]
            assert torch.equal(eng.reconstruct_by_bone_lengths(c25, k.cuda()), ref)
            assert torch.equal(eng.reconstruct_by_bone_lengths(c25, k.cuda()), ref)  # run to run
        else:
            assert torch.equal(eng.head_decode(eng.backbone(crops.cuda()))[1], ref)
        for _ in range(3):  # the library captures its own graph on the second call with the same buffers
            cb, kb, ob = crops.cuda(), kk, torch.empty_like(ref)
            eng.forward(cb, kb, out=ob)
        assert torch.equal(ob, ref)
        g = eng.capture_forward(cb, kb, ob)
        ob.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(ob, ref), cls
        host = eng.forward_host(crops, None if cls == 'metro' else k)
        assert torch.equal(host, ref.cpu())
        out_host = torch.empty(6, J, 3).pin_memory()
        eng.forward_host_submit(crops.pin_memory(), k.pin_memory(), out_host, 0)
        eng.forward_host_wait(0)
        assert torch.equal(out_host, ref.cpu())
        eng.comm_init(0, 1, lambda raw: raw)
        assert torch.equal(eng.forward_sharded(crops.cuda(), kk), ref), cls


def test_metrabs_handles_unchanged_by_the_class_entry_points():
    """A MeTRAbs handle: mtb_reconstruct_by_bone_lengths refuses it and its scratch size is 0."""
    from tests import helpers
    pcfg = port.PathConfig(proc_side=64)
    sd = port.make_effnet_state_dict(port.effnet_spec('efficientnetv2-tiny'), pcfg, J, seed=0)
    eng = helpers.device_model('efficientnetv2-tiny', pcfg, J, sd).engine()
    assert _lib.lib().mtb_bone_lengths_scratch_bytes(eng._h, 4) == 0
    with pytest.raises(_lib.MetrabsB200Error, match='not a Model25D'):
        eng.reconstruct_by_bone_lengths(torch.zeros(4, J, 3).cuda(), torch.eye(3).expand(4, 3, 3).cuda())


def test_set_model_class_rejects_invalid_arguments():
    from metrabs_b200.engine import Engine, make_config
    from metrabs_b200.backbones import efficientnet as E
    lib = _lib.lib()
    pcfg, sd, *_ = oracle_setup('efficientnetv2-tiny@64')
    feats = E.EfficientNet('tiny').features

    def handle(**kw):
        cfg = metrabs_b200.Config(**{**dataclasses.asdict(pcfg), **kw})
        return Engine(make_config(cfg, J, stages=feats.stages, last_channel=feats.last_channel, arch=feats.arch))

    eng = handle()
    e = np.asarray(EDGES, np.int32)
    good = np.asarray(LENGTHS, np.float32)

    def call(h, cls, edges=e, lengths=good, n=len(EDGES), mean_rel=1):
        ep = edges.ctypes.data_as(C.c_void_p) if edges is not None else None
        lp = lengths.ctypes.data_as(C.c_void_p) if lengths is not None else None
        return lib.mtb_set_model_class(h._h, cls, ep, lp, n, mean_rel)

    assert call(eng, 3) == -1 and call(eng, -1) == -1
    bad_e = e.copy()
    bad_e[2, 1] = J
    assert call(eng, _lib.MODEL_25D, edges=bad_e) == -1
    bad_e[2, 1] = -1
    assert call(eng, _lib.MODEL_25D, edges=bad_e) == -1
    for v in (0.0, -1.0, np.nan, np.inf):
        bl = good.copy()
        bl[1] = v
        assert call(eng, _lib.MODEL_25D, lengths=bl) == -1
    assert call(eng, _lib.MODEL_25D, edges=None) == -1 and call(eng, _lib.MODEL_25D, n=0) == -1
    assert call(eng, _lib.MODEL_METRO, edges=None, lengths=None, n=0) == 0  # Metro takes no bones
    assert call(handle(legacy_centered_stride_bug=True), _lib.MODEL_METRO) == -1
    lat = handle()
    w = torch.eye(J)
    assert lib.mtb_set_latent_recombination(lat._h, C.c_void_p(w.data_ptr()), J, J) == 0
    assert call(lat, _lib.MODEL_25D) == -1
    cls_h = handle()
    assert call(cls_h, _lib.MODEL_25D) == 0
    assert lib.mtb_set_latent_recombination(cls_h._h, C.c_void_p(w.data_ptr()), J, J) == -1
    head_only = Engine(make_config(metrabs_b200.Config(proc_side=64), J, arch=_lib.ARCH_HEAD_ONLY, feature_channels=64))
    assert call(head_only, _lib.MODEL_METRO) == -1
    done = device_model('25d', 'efficientnetv2-tiny@64', 'fp32').engine()
    assert call(done, _lib.MODEL_25D) == -1  # finalized


def test_pose_estimator_with_a_25d_model():
    """Pose3dEstimator drives a Model25D as it drives a Metrabs model: the crop model sees what the estimator passes and
    returns the restated Model25D's joints on them, and the estimator's result equals its own composition around a crop model
    that returns those restated joints."""
    from metrabs_b200.multiperson import Pose3dEstimator
    name = 'efficientnetv2-tiny@64'
    pcfg, sd, features_fn, *_ = oracle_setup(name)
    m = device_model('25d', name, 'fp32')
    seen = []

    class Recorder(torch.nn.Module):
        def __init__(self, inner, replay=None):
            super().__init__()
            self.inner, self.replay = inner, replay
            self.joint_names, self.joint_edges, self.input_resolution = inner.joint_names, inner.joint_edges, inner.input_resolution

        def forward(self, inp):
            if self.replay is not None:
                return self.replay.cuda()
            out = self.inner(inp)
            seen.append((inp[0].cpu(), inp[1].cpu(), out.cpu()))
            return out

    skel = {'': dict(indices=list(range(J)), names=[f'j{i}' for i in range(J)], edges=[list(e) for e in EDGES])}
    frames = torch.randint(0, 256, (1, 3, 120, 160), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda()
    boxes = [torch.tensor([[20., 10., 60., 90.], [70., 20., 50., 80.]])]
    res = Pose3dEstimator(Recorder(m), skel, None).estimate_poses_batched(frames, boxes, num_aug=3)
    crops, k, out = seen[0]
    ref = pm.model25d_forward(sd, features_fn, pcfg, J, crops, k, LENGTHS, EDGES)
    err = rel(out, ref)
    print(f'estimator crop batch {tuple(crops.shape)}: Model25D vs restatement {err:.2e}')
    assert err < 1e-3
    res_ref = Pose3dEstimator(Recorder(m, replay=ref), skel, None).estimate_poses_batched(frames, boxes, num_aug=3)
    for key in ('poses3d', 'poses2d'):
        e = rel(res[key][0], res_ref[key][0])
        assert e < 1e-3, (key, e)
