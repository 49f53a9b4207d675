"""GPU parity tests proper: the CUDA path (through the C ABI) against the oracle port on the same seeded inputs and
against the committed goldens produced by the unmodified reference.  Tolerance: 1e-3 relative on fp32 joints
(BASELINE.json north_star), tighter where the arithmetic allows."""
import os

import numpy as np
import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


# ------------------------------------------------------------------------------------------- decode kernels
def test_soft_argmax_reference_layout(H, golden_dir):
    from metrabs_b200 import ptu
    g = _golden(golden_dir, 'decode_functions.npz')
    for i in range(int(g['n_sa3d'])):
        x = torch.from_numpy(g[f'sa3d_{i}_in']).cuda()
        out = ptu.soft_argmax(x, dim=(4, 3, 1))
        np.testing.assert_allclose(out.cpu().numpy(), g[f'sa3d_{i}_out'], rtol=0, atol=5e-6)
    for i in range(int(g['n_sa2d'])):
        x = torch.from_numpy(g[f'sa2d_{i}_in']).cuda()
        out = ptu.soft_argmax(x, dim=(3, 2))
        np.testing.assert_allclose(out.cpu().numpy(), g[f'sa2d_{i}_out'], rtol=0, atol=5e-6)


@pytest.mark.parametrize('shape', [(3, 8, 24, 8, 8), (2, 8, 122, 8, 8), (2, 32, 24, 32, 32), (1, 8, 5, 12, 12),
                                   (2, 4, 3, 5, 7)])
def test_soft_argmax_layouts_vs_oracle(H, shape):
    from metrabs_b200 import _lib
    from metrabs_b200.engine import soft_argmax_device
    b, d, j, h, w = shape
    g = torch.Generator().manual_seed(5)
    l3 = torch.randn(b, d, j, h, w, generator=g) * 5
    l2 = torch.randn(b, j, h, w, generator=g) * 5
    ref3 = port.soft_argmax(l3, (4, 3, 1))
    ref2 = port.soft_argmax(l2, (3, 2))
    _, out3 = soft_argmax_device(l3.cuda(), _lib.LAYOUT_BDJHW, j, d, h, w)
    assert (out3.cpu() - ref3).abs().max() < 5e-6
    # bf16 storage of the same values
    _, out3b = soft_argmax_device(l3.bfloat16().cuda(), _lib.LAYOUT_BDJHW, j, d, h, w)
    assert (out3b.cpu() - port.soft_argmax(l3.bfloat16().float(), (4, 3, 1))).abs().max() < 5e-6
    # fp16 storage: what the reference's head emits under its autocast (multiperson_model.py:241, models/metrabs.py:80 `.float()`)
    _, out3h = soft_argmax_device(l3.half().cuda(), _lib.LAYOUT_BDJHW, j, d, h, w)
    assert (out3h.cpu() - port.soft_argmax(l3.half().float(), (4, 3, 1))).abs().max() < 5e-6
    out2h, _ = soft_argmax_device(l2.half().cuda(), _lib.LAYOUT_BDJHW, j, 0, h, w)
    assert (out2h.cpu() - port.soft_argmax(l2.half().float(), (3, 2))).abs().max() < 5e-6
    # internal NHWC layout: channel n = J + d*J + j
    nhwc = torch.cat([l2, l3.reshape(b, d * j, h, w)], dim=1).permute(0, 2, 3, 1).contiguous()
    out2n, out3n = soft_argmax_device(nhwc.cuda(), _lib.LAYOUT_BHWN, j, d, h, w)
    assert (out3n.cpu() - ref3).abs().max() < 5e-6
    assert (out2n.cpu() - ref2).abs().max() < 5e-6


def test_soft_argmax_idempotent_on_delta(H):
    """Size-independent property at the full c5b row size: a one-hot (huge logit) volume decodes to its index."""
    from metrabs_b200 import ptu
    b, d, j, h, w = 2, 32, 24, 32, 32
    x = torch.zeros(b, d, j, h, w)
    idx = torch.randint(0, 32, (b, j, 3), generator=torch.Generator().manual_seed(1))
    for bi in range(b):
        for ji in range(j):
            x[bi, idx[bi, ji, 2], ji, idx[bi, ji, 1], idx[bi, ji, 0]] = 200.0
    out = ptu.soft_argmax(x.cuda(), dim=(4, 3, 1)).cpu()
    assert (out - idx.float() / 31).abs().max() < 1e-6


def test_reconstruct_absolute_goldens(H, golden_dir):
    import metrabs_b200
    from metrabs_b200 import ptu3d
    g = _golden(golden_dir, 'decode_functions.npz')
    for ci, (s, st, cs, lb) in enumerate(g['geo_cfgs']):
        metrabs_b200.set_config(metrabs_b200.Config(proc_side=int(s), stride_test=int(st), centered_stride=bool(cs),
                                                    legacy_centered_stride_bug=bool(lb)))
        for nb, nj in [(3, 24), (1, 8), (5, 122)]:
            tag = f'geo_{ci}_{nb}_{nj}'
            c2d, c3d, k = (torch.from_numpy(g[tag + n]).cuda() for n in ('_c2d', '_c3d', '_k'))
            out = ptu3d.reconstruct_absolute(c2d, c3d, k, mix_3d_inside_fov=0.5)
            assert H.rel_err(out, g[tag + '_out']) < 2e-5, tag
            out = ptu3d.reconstruct_absolute(c2d, c3d, k, mix_3d_inside_fov=None)
            assert H.rel_err(out, g[tag + '_out_nomix']) < 2e-5, tag


# ------------------------------------------------------------------------------------------------ backbone
def _layer_report(H, m, sd, spec, crops):
    """Layer-by-layer comparison against the oracle taps; returns [(op name, rel err)]."""
    tap = {}
    with torch.inference_mode():
        port.effnet_features(sd, spec, crops, tap=tap)
    eng = m.engine()
    rows = []
    for i, name in enumerate(eng.op_names()):
        if name.endswith(('.avgpool', '.fc1', '.fc2')):
            continue
        out = eng.debug_run_ops(crops.cuda(), i + 1).permute(0, 3, 1, 2).cpu()
        cands = [tap[name]]
        blk = name.rsplit('.block.', 1)[0]
        if blk in tap and tap[blk].shape == out.shape:
            cands.append(tap[blk])
        rows.append((name, min(port.relative_error(out, c) for c in cands)))
    return rows


@pytest.mark.parametrize('fname', ['tiny_s64_j8.npz', 'tiny_s128_j8_legacy.npz'])
def test_tiny_model_golden(H, golden_dir, fname):
    g = _golden(golden_dir, fname)
    pcfg = port.PathConfig(proc_side=int(g['proc_side']), centered_stride=bool(g['centered_stride']),
                           legacy_centered_stride_bug=bool(g['legacy_centered_stride_bug']))
    name, j = str(g['name']), int(g['n_joints'])
    spec = port.effnet_spec(name, centered_stride=pcfg.centered_stride)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith('sd/')}
    m = H.device_model(name, pcfg, j, sd)
    crops, k = torch.from_numpy(g['crops']), torch.from_numpy(g['intrinsics'])
    rows = _layer_report(H, m, sd, spec, crops)
    bad = [(n, e) for n, e in rows if not e < 1e-4]
    assert not bad, f'first diverging layers: {bad[:5]}'
    eng = m.engine()
    feats = eng.backbone(crops.cuda())
    assert H.rel_err(feats.permute(0, 3, 1, 2).reshape(crops.shape[0], -1), g['features']) < 1e-4
    c2d, c3d = eng.head_decode(feats)
    assert H.rel_err(c2d, g['coords2d']) < 1e-4
    assert H.rel_err(c3d, g['coords3d_rel']) < 1e-4
    out = m((crops.cuda(), k.cuda()))
    assert H.rel_err(out, g['coords3d_abs']) < 1e-3
    # the reference-layout sub-module call and the host-buffer entry point agree with the fused forward
    c2d_b, c3d_b = m.heatmap_heads(feats.permute(0, 3, 1, 2))
    assert torch.equal(c2d_b, c2d) and torch.equal(c3d_b, c3d)
    out_h = eng.forward_host(crops.pin_memory(), k.pin_memory())
    assert torch.equal(out_h, out.cpu())  # the path is deterministic (split-K partials are summed in a fixed order)
    assert eng.last_launch_count > 0
    # pipelined host entry points (two slots, copy stream): the next batch is submitted before the previous one is waited
    # for, slots are reused, and every batch's joints equal the synchronous call's bit for bit
    ch, kh = crops.float().contiguous().pin_memory(), k.float().contiguous().pin_memory()
    outs = [torch.empty(out_h.shape, dtype=torch.float32).pin_memory() for _ in range(2)]
    eng.forward_host_submit(ch, kh, outs[0], 0)
    eng.forward_host_submit(ch, kh, outs[1], 1)
    eng.forward_host_wait(0)
    eng.forward_host_wait(1)
    eng.forward_host_wait(0)  # waiting twice is harmless
    assert torch.equal(outs[0], out_h) and torch.equal(outs[1], out_h)
    outs[0].zero_()
    eng.forward_host_submit(ch, kh, outs[0], 0)
    eng.forward_host_wait(0)
    assert torch.equal(outs[0], out_h)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('name,side,j,batch,fname', [
    ('efficientnetv2-s', 256, 24, 3, 'effnetv2s_s256_j24.npz'),
    ('efficientnetv2-s', 256, 122, 2, 'effnetv2s_s256_j122.npz'),
    ('efficientnetv2-l', 256, 24, 2, 'effnetv2l_s256_j24.npz'),
    ('efficientnetv2-l', 384, 24, 1, 'effnetv2l_s384_j24.npz'),
])
def test_full_models_parity_modes(H, golden_dir, name, side, j, batch, fname, precision):
    """The two modes that must meet BASELINE.json's 1e-3 bar - 'fp32' (CUDA-core FMA) and 'tf32x3' (wgmma tf32, three
    split products, fp32 accumulate) - against the oracle port on the same weights/inputs AND against the goldens the
    unmodified reference produced (/root/reference/metrabs_pytorch/models/metrabs.py:47-64), the latter at the golden's
    own batch size (reconstruct_ref_fullpersp normalises with batch-global RMS, ptu3d.py:71-74)."""
    g = _golden(golden_dir, fname)
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, j, seed=0)
    crops, k = port.synthetic_inputs(batch, side, seed=0)
    stages = {}
    with torch.inference_mode():
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    m = H.device_model(name, pcfg, j, sd, precision=precision)
    eng = m.engine()
    feats = eng.backbone(crops.cuda())
    e_feat = H.rel_err(feats.permute(0, 3, 1, 2), stages['features'])
    out = m((crops.cuda(), k.cuda()))
    e_out = H.rel_err(out, ref)
    assert e_feat < 1e-3
    assert e_out < 1e-3
    gb = int(g['batch'])
    gcrops, gk = port.synthetic_inputs(gb, side, seed=int(g['seed']))
    gout = m((gcrops.cuda(), gk.cuda()))
    e_gold = H.rel_err(gout, g['coords3d_abs'])
    e_gfeat = H.rel_err(eng.backbone(gcrops.cuda()).permute(0, 3, 1, 2).reshape(gb, -1)[:, ::int(g['feature_stride'])], g['features'])
    print(f'{name}@{side} J={j} [{precision}]: vs oracle features {e_feat:.2e} joints {e_out:.2e}; vs reference goldens '
          f'features {e_gfeat:.2e} joints {e_gold:.2e}; launches {eng.last_launch_count}')
    assert e_gfeat < 1e-3
    assert e_gold < 1e-3


@pytest.mark.parametrize('kind,cfgkw,j,batch', [
    ('mobilenetv3-small', dict(proc_side=256, stride_test=32, depth=8), 8, 4),   # BASELINE config c1
    ('resnet50', dict(proc_side=256, stride_test=8, depth=32), 24, 2),           # BASELINE config c2 (small batch)
    ('resnet50', dict(proc_side=256, stride_test=32, depth=8, centered_stride=False), 24, 2),
])
def test_tf_only_backbones_fp32(H, kind, cfgkw, j, batch):
    """ResNet-50 V1 / MobileNetV3-Small: device vs the build's own torch restatement of the Keras code (PARITY
    UNPINNED by the reference: no tests, no importable implementation - oracle/port_tf_backbones.py)."""
    from oracle import port_tf_backbones as tfb
    pcfg = port.PathConfig(**cfgkw)
    spec = tfb.ResNet50Spec(pcfg) if kind == 'resnet50' else tfb.MobileNetV3SmallSpec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, pcfg.proc_side, seed=0)
    tap, stages = {}, {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    m = H.device_model_tf(kind, pcfg, j, sd)
    eng = m.engine()
    bad = []
    for i, name in enumerate(eng.op_names()):
        if name.endswith(('.avgpool', '.fc1', '.fc2')) or name not in tap:
            continue
        out = eng.debug_run_ops(crops.cuda(), i + 1).permute(0, 3, 1, 2).cpu()
        err = port.relative_error(out, tap[name])
        if not err < 1e-4:
            bad.append((name, err))
    assert not bad, f'first diverging layers: {bad[:5]}'
    out = m((crops.cuda(), k.cuda()))
    e_feat = H.rel_err(eng.backbone(crops.cuda()).permute(0, 3, 1, 2), stages['features'])
    e_out = H.rel_err(out, ref)
    print(f'{kind} {cfgkw}: features {e_feat:.2e}, joints {e_out:.2e}, {eng.backbone_flops_per_crop / 1e9:.2f} GFLOP/crop')
    assert e_feat < 1e-3 and e_out < 1e-3


def test_batch_global_rms_is_reproduced(H):
    """reconstruct_ref_fullpersp normalises by batch-global RMS (ptu3d.py:71-74): solving crops alone vs inside a
    larger batch differs slightly in the reference; the device must follow the SAME batch composition."""
    from metrabs_b200 import ptu3d
    import metrabs_b200
    metrabs_b200.set_config(metrabs_b200.Config())
    pcfg = port.PathConfig()
    g = torch.Generator().manual_seed(9)
    c2d = 40 + 170 * torch.rand(6, 24, 2, generator=g)
    c3d = torch.randn(6, 24, 3, generator=g) * 300
    _, k = port.synthetic_inputs(6, 256)
    for sl in (slice(0, 6), slice(0, 2), slice(3, 4)):
        ref = port.reconstruct_absolute(c2d[sl], c3d[sl], k[sl], pcfg)
        out = ptu3d.reconstruct_absolute(c2d[sl].cuda(), c3d[sl].cuda(), k[sl].cuda(), mix_3d_inside_fov=0.5)
        assert H.rel_err(out, ref) < 2e-5
    # batches past one CTA's strided reduction (128 threads), joints past one pass of the crop loop, crops whose joints
    # are all outside the field of view, joints exactly on its inclusive bounds, mixing on and off: per crop, max |dev-ref|
    # over its joints relative to its largest joint, against the fp64 reconstruction on the same fp32 inputs
    lo, hi = pcfg.stride_train * 0.75, pcfg.proc_side - pcfg.stride_train * 0.75  # is_within_fov, centered stride
    worst = 0.0
    for b, j in ((129, 24), (256, 129), (1000, 24), (256, 1024)):
        c2d = 40 + 170 * torch.rand(b, j, 2, generator=g)
        c3d = torch.randn(b, j, 3, generator=g) * 300
        c3d[..., 2] += 3000
        c2d[1] = 300 + 10 * torch.rand(j, 2, generator=g)  # every joint of crop 1 outside the field of view
        c2d[2, :, 0] = lo                                   # crop 2 on the lower bound in x, the upper in y
        c2d[2, :, 1] = hi
        c2d[b - 1, ::2] = hi                                # half of the last crop's joints on the upper corner
        _, k = port.synthetic_inputs(b, 256, seed=b + j)
        for mix in (0.5, None):
            ref = port.reconstruct_absolute(c2d.double(), c3d.double(), k.double(), pcfg, mix_3d_inside_fov=mix)
            out = ptu3d.reconstruct_absolute(c2d.cuda(), c3d.cuda(), k.cuda(), mix_3d_inside_fov=mix).double().cpu()
            per_crop = (out - ref).abs().amax(dim=(1, 2)) / ref.abs().amax(dim=(1, 2))
            worst = max(worst, float(per_crop.max()))
            assert float(per_crop.max()) < 2e-5, (b, j, mix, int(per_crop.argmax()), float(per_crop.max()))
    print(f'reconstruction per crop: worst max|dev-ref| / max|ref| {worst:.1e}')


def test_errors_are_loud(H):
    import metrabs_b200
    from metrabs_b200._lib import MetrabsB200Error
    pcfg = port.PathConfig(proc_side=64)
    sd = port.make_effnet_state_dict(port.effnet_spec('efficientnetv2-tiny'), pcfg, 8)
    m = H.device_model('efficientnetv2-tiny', pcfg, 8, sd)
    with pytest.raises(MetrabsB200Error):
        m.engine().forward(torch.rand(1, 3, 64, 64), torch.eye(3)[None])  # CPU tensors: no fallback
    sd.pop('backbone.1.3.0.block.1.1.running_var')
    from metrabs_b200.engine import Engine, make_config
    from metrabs_b200.backbones.efficientnet import stage_table
    stages, last = stage_table('tiny', True)
    eng = Engine(make_config(metrabs_b200.get_config(), 8, stages=stages, last_channel=last))
    with pytest.raises(MetrabsB200Error, match='backbone.1.3.0.block.1.1'):
        eng.load_state_dict(sd)


def test_checkpoint_file_round_trip(H, golden_dir, tmp_path):
    """SURVEY.md 8f-3: the on-disk format.  tests/golden/tiny_ckpt.pt is ``torch.save(model.state_dict())`` of the REFERENCE
    Metrabs object (scripts/demo_image.py:59-74 loads exactly this); it must load with strict=True through the reference key
    schema (BN fold + NHWC / K-major repack inside mtb_load_weight) and reproduce the reference's own outputs.  A half-precision
    copy of the file (how released checkpoints are often stored) goes through the F16 loader path.  No trained weights exist
    offline, so the fast-mode deviation on TRAINED weights cannot be measured here - said so instead of guessed."""
    g = _golden(golden_dir, 'tiny_s64_j8.npz')
    sd = torch.load(os.path.join(golden_dir, 'tiny_ckpt.pt'), weights_only=True)
    assert any(k.endswith('num_batches_tracked') for k in sd)  # the real file carries keys the engine must ignore
    pcfg = port.PathConfig(proc_side=64)
    crops, k = torch.from_numpy(g['crops']), torch.from_numpy(g['intrinsics'])
    m = H.device_model('efficientnetv2-tiny', pcfg, 8, sd)
    out = m((crops.cuda(), k.cuda()))
    assert H.rel_err(out, g['coords3d_abs']) < 1e-3
    # save / load cycle of THIS package's module: identical bits
    path = tmp_path / 'ckpt.pt'
    torch.save(m.state_dict(), path)
    m2 = H.device_model('efficientnetv2-tiny', pcfg, 8, torch.load(path, weights_only=True))
    assert torch.equal(m2((crops.cuda(), k.cuda())), out)
    # fp16 file: the engine converts on load; the result equals the fp32 engine fed the fp16-rounded weights
    sd16 = {kk: (v.half() if v.is_floating_point() else v) for kk, v in sd.items()}
    torch.save(sd16, path)
    ld = torch.load(path, weights_only=True)
    from metrabs_b200.engine import Engine, make_config
    import metrabs_b200
    from metrabs_b200.backbones.efficientnet import stage_table
    stages, last = stage_table('tiny', True)
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=64))
    e16 = Engine(make_config(metrabs_b200.get_config(), 8, stages=stages, last_channel=last))
    e16.load_state_dict(ld)  # fp16 tensors straight into mtb_load_weight (MTB_DTYPE_F16)
    m3 = H.device_model('efficientnetv2-tiny', pcfg, 8, {kk: (v.float() if v.is_floating_point() else v) for kk, v in sd16.items()})
    assert torch.equal(e16.forward(crops.cuda(), k.cuda()), m3((crops.cuda(), k.cuda())))
