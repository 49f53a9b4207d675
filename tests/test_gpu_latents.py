"""GPU: latent-point MeTRAbs models (affine-combining autoencoder heads) on the device.

- ``transform_coords`` and ``predict_all_and_latents`` on the tiny model against the reference's golden
  (tests/golden/latents_tiny_s64.npz) and the oracle port, in every arithmetic mode;
- the sliced head of ``predict_all_and_latents`` is the reference head restricted to the latents;
- mtb_linear_combine_points against an fp64 einsum; mtb_set_latent_recombination argument checks;
- the host-buffer, pipelined and graph-captured entry points, the multiperson caller and (>= 2 GPUs) the sharded
  forward on a latent-point model."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from metrabs_b200 import _lib
from metrabs_b200._lib import lib
from metrabs_b200.engine import Engine, linear_combine_points, make_config
from oracle import port, port_latents

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'latents_tiny_s64.npz')
OPTIONS = ('transform_coords', 'predict_all_and_latents')
G = np.load(GOLDEN)
J, L, B, S = int(G['n_joints']), int(G['n_latents']), int(G['batch']), int(G['proc_side'])
SPEC = port.effnet_spec('efficientnetv2-tiny')


def n_raw_points(option):
    return L if option == 'transform_coords' else L + J


@pytest.fixture(scope='module')
def affine_path(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('affine') / 'affine_tiny.npz')
    np.savez(path, w1=G['w1'], w2=G['w2'])
    return path


def latent_model(option, precision, affine_path):
    from tests import helpers
    pcfg = port.PathConfig(proc_side=S, affine_weights=affine_path, **{option: True})
    sd = port.make_effnet_state_dict(SPEC, port.PathConfig(proc_side=S), n_raw_points(option), seed=0)
    return helpers.device_model('efficientnetv2-tiny', pcfg, J, sd, precision=precision), sd


def oracle(option, sd, crops, k, stages=None):
    with torch.inference_mode():
        return port_latents.metrabs_forward(sd, SPEC, port.PathConfig(proc_side=S), n_raw_points(option), crops, k,
                                            G['w2'], L, stages=stages)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'bf16'])
@pytest.mark.parametrize('option', OPTIONS)
def test_latent_forward_vs_golden_and_oracle(affine_path, option, precision):
    m, sd = latent_model(option, precision, affine_path)
    crops, k = port.synthetic_inputs(B, S, seed=0)
    ref = oracle(option, sd, crops, k)
    out = m((crops.cuda(), k.cuda()))
    torch.cuda.synchronize()
    assert out.shape == (B, J, 3)
    assert torch.isfinite(out).all()
    eng = m.engine()
    assert eng.n_points == L and eng.n_out == J
    e_gold = port.relative_error(out.cpu(), G[f'{option}/joints'])
    e_ref = port.relative_error(out.cpu(), ref)
    print(f'[{option} {precision}] joints rel err: vs golden {e_gold:.2e}, vs oracle {e_ref:.2e}, '
          f'launches {eng.last_launch_count}')
    if precision != 'bf16':
        assert e_gold < 1e-3 and e_ref < 1e-3, (e_gold, e_ref)


def test_sliced_head_is_the_reference_head(affine_path):
    """predict_all_and_latents: the device keeps only the latents' head channels; on the oracle's features its decode
    equals the first L points of the full (L + J)-point head."""
    option = 'predict_all_and_latents'
    m, sd = latent_model(option, 'fp32', affine_path)
    crops, _ = port.synthetic_inputs(B, S, seed=0)
    with torch.inference_mode():
        feats = port.effnet_features(sd, SPEC, crops)
        full2d, full3d = port.heads(sd, feats, port.PathConfig(proc_side=S), L + J)
    c2d, c3d = m.heatmap_heads(feats.cuda())
    torch.cuda.synchronize()
    assert c2d.shape == (B, L, 2) and c3d.shape == (B, L, 3)
    assert port.relative_error(c2d.cpu(), full2d[:, :L]) < 1e-5
    assert port.relative_error(c3d.cpu(), full3d[:, :L]) < 1e-5
    assert port.relative_error(full2d, G[f'{option}/coords2d']) < 1e-5


@pytest.mark.parametrize('batch,n_in,n_out', [(256, 48, 555), (4, 1, 1), (7, 13, 300)])
def test_linear_combine_points_vs_fp64(batch, n_in, n_out):
    g = torch.Generator().manual_seed(batch + n_in + n_out)
    pts = torch.randn(batch, n_in, 3, generator=g) * torch.tensor([400., 400., 300.]) + torch.tensor([0., 0., 4000.])
    w = torch.randn(n_in, n_out, generator=g) if n_in > 1 else torch.rand(n_in, n_out, generator=g)
    out = linear_combine_points(pts.cuda(), w.cuda())
    torch.cuda.synchronize()
    ref = torch.einsum('bjc,jJ->bJc', pts.double(), w.double())
    assert out.shape == (batch, n_out, 3)
    assert port.relative_error(out.cpu(), ref) < 1e-6


def test_set_latent_recombination_rejects_invalid_arguments(affine_path):
    import metrabs_b200
    from metrabs_b200.backbones.efficientnet import stage_table
    stages, last = stage_table('tiny', True)
    cfg = metrabs_b200.Config(proc_side=S)
    n_raw = L + J
    eng = Engine(make_config(cfg, n_raw, stages=stages, last_channel=last))
    w = np.ascontiguousarray(G['w2'], np.float32)
    wp = C.c_void_p(w.ctypes.data)
    h = eng._h
    bad = np.ascontiguousarray(w.copy())
    bad[2, 3] = np.nan
    inf = np.ascontiguousarray(w.copy())
    inf[0, 0] = np.inf
    big = np.zeros((L, 4097), np.float32)
    inv = _lib.lib().mtb_set_latent_recombination
    for args in [(wp, 0, J), (wp, n_raw + 1, J), (wp, L, 0), (C.c_void_p(big.ctypes.data), L, 4097), (None, L, J),
                 (C.c_void_p(bad.ctypes.data), L, J), (C.c_void_p(inf.ctypes.data), L, J)]:
        assert inv(h, *args) == -1, args  # MTB_ERR_INVALID_ARG
        assert lib().mtb_last_error(h)
    assert inv(None, wp, L, J) == -1
    assert lib().mtb_output_joints(h) == n_raw  # nothing was set
    # a second call before finalize replaces the first
    assert inv(h, wp, L, 3) == 0 and lib().mtb_output_joints(h) == 3
    sd = port.make_effnet_state_dict(SPEC, port.PathConfig(proc_side=S), n_raw, seed=0)
    eng.set_latent_recombination(G['w2'])
    eng.load_state_dict(sd)
    assert lib().mtb_output_joints(h) == J
    assert inv(h, wp, L, J) == -1  # finalized handle
    crops, k = port.synthetic_inputs(B, S, seed=0)
    out = eng.forward(crops.cuda(), k.cuda())
    torch.cuda.synchronize()
    assert port.relative_error(out.cpu(), G['predict_all_and_latents/joints']) < 1e-3
    head = Engine(make_config(cfg, n_raw, arch=_lib.ARCH_HEAD_ONLY, feature_channels=64))
    assert inv(head._h, wp, L, J) == -1  # head-only handle


def test_latent_entry_points_bit_equal(affine_path):
    m, _ = latent_model('predict_all_and_latents', 'bf16', affine_path)
    eng = m.engine()
    crops, k = port.synthetic_inputs(8, S, seed=1)
    cd, kd = crops.cuda(), k.cuda()
    out = eng.forward(cd, kd)
    out2 = eng.forward(cd, kd)  # second sighting: captured and replayed as a graph inside mtb_forward
    out3 = eng.forward(cd, kd, out=out2)
    torch.cuda.synchronize()
    assert out.shape == (8, J, 3) and torch.equal(out, out3)
    out_h = eng.forward_host(crops.pin_memory(), k.pin_memory())
    assert out_h.shape == (8, J, 3) and torch.equal(out_h, out.cpu())
    ch, kh = crops.contiguous().pin_memory(), k.contiguous().pin_memory()
    outs = [torch.empty(out_h.shape, dtype=torch.float32).pin_memory() for _ in range(2)]
    eng.forward_host_submit(ch, kh, outs[0], 0)
    eng.forward_host_submit(ch, kh, outs[1], 1)
    eng.forward_host_wait(0)
    eng.forward_host_wait(1)
    assert torch.equal(outs[0], out_h) and torch.equal(outs[1], out_h)
    buf = torch.empty(8, eng.n_out, 3, device='cuda')
    eng.forward(cd, kd, out=buf)
    graph = eng.capture_forward(cd, kd, buf)
    buf.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(buf, out)
    # the recombination is one more launch, timed under its own profiler class
    eng.profile_begin()
    eng.forward(cd, kd)
    prof = eng.profile_end()
    assert prof['combine_points_kernel']['launches'] == 1
    # TF method names, on the device
    lat = torch.randn(8, L, 3, device='cuda') * 300
    torch.testing.assert_close(m.latent_points_to_joints(lat).cpu(),
                               torch.einsum('blc,lJ->bJc', lat.cpu().double(), torch.from_numpy(G['w2']).double()).float(),
                               rtol=1e-5, atol=1e-3)
    jts = m.latent_points_to_joints(lat)
    assert m.joints_to_latent_points(jts).shape == (8, L, 3)
    assert m.joints_to_joints(jts).shape == (8, J, 3)


def test_plain_model_launches_unchanged(affine_path):
    """A model without recombination launches no combine kernel and writes cfg.n_joints joints; the latent-point model
    of the same backbone launches exactly one kernel more."""
    from tests import helpers
    pcfg = port.PathConfig(proc_side=S)
    sd = port.make_effnet_state_dict(SPEC, pcfg, 8, seed=0)
    crops, k = port.synthetic_inputs(4, S, seed=0)
    m = helpers.device_model('efficientnetv2-tiny', pcfg, 8, sd, precision='bf16')
    eng = m.engine()
    eng.profile_begin()
    eng.forward(crops.cuda(), k.cuda())
    prof = eng.profile_end()
    plain_launches = eng.last_launch_count
    assert 'combine_points_kernel' not in prof
    assert eng.n_out == eng.n_points == 8
    lm, _ = latent_model('predict_all_and_latents', 'bf16', affine_path)
    leng = lm.engine()
    leng.forward(crops.cuda(), k.cuda())
    torch.cuda.synchronize()
    assert leng.last_launch_count == plain_launches + 1


def test_pose_estimator_on_latent_model(affine_path):
    from metrabs_b200.multiperson import Pose3dEstimator
    m, _ = latent_model('transform_coords', 'fp32', affine_path)
    names = [f'j{i}' for i in range(J)]
    est = Pose3dEstimator(m, {'': dict(indices=list(range(J)), names=names, edges=[[0, 1]])}, None)
    frames = torch.randint(0, 256, (1, 3, 120, 160), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    res = est.estimate_poses_batched(frames.cuda(), [torch.tensor([[20., 10., 60., 90.], [70., 20., 50., 80.]])],
                                     num_aug=3)
    torch.cuda.synchronize()
    assert res['poses3d'][0].shape == (2, J, 3) and torch.isfinite(res['poses3d'][0]).all()


def _worker(rank, world, port_no, affine, out_dir):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port_no)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from metrabs_b200 import parallel
    m, _ = latent_model('predict_all_and_latents', 'fp32', affine)
    m = m.to(dev)
    eng = m.engine(dev)

    def bcast(raw):
        t = torch.tensor(list(raw) if raw is not None else [0] * 128, dtype=torch.uint8, device=dev)
        dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())
    eng.comm_init(rank, world, bcast)
    sh = parallel.ShardedMetrabs(m, rank, world)
    res = {}
    for n_total in (8, 5, 1):  # equal shards (mtb_forward_sharded), ragged, fewer crops than ranks
        crops, k = port.synthetic_inputs(n_total, S, seed=3)
        crops, k = crops.to(dev), k.to(dev)
        out = sh.forward(crops, k)
        ref = eng.forward(crops, k)
        torch.cuda.synchronize()
        res[n_total] = (out.cpu(), ref.cpu())
    torch.save(res, os.path.join(out_dir, f'r{rank}.pt'))
    dist.destroy_process_group()


def test_sharded_latent_model_equals_unsharded_nccl(tmp_path, affine_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 CUDA devices')
    world = 2
    port_no = 37500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(world, port_no, affine_path, str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f'r{r}.pt') for r in range(world)]
    for n_total in (8, 5, 1):
        for r in range(world):
            out, ref = outs[r][n_total]
            assert out.shape == (n_total, J, 3)
            err = float((out - ref).abs().max() / ref.abs().max())
            assert err <= 1e-6, (n_total, r, err)
        assert torch.equal(outs[0][n_total][0], outs[1][n_total][0])
