"""CPU: latent-point MeTRAbs models (affine-combining autoencoder heads).

- the oracle port's latent forward against tests/golden/latents_tiny_s64.npz, which the unmodified reference produced
  (oracle/gen_golden_latents.py) for ``transform_coords`` and ``predict_all_and_latents``;
- the ``Metrabs`` constructor: flag handling, file resolution, weight validation, state_dict schema (no device needed);
- the ragged ``ShardedMetrabs`` path of a latent-point model over gloo: it gathers latents and recombines them after
  the full-batch reconstruction."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import metrabs_b200
from metrabs_b200.backbones import efficientnet as E
from metrabs_b200.models.metrabs import Metrabs
from oracle import port, port_latents

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'latents_tiny_s64.npz')
OPTIONS = ('transform_coords', 'predict_all_and_latents')


def _golden():
    return np.load(GOLDEN)


def n_raw_points(option, g):
    return int(g['n_latents']) if option == 'transform_coords' else int(g['n_latents']) + int(g['n_joints'])


def _joint_info(n):
    return types.SimpleNamespace(names=[f'j{i}' for i in range(n)], stick_figure_edges=[(0, 1)], n_joints=n)


def _write_affine(tmp_path, w1, w2, name='affine.npz'):
    path = os.path.join(str(tmp_path), name)
    np.savez(path, w1=w1, w2=w2)
    return path


def _model(**cfg_kwargs):
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=64, **cfg_kwargs))
    return Metrabs(torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet('tiny').features), _joint_info(10))


@pytest.fixture(autouse=True)
def _restore_config():
    saved = metrabs_b200.get_config()
    yield
    metrabs_b200.set_config(saved)


@pytest.mark.parametrize('option', OPTIONS)
def test_oracle_port_matches_reference_golden(option):
    g = _golden()
    n_lat, n_raw = int(g['n_latents']), n_raw_points(option, g)
    w1, w2 = port_latents.make_affine_weights(int(g['n_joints']), n_lat, seed=0)
    assert np.array_equal(w1, g['w1']) and np.array_equal(w2, g['w2'])
    cfg = port.PathConfig(proc_side=int(g['proc_side']))
    spec = port.effnet_spec(str(g['name']))
    sd = port.make_effnet_state_dict(spec, cfg, n_raw, seed=0)
    crops, k = port.synthetic_inputs(int(g['batch']), int(g['proc_side']), seed=0)
    stages = {}
    with torch.inference_mode():
        out = port_latents.metrabs_forward(sd, spec, cfg, n_raw, crops, k, w2, n_lat, stages=stages)
    assert stages['coords2d'].shape == (int(g['batch']), n_raw, 2)
    assert port.relative_error(stages['coords2d'], g[f'{option}/coords2d']) < 1e-5
    assert port.relative_error(stages['coords3d_rel'], g[f'{option}/coords3d_rel']) < 1e-5
    assert port.relative_error(stages['latents_abs'], g[f'{option}/latents_abs']) < 1e-4
    assert out.shape == (int(g['batch']), int(g['n_joints']), 3)
    assert port.relative_error(out, g[f'{option}/joints']) < 1e-4


def test_affine_weights_are_affine():
    w1, w2 = port_latents.make_affine_weights(555, 48, seed=0)
    assert w1.shape == (555, 48) and w2.shape == (48, 555)
    np.testing.assert_allclose(w1.sum(axis=0), 1.0, rtol=1e-5)
    np.testing.assert_allclose(w2.sum(axis=0), 1.0, rtol=1e-5)


def test_affine_weights_without_a_flag_raise(tmp_path):
    w1, w2 = port_latents.make_affine_weights(10, 6)
    with pytest.raises(ValueError, match='none of transform_coords'):
        _model(affine_weights=_write_affine(tmp_path, w1, w2))


def test_missing_affine_file_raises(tmp_path, monkeypatch):
    monkeypatch.setenv('DATA_ROOT', str(tmp_path))
    with pytest.raises(FileNotFoundError, match='huge8_missing'):
        _model(affine_weights='huge8_missing', transform_coords=True)


def test_affine_name_resolves_under_data_root(tmp_path, monkeypatch):
    w1, w2 = port_latents.make_affine_weights(10, 6)
    os.makedirs(tmp_path / 'skeleton_conversion')
    _write_affine(tmp_path / 'skeleton_conversion', w1, w2, name='huge8_tiny.npz')
    monkeypatch.setenv('DATA_ROOT', str(tmp_path))
    m = _model(affine_weights='huge8_tiny', transform_coords=True)
    assert m.n_latents == 6 and m.heatmap_heads.n_points == 6
    np.testing.assert_array_equal(m.recombination_weights.numpy(), w2)
    np.testing.assert_array_equal(m.encoder_weights.numpy(), w1)
    torch.testing.assert_close(m.reconstruction_weights, torch.from_numpy(w1) @ torch.from_numpy(w2))


@pytest.mark.parametrize('bad', ['w2_joints', 'w1_joints', 'latents'])
def test_affine_shape_mismatch_raises(tmp_path, bad):
    w1, w2 = port_latents.make_affine_weights(10, 6)
    if bad == 'w2_joints':
        w2 = w2[:, :9]
    elif bad == 'w1_joints':
        w1 = w1[:9]
    else:
        w1 = w1[:, :5]
    with pytest.raises(ValueError, match='expected w1'):
        _model(affine_weights=_write_affine(tmp_path, w1, w2), transform_coords=True)


def test_regularize_to_manifold_builds_a_joint_head(tmp_path):
    w1, w2 = port_latents.make_affine_weights(10, 6)
    m = _model(affine_weights=_write_affine(tmp_path, w1, w2), regularize_to_manifold=True)
    assert m.heatmap_heads.n_points == 10 and m.n_latents == 6
    assert not m._latent_forward  # identical to a plain model at inference
    assert m.heatmap_heads.conv_final.weight.shape == (10 * 9, 64, 1, 1)


@pytest.mark.parametrize('option', OPTIONS)
def test_state_dict_schema_equals_reference(tmp_path, option):
    """Same keys and shapes as the reference's state_dict (port.make_effnet_state_dict follows its key schema and
    loads into the reference with strict=True, oracle/gen_golden_latents.py); the autoencoder weights stay outside."""
    g = _golden()
    n_raw = n_raw_points(option, g)
    w1, w2 = port_latents.make_affine_weights(10, 6)
    m = _model(affine_weights=_write_affine(tmp_path, w1, w2), **{option: True})
    sd = port.make_effnet_state_dict(port.effnet_spec('efficientnetv2-tiny'), port.PathConfig(proc_side=64), n_raw)
    ours = m.state_dict()
    assert set(ours) == set(sd)
    assert ours['heatmap_heads.conv_final.weight'].shape == (n_raw * 9, 64, 1, 1)
    assert all(ours[key].shape == sd[key].shape for key in sd)
    m.load_state_dict(sd, strict=True)


class _LatentOracleEngine:
    """Engine-shaped adapter over the oracle port + gloo for a latent-point model (head of n_raw points, the first
    n_latents reconstructed), so ShardedMetrabs.forward itself runs on the CPU."""

    def __init__(self, sd, spec, pcfg, world, n_raw, w2):
        self.sd, self.spec, self.pcfg, self.world, self.n_raw, self.w2 = sd, spec, pcfg, world, n_raw, w2
        self.n_joints, self.n_points = n_raw, w2.shape[0]

    def backbone(self, crops):
        return port.effnet_features(self.sd, self.spec, crops)

    def head_decode(self, feats):
        c2d, c3d = port.heads(self.sd, feats, self.pcfg, self.n_raw)
        return c2d[:, :self.n_points], c3d[:, :self.n_points]

    def allgather(self, t):
        outs = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(outs, t)
        return torch.stack(outs)

    def reconstruct_absolute(self, c2d, c3d, k):
        return port.reconstruct_absolute(c2d, c3d, k, self.pcfg)

    def combine_latents(self, points):
        return port_latents.linear_combine_points(points, self.w2)


def _worker_sharded(rank, world, port_no, n_total, option, out_dir):
    sys.path.insert(0, ROOT)
    from metrabs_b200 import parallel
    from oracle import port as oport
    from oracle import port_latents as olat
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port_no)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(2)
    g = np.load(GOLDEN)
    n_lat, n_raw = int(g['n_latents']), n_raw_points(option, g)
    w2 = torch.from_numpy(g['w2'])
    pcfg = oport.PathConfig(proc_side=64)
    spec = oport.effnet_spec('efficientnetv2-tiny')
    sd = oport.make_effnet_state_dict(spec, pcfg, n_raw, seed=0)
    crops, k = oport.synthetic_inputs(n_total, 64, seed=3)
    eng = _LatentOracleEngine(sd, spec, pcfg, world, n_raw, w2)
    with torch.inference_mode():
        out = parallel.ShardedMetrabs(None, rank, world, engine=eng).forward(crops, k)
        ref = olat.metrabs_forward(sd, spec, pcfg, n_raw, crops, k, w2, n_lat)
    torch.save(dict(out=out, ref=ref), os.path.join(out_dir, f'r{rank}.pt'))
    dist.destroy_process_group()


@pytest.mark.parametrize('option', OPTIONS)
def test_sharded_latent_model_equals_unsharded(tmp_path, option):
    world, n_total = 2, 5  # ragged: 3 + 2 crops
    port_no = 35500 + (os.getpid() % 2000) + OPTIONS.index(option)
    mp.spawn(_worker_sharded, args=(world, port_no, n_total, option, str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f'r{r}.pt') for r in range(world)]
    for o in outs:
        assert o['out'].shape == (n_total, 10, 3)
        assert (o['out'] - o['ref']).abs().max() / o['ref'].abs().max() < 1e-5
    assert torch.equal(outs[0]['out'], outs[1]['out'])
