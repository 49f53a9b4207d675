"""CPU: the restatement of the reference's Metro and Model25D classes (oracle/port_model_classes.py) - the bone-length solve
recovers a known depth, its bone weights and batch-coupled accept rule, the Metro head as the 3D part of a MeTRAbs head,
the refusals of the Python classes, and the header / ctypes agreement of the new entry points."""
import os
import re
import types

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib
from oracle import port
from oracle import port_model_classes as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_solve_recovers_known_depth():
    """2.5D coordinates by exact projection of one skeleton at four depths and offsets, bone lengths measured on it: the
    solve returns the camera-space joints, so z_ref, to 1e-4 relative."""
    cfg = port.PathConfig(proc_side=256)
    j = 16
    edges = pm.tree_edges(j)
    pose, k, _ = pm.synthetic_pose_25d(1, j, cfg, seed=0)
    shift = torch.tensor([[0., 0., 0.], [150., -80., 900.], [-120., 60., -700.], [40., 30., 1500.]])
    poses = pose + shift[:, None]
    kk = k.expand(4, 3, 3).contiguous()
    proj = poses @ kk.transpose(1, 2)
    c25 = torch.cat([proj[..., :2] / proj[..., 2:], poses[..., 2:] - 5000.0], dim=-1)
    assert pm.port.is_within_fov(c25[..., :2], cfg).all()
    lengths = pm.bone_lengths_of(pose[0], edges)
    for mean_relative in (True, False):
        out = pm.reconstruct_by_bone_lengths(c25, kk, lengths, edges, cfg, mean_relative=mean_relative)
        err = port.relative_error(out, poses)
        assert err < 1e-4, (mean_relative, err)
        z_ref = poses[..., 2].mean(1) if mean_relative else poses[:, -1, 2]
        n2d, z_rel, _, _ = pm.bone_problem(c25, kk, edges, cfg, mean_relative)
        assert torch.allclose(out[..., 2] - z_rel, z_ref[:, None].expand_as(z_rel), rtol=1e-4)


def test_out_of_fov_joints_give_negligible_bone_weights():
    cfg = port.PathConfig(proc_side=256)
    j = 8
    edges = pm.tree_edges(j)
    _, k, c25 = pm.synthetic_pose_25d(2, j, cfg, seed=1)
    c25 = c25.clone()
    c25[0, 3, 0] = -40.0  # joint 3 of crop 0 outside the field of view (lower bound 24 px at stride_train 32)
    c25[1, 5, 1] = 250.0  # joint 5 of crop 1 beyond the upper bound 232 px
    _, _, (c, d, e, w), _ = pm.bone_problem(c25, k, edges, cfg)
    touches = lambda jt: torch.tensor([jt in ed for ed in edges])  # noqa: E731
    assert torch.all(w[0][touches(3)] == np.float32(1e-8))
    assert torch.all(w[0][~touches(3)] == np.float32(1.0) + np.float32(1e-8))
    assert torch.all(w[1][touches(5)] == np.float32(1e-8))
    assert torch.all(w[1][~touches(5)] == np.float32(1.0) + np.float32(1e-8))


def test_step_that_raises_the_batch_objective_moves_no_crop():
    """Crop 0: r = atan(z) from 2, where the Gauss-Newton step overshoots; crop 1: r = z - 1 from 1.1, which one step
    solves.  The batch objective rises, so the first iteration keeps both crops and raises lam; once lam damps crop 0's step
    enough, both crops move together."""
    res = lambda z: torch.stack([torch.atan(z[0]), z[1] - 1])[:, None]  # noqa: E731
    jac = lambda z: torch.stack([1 / (1 + z[0] ** 2), torch.ones_like(z[1])])[:, None]  # noqa: E731
    z0 = torch.tensor([2.0, 1.1])
    trace = []
    z = pm.levenberg_marquardt(res, jac, z0, max_iter=40, trace=trace)
    first = trace[0]
    assert not first['accepted'] and first['new_objective'] > first['objective']
    assert abs(float(first['candidate'][1]) - 1.0) < 1e-6  # alone, crop 1 would have been solved
    assert torch.equal(first['z'], z0)
    assert trace[1]['lam'] == pytest.approx(1e-19, rel=1e-6)
    accepted = [t['accepted'] for t in trace]
    n_rejected = accepted.index(True)
    assert n_rejected > 1 and all(torch.equal(t['z'], z0) for t in trace[:n_rejected])
    assert abs(float(z[0])) < 0.05 and abs(float(z[1]) - 1) < 1e-6


def test_metro_head_is_the_3d_part_of_a_metrabs_head():
    """Same D*J weights, zero 2D weights: Metro's output equals the coords3d_rel of the MeTRAbs head."""
    for hw, channels, j, depth in ((8, 64, 6, 8), (6, 32, 5, 4)):
        cfg = port.PathConfig(proc_side=hw * 32, depth=depth)
        feats, sd = port.head_only_inputs(3, channels, hw, j, depth, seed=2)
        w3, b3 = sd['heatmap_heads.conv_final.weight'][j:], sd['heatmap_heads.conv_final.bias'][j:]
        metrabs_sd = {'heatmap_heads.conv_final.weight': torch.cat([torch.zeros_like(w3[:j]), w3]),
                      'heatmap_heads.conv_final.bias': torch.cat([torch.zeros(j), b3])}
        _, c3d = port.heads(metrabs_sd, feats, cfg, j)
        metro = pm.metro_head(pm.to_volumetric_state_dict(metrabs_sd, j), feats, cfg, j)
        assert torch.allclose(metro, c3d, rtol=0, atol=1e-5 * float(c3d.abs().max())), (hw, depth)


def test_one_long_axis_decodes_to_zero():
    """tf.linspace(0, 1, 1) is [0]: a 1x1 heatmap with D = 1 decodes to the receptive-field offset, unlike ptu's 0.5."""
    cfg = port.PathConfig(proc_side=32, stride_test=32, depth=1)
    feats = torch.randn(2, 16, 1, 1)
    sd = {pm.HEAD_KEY + '.weight': torch.randn(3, 16, 1, 1), pm.HEAD_KEY + '.bias': torch.zeros(3)}
    coords = pm.head_heatmap_coords(sd, feats, cfg, 3)
    assert torch.equal(coords, torch.zeros(2, 3, 3))
    c25 = pm.head_25d(sd, feats, cfg, 3)
    assert torch.equal(c25[..., :2], torch.full((2, 3, 2), 16.0)) and torch.equal(c25[..., 2], torch.zeros(2, 3))


def _tiny_backbone():
    from metrabs_b200.backbones import efficientnet as E
    return torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet('tiny').features)


def _joint_info(n, edges):
    return types.SimpleNamespace(names=[f'j{i}' for i in range(n)], stick_figure_edges=edges, n_joints=n)


@pytest.fixture
def config():
    import metrabs_b200
    old = metrabs_b200.util.get_config()
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=64))
    yield metrabs_b200
    metrabs_b200.set_config(old)


def test_key_schema_and_attributes(config):
    from metrabs_b200.models.metro import Metro
    from metrabs_b200.models.twofive import Model25D
    ji = _joint_info(8, pm.tree_edges(8))
    for m in (Metro(_tiny_backbone(), ji), Model25D(_tiny_backbone(), ji, np.full(7, 300.0))):
        keys = list(m.state_dict())
        assert all(k.startswith('backbone.') or k.startswith('heatmap_head.conv_final.') for k in keys)
        assert tuple(m.state_dict()['heatmap_head.conv_final.weight'].shape) == (8 * 8, 64, 1, 1)
        assert list(m.joint_names) == ji.names and m.joint_edges.shape == (7, 2) and int(m.input_resolution) == 64


def test_refusals(config):
    from metrabs_b200.models.metro import Metro
    from metrabs_b200.models.twofive import Model25D
    from metrabs_b200.multiperson import Pose3dEstimator
    ji = _joint_info(8, pm.tree_edges(8))
    for flag in (dict(transform_coords=True), dict(predict_all_and_latents=True), dict(affine_weights='x'),
                 dict(legacy_centered_stride_bug=True)):
        config.set_config(config.Config(proc_side=64, **flag))
        with pytest.raises(ValueError):
            Metro(_tiny_backbone(), ji)
        with pytest.raises(ValueError):
            Model25D(_tiny_backbone(), ji, np.full(7, 300.0))
    config.set_config(config.Config(proc_side=64))
    with pytest.raises(ValueError):
        Model25D(_tiny_backbone(), ji, np.full(6, 300.0))  # one length per edge
    for bad in (0.0, -5.0, np.nan, np.inf):
        lengths = np.full(7, 300.0)
        lengths[2] = bad
        with pytest.raises(ValueError):
            Model25D(_tiny_backbone(), ji, lengths)
    with pytest.raises(ValueError):
        Model25D(_tiny_backbone(), _joint_info(8, [(0, 1), (1, 8)]), np.full(2, 300.0))
    with pytest.raises(ValueError, match='no absolute output'):
        Pose3dEstimator(Metro(_tiny_backbone(), ji), {'': dict(indices=list(range(8)), names=ji.names, edges=[[0, 1]])}, None)
    Pose3dEstimator(Model25D(_tiny_backbone(), ji, np.full(7, 300.0)),
                    {'': dict(indices=list(range(8)), names=ji.names, edges=[[0, 1]])}, None)
    with pytest.raises(ValueError):
        pm.head_heatmap_coords({}, torch.zeros(1, 4, 2, 2), port.PathConfig(legacy_centered_stride_bug=True), 1)


def test_header_and_binding_agree():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    values = {m[0]: int(m[1]) for m in re.findall(r'MTB_MODEL_([A-Z0-9_]+) = (\d+)', src)}
    assert values == {'METRABS': _lib.MODEL_METRABS, 'METRO': _lib.MODEL_METRO, '25D': _lib.MODEL_25D} == \
        {'METRABS': 0, 'METRO': 1, '25D': 2}
    flat = re.sub(r'\s+', ' ', re.sub(r'/\*.*?\*/', '', src, flags=re.S))
    protos = {
        'mtb_set_model_class': 'int mtb_set_model_class(mtb_handle* h, int model_class, const int32_t* edges, '
                               'const float* bone_lengths, int n_bones, int mean_relative);',
        'mtb_bone_lengths_scratch_bytes': 'size_t mtb_bone_lengths_scratch_bytes(const mtb_handle* h, int batch);',
        'mtb_reconstruct_by_bone_lengths': 'int mtb_reconstruct_by_bone_lengths(mtb_handle* h, const float* coords25d, '
                                           'const float* intrinsics, int batch, float* coords3d_abs, void* scratch, '
                                           'void* stream);'}
    import ctypes as C
    for name, proto in protos.items():
        assert proto in flat, name
        assert name in _lib.EXPORTED_SYMBOLS
        n_args = proto.count(',') + 1
        restype, argtypes = _lib._SIGNATURES[name]
        assert len(argtypes) == n_args and restype == (C.c_size_t if proto.startswith('size_t') else C.c_int), name


def test_sharded_host_path_of_the_model_classes():
    """ShardedMetrabs without the one-call path: a Metro gathers its decoded joints, a Model25D gathers coords25d and
    solves the whole batch (driven through a host-side engine)."""
    from metrabs_b200 import parallel
    cfg = port.PathConfig(proc_side=256)
    _, k, c25 = pm.synthetic_pose_25d(5, 6, cfg, seed=3)
    edges, lengths = pm.tree_edges(6), pm.seeded_bone_lengths(5)

    class Eng:
        n_joints = 6

        def __init__(self, model_class):
            self.model_class = model_class

        def backbone(self, crops):
            return crops

        def head_decode(self, idx):
            return c25[idx.long(), :, :2], c25[idx.long()]

        def allgather(self, t):
            return t[None]

        def reconstruct_by_bone_lengths(self, coords, intrinsics):
            return pm.reconstruct_by_bone_lengths(coords, intrinsics, lengths, edges, cfg)

    idx = torch.arange(5).float()
    out = parallel.ShardedMetrabs(None, 0, 1, engine=Eng(_lib.MODEL_METRO)).forward(idx, None)
    assert torch.equal(out, c25)
    out = parallel.ShardedMetrabs(None, 0, 1, engine=Eng(_lib.MODEL_25D)).forward(idx, k)
    assert torch.equal(out, pm.reconstruct_by_bone_lengths(c25, k, lengths, edges, cfg))
