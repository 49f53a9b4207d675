"""CPU: EfficientNet-B0..B7.  The restatement (oracle/port_effnet_b.py) against the goldens the unmodified reference
produced through its public efficientnet_bN() (tests/golden/effnetb*.npz, oracle/gen_golden_effnet_b.py); its tables and
BatchNorm eps against the reference's _efficientnet_conf and BN modules (skipped without the reference tree); the parameter
holders of metrabs_b200.backbones.efficientnet against the reference's key schema; and the C ABI values."""
import os
import re

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import efficientnet as E
from oracle import port, port_effnet_b
from oracle.gen_golden import state_dict_checksum
from oracle.ref_import import import_reference, reference_available, set_reference_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = range(8)
# stem, last conv, BN eps, 5x5 depthwise convs, convs (SE fcs included): counted on the reference's constructors
COUNTS = {0: (32, 1280, 1e-5, 9, 81), 1: (32, 1280, 1e-5, 12, 115), 2: (32, 1408, 1e-5, 12, 115),
          3: (40, 1536, 1e-5, 14, 130), 4: (48, 1792, 1e-5, 18, 160), 5: (48, 2048, 1e-3, 21, 194),
          6: (56, 2304, 1e-3, 25, 224), 7: (64, 2560, 1e-3, 30, 273)}
GOLDENS = [('efficientnet-b0', 256, 24, True, 'effnetb0_s256_j24.npz'),
           ('efficientnet-b3', 384, 24, False, 'effnetb3_s384_j24_nocenter.npz'),
           ('efficientnet-b5', 256, 24, True, 'effnetb5_s256_j24.npz')]

needs_reference = pytest.mark.skipif(not reference_available(), reason='reference tree not present')


def _rows(spec):
    return [(s.expand, s.kernel, s.stride, s.cin, s.cout, s.layers, s.bottomright) for s in spec.stages]


def _features(v, centered=True):
    """metrabs_b200's parameter tree of B<v>, on the meta device."""
    stages, last, eps = E.b_stage_table(f'b{v}', centered_stride=centered)
    with torch.device('meta'):
        return E.Features(stages, last, eps)


@pytest.fixture(scope='module')
def R():
    return import_reference(port.PathConfig().as_reference_dict())


@needs_reference
@pytest.mark.parametrize('centered', [True, False])
@pytest.mark.parametrize('v', VARIANTS)
def test_tables_and_eps_equal_the_reference(R, v, centered):
    set_reference_config(port.PathConfig(centered_stride=centered).as_reference_dict())
    width, depth, eps = port_effnet_b.B_VARIANTS[v]
    conf, last = R.effnet._efficientnet_conf(f'efficientnet_b{v}', width_mult=width, depth_mult=depth)
    spec = port_effnet_b.effnet_b_spec(f'efficientnet-b{v}', centered_stride=centered)
    assert _rows(spec) == [(c.expand_ratio, c.kernel, c.stride, c.input_channels, c.out_channels, c.num_layers,
                            bool(c.bottomright_stride)) for c in conf]
    assert all(isinstance(c, R.effnet.MBConvConfig) for c in conf) and last is None
    with torch.device('meta'):
        ref = getattr(R.effnet, f'efficientnet_b{v}')()
    assert {m.eps for m in ref.modules() if isinstance(m, torch.nn.BatchNorm2d)} == {spec.bn_eps}
    # the multipliers above are the constructor's own: its features have the spec's shapes
    ref_shapes = {k: tuple(t.shape) for k, t in ref.features.state_dict().items()}
    ours = _features(v, centered)
    assert ref_shapes == {k: tuple(t.shape) for k, t in ours.state_dict().items()}
    assert {m.eps for m in ours.modules() if isinstance(m, torch.nn.BatchNorm2d)} == {spec.bn_eps}
    stem, last_ch, eps_, n5, nconv = COUNTS[v]
    convs = [m for m in ref.features.modules() if isinstance(m, torch.nn.Conv2d)]
    assert (spec.stem_channels, spec.last_channel, spec.bn_eps) == (stem, last_ch, eps_)
    assert (sum(m.kernel_size == (5, 5) for m in convs), len(convs)) == (n5, nconv)


@pytest.mark.parametrize('centered', [True, False])
@pytest.mark.parametrize('v', VARIANTS)
def test_backbone_tables_equal_the_restatement(v, centered):
    stages, last, eps = E.b_stage_table(f'b{v}', centered_stride=centered)
    spec = port_effnet_b.effnet_b_spec(f'efficientnet-b{v}', centered_stride=centered)
    assert [(s['expand'], s['kernel'], s['stride'], s['cin'], s['cout'], s['layers'], s['bottomright']) for s in stages] == \
        _rows(spec)
    assert all(s['block'] == 'mb' for s in stages)
    assert (last, eps) == (spec.last_channel, spec.bn_eps)
    assert all(c % 8 == 0 for s in stages for c in (s['cin'], s['cout']))
    assert [s['bottomright'] for s in stages] == [False] * 5 + [centered, False]
    f = _features(v, centered)
    assert f.arch == (_lib.ARCH_EFFNET_EPS1E5 if v < 5 else _lib.ARCH_EFFNET) and f.bn_eps == eps
    # stage 1 has expand 1: no expand conv, keys block.0 dw, .1 SE, .2 project
    keys = set(f.state_dict())
    assert {'1.0.block.0.0.weight', '1.0.block.1.fc1.weight', '1.0.block.2.0.weight'} <= keys
    assert '1.0.block.3.0.weight' not in keys and '2.0.block.3.0.weight' in keys


@pytest.mark.parametrize('name,side', [('efficientnet-b0', 64), ('efficientnet-b3', 96)])
def test_state_dict_loads_strict(name, side):
    """The restatement's state dict, a stand-in for a checkpoint of Metrabs(Sequential(PreprocLayer(), efficientnet_bN()
    .features), ji) (the golden generator loads the same dict into that reference model with strict=True), loads into
    metrabs_b200's model with strict=True."""
    import types
    from metrabs_b200.models.metrabs import Metrabs
    import metrabs_b200
    pcfg = port.PathConfig(proc_side=side)
    spec = port_effnet_b.effnet_b_spec(name)
    sd = port_effnet_b.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=side))
    bb = getattr(E, 'efficientnet_' + name.split('-')[1])()
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(8)], stick_figure_edges=[(0, 1)], n_joints=8)
    m = Metrabs(torch.nn.Sequential(E.PreprocLayer(), bb.features), ji)
    m.load_state_dict(sd, strict=True)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in sd.items()}


@pytest.mark.parametrize('name,side,j,centered,fname', GOLDENS)
def test_port_matches_reference_goldens(golden_dir, name, side, j, centered, fname):
    g = np.load(os.path.join(golden_dir, fname), allow_pickle=False)
    assert str(g['name']) == name and int(g['proc_side']) == side and bool(g['centered_stride']) == centered
    pcfg = port.PathConfig(proc_side=side, centered_stride=centered)
    spec = port_effnet_b.effnet_b_spec(name, centered_stride=centered)
    assert float(g['bn_eps']) == spec.bn_eps
    sd = port_effnet_b.make_state_dict(spec, pcfg, j, seed=int(g['seed']))
    assert abs(state_dict_checksum(sd) - float(g['state_dict_checksum'])) <= 1e-9 * float(g['state_dict_checksum'])
    batch = int(g['batch'])
    crops, k = port.synthetic_inputs(batch, side, seed=int(g['seed']))
    stages = {}
    with torch.inference_mode():
        out = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    feats = stages['features'].reshape(batch, -1)[:, ::int(g['feature_stride'])]
    assert port.relative_error(feats, g['features']) < 1e-5
    assert port.relative_error(stages['coords2d'], g['coords2d']) < 1e-5
    assert port.relative_error(stages['coords3d_rel'], g['coords3d_rel']) < 1e-5
    assert port.relative_error(out, g['coords3d_abs']) < 1e-4


def test_header_values():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    assert int(re.search(r'MTB_ARCH_EFFNET_EPS1E5 = (\d+)', src).group(1)) == _lib.ARCH_EFFNET_EPS1E5 == 9
    assert 'MTB_DW_5X5_POOL_16B = MTB_DW_5X5_16B + 1' in src
    assert _lib.DW_5X5_POOL_16B == _lib.DW_5X5_16B + 1 == 5


@pytest.mark.parametrize('row', [dict(block='fused'), dict(kernel=7), dict(stride=3)])
def test_eps1e5_arch_rejects_other_rows(row):
    """MTB_ARCH_EFFNET_EPS1E5 takes MBConv rows with kernel 3 or 5 and stride 1 or 2 only (checked before any device
    is needed)."""
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libmetrabs_b200.so not built')
    import metrabs_b200
    from metrabs_b200.engine import Engine, make_config
    stages, last, _eps = E.b_stage_table('b0', centered_stride=True)
    stages[2] = dict(stages[2], **row)
    with pytest.raises(_lib.MetrabsB200Error, match='only MBConv rows'):
        Engine(make_config(metrabs_b200.Config(proc_side=64), 8, stages=stages, last_channel=last,
                           arch=_lib.ARCH_EFFNET_EPS1E5))
