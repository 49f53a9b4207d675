"""CPU: EfficientNetV2-B0..B3 and -XL.  The stage tables of metrabs_b200.backbones.efficientnet and of the restatement
(oracle/port_effnet_v2_variants.py) equal the TF reference's ``efficientnetv2-b0`` .. ``-b3`` / ``-xl`` block strings after
TF rounding (read from the reference tree, skipped without it); the tables are the ones worked out by hand; other output
strides are refused; the B names stay the V1 nets; the seeded state dicts load strictly into metrabs_b200's model and
the reference's PyTorch module; and the restatement meets the goldens the reference module produced
(tests/golden/effnetv2{b0,b3,xl}_*.npz, oracle/gen_golden_effnet_v2_variants.py)."""
import ast
import math
import os
import types

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import efficientnet as E
from oracle import port
from oracle import port_effnet_v2_variants as V
from oracle.gen_golden import state_dict_checksum
from oracle.ref_import import import_reference, reference_available, set_reference_config
from tests.test_oracle_effnet_dilated import KEYS, TF_CONFIGS, reference_blocks

SIZES = {'efficientnetv2-b0': 'v2-b0', 'efficientnetv2-b1': 'v2-b1', 'efficientnetv2-b2': 'v2-b2',
         'efficientnetv2-b3': 'v2-b3', 'efficientnetv2-xl': 'xl'}
# stem, stage couts, repeats, head, identity-shaped FusedMBConv blocks (Cin, Cexp): worked out by hand from the TF tables
EXPECTED = {'efficientnetv2-b0': (32, [16, 32, 48, 96, 112, 192], [1, 2, 2, 3, 5, 8], 1280, [(32, 128), (48, 192)]),
            'efficientnetv2-b1': (32, [16, 32, 48, 96, 112, 192], [2, 3, 3, 4, 6, 9], 1280, [(32, 128), (48, 192)]),
            'efficientnetv2-b2': (32, [16, 32, 56, 104, 120, 208], [2, 3, 3, 4, 6, 10], 1408, [(32, 128), (56, 224)]),
            'efficientnetv2-b3': (40, [16, 40, 56, 112, 136, 232], [2, 3, 3, 5, 7, 12], 1536, [(40, 160), (56, 224)]),
            'efficientnetv2-xl': (32, [32, 64, 96, 192, 256, 512, 640], [4, 8, 8, 16, 24, 32, 8], 1280,
                                  [(64, 256), (96, 384)])}
GOLDENS = ['effnetv2b0_s224_j24.npz', 'effnetv2b3_s256_j24.npz', 'effnetv2xl_s256_j24.npz']

needs_reference = pytest.mark.skipif(not reference_available(), reason='reference tree not present')


def tf_params(name):
    """(block list name, width, depth) of ``name`` in effnetv2_configs.efficientnetv2_params, read with ast."""
    tree = ast.parse(open(TF_CONFIGS).read())
    params = next(n.value for n in tree.body
                  if isinstance(n, ast.Assign) and any(getattr(t, 'id', None) == 'efficientnetv2_params' for t in n.targets))
    for k, v in zip(params.keys, params.values):
        if ast.literal_eval(k) == name:
            return v.elts[0].id, ast.literal_eval(v.elts[1]), ast.literal_eval(v.elts[2])
    raise KeyError(name)


def tf_round_filters(filters, multiplier, divisor=8):
    filters *= multiplier
    return int(max(divisor, int(filters + divisor / 2) // divisor * divisor))


def tf_table(name, centered):
    """The TF model's scaled stage dicts (effnetv2_model.py:574-600: round_filters on input and output filters,
    round_repeats on the repeats) and its head width (:479)."""
    block, width, depth = tf_params(name)
    rows = reference_blocks(block, centered)
    for r in rows:
        r.update(cin=tf_round_filters(r['cin'], width), cout=tf_round_filters(r['cout'], width),
                 layers=int(math.ceil(depth * r['layers'])))
    return rows, tf_round_filters(1280, width)


@pytest.mark.parametrize('centered', [True, False])
@pytest.mark.parametrize('name', list(SIZES))
def test_tables_equal_the_tf_reference(name, centered):
    if not os.path.exists(TF_CONFIGS):
        pytest.skip('reference tree not present')
    rows, head = tf_table(name, centered)
    stages, last = E.stage_table(SIZES[name], centered)
    assert [{k: st[k] for k in KEYS} for st in stages] == rows
    assert last == head
    spec = V.effnet_spec(name, centered)
    assert [(s.block, s.expand, s.kernel, s.stride, s.cin, s.cout, s.layers, s.bottomright) for s in spec.stages] == [
        tuple(r[k] for k in KEYS[:8]) for r in rows]
    assert spec.last_channel == head and spec.stem_channels == tf_round_filters(32, tf_params(name)[1])


@pytest.mark.parametrize('name', list(SIZES))
def test_tables_are_the_hand_derived_ones(name):
    stem, couts, repeats, head, fused = EXPECTED[name]
    stages, last = E.stage_table(SIZES[name], True)
    assert (stages[0]['cin'], [s['cout'] for s in stages], [s['layers'] for s in stages], last) == (stem, couts, repeats, head)
    assert [s['bottomright'] for s in stages] == [s['stride'] == 2 and i == max(
        j for j, t in enumerate(stages) if t['stride'] == 2) for i, s in enumerate(stages)]
    spec = V.effnet_spec(name)
    assert V.identity_fused_blocks(spec) == fused
    feats = E.EfficientNet(SIZES[name]).features
    assert feats.arch == _lib.ARCH_EFFNET and feats.bn_eps == 1e-3 and feats.output_stride == 32
    assert {m.eps for m in feats.modules() if isinstance(m, torch.nn.BatchNorm2d)} == {1e-3}
    # SE width max(1, int(block input * 0.25)) on every MBConv block
    for si, st in enumerate(stages):
        for bi in range(st['layers']):
            if st['block'] == 'mb':
                cin = st['cin'] if bi == 0 else st['cout']
                assert feats._modules[str(si + 1)][bi].block[2 if st['expand'] != 1 else 1].fc1.out_channels == max(1, int(cin * 0.25))
    if name == 'efficientnetv2-xl':
        assert sum(s['layers'] for s in stages) == 100


def test_constructors():
    for fn, size in [(E.efficientnet_v2_xl, 'xl'), (E.efficientnet_v2_b0, 'v2-b0'), (E.efficientnet_v2_b1, 'v2-b1'),
                     (E.efficientnet_v2_b2, 'v2-b2'), (E.efficientnet_v2_b3, 'v2-b3')]:
        m = fn()
        assert m.size == size and m.features.stages == E.stage_table(size)[0]
    # 'b0'..'b7' stay EfficientNet-B (V1: MBConv rows only, torchvision's 0.9 rounding, BN eps 1e-5 up to B4)
    for v in range(8):
        f = E.EfficientNet(f'b{v}').features
        assert f.stages == E.b_stage_table(f'b{v}')[0] and all(s['block'] == 'mb' for s in f.stages)
    assert E.EfficientNet('b3').features.stages[0]['cin'] == 40 and E.EfficientNet('b3').features.bn_eps == 1e-5


@pytest.mark.parametrize('output_stride', [16, 8, 4])
@pytest.mark.parametrize('size', ['v2-b0', 'v2-b1', 'v2-b2', 'v2-b3', 'xl'])
def test_other_output_strides_raise(size, output_stride):
    with pytest.raises(ValueError):
        E.EfficientNet(size, output_stride)
    with pytest.raises(ValueError):
        E.stage_table(size, True, output_stride=output_stride)


def _crop_model(size, side, n_joints):
    import metrabs_b200
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=side))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(n_joints)], stick_figure_edges=[(0, 1)], n_joints=n_joints)
    return Metrabs(torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet(size).features), ji)


@pytest.mark.parametrize('name', list(SIZES))
def test_state_dict_loads_strict(name):
    """The seeded state dict (a stand-in for a checkpoint of the reference model; the golden generator loads the same
    kind of dict into the reference's PyTorch module with strict=True) loads into metrabs_b200's model with strict=True."""
    side = 64
    pcfg = port.PathConfig(proc_side=side)
    spec = V.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    m = _crop_model(SIZES[name], side, 8)
    m.load_state_dict(sd, strict=True)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in sd.items()}


@needs_reference
@pytest.mark.parametrize('name', list(SIZES))
def test_state_dict_loads_strict_into_the_reference_module(name):
    from oracle.gen_golden import build_reference_model
    side = 64
    pcfg = port.PathConfig(proc_side=side)
    R = import_reference(pcfg.as_reference_dict())
    set_reference_config(pcfg.as_reference_dict())
    spec = V.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    m = build_reference_model(R, spec, 8, side)
    m.load_state_dict(sd, strict=True)
    assert {k for k in m.state_dict()} == set(sd)


@pytest.mark.parametrize('fname', GOLDENS)
def test_port_matches_reference_goldens(golden_dir, fname):
    """Weights regenerated from the seed (the init runs a BN calibration forward whose summation order may differ across
    machines, so the state dict is pinned by its checksum and the outputs to 1e-5 relative)."""
    g = np.load(os.path.join(golden_dir, fname), allow_pickle=False)
    name, side, j, b = str(g['name']), int(g['proc_side']), int(g['n_joints']), int(g['batch'])
    pcfg = port.PathConfig(proc_side=side)
    spec = V.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, j, seed=int(g['seed']), calib_batch=int(g['calib_batch']))
    chk = state_dict_checksum(sd)
    assert abs(chk - float(g['state_dict_checksum'])) < 1e-6 * abs(chk)
    crops, k = port.synthetic_inputs(b, side, seed=int(g['seed']))
    stages = {}
    with torch.inference_mode():
        out = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=stages)
    assert stages['features'].shape[-1] == side // 32
    feats = stages['features'].numpy().reshape(b, -1)[:, ::int(g['feature_stride'])]
    assert port.relative_error(feats, g['features']) < 1e-5
    assert port.relative_error(stages['coords2d'], g['coords2d']) < 1e-5
    assert port.relative_error(stages['coords3d_rel'], g['coords3d_rel']) < 1e-5
    assert port.relative_error(out, g['coords3d_abs']) < 1e-5
