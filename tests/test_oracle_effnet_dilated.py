"""CPU: EfficientNetV2 at output stride 16 and 8.  The derived stage tables equal the TF reference's
``efficientnetv2-{s,l}-stride{16,8}`` block strings; the stride-32 tables are unchanged; the refusals raise; the oracle
restatement (oracle/port_effnet_dilated.py) meets the fixtures of the reference's dilated modules; and the ctypes
``MtbStage`` matches the header struct."""
import ast
import os
import re

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib
from metrabs_b200.backbones import efficientnet as E
from oracle import port
from oracle import port_effnet_dilated as D
from oracle.ref_import import REFERENCE_ROOT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
TF_CONFIGS = os.path.join(REFERENCE_ROOT, 'metrabs_tf', 'backbones', 'efficientnet', 'effnetv2_configs.py')
KEYS = ('block', 'expand', 'kernel', 'stride', 'cin', 'cout', 'layers', 'bottomright', 'dilation_in', 'dilation_out')


def reference_blocks(name, centered_stride):
    """The block list ``name`` of effnetv2_configs.py, decoded like BlockDecoder._decode_block_string (:26-50) into stage
    dicts.  Read with ast: importing the file pulls in TF-side modules."""
    if not os.path.exists(TF_CONFIGS):
        pytest.skip('reference tree not present')
    tree = ast.parse(open(TF_CONFIGS).read())
    rows = next(ast.literal_eval(n.value) for n in tree.body
                if isinstance(n, ast.Assign) and any(getattr(t, 'id', None) == name for t in n.targets))
    stages = []
    for s in rows:
        ops = s.split('_')
        o = {}
        for op in ops:
            parts = re.split(r'(\d.*)', op)
            if len(parts) >= 2:
                o[parts[0]] = parts[1]
        stages.append(dict(block='fused' if int(o.get('c', 0)) == 1 else 'mb', expand=int(o['e']), kernel=int(o['k']),
                           stride=int(o['s']), cin=int(o['i']), cout=int(o['o']), layers=int(o['r']),
                           bottomright='br' in ops and centered_stride, dilation_in=int(o['din']),
                           dilation_out=int(o['dout'])))
    return stages


@pytest.mark.parametrize('centered', [True, False])
@pytest.mark.parametrize('size,output_stride,ref', [
    ('s', 16, 'v2_s_block_stride16'), ('s', 8, 'v2_s_block_stride8'), ('s', 32, 'v2_s_block'),
    ('l', 16, 'v2_l_block_stride16'), ('l', 8, 'v2_l_block_stride8'), ('l', 32, 'v2_l_block'), ('m', 32, 'v2_m_block')])
def test_stage_table_equals_the_reference(size, output_stride, ref, centered):
    stages, last = E.stage_table(size, centered, output_stride=output_stride)
    assert [{k: st[k] for k in KEYS} for st in stages] == reference_blocks(ref, centered)
    assert last == 1280
    spec = D.effnet_spec(f'efficientnetv2-{size}', centered, output_stride)  # the oracle applies the same rule
    assert [tuple(getattr(s, k) for k in KEYS) for s in spec.stages] == [tuple(st[k] for k in KEYS) for st in stages]


@pytest.mark.parametrize('centered', [True, False])
def test_stride32_tables_are_unchanged(centered):
    for size in ('s', 'm', 'l', 'tiny'):
        stages, _ = E.stage_table(size, centered)
        assert stages == E.stage_table(size, centered, output_stride=32)[0]
        assert stages == E.dilate_stages(stages, 32, centered)  # the rule is the identity at 32
        assert all(st['dilation_in'] == st['dilation_out'] == 1 for st in stages)
        base = port.effnet_spec(f'efficientnetv2-{size}', centered).stages
        assert [tuple(st[k] for k in KEYS[:8]) for st in stages] == [
            (s.block, s.expand, s.kernel, s.stride, s.cin, s.cout, s.layers, s.bottomright) for s in base]
    for v in range(8):
        stages, _, _ = E.b_stage_table(f'b{v}', centered)
        assert all(st['dilation_in'] == st['dilation_out'] == 1 for st in stages)


def test_output_stride_reaches_the_features():
    for size, output_stride, side in [('s', 16, 16), ('l', 8, 32), ('tiny', 8, 8)]:
        feats = E.EfficientNet(size, output_stride).features
        assert feats.output_stride == output_stride
    assert E.efficientnet_v2_s(output_stride=16).features.output_stride == 16
    assert E.efficientnet_v2_l(output_stride=8).features.output_stride == 8
    assert E.efficientnet_v2_tiny(output_stride=16).features.output_stride == 16
    assert E.EfficientNet('l').features.output_stride == 32
    assert E.EfficientNet('b0').features.output_stride == 32


@pytest.mark.parametrize('size,output_stride', [('m', 16), ('m', 8), ('b0', 16), ('b3', 8), ('b7', 16), ('s', 4),
                                                ('l', 4), ('s', 12), ('l', 64)])
def test_refusals(size, output_stride):
    with pytest.raises(ValueError):
        E.EfficientNet(size, output_stride)
    if size in ('s', 'l', 'm'):
        with pytest.raises(ValueError):
            E.stage_table(size, True, output_stride=output_stride)


@pytest.mark.parametrize('fname', ['tiny_s64_j8_os16.npz', 'tiny_s64_j8_os8.npz'])
def test_tiny_oracle_meets_the_reference(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    os_ = int(g['output_stride'])
    cfg = port.PathConfig(proc_side=int(g['proc_side']), stride_test=os_)
    spec = D.effnet_spec(str(g['name']), output_stride=os_)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith('sd/')}
    stages = {}
    with torch.inference_mode():
        out = port.metrabs_forward(sd, spec, cfg, int(g['n_joints']), torch.from_numpy(g['crops']),
                                   torch.from_numpy(g['intrinsics']), stages=stages)
    assert stages['features'].shape[-1] == cfg.proc_side // os_
    assert port.relative_error(stages['features'].numpy().reshape(int(g['batch']), -1), g['features']) < 1e-5
    assert port.relative_error(stages['coords2d'], g['coords2d']) < 1e-5
    assert port.relative_error(stages['coords3d_rel'], g['coords3d_rel']) < 1e-5
    assert port.relative_error(out, g['coords3d_abs']) < 1e-5
    sd2 = D.make_state_dict(spec, cfg, int(g['n_joints']), seed=0)  # the committed weights are the seeded init
    assert sd2.keys() == sd.keys()
    for k in sd:
        assert port.relative_error(sd2[k].float(), sd[k].float()) < 1e-4, k


@pytest.mark.parametrize('fname', ['effnetv2s_s256_j24_os16.npz', 'effnetv2l_s256_j24_os8.npz'])
def test_full_models_meet_the_reference(fname):
    """Weights regenerated from the seed (the init runs a BN calibration forward, whose summation order may differ across
    machines by ~1e-5, so the state dict is pinned by its checksum and the outputs to 1e-5 relative)."""
    g = np.load(os.path.join(GOLDEN, fname))
    s, j, b, os_ = int(g['proc_side']), int(g['n_joints']), int(g['batch']), int(g['output_stride'])
    cfg = port.PathConfig(proc_side=s, stride_test=os_)
    spec = D.effnet_spec(str(g['name']), output_stride=os_)
    sd = D.make_state_dict(spec, cfg, j, seed=0, calib_batch=2 if b < 3 else 4)
    chk = float(sum(v.double().abs().sum() for k, v in sorted(sd.items()) if v.ndim > 0))
    assert abs(chk - float(g['state_dict_checksum'])) < 1e-6 * abs(chk)
    crops, k = port.synthetic_inputs(b, s, seed=0)
    stages = {}
    with torch.inference_mode():
        out = port.metrabs_forward(sd, spec, cfg, j, crops, k, stages=stages)
    feats = stages['features'].numpy().reshape(b, -1)[:, ::int(g['feature_stride'])]
    assert port.relative_error(feats, g['features']) < 1e-5
    assert port.relative_error(stages['coords2d'], g['coords2d']) < 1e-5
    assert port.relative_error(stages['coords3d_rel'], g['coords3d_rel']) < 1e-5
    assert port.relative_error(out, g['coords3d_abs']) < 1e-5


def test_mtb_stage_matches_the_header():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    body = re.search(r'typedef struct \{(.*?)\} mtb_stage;', src, re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = [n.strip() for decl in body.split(';') if decl.strip() for n in decl.strip()[len('int32_t'):].split(',')]
    assert [f for f, _ in _lib.MtbStage._fields_] == fields
    assert fields[-2:] == ['dilation_in', 'dilation_out']
    assert re.search(r'#define MTB_ABI_VERSION (\d+)', src).group(1) == str(_lib.MTB_ABI_VERSION) == '2'


def test_make_config_fills_the_dilations():
    import metrabs_b200
    from metrabs_b200.engine import make_config
    stages, last = E.stage_table('l', True, output_stride=8)
    c = make_config(metrabs_b200.Config(proc_side=256, stride_test=8), 24, stages=stages, last_channel=last)
    assert [(c.stages[i].stride, c.stages[i].dilation_in, c.stages[i].dilation_out) for i in range(c.n_stages)] == [
        (st['stride'], st['dilation_in'], st['dilation_out']) for st in stages]


def _create(stages, last, stride_test):
    import metrabs_b200
    from metrabs_b200.engine import Engine, make_config
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libmetrabs_b200.so not built')
    return Engine(make_config(metrabs_b200.Config(proc_side=256, stride_test=stride_test), 24, stages=stages,
                              last_channel=last))


@pytest.mark.parametrize('size,output_stride,stride_test', [('l', 8, 32), ('l', 8, 16), ('s', 16, 32), ('s', 16, 8)])
def test_create_rejects_a_table_off_stride_test(size, output_stride, stride_test):
    """A dilated table decodes with stride_test's geometry, so the two must agree (checked before any device is needed)."""
    stages, last = E.stage_table(size, True, output_stride=output_stride)
    with pytest.raises(_lib.MetrabsB200Error, match=f'output stride {output_stride} but stride_test is {stride_test}'):
        _create(stages, last, stride_test)


@pytest.mark.parametrize('stage,row', [(1, dict(dilation_in=2, dilation_out=2)), (2, dict(dilation_out=2)),
                                       (5, dict(dilation_in=0)), (5, dict(dilation_out=16))])
def test_create_rejects_unsupported_dilations(stage, row):
    """FusedMBConv rows are never dilated (output stride 4 is not built); dilations outside 1..8 are refused."""
    stages, last = E.stage_table('s', True, output_stride=16)
    stages[stage] = dict(stages[stage], **row)
    with pytest.raises(_lib.MetrabsB200Error, match='dilation'):
        _create(stages, last, 16)
