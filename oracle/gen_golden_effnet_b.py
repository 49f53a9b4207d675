"""TEST INFRASTRUCTURE ONLY - generates the EfficientNet-B fixtures tests/golden/effnetb*.npz by running the UNMODIFIED
reference (oracle/ref_import.py) on torch-cpu.  It writes only these files; the other fixtures are gen_golden.py's.

Run in the build container only:  ``python oracle/gen_golden_effnet_b.py``.  The reference model is built through its
public constructor ``efficientnet_bN()`` (``Metrabs(Sequential(PreprocLayer(), efficientnet_bN().features), ji)``), so the
table, the channel rounding and the BatchNorm eps (1e-5 for B0-B4, 1e-3 for B5-B7) are the reference's own.  The weights
are ``oracle/port_effnet_b.make_state_dict`` (conditioned random init, deterministic from the seed) loaded with
``load_state_dict(strict=True)``, which pins the key schema and every shape.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import port, port_effnet_b  # noqa: E402
from oracle.gen_golden import OUT, state_dict_checksum  # noqa: E402
from oracle.ref_import import import_reference, set_reference_config  # noqa: E402

# (variant, proc_side, n_joints, batch, centered_stride, file)
FIXTURES = [(0, 256, 24, 2, True, 'effnetb0_s256_j24.npz'),
            (3, 384, 24, 1, False, 'effnetb3_s384_j24_nocenter.npz'),
            (5, 256, 24, 2, True, 'effnetb5_s256_j24.npz')]


def reference_b_model(R, variant, n_joints, proc_side):
    """The reference crop model on efficientnet_bN().features (the config must already be set: _efficientnet_conf reads
    centered_stride when the backbone is constructed)."""
    E = R.effnet
    bb = getattr(E, f'efficientnet_b{variant}')()
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(n_joints)], stick_figure_edges=[(0, 1)], n_joints=n_joints)
    m = R.metrabs.Metrabs(torch.nn.Sequential(E.PreprocLayer(), bb.features), ji).eval()
    with torch.inference_mode():  # materialise LazyConv2d (scripts/demo_image.py:69-72)
        m((torch.rand(1, 3, proc_side, proc_side), torch.eye(3)[None]))
    return m


def b_golden(R, variant, proc_side, n_joints, batch, centered_stride, fname, feature_stride=16):
    cfg = port.PathConfig(proc_side=proc_side, centered_stride=centered_stride)
    set_reference_config(cfg.as_reference_dict())
    name = f'efficientnet-b{variant}'
    spec = port_effnet_b.effnet_b_spec(name, centered_stride=centered_stride)
    sd = port_effnet_b.make_state_dict(spec, cfg, n_joints, seed=0)
    m = reference_b_model(R, variant, n_joints, proc_side)
    m.load_state_dict(sd, strict=True)
    eps = {mod.eps for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)}
    assert eps == {spec.bn_eps}, (name, eps)
    crops, k = port.synthetic_inputs(batch, proc_side, seed=0)
    with torch.inference_mode():
        feats = m.backbone(crops)
        c2d, c3d = m.heatmap_heads(feats)
        out = m((crops, k))
    np.savez_compressed(os.path.join(OUT, fname), **dict(
        name=name, proc_side=proc_side, n_joints=n_joints, batch=batch, seed=0, centered_stride=centered_stride,
        legacy_centered_stride_bug=False, feature_stride=feature_stride, bn_eps=spec.bn_eps,
        state_dict_checksum=state_dict_checksum(sd),
        features=feats.numpy().reshape(batch, -1)[:, ::feature_stride].copy(), features_absmean=float(feats.abs().mean()),
        coords2d=c2d.numpy(), coords3d_rel=c3d.numpy(), coords3d_abs=out.numpy()))
    print(fname, 'abs range', float(out.min()), float(out.max()), 'checksum', state_dict_checksum(sd))


def main():
    torch.set_num_threads(8)
    R = import_reference(port.PathConfig().as_reference_dict())
    for variant, side, j, batch, centered, fname in FIXTURES:
        b_golden(R, variant, side, j, batch, centered, fname)


if __name__ == '__main__':
    main()
