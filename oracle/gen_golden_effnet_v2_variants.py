"""TEST INFRASTRUCTURE ONLY - generates the EfficientNetV2-B0..B3 / -XL fixtures
tests/golden/{effnetv2b0_s224_j24, effnetv2b3_s256_j24, effnetv2xl_s256_j24}.npz on torch-cpu.  It writes only these files.

Run where the reference tree is present:  ``python oracle/gen_golden_effnet_v2_variants.py``.

What the fixtures pin: these backbones are TF-only in the reference (``efficientnetv2-b0`` .. ``-b3``, ``efficientnetv2-xl``,
``metrabs_tf/backbones/efficientnet/effnetv2_configs.py`` :249-282), and the TF model cannot run without TensorFlow.  So
this script builds the reference's own PyTorch ``EfficientNet`` (``metrabs_pytorch/backbones/efficientnet.py`` :238-330)
from ``FusedMBConvConfig`` / ``MBConvConfig`` rows with the channels, layer counts, ``bottomright_stride`` flags and
``last_channel`` of ``oracle/port_effnet_v2_variants.effnet_spec`` (TF rounding), BatchNorm eps 1e-3.  The weights are
``port.make_effnet_state_dict`` (conditioned random init, deterministic from the seed) loaded with
``load_state_dict(strict=True)``.  Like the existing full-model fixtures, each file stores a state-dict checksum and
subsampled features, not the weights.  V2-B0 runs at 224, its eval size; V2-B3 at 256 with two crops; XL at 256 with one.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import port, port_effnet_v2_variants as V  # noqa: E402
from oracle.gen_golden import OUT, build_reference_model, state_dict_checksum  # noqa: E402
from oracle.ref_import import import_reference, set_reference_config  # noqa: E402

# (name, proc_side, n_joints, batch, calib_batch, feature_stride, file)
FIXTURES = [('efficientnetv2-b0', 224, 24, 2, 2, 16, 'effnetv2b0_s224_j24.npz'),
            ('efficientnetv2-b3', 256, 24, 2, 2, 16, 'effnetv2b3_s256_j24.npz'),
            ('efficientnetv2-xl', 256, 24, 1, 2, 16, 'effnetv2xl_s256_j24.npz')]


def golden(R, name, proc_side, n_joints, batch, calib_batch, feature_stride, fname):
    cfg = port.PathConfig(proc_side=proc_side)
    set_reference_config(cfg.as_reference_dict())
    spec = V.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, cfg, n_joints, seed=0, calib_batch=calib_batch)
    m = build_reference_model(R, spec, n_joints, proc_side)
    m.load_state_dict(sd, strict=True)
    crops, k = port.synthetic_inputs(batch, proc_side, seed=0)
    with torch.inference_mode():
        feats = m.backbone(crops)
        c2d, c3d = m.heatmap_heads(feats)
        out = m((crops, k))
    np.savez_compressed(os.path.join(OUT, fname), **dict(
        name=name, proc_side=proc_side, n_joints=n_joints, batch=batch, seed=0, calib_batch=calib_batch,
        centered_stride=True, legacy_centered_stride_bug=False, feature_stride=feature_stride,
        state_dict_checksum=state_dict_checksum(sd),
        features=feats.numpy().reshape(batch, -1)[:, ::feature_stride].copy(), features_absmean=float(feats.abs().mean()),
        coords2d=c2d.numpy(), coords3d_rel=c3d.numpy(), coords3d_abs=out.numpy()))
    print(fname, f'features {tuple(feats.shape)}, abs range', float(out.min()), float(out.max()),
          'checksum', state_dict_checksum(sd))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    R = import_reference(port.PathConfig().as_reference_dict())
    for f in FIXTURES:
        golden(R, *f)


if __name__ == '__main__':
    main()
