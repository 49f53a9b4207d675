"""TEST INFRASTRUCTURE ONLY - generates the fixtures of EfficientNetV2 at output stride 16 and 8,
tests/golden/{tiny_s64_j8_os16, tiny_s64_j8_os8, effnetv2s_s256_j24_os16, effnetv2l_s256_j24_os8}.npz, on torch-cpu.  It writes
only these files.

Run where the reference tree is present:  ``python oracle/gen_golden_effnet_dilated.py``.

What the fixtures pin: the dilated backbones are TF-only in the reference (``efficientnetv2-{s,l}-stride{16,8}``,
``metrabs_tf/backbones/efficientnet/effnetv2_configs.py`` :163-228), and the TF model cannot run without TensorFlow.  So this
script builds the reference's own PyTorch modules, re-strided and dilated per the TF tables:

* ``EfficientNet`` (``metrabs_pytorch/backbones/efficientnet.py``) from ``MBConvConfig`` / ``FusedMBConvConfig`` rows with the
  strides and ``bottomright_stride`` of ``oracle/port_effnet_dilated.effnet_spec``;
* in each block with dilation d > 1, its depthwise ``Conv2d.dilation = (d, d)`` and its ``padding`` module replaced by the
  reference's ``fixed_padding_layer(k, rate=d)``.

The weights are ``port_effnet_dilated.make_state_dict`` (conditioned random init, deterministic from the seed) loaded with
``load_state_dict(strict=True)``.  The tiny fixtures carry their weights; the S and L ones store a checksum and features
subsampled like the existing full-model fixtures.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import port, port_effnet_dilated as D  # noqa: E402
from oracle.gen_golden import OUT, build_reference_model, state_dict_checksum  # noqa: E402
from oracle.ref_import import import_reference, set_reference_config  # noqa: E402

# (name, output_stride, proc_side, n_joints, batch, store_weights, feature_stride, file)
FIXTURES = [('efficientnetv2-tiny', 16, 64, 8, 3, True, 1, 'tiny_s64_j8_os16.npz'),
            ('efficientnetv2-tiny', 8, 64, 8, 3, True, 1, 'tiny_s64_j8_os8.npz'),
            ('efficientnetv2-s', 16, 256, 24, 2, False, 16, 'effnetv2s_s256_j24_os16.npz'),
            ('efficientnetv2-l', 8, 256, 24, 1, False, 64, 'effnetv2l_s256_j24_os8.npz')]


def dilate_reference_model(m, spec):
    """Dilates the depthwise conv of every block of the reference model ``m`` whose dilation is > 1, with the reference's
    fixed_padding_layer(k, rate=d) in front of it (efficientnet.py:1127-1161)."""
    R_eff = sys.modules['metrabs_pytorch.backbones.efficientnet']
    feats = m.backbone[1]
    n = 0
    for b in D.block_list(spec):
        si, bi = (int(v) for v in b['key'].split('.'))
        blk = feats._modules[str(si)][bi].block
        if b['dil'] == 1:
            continue
        dw = [mod for mod in blk.modules() if isinstance(mod, torch.nn.Conv2d) and mod.groups > 1]
        assert len(dw) == 1 and 'padding' in blk._modules, b
        dw[0].dilation = (b['dil'], b['dil'])
        blk._modules['padding'] = R_eff.fixed_padding_layer(b['kernel'], rate=b['dil'], shifts=(b['shift'], b['shift']))
        n += 1
    return n


def golden(R, name, output_stride, proc_side, n_joints, batch, store_weights, feature_stride, fname):
    cfg = port.PathConfig(proc_side=proc_side, stride_test=output_stride)
    set_reference_config(cfg.as_reference_dict())
    spec = D.effnet_spec(name, output_stride=output_stride)
    sd = D.make_state_dict(spec, cfg, n_joints, seed=0, calib_batch=2 if batch < 3 else 4)
    m = build_reference_model(R, spec, n_joints, proc_side)
    n_dil = dilate_reference_model(m, spec)
    m.load_state_dict(sd, strict=True)
    crops, k = port.synthetic_inputs(batch, proc_side, seed=0)
    with torch.inference_mode():
        feats = m.backbone(crops)
        c2d, c3d = m.heatmap_heads(feats)
        out = m((crops, k))
    assert feats.shape[-1] == proc_side // output_stride, feats.shape
    data = dict(name=name, output_stride=output_stride, proc_side=proc_side, n_joints=n_joints, batch=batch, seed=0,
                centered_stride=True, legacy_centered_stride_bug=False, feature_stride=feature_stride,
                state_dict_checksum=state_dict_checksum(sd),
                features=feats.numpy().reshape(batch, -1)[:, ::feature_stride].copy(),
                features_absmean=float(feats.abs().mean()),
                coords2d=c2d.numpy(), coords3d_rel=c3d.numpy(), coords3d_abs=out.numpy())
    if store_weights:
        data['crops'] = crops.numpy()
        data['intrinsics'] = k.numpy()
        for key, v in sd.items():
            data['sd/' + key] = v.numpy()
    np.savez_compressed(os.path.join(OUT, fname), **data)
    print(fname, f'{n_dil} dilated blocks, features {tuple(feats.shape)}, abs range', float(out.min()), float(out.max()))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    R = import_reference(port.PathConfig().as_reference_dict())
    for f in FIXTURES:
        golden(R, *f)


if __name__ == '__main__':
    main()
