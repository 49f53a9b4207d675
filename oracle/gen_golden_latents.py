"""TEST INFRASTRUCTURE ONLY - generates tests/golden/latents_tiny_s64.npz by running the UNMODIFIED reference
(imported from /root/reference via oracle/ref_import.py) on torch-cpu, for the two latent-point model options that
change inference: ``transform_coords`` (the head predicts L latents) and ``predict_all_and_latents`` (L + J points, the
first L are reconstructed).

Run in the build container only:  ``python oracle/gen_golden_latents.py``.  The reference's own ``Metrabs`` constructor
reads a temporary affine-weights ``.npz`` (``oracle/port_latents.make_affine_weights``) and sizes its head from it; its
``heatmap_heads``, ``ptu3d.reconstruct_absolute`` and ``forward`` then run as they are.  The one restated piece is
``latent_points_to_joints``, which only the reference's TF model defines (metrabs_tf/models/metrabs.py:80-81 ->
tfu3d.linear_combine_points, metrabs_tf/tfu3d.py:48-49): it is attached to the model instance as that one-line einsum.
Weights regenerate from ``port.make_effnet_state_dict(spec, cfg, n_raw, seed=0)``; inputs from
``port.synthetic_inputs(BATCH, 64, seed=0)``.
"""
import os
import sys
import tempfile
import types
from functools import partial

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import port, port_latents  # noqa: E402
from oracle.ref_import import import_reference, set_reference_config  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
NAME, PROC_SIDE, N_JOINTS, N_LATENTS, BATCH = 'efficientnetv2-tiny', 64, 10, 6, 3
OPTIONS = ('transform_coords', 'predict_all_and_latents')


def n_raw_points(option):
    return N_LATENTS if option == 'transform_coords' else N_LATENTS + N_JOINTS


def build_reference_latent_model(R, spec, proc_side):
    E = R.effnet
    rows = []
    for st in spec.stages:
        C = E.FusedMBConvConfig if st.block == 'fused' else E.MBConvConfig
        rows.append(C(st.expand, st.kernel, st.stride, st.cin, st.cout, st.layers, bottomright_stride=st.bottomright))
    bb = E.EfficientNet(rows, 0.2, last_channel=spec.last_channel, norm_layer=partial(torch.nn.BatchNorm2d, eps=1e-3))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(N_JOINTS)], stick_figure_edges=[(0, 1)], n_joints=N_JOINTS)
    m = R.metrabs.Metrabs(torch.nn.Sequential(E.PreprocLayer(), bb.features), ji).eval()
    # THE ONLY RESTATED LINE: tfu3d.linear_combine_points with the recombination weights the reference constructor loaded
    m.latent_points_to_joints = lambda points: torch.einsum('bjc,jJ->bJc', points, m.recombination_weights)
    with torch.inference_mode():  # materialise LazyConv2d (scripts/demo_image.py:69-72)
        m((torch.rand(1, 3, proc_side, proc_side), torch.eye(3)[None]))
    return m


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    R = import_reference(port.PathConfig().as_reference_dict())
    w1, w2 = port_latents.make_affine_weights(N_JOINTS, N_LATENTS, seed=0)
    spec = port.effnet_spec(NAME)
    crops, k = port.synthetic_inputs(BATCH, PROC_SIDE, seed=0)
    data = dict(name=NAME, proc_side=PROC_SIDE, n_joints=N_JOINTS, n_latents=N_LATENTS, batch=BATCH, seed=0, w1=w1, w2=w2)
    with tempfile.TemporaryDirectory() as tmp:
        affine_path = os.path.join(tmp, 'affine_tiny.npz')
        np.savez(affine_path, w1=w1, w2=w2)
        for option in OPTIONS:
            cfg = port.PathConfig(proc_side=PROC_SIDE, affine_weights=affine_path, **{option: True})
            set_reference_config(cfg.as_reference_dict())
            n_raw = n_raw_points(option)
            sd = port.make_effnet_state_dict(spec, cfg, n_raw, seed=0)
            m = build_reference_latent_model(R, spec, PROC_SIDE)
            assert m.heatmap_heads.n_points == n_raw and m.n_latents == N_LATENTS
            m.load_state_dict(sd, strict=True)
            with torch.inference_mode():
                c2d, c3d = m.heatmap_heads(m.backbone(crops))
                latents = R.ptu3d.reconstruct_absolute(c2d[:, :N_LATENTS], c3d[:, :N_LATENTS], k,
                                                       mix_3d_inside_fov=cfg.mix_3d_inside_fov)
                joints = m((crops, k))
            assert joints.shape == (BATCH, N_JOINTS, 3)
            data[f'{option}/coords2d'] = c2d.numpy()
            data[f'{option}/coords3d_rel'] = c3d.numpy()
            data[f'{option}/latents_abs'] = latents.numpy()
            data[f'{option}/joints'] = joints.numpy()
            print(option, 'n_raw', n_raw, 'joints range', float(joints.min()), float(joints.max()))
    np.savez_compressed(os.path.join(OUT, 'latents_tiny_s64.npz'), **data)


if __name__ == '__main__':
    main()
