"""The crop model: host-side mirror of /root/reference/metrabs_pytorch/models/metrabs.py (``Metrabs`` :12-64,
``MetrabsHeads`` :67-85) whose forward runs in libmetrabs_b200.so.

Drop-in contract (SURVEY.md 8b): ``Metrabs(backbone, joint_info)``; ``forward((image[B,3,S,S] fp32 in [0,1],
intrinsics[B,3,3])) -> coords3d_abs[B,J,3] fp32``; attributes ``joint_names``, ``joint_edges``,
``input_resolution``, ``joint_info``, ``heatmap_heads``; ``load_state_dict`` with the reference key schema
(``backbone.1.<stage>...``, ``heatmap_heads.conv_final.{weight,bias}``).  The consumer is
``Pose3dEstimator._predict_single_batch`` (multiperson/multiperson_model.py:240-242).

Latent-point models (``affine_weights`` with ``transform_coords``, ``predict_all_and_latents`` or
``regularize_to_manifold``, models/metrabs.py:23-45) are built like the reference builds them; their forward maps the
reconstructed latents to joints on the device, which the reference's PyTorch forward cannot do (it calls an undefined
``latent_points_to_joints``, :61-62; the TF model defines it, metrabs_tf/models/metrabs.py:80-87).
"""
import os

import numpy as np
import torch
from torch import nn

from metrabs_b200 import _lib
from metrabs_b200.engine import Engine, linear_combine_points, make_config
from metrabs_b200.util import get_config


def resolve_affine_weights(name):
    """``affine_weights`` as a file path, else ``$DATA_ROOT/skeleton_conversion/<name>.npz`` (models/metrabs.py:24-27)."""
    if os.path.exists(name):
        return name
    data_root = os.environ.get('DATA_ROOT', '')
    path = f'{data_root}/skeleton_conversion/{name}.npz'
    if not os.path.exists(path):
        raise FileNotFoundError(f'affine_weights {name!r}: neither {name!r} nor {path!r} exists')
    return path


def _find_features(backbone):
    for m in backbone.modules():
        if hasattr(m, 'arch') and hasattr(m, 'last_channel') and hasattr(m, 'stages'):
            return m
    raise TypeError('backbone must contain a metrabs_b200.backbones.*.Features module '
                    '(e.g. Sequential(PreprocLayer(), efficientnet_v2_s().features))')


class MetrabsHeads(nn.Module):
    """1x1 conv (J + D*J channels, bias) + 2D / volumetric soft-argmax + metric scaling, fused on the device."""

    def __init__(self, n_points, in_channels, owner=None):
        super().__init__()
        cfg = get_config()
        self.n_points = n_points
        self.n_outs = [n_points, cfg.depth * n_points]
        self.conv_final = nn.Conv2d(in_channels, sum(self.n_outs), kernel_size=1)
        self._owner = [owner]  # list: keep the parent out of the module tree

    def forward(self, inp):
        """features NCHW [B,C,H,W] (reference layout) -> (coords2d [B,J,2] px, coords3d_rel [B,J,3] mm)."""
        eng = self._owner[0].engine()
        nhwc = inp.permute(0, 2, 3, 1).contiguous().to(eng.feature_dtype)
        return eng.head_decode(nhwc)


class Metrabs(nn.Module):
    def __init__(self, backbone, joint_info):
        super().__init__()
        cfg = get_config()
        self.backbone = backbone
        self.joint_names = np.array(joint_info.names)
        self.joint_edges = np.array([[i, j] for i, j in joint_info.stick_figure_edges])
        self.input_resolution = np.int32(cfg.proc_side)
        self.joint_info = joint_info
        self._features = [_find_features(backbone)]
        feats = self._features[0]
        # plain tensors, not buffers: state_dict() keeps the reference's keys (the autoencoder ships as its own file)
        self.n_latents = None
        self.recombination_weights = self.encoder_weights = self.reconstruction_weights = None
        n_raw_points = joint_info.n_joints
        if cfg.affine_weights:
            ws = np.load(resolve_affine_weights(cfg.affine_weights))
            w1, w2 = np.asarray(ws['w1'], np.float32), np.asarray(ws['w2'], np.float32)
            j = joint_info.n_joints
            if w1.ndim != 2 or w2.ndim != 2 or w1.shape[0] != j or w2.shape[1] != j or w1.shape[1] != w2.shape[0]:
                raise ValueError(f'affine weights {cfg.affine_weights!r}: expected w1 [{j}, L] and w2 [L, {j}] for '
                                 f'{j} joints, got w1 {w1.shape} and w2 {w2.shape}')
            self.n_latents = w2.shape[0]
            self.recombination_weights = torch.from_numpy(w2).float()
            self.encoder_weights = torch.from_numpy(w1).float()
            self.reconstruction_weights = self.encoder_weights @ self.recombination_weights
            if cfg.transform_coords:
                n_raw_points = self.n_latents
            elif cfg.predict_all_and_latents:
                n_raw_points = self.n_latents + joint_info.n_joints
            elif cfg.regularize_to_manifold:
                n_raw_points = joint_info.n_joints
            else:
                # models/metrabs.py:40-41
                raise ValueError('affine_weights is set but none of transform_coords, predict_all_and_latents, '
                                 'regularize_to_manifold uses it')
        self._latent_forward = bool(cfg.affine_weights) and bool(cfg.transform_coords or cfg.predict_all_and_latents)
        self._device_weights = {}
        self.heatmap_heads = MetrabsHeads(n_points=n_raw_points, in_channels=feats.last_channel, owner=self)
        self._cfg = cfg
        self._engine = None
        self._dirty = True
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.mark_weights_changed())

    def mark_weights_changed(self):
        self._dirty = True

    def engine(self, device=None):
        """Builds the C handle lazily on the module's CUDA device and (re)uploads the weights when they changed."""
        if device is None:
            device = self.heatmap_heads.conv_final.weight.device
        if device.type != 'cuda':
            raise _lib.MetrabsB200Error('metrabs_b200.Metrabs runs on CUDA only: call .cuda() first (no CPU fallback)')
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._engine is None or self._engine.cfg.device != index:
            feats = self._features[0]
            self._engine = Engine(make_config(self._cfg, self.heatmap_heads.n_points, stages=feats.stages,
                                              last_channel=feats.last_channel, arch=feats.arch, device=index))
            if self._latent_forward:
                self._engine.set_latent_recombination(self.recombination_weights)
            self._dirty = True
        if self._dirty:
            self._engine.load_state_dict(self.state_dict())
            self._dirty = False
        return self._engine

    def forward(self, inp):
        image, intrinsics = inp
        eng = self.engine(image.device)
        return eng.forward(image.float(), intrinsics.float())

    # ---- latent points <-> joints (metrabs_tf/models/metrabs.py:80-87), on the device ---------------------------------
    def _weights_on(self, name, device):
        w = getattr(self, name)
        if w is None:
            raise ValueError('this model has no affine weights (Config.affine_weights)')
        key = (name, device)
        if key not in self._device_weights:
            self._device_weights[key] = w.to(device)
        return self._device_weights[key]

    def latent_points_to_joints(self, points):
        """[B, L, 3] -> [B, J, 3] with the recombination weights w2 (CUDA tensors only)."""
        return linear_combine_points(points, self._weights_on('recombination_weights', points.device))

    def joints_to_latent_points(self, points):
        """[B, J, 3] -> [B, L, 3] with the encoder weights w1 (CUDA tensors only)."""
        return linear_combine_points(points, self._weights_on('encoder_weights', points.device))

    def joints_to_joints(self, points):
        """[B, J, 3] -> [B, J, 3] through the latent space, w1 @ w2 (CUDA tensors only)."""
        return linear_combine_points(points, self._weights_on('reconstruction_weights', points.device))
