"""The Metro crop model: host-side mirror of the reference's TF-only ``Metro`` (metrabs_tf/models/metro.py:13-45) whose
forward runs in libmetrabs_b200.so.

``Metro(backbone, joint_info)``; ``forward(image[B,3,S,S] fp32 in [0,1]) -> coords3d_rel[B,J,3]`` in mm, relative to the crop
box (heatmap_to_metric of the head; not root-centred: ``center_relative_pose`` appears only in the reference's trainer loss).
Attributes ``joint_names``, ``joint_edges``, ``input_resolution``, ``joint_info``, ``heatmap_head``; ``load_state_dict`` with
the keys ``backbone.*`` (as for ``Metrabs``) and ``heatmap_head.conv_final.{weight,bias}``, weight ``[D*J, C, 1, 1]``.

The head (``Head3D``, :34-44, shared with ``Model25D``) is the 3D part of the MeTRAbs head without its J leading 2D channels:
channel ``d*J + j``, soft-argmax jointly over (W, H, D) in fp32 with ``tf.linspace(0, 1, n)``, which decodes a one-long axis
to 0 (``ptu.linspace`` would give 0.5).
"""
import numpy as np
import torch
from torch import nn

from metrabs_b200 import _lib
from metrabs_b200.engine import Engine, make_config
from metrabs_b200.models.metrabs import _find_features
from metrabs_b200.util import get_config


class Head3D(nn.Module):
    """1x1 conv (D*J channels, bias) + volumetric soft-argmax + the class's scaling, fused on the device."""

    def __init__(self, n_points, in_channels, owner=None):
        super().__init__()
        cfg = get_config()
        self.n_points = n_points
        self.conv_final = nn.Conv2d(in_channels, cfg.depth * n_points, kernel_size=1)
        self._owner = [owner]  # list: keep the parent out of the module tree

    def forward(self, inp):
        """features NCHW [B,C,H,W] -> [B,J,3]: Metro mm (heatmap_to_metric), Model25D (x px, y px, z mm)."""
        eng = self._owner[0].engine()
        nhwc = inp.permute(0, 2, 3, 1).contiguous().to(eng.feature_dtype)
        return eng.head_decode(nhwc)[1]


class VolumetricHeadModel(nn.Module):
    """What Metro and Model25D share: the backbone, the D*J-channel head, the C handle and the config checks."""
    model_class = None

    def __init__(self, backbone, joint_info):
        super().__init__()
        cfg = get_config()
        name = type(self).__name__
        # twofive.py:21,42-43 reads a recombination_weights its __init__ never sets; Metro has no latent points at all
        for flag in ('affine_weights', 'transform_coords', 'predict_all_and_latents'):
            if getattr(cfg, flag):
                raise ValueError(f'{name} does not support Config.{flag}: latent points are a Metrabs feature (the reference '
                                 f'Model25D reads recombination weights it never sets)')
        if cfg.legacy_centered_stride_bug:
            raise ValueError(f'{name} decodes with the TF heatmap_to_image, which has no legacy_centered_stride_bug term '
                             '(metrabs_tf/models/util.py:8-18): set Config(legacy_centered_stride_bug=False)')
        self.backbone = backbone
        self.joint_names = np.array(joint_info.names)
        self.joint_edges = np.array([[i, j] for i, j in joint_info.stick_figure_edges])
        self.input_resolution = np.int32(cfg.proc_side)
        self.joint_info = joint_info
        self._features = [_find_features(backbone)]
        self.heatmap_head = Head3D(n_points=joint_info.n_joints, in_channels=self._features[0].last_channel, owner=self)
        self._cfg = cfg
        self._engine = None
        self._dirty = True
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.mark_weights_changed())

    def mark_weights_changed(self):
        self._dirty = True

    def _set_class(self, eng):
        eng.set_model_class(self.model_class)

    def engine(self, device=None):
        """Builds the C handle lazily on the module's CUDA device and (re)uploads the weights when they changed."""
        if device is None:
            device = self.heatmap_head.conv_final.weight.device
        if device.type != 'cuda':
            raise _lib.MetrabsB200Error(f'metrabs_b200.{type(self).__name__} runs on CUDA only: call .cuda() first '
                                        '(no CPU fallback)')
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._engine is None or self._engine.cfg.device != index:
            feats = self._features[0]
            self._engine = Engine(make_config(self._cfg, self.heatmap_head.n_points, stages=feats.stages,
                                              last_channel=feats.last_channel, arch=feats.arch, device=index))
            self._set_class(self._engine)
            self._dirty = True
        if self._dirty:
            self._engine.load_state_dict(self.state_dict())
            self._dirty = False
        return self._engine


class Metro(VolumetricHeadModel):
    model_class = _lib.MODEL_METRO
    # Pose3dEstimator needs camera-space joints: Metro's are relative to the crop box
    has_absolute_output = False

    def forward(self, image):
        """[B,3,S,S] -> root-relative joints [B,J,3] in mm (Metro.call / predict_multi, metro.py:24-31)."""
        eng = self.engine(image.device)
        return eng.forward(image.float(), None)
