"""The 2.5D crop model: host-side mirror of the reference's TF-only ``Model25D`` (metrabs_tf/models/twofive.py:14-57) whose
forward runs in libmetrabs_b200.so.

``Model25D(backbone, joint_info, bone_lengths_ideal)``; ``forward((image[B,3,S,S], intrinsics[B,3,3])) -> coords3d_abs[B,J,3]``
in camera space (mm), the call signature of ``Metrabs``, so it drives ``Pose3dEstimator`` as a MeTRAbs model does.  The head
is Metro's ``Head3D`` decoded by ``heatmap_to_25d`` (models/util.py:21-23: x, y in crop pixels, z in mm); the absolute depth
of each crop comes from ``reconstruct_absolute_by_bone_lengths`` (metrabs_tf/tfu3d.py:219-269) over the bones
``joint_info.stick_figure_edges`` with ``bone_lengths_ideal`` [E] mm, depths relative to the mean joint when
``Config.mean_relative`` (the reference default), else to the last joint.

That solve is a Levenberg-Marquardt fit whose steps are accepted on the objective of the WHOLE batch, so a crop's absolute
joints depend on the batch it runs in, as in the reference; its features and decoded coords25d do not.
"""
import numpy as np

from metrabs_b200 import _lib
from metrabs_b200.models.metro import Head3D, VolumetricHeadModel

Head25D = Head3D  # the reference's Head25D (twofive.py:46-56) is Head3D with another decode scale, which the handle applies


class Model25D(VolumetricHeadModel):
    model_class = _lib.MODEL_25D

    def __init__(self, backbone, joint_info, bone_lengths_ideal):
        super().__init__(backbone, joint_info)
        self.edges = [tuple(e) for e in joint_info.stick_figure_edges]
        lengths = np.asarray(bone_lengths_ideal, dtype=np.float32).reshape(-1)
        if lengths.shape[0] != len(self.edges) or len(self.edges) == 0:
            raise ValueError(f'bone_lengths_ideal has {lengths.shape[0]} entries for {len(self.edges)} edges of '
                             'joint_info.stick_figure_edges (one per edge, at least one)')
        if not np.all(np.isfinite(lengths)) or not np.all(lengths > 0):
            raise ValueError('bone_lengths_ideal must be finite and positive (mm)')
        n = joint_info.n_joints
        if any(not (0 <= i < n and 0 <= j < n) for i, j in self.edges):
            raise ValueError(f'stick_figure_edges has a joint index outside [0, {n})')
        self.bone_lengths_ideal = lengths

    def _set_class(self, eng):
        eng.set_model_class(self.model_class, np.asarray(self.edges, dtype=np.int32), self.bone_lengths_ideal,
                            mean_relative=self._cfg.mean_relative)

    def forward(self, inp):
        image, intrinsics = inp
        eng = self.engine(image.device)
        return eng.forward(image.float(), intrinsics.float())
