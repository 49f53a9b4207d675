"""``Pose3dEstimator``: host-side mirror of /root/reference/metrabs_pytorch/multiperson/multiperson_model.py (:16-407).

Same constructor and method names; the data path is device-resident:

    frames u8 [N,3,H,W] --mtb_image_pyramid--> pyramid
    boxes --mtb_crop_setup--> per-crop matrices --mtb_warp_crops--> crops [A*n,3,res,res] (ONE launch, not a Python loop)
    --crop_model (mtb_forward)--> poses [A*n,J,3] --mtb_tta_merge--> poses3d / poses2d per box (--mtb_filter_poses-->)

Differences from the reference, all deliberate: the person detector is third-party (ultralytics YOLO, person_detector.py)
and out of scope, so ``detect_poses*`` take a ``detector`` callable; ``JointInfo`` comes from the un-vendored posepile
(stand-in in joint_info.py); the public ``estimate_poses*`` of the reference crash on their tuple defaults (SURVEY.md 3.4)
- here they work; the plausibility filter, commented out in the PyTorch reference (:158-163), runs when bone statistics
are supplied.

``antialias_factor`` (every public method): 1, 2, 4 or 5..16, the factors the reference accepts except 3, for which it
has no shrink step (:309-315).  At 2 and 4 the res*f render is box-averaged, above 4 it is shrunk with the antialiased
bilinear resize, as in the reference; other factors raise MetrabsB200Error."""
import ctypes as C

import numpy as np
import torch

from metrabs_b200 import _lib
from metrabs_b200._lib import check, lib
from metrabs_b200.multiperson import plausibility_check, warping
from metrabs_b200.multiperson.joint_info import JointInfo
from metrabs_b200.multiperson.warping import _ptr, _stream

UNKNOWN_INTRINSIC_MATRIX = ((-1, -1, -1), (-1, -1, -1), (-1, -1, -1))
DEFAULT_EXTRINSIC_MATRIX = ((1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1))
DEFAULT_DISTORTION = (0, 0, 0, 0, 0)
DEFAULT_WORLD_UP = (0, -1, 0)


def _linspace(start, stop, num, endpoint=True):
    """ptu.linspace (ptu.py:78-92)."""
    start = torch.as_tensor(start, dtype=torch.float32)
    stop = torch.as_tensor(stop, dtype=torch.float32)
    if endpoint:
        if num == 1:
            return torch.mean(torch.stack([start, stop], dim=0), dim=0, keepdim=True)
        return torch.linspace(start, stop, num)
    if num > 1:
        step = (stop - start) / num
        return torch.linspace(start, stop - step, num)
    return torch.linspace(start, stop, num)


def _rotation_mat_z(angle):
    """ptu3d.rotation_mat(angle, 'z')."""
    sin, cos = torch.sin(angle), torch.cos(angle)
    _0, _1 = torch.zeros_like(angle), torch.ones_like(angle)
    return torch.stack([torch.stack([cos, -sin, _0], dim=-1), torch.stack([sin, cos, _0], dim=-1),
                        torch.stack([_0, _0, _1], dim=-1)], dim=-2)


def intrinsic_matrix_from_field_of_view(fov_degrees, imshape):
    """ptu3d.intrinsic_matrix_from_field_of_view."""
    imshape = torch.tensor(imshape, dtype=torch.float32)
    fov_radians = fov_degrees * torch.tensor(np.pi / 180, dtype=torch.float32)
    focal = torch.max(imshape) / (torch.tan(fov_radians / 2) * 2)
    return torch.tensor([[focal, 0, imshape[1] / 2], [0, focal, imshape[0] / 2], [0, 0, 1]], dtype=torch.float32).unsqueeze(0)


def aug_parameters(num_aug):
    """The test-time augmentation plan of _estimate_poses_batched (multiperson_model.py:108-141): gammas, scales, flips and
    the combined rotation/flip matrices."""
    aug_gammas = _linspace(np.float32(0.6), np.float32(1.0), num_aug)
    aug_angle_range = np.float32(np.deg2rad(25))
    aug_angles = _linspace(-aug_angle_range, aug_angle_range, num_aug)
    aug_scales = torch.cat([_linspace(0.8, 1.0, num_aug // 2, endpoint=False),
                            torch.linspace(1.0, 1.1, num_aug - num_aug // 2)], dim=0)
    aug_should_flip = (torch.arange(0, num_aug) - num_aug // 2) % 2 != 0
    aug_flipmat = torch.tensor([[-1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=torch.float32)
    aug_maybe_flipmat = torch.where(aug_should_flip[:, np.newaxis, np.newaxis], aug_flipmat, torch.eye(3))
    aug_rotflipmat = aug_maybe_flipmat @ _rotation_mat_z(-aug_angles)
    return aug_gammas, aug_scales, aug_should_flip, aug_rotflipmat


class Pose3dEstimator(torch.nn.Module):
    def __init__(self, crop_model, skeleton_infos, joint_transform_matrix, detector=None, joint_info=None,
                 mean_bone_lengths=None):
        super().__init__()
        if getattr(crop_model, 'has_absolute_output', True) is False:
            raise ValueError(f'{type(crop_model).__name__} has no absolute output: its joints are relative to the crop box, '
                             'and the estimator needs camera-space joints (use Metrabs or Model25D)')
        self.crop_model = crop_model
        self.joint_names = self.crop_model.joint_names
        self.joint_edges = self.crop_model.joint_edges
        self.joint_info = joint_info if joint_info is not None else JointInfo(self.joint_names, self.joint_edges)
        self.detector = detector
        self.joint_transform_matrix = (torch.as_tensor(joint_transform_matrix, dtype=torch.float32)
                                       if joint_transform_matrix is not None else None)
        self.per_skeleton_indices = {k: torch.tensor(v['indices'], dtype=torch.int32) for k, v in skeleton_infos.items()}
        self.per_skeleton_joint_names = {k: v['names'] for k, v in skeleton_infos.items()}
        self.per_skeleton_joint_edges = {k: torch.tensor(v['edges'], dtype=torch.int32) for k, v in skeleton_infos.items()}
        self.skeleton_joint_indices_table = {k: v['indices'] for k, v in skeleton_infos.items()}
        self.mean_bone_lengths = mean_bone_lengths  # per edge of joint_info.stick_figure_edges, mm (plausibility filter)

    # ---------------------------------------------------------------------------------------------- public API
    def detect_poses_batched(self, images, intrinsic_matrix=np.array([UNKNOWN_INTRINSIC_MATRIX]),
                             distortion_coeffs=np.array([DEFAULT_DISTORTION]),
                             extrinsic_matrix=np.array([DEFAULT_EXTRINSIC_MATRIX]), world_up_vector=DEFAULT_WORLD_UP,
                             default_fov_degrees=55, internal_batch_size=64, antialias_factor=1, num_aug=5,
                             average_aug=True, skeleton='', detector_threshold=0.3, detector_nms_iou_threshold=0.7,
                             max_detections=None, detector_flip_aug=False, suppress_implausible_poses=True):
        if self.detector is None:
            raise NotImplementedError('the person detector (ultralytics YOLO in the reference) is outside this package: pass '
                                      'detector=callable(images, threshold, nms_iou_threshold, max_detections) -> list of [n,5]')
        boxes = self.detector(images=images, threshold=detector_threshold, nms_iou_threshold=detector_nms_iou_threshold,
                              max_detections=max_detections)
        return self._estimate_poses_batched(images, boxes, intrinsic_matrix, distortion_coeffs, extrinsic_matrix,
                                            world_up_vector, default_fov_degrees, internal_batch_size, antialias_factor,
                                            num_aug, average_aug, skeleton, suppress_implausible_poses)

    def estimate_poses_batched(self, images, boxes, intrinsic_matrix=(UNKNOWN_INTRINSIC_MATRIX,),
                               distortion_coeffs=(DEFAULT_DISTORTION,), extrinsic_matrix=(DEFAULT_EXTRINSIC_MATRIX,),
                               world_up_vector=DEFAULT_WORLD_UP, default_fov_degrees=55, internal_batch_size=64,
                               antialias_factor=1, num_aug=5, average_aug=True, skeleton=''):
        boxes = [torch.cat([torch.as_tensor(b, dtype=torch.float32)[..., :4],
                            torch.ones_like(torch.as_tensor(b, dtype=torch.float32)[..., :1])], dim=-1) for b in boxes]
        pred = self._estimate_poses_batched(images, boxes, intrinsic_matrix, distortion_coeffs, extrinsic_matrix,
                                            world_up_vector, default_fov_degrees, internal_batch_size, antialias_factor,
                                            num_aug, average_aug, skeleton, suppress_implausible_poses=False)
        del pred['boxes']
        return pred

    def detect_poses(self, image, intrinsic_matrix=UNKNOWN_INTRINSIC_MATRIX, distortion_coeffs=DEFAULT_DISTORTION,
                     extrinsic_matrix=DEFAULT_EXTRINSIC_MATRIX, world_up_vector=DEFAULT_WORLD_UP, default_fov_degrees=55,
                     internal_batch_size=64, antialias_factor=1, num_aug=5, average_aug=True, skeleton='',
                     detector_threshold=0.3, detector_nms_iou_threshold=0.7, max_detections=-1, detector_flip_aug=False,
                     suppress_implausible_poses=True):
        result = self.detect_poses_batched(
            image[np.newaxis], torch.as_tensor(intrinsic_matrix, dtype=torch.float32)[np.newaxis],
            torch.as_tensor(distortion_coeffs, dtype=torch.float32)[np.newaxis],
            torch.as_tensor(extrinsic_matrix, dtype=torch.float32)[np.newaxis], world_up_vector, default_fov_degrees,
            internal_batch_size, antialias_factor, num_aug, average_aug, skeleton, detector_threshold,
            detector_nms_iou_threshold, max_detections, detector_flip_aug, suppress_implausible_poses)
        return {k: v[0] for k, v in result.items()}

    def estimate_poses(self, image, boxes, intrinsic_matrix=UNKNOWN_INTRINSIC_MATRIX, distortion_coeffs=DEFAULT_DISTORTION,
                       extrinsic_matrix=DEFAULT_EXTRINSIC_MATRIX, world_up_vector=DEFAULT_WORLD_UP, default_fov_degrees=55,
                       internal_batch_size=64, antialias_factor=1, num_aug=5, average_aug=True, skeleton=''):
        result = self.estimate_poses_batched(
            image[np.newaxis], [boxes], torch.as_tensor(intrinsic_matrix, dtype=torch.float32)[np.newaxis],
            torch.as_tensor(distortion_coeffs, dtype=torch.float32)[np.newaxis],
            torch.as_tensor(extrinsic_matrix, dtype=torch.float32)[np.newaxis], world_up_vector, default_fov_degrees,
            internal_batch_size, antialias_factor, num_aug, average_aug, skeleton)
        return {k: v[0] for k, v in result.items()}

    # ------------------------------------------------------------------------------------------------ the path
    def _device(self):
        cm = self.crop_model
        if hasattr(cm, 'heatmap_heads'):
            return cm.heatmap_heads.conv_final.weight.device
        for t in list(cm.parameters()) + list(cm.buffers()):
            return t.device
        return torch.device(getattr(cm, 'device', 'cuda'))

    def _estimate_poses_batched(self, images, boxes, intrinsic_matrix, distortion_coeffs, extrinsic_matrix, world_up_vector,
                                default_fov_degrees, internal_batch_size, antialias_factor, num_aug, average_aug, skeleton,
                                suppress_implausible_poses):
        dev = self._device()
        if dev.type != 'cuda':
            raise _lib.MetrabsB200Error('Pose3dEstimator runs on CUDA only (no CPU fallback): call .cuda() on the crop model')
        images = torch.as_tensor(images)
        if images.dtype != torch.uint8:
            raise TypeError('images must be uint8 [N,3,H,W] (the reference decodes them as (images / 255) ** 2.2)')
        images = images.to(dev).contiguous()
        intrinsic_matrix = torch.as_tensor(np.asarray(intrinsic_matrix, dtype=np.float32) if not torch.is_tensor(intrinsic_matrix)
                                           else intrinsic_matrix, dtype=torch.float32).cpu()
        distortion_coeffs = torch.as_tensor(np.asarray(distortion_coeffs, dtype=np.float32) if not torch.is_tensor(distortion_coeffs)
                                            else distortion_coeffs, dtype=torch.float32).cpu()
        extrinsic_matrix = torch.as_tensor(np.asarray(extrinsic_matrix, dtype=np.float32) if not torch.is_tensor(extrinsic_matrix)
                                           else extrinsic_matrix, dtype=torch.float32).cpu()
        world_up_vector = torch.as_tensor(world_up_vector, dtype=torch.float32).cpu()
        boxes = [torch.as_tensor(b, dtype=torch.float32).cpu().reshape(-1, 5) for b in boxes]
        n_images = len(images)
        # camera parameters: one set repeated over the images, then over each image's boxes (:87-106)
        if len(intrinsic_matrix) == 1:
            if torch.all(intrinsic_matrix == -1):
                intrinsic_matrix = intrinsic_matrix_from_field_of_view(default_fov_degrees, images.shape[2:4])
            intrinsic_matrix = torch.repeat_interleave(intrinsic_matrix, n_images, dim=0)
        if len(distortion_coeffs) == 1:
            distortion_coeffs = torch.repeat_interleave(distortion_coeffs, n_images, dim=0)
        if len(extrinsic_matrix) == 1:
            extrinsic_matrix = torch.repeat_interleave(extrinsic_matrix, n_images, dim=0)
        n_box_per_image = torch.tensor([len(b) for b in boxes])
        n_total = int(n_box_per_image.sum())
        counts = [int(c) for c in n_box_per_image]
        if n_total == 0:
            js = len(self.skeleton_joint_indices_table[skeleton]) if skeleton in self.skeleton_joint_indices_table else 0
            shape3 = (0, js, 3) if average_aug else (0, num_aug, js, 3)
            shape2 = shape3[:-1] + (2,)
            return dict(boxes=boxes, poses3d=[torch.zeros(shape3, device=dev) for _ in boxes],
                        poses2d=[torch.zeros(shape2, device=dev) for _ in boxes])
        k_box = torch.repeat_interleave(intrinsic_matrix, n_box_per_image, dim=0)
        d_box = torch.repeat_interleave(distortion_coeffs, n_box_per_image, dim=0)
        camspace_up = torch.einsum('c,bCc->bC', world_up_vector, extrinsic_matrix[..., :3, :3])
        camspace_up = torch.repeat_interleave(camspace_up, n_box_per_image, dim=0)
        ext_inv_box = torch.repeat_interleave(torch.linalg.inv(extrinsic_matrix), n_box_per_image, dim=0)
        image_id_per_box = torch.repeat_interleave(torch.arange(len(boxes)), n_box_per_image)
        aug_gammas, aug_scales, aug_should_flip, aug_rotflipmat = aug_parameters(num_aug)

        boxes_flat = torch.cat(boxes, dim=0).to(dev)
        k_box, d_box, camspace_up, ext_inv_box = (t.to(dev).contiguous() for t in (k_box, d_box, camspace_up, ext_inv_box))
        image_id_per_box = image_id_per_box.int().to(dev)
        pyramid = warping.build_pyramid(images)  # gamma decoding + box-filter levels (:200, warping.py:9-13)

        skel = self.skeleton_joint_indices_table[skeleton]
        n_skel = len(skel)
        shape3 = (n_total, n_skel, 3) if average_aug else (n_total, num_aug, n_skel, 3)
        poses3d = torch.empty(shape3, dtype=torch.float32, device=dev)
        poses2d = torch.empty(shape3[:-1] + (2,), dtype=torch.float32, device=dev)
        want_filter = bool(suppress_implausible_poses) and self.mean_bone_lengths is not None and num_aug >= 2
        j2 = self.joint_transform_matrix.shape[1] if self.joint_transform_matrix is not None else self.joint_info.n_joints
        cam3d = torch.empty(n_total, num_aug, j2, 3, dtype=torch.float32, device=dev) if want_filter else None
        cam2d = torch.empty(n_total, num_aug, j2, 2, dtype=torch.float32, device=dev) if want_filter else None
        eye4 = torch.eye(4, device=dev).expand(n_total, 4, 4).contiguous() if want_filter else None

        boxes_per_batch = internal_batch_size // num_aug  # (:190) 0 = everything as one batch
        step = n_total if boxes_per_batch == 0 else boxes_per_batch
        for s in range(0, n_total, step):
            sl = slice(s, min(s + step, n_total))
            poses_flat, rot = self._predict_single_batch(images, pyramid, k_box[sl], d_box[sl], camspace_up[sl], boxes_flat[sl],
                                                         image_id_per_box[sl], aug_rotflipmat, aug_should_flip, aug_scales,
                                                         aug_gammas, antialias_factor)
            self._tta_merge(poses_flat, rot, aug_should_flip, k_box[sl], d_box[sl], ext_inv_box[sl], skel, average_aug,
                            poses3d[sl], poses2d[sl])
            if want_filter:  # camera-space poses of every augmentation, all joints, for the plausibility checks
                self._tta_merge(poses_flat, rot, aug_should_flip, k_box[sl], d_box[sl], eye4[sl], None, False, cam3d[sl], cam2d[sl])

        result_boxes = boxes
        poses3d = list(torch.split(poses3d, counts))
        poses2d = list(torch.split(poses2d, counts))
        if want_filter:
            _, keep = plausibility_check.filter_poses(cam3d, cam2d, boxes_flat, counts, self.joint_info.stick_figure_edges,
                                                      self.mean_bone_lengths)
            keeps = torch.split(keep.cpu(), counts)
            result_boxes = [b[k] for b, k in zip(boxes, keeps)]
            poses3d = [p[k.to(dev)] for p, k in zip(poses3d, keeps)]
            poses2d = [p[k.to(dev)] for p, k in zip(poses2d, keeps)]
        return dict(boxes=result_boxes, poses3d=poses3d, poses2d=poses2d)

    def _get_crops(self, images, pyramid, intrinsic_matrix, distortion_coeffs, camspace_up, boxes, image_ids, aug_rotflipmat,
                   aug_scales, aug_gammas, antialias_factor):
        """-> crops [A*n,3,res,res], new_intrinsic_matrix [A,n,3,3], R [A,n,3,3]  (multiperson_model.py:264-319)."""
        res = int(self.crop_model.input_resolution)
        num_aug = aug_gammas.shape[0]
        new_k, rot, inv, lev = warping.crop_setup(boxes, intrinsic_matrix, distortion_coeffs, camspace_up, aug_rotflipmat,
                                                  aug_scales, res, antialias_factor)
        crops = warping.warp_images_with_pyramid(images, pyramid, intrinsic_matrix, inv, distortion_coeffs, lev,
                                                 aug_gammas / 2.2, res, image_ids, num_aug, antialias_factor)
        return crops, new_k, rot

    def _predict_single_batch(self, images, pyramid, intrinsic_matrix, distortion_coeffs, camspace_up, boxes, image_ids,
                              aug_rotflipmat, aug_should_flip, aug_scales, aug_gammas, antialias_factor):
        crops_flat, new_k, rot = self._get_crops(images, pyramid, intrinsic_matrix, distortion_coeffs, camspace_up, boxes,
                                                 image_ids, aug_rotflipmat, aug_scales, aug_gammas, antialias_factor)
        poses_flat = self.crop_model((crops_flat, new_k.reshape(-1, 3, 3)))  # [A*n, J, 3]  (:240-242)
        return poses_flat, rot

    def _tta_merge(self, poses_flat, rot, aug_should_flip, k_box, d_box, ext_inv_box, skeleton_indices, average_aug, out3d,
                   out2d):
        """Mirror swap, poses @ R, joint transform, projection, extrinsics, skeleton gather, mean (:246-259, :143-182)."""
        dev = poses_flat.device
        num_aug, n = rot.shape[0], rot.shape[1]
        j = self.joint_info.n_joints
        flip = aug_should_flip.to(torch.uint8).to(dev).contiguous()
        mirror = torch.as_tensor(self.joint_info.mirror_mapping, dtype=torch.int32).to(dev)
        jt = self.joint_transform_matrix.to(dev).contiguous() if self.joint_transform_matrix is not None else None
        skel = (torch.as_tensor(skeleton_indices, dtype=torch.int32).to(dev).contiguous()
                if skeleton_indices is not None else None)
        poses_flat = poses_flat.contiguous()
        rot = rot.contiguous()
        k_box, d_box, ext_inv_box = k_box.contiguous(), d_box.contiguous(), ext_inv_box.contiguous()
        assert out3d.is_contiguous() and out2d.is_contiguous()
        args = _lib.MtbTtaArgs(_ptr(poses_flat), _ptr(rot), _ptr(flip), _ptr(mirror), _ptr(jt), _ptr(skel), _ptr(k_box), _ptr(d_box),
                               d_box.shape[1], _ptr(ext_inv_box), n, num_aug, j, jt.shape[1] if jt is not None else j,
                               skel.shape[0] if skel is not None else 0, int(bool(average_aug)), _ptr(out3d), _ptr(out2d))
        with torch.cuda.device(dev):
            check(lib().mtb_tta_merge(C.byref(args), _stream(dev)))
        return out3d, out2d
