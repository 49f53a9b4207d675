"""Device mirror of /root/reference/metrabs_pytorch/multiperson/warping.py: ``warp_images_with_pyramid`` (:6-28) as ONE
kernel launch for all crops (the reference loops over crops in Python, :23-28), ``distort_points`` inside it."""
import ctypes as C

import torch

from metrabs_b200 import _lib
from metrabs_b200._lib import check, lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _dev_f32(t, device):
    return torch.as_tensor(t, dtype=torch.float32).to(device).contiguous()


def build_pyramid(images):
    """images u8 [N,3,H,W] on the GPU -> (level1, level2) gamma-decoded fp32 box-filter levels (warping.py:9-13)."""
    if not images.is_cuda or images.dtype != torch.uint8:
        raise _lib.MetrabsB200Error('build_pyramid takes a uint8 CUDA tensor [N,3,H,W] (no CPU fallback)')
    images = images.contiguous()
    n, c, h, w = images.shape
    assert c == 3
    l1 = torch.empty(n, 3, h // 2, w // 2, dtype=torch.float32, device=images.device)
    l2 = torch.empty(n, 3, h // 4, w // 4, dtype=torch.float32, device=images.device)
    with torch.cuda.device(images.device):
        check(lib().mtb_image_pyramid(images.data_ptr(), n, h, w, l1.data_ptr(), l2.data_ptr(), _stream(images.device)))
    return l1, l2


def crop_setup(boxes, intrinsic_matrix, distortion_coeffs, camspace_up, aug_rotflipmat, aug_scales, resolution,
               antialias_factor=1):
    """_get_new_rotation_and_scale + the matrices of _get_crops (multiperson_model.py:264-293, :321-355).
    -> new_intrinsic_matrix [A,n,3,3], R [A,n,3,3], new_invprojmat [A*n,3,3], pyramid levels [A*n] (device tensors).
    ``antialias_factor``: 1, 2, 4 or 5..16, as for warp_images_with_pyramid; others raise MetrabsB200Error."""
    dev = boxes.device
    n, a = boxes.shape[0], aug_scales.shape[0]
    boxes = boxes.float().contiguous()
    k = _dev_f32(intrinsic_matrix, dev)
    d = _dev_f32(distortion_coeffs, dev)
    up = _dev_f32(camspace_up, dev)
    rf = _dev_f32(aug_rotflipmat, dev)
    sc = _dev_f32(aug_scales, dev)
    new_k = torch.empty(a, n, 3, 3, dtype=torch.float32, device=dev)
    rot = torch.empty(a, n, 3, 3, dtype=torch.float32, device=dev)
    inv = torch.empty(a * n, 3, 3, dtype=torch.float32, device=dev)
    lev = torch.empty(a * n, dtype=torch.int32, device=dev)
    args = _lib.MtbCropSetupArgs(_ptr(boxes), boxes.shape[1], _ptr(k), _ptr(d), d.shape[1], _ptr(up), _ptr(rf), _ptr(sc), n, a,
                                 int(resolution), int(antialias_factor), _ptr(new_k), _ptr(rot), _ptr(inv), _ptr(lev))
    with torch.cuda.device(dev):
        check(lib().mtb_crop_setup(C.byref(args), _stream(dev)))
    return new_k, rot, inv, lev


def warp_images_with_pyramid(images, pyramid, intrinsic_matrix, new_invprojmats, distortion_coeffs, pyramid_levels,
                             gamma_exponents, resolution, image_ids, num_aug, antialias_factor=1, out=None):
    """All ``num_aug * n_boxes`` crops in one launch (warping.py:6-52 + the gamma of multiperson_model.py:318), as the fp32
    NCHW tensor the crop model reads.  ``intrinsic_matrix`` / ``distortion_coeffs`` / ``image_ids`` are per BOX (the
    reference tiles them over the augmentations, multiperson_model.py:299-305).

    ``antialias_factor`` f renders each crop at res * f: at 2 and 4 it is box-averaged (the reference's avg_pool2d), at
    5..16 shrunk with the antialiased bilinear resize (torchvision's resize(BILINEAR, antialias=True), :311-314) inside the
    kernel, without the render reaching device memory.  3 (the reference has no shrink for it), 0 and above 16 raise
    MetrabsB200Error."""
    dev = images.device
    n = intrinsic_matrix.shape[0]
    images = images.contiguous()
    k = _dev_f32(intrinsic_matrix, dev)
    d = _dev_f32(distortion_coeffs, dev)
    ids = torch.as_tensor(image_ids, dtype=torch.int32).to(dev).contiguous()
    ge = _dev_f32(gamma_exponents, dev)
    if out is None:
        out = torch.empty(num_aug * n, 3, resolution, resolution, dtype=torch.float32, device=dev)
    args = _lib.MtbWarpArgs(_ptr(images), _ptr(pyramid[0]), _ptr(pyramid[1]), images.shape[0], images.shape[2], images.shape[3],
                            _ptr(k), _ptr(d), d.shape[1], _ptr(ids), _ptr(new_invprojmats), _ptr(pyramid_levels), _ptr(ge), n,
                            int(num_aug), int(resolution), int(antialias_factor), _ptr(out))
    with torch.cuda.device(dev):
        check(lib().mtb_warp_crops(C.byref(args), _stream(dev)))
    return out
