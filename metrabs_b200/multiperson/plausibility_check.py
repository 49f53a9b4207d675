"""Device mirror of /root/reference/metrabs_pytorch/multiperson/plausibility_check.py (:8-119): the three plausibility
checks and the pose-similarity NMS in one launch per batch of images (``mtb_filter_poses``).  The reference reads the
mean bone lengths from a posepile dataset (:12-16); here they are an explicit argument."""
import ctypes as C

import torch

from metrabs_b200 import _lib
from metrabs_b200._lib import check, lib
from metrabs_b200.multiperson.warping import _ptr, _stream


def filter_poses(poses3d, poses2d, boxes, n_box_per_image, joint_edges, mean_bones):
    """poses3d [n,A,J,3] (camera space), poses2d [n,A,J,2], boxes [n,5] (x,y,w,h,score), all on the GPU.
    -> (plausible [n] bool, keep [n] bool): ``keep`` = plausible and surviving pose_non_max_suppression per image.
    Any number of boxes per image up to what one block's shared memory holds (about 16,000 per call on an H100); beyond
    that the call raises ``MetrabsB200Error`` rather than drop boxes."""
    dev = poses3d.device
    n, a, j, _ = poses3d.shape
    if sum(int(c) for c in n_box_per_image) != n or any(int(c) < 0 for c in n_box_per_image):
        raise ValueError(f'n_box_per_image {list(n_box_per_image)} does not partition the {n} boxes')
    poses3d = poses3d.float().contiguous()
    poses2d = poses2d.float().contiguous()
    boxes = boxes.float().contiguous()
    bones = torch.as_tensor(joint_edges, dtype=torch.int32).reshape(-1, 2).to(dev).contiguous()
    mb = torch.as_tensor(mean_bones, dtype=torch.float32).to(dev).contiguous()
    counts = torch.as_tensor(n_box_per_image, dtype=torch.int64)
    start = torch.zeros(len(counts) + 1, dtype=torch.int32)
    start[1:] = torch.cumsum(counts, 0).int()
    start = start.to(dev)
    plausible = torch.empty(n, dtype=torch.uint8, device=dev)
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    scratch = torch.empty(n, j, 3, dtype=torch.float32, device=dev)
    args = _lib.MtbFilterArgs(_ptr(poses3d), _ptr(poses2d), _ptr(boxes), boxes.shape[1], _ptr(bones), _ptr(mb), bones.shape[0],
                              _ptr(start), len(counts), n, a, j, _ptr(plausible), _ptr(keep), _ptr(scratch))
    with torch.cuda.device(dev):
        check(lib().mtb_filter_poses(C.byref(args), _stream(dev)))
    return plausible.bool(), keep.bool()
