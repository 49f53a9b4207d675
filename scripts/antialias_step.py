"""Cost of the antialias factor in crop generation.  From 4 frames of 3840 x 2160 with 51 person boxes x 5 augmentations =
255 crops (bench.py's frames leg, at 4K): the warp launch alone (mtb_warp_crops: warp_crops_kernel for f = 1, 2, 4,
warp_crops_aa_kernel above 4) per batch and in render supersamples per second, for f in 1, 2, 4, 5, 8, 16 at res 256 and
384; and the step of Pose3dEstimator._estimate_poses_batched (pyramid, setup, warp, EfficientNetV2-L@256 bf16 crop model,
TTA merge) at f = 1 and 8.  CUDA events around back-to-back launches and a synchronise; the factors alternate within
each round and the medians over rounds are reported.  Prints one JSON line with the card's name and power limit.

  python scripts/antialias_step.py [--rounds 5] [--steps 5]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from scripts.latent_step import card  # noqa: E402

FACTORS = (1, 2, 4, 5, 8, 16)


def scene(device):
    g = torch.Generator().manual_seed(11)
    n_img, h, w = 4, 2160, 3840
    frames = torch.randint(0, 256, (n_img, 3, h, w), generator=g, dtype=torch.uint8).to(device)
    counts = [13, 12, 13, 13]
    boxes = []
    for c in counts:
        xy = torch.rand(c, 2, generator=g) * torch.tensor([w - 1200., h - 1500.])
        wh = torch.tensor([540., 1200.]) * (0.6 + 0.8 * torch.rand(c, 2, generator=g))
        boxes.append(torch.cat([xy, wh, torch.rand(c, 1, generator=g)], dim=1))
    k = torch.tensor([[[3300., 0, w / 2], [0, 3300., h / 2], [0, 0, 1]]])
    dist = torch.tensor([[-0.05, 0.01, 0.0005, -0.0005, 0.001]])
    return frames, boxes, counts, k, dist


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--no-pose-step', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('antialias_step.py measures on the GPU and needs a CUDA device')
    from metrabs_b200.multiperson import Pose3dEstimator, warping
    from metrabs_b200.multiperson.multiperson_model import aug_parameters
    dev = torch.device('cuda', 0)
    frames, boxes, counts, k, dist = scene(dev)
    n_box, num_aug = sum(counts), 5
    n_crops = n_box * num_aug
    pyr = warping.build_pyramid(frames)
    k_box = k.repeat(n_box, 1, 1).to(dev)
    d_box = dist.repeat(n_box, 1).to(dev)
    up = torch.tensor([[0., -1., 0.]]).repeat(n_box, 1).to(dev)
    ids = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    boxes_flat = torch.cat(boxes).to(dev)
    gam, sc, fl, rf = aug_parameters(num_aug)
    ge = (gam / 2.2).float()
    warps = {}
    for res in (256, 384):
        out = torch.empty(n_crops, 3, res, res, device=dev)
        for f in FACTORS:
            _, _, inv, lev = warping.crop_setup(boxes_flat, k_box, d_box, up, rf, sc, res, f)

            def run(inv=inv, lev=lev, res=res, f=f, out=out):
                warping.warp_images_with_pyramid(frames, pyr, k_box, inv, d_box, lev, ge, res, ids, num_aug, f, out=out)
            run()
            warps[(res, f)] = dict(run=run, ms=[], levels=sorted(set(lev.tolist())))
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for w in warps.values():
            w['ms'].append(timed(w['run'], args.steps))
    warp_res = {}
    for (res, f), w in warps.items():
        ms = statistics.median(w['ms'])
        warp_res[f'res{res}_f{f}'] = dict(ms_per_batch=ms, ms=w['ms'], levels=w['levels'],
                                          gsupersamples_per_s=n_crops * (res * f) ** 2 / ms / 1e6,
                                          output_pixels_per_s_g=n_crops * res * res / ms / 1e6)
    result = dict(workload=f'4 frames 3840x2160, {n_box} boxes x {num_aug} augmentations = {n_crops} crops', **card(),
                  warp=warp_res, rounds=args.rounds, steps=args.steps)
    if not args.no_pose_step:
        model = bench.build_model(argparse.Namespace(side=256, precision='bf16', joints=24, size='l'), dev)
        model.joint_names, model.joint_edges = [f'j{i}' for i in range(24)], [[0, 1]]
        est = Pose3dEstimator(model, {'': dict(indices=list(range(24)), names=model.joint_names, edges=[[0, 1]])}, None)
        kw = dict(intrinsic_matrix=k, distortion_coeffs=dist, extrinsic_matrix=torch.eye(4)[None],
                  world_up_vector=torch.tensor([0., -1., 0.]), default_fov_degrees=55, internal_batch_size=0, num_aug=num_aug,
                  average_aug=True, skeleton='', suppress_implausible_poses=False)
        steps = {f: [] for f in (1, 8)}
        for f in steps:
            for _ in range(2):
                est._estimate_poses_batched(frames, boxes, antialias_factor=f, **kw)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for f in steps:
                steps[f].append(timed(lambda f=f: est._estimate_poses_batched(frames, boxes, antialias_factor=f, **kw), args.steps))
        result['pose_step'] = {f'f{f}': dict(ms_median=statistics.median(v), ms=v,
                                             crops_per_s=n_crops / statistics.median(v) * 1e3) for f, v in steps.items()}
        result['pose_step_model'] = 'EfficientNetV2-L@256, 24 joints, bf16'
    print(json.dumps(result), flush=True)


if __name__ == '__main__':
    main()
