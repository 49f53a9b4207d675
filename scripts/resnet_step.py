"""Step time of the ResNet family (ResNet-18, -34, -50, -101, -152 V1) at proc_side 256, output stride 32 (D=8) and 8
(D=32), in the 'bf16' and 'fp16' tensor-core modes: device buffers, mtb_forward with its captured graph, the same
conditioned random weights bench.py uses (its `--size resnet50` model is the ResNet-50 here).  After a warm-up, every
configuration is timed for --steps steps in each of --rounds alternating rounds in one process; the JSON line reports the
median and the spread (min, max) of the rounds, crops/s, the backbone FLOPs per crop (mtb_backbone_flops_per_crop) and
the whole-step rate (backbone + head FLOPs over the whole step time, decode and reconstruction included) over the 989
TFLOP/s dense 16-bit data-sheet figure of the H100 SXM: a whole-program rate, not a kernel's share of peak.  The
per-kernel-class device times come from the library's CUDA-event profiler in a separate pass (plain launches, no graph).
Prints one JSON line with the card's name, power limit and max SM clock.

  python scripts/resnet_step.py [--batch 128] [--steps 20] [--rounds 5] [--depths 18,34,50,101,152]"""
import argparse
import json
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from scripts.latent_step import card, step_ms  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16 / FP16, 700 W
STRIDES = ((32, 8), (8, 32))  # (stride_test, heatmap depth D)
MODES = ('bf16', 'fp16')


def build(depth, stride, d, precision, joints, device):
    """bench.build_model with the backbone of `depth`: same config, same conditioned_random_init_."""
    import metrabs_b200
    from metrabs_b200.backbones import resnet
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision=precision, stride_test=stride, depth=d))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    model = Metrabs(resnet.Features(depth), ji).eval()
    conditioned_random_init_(model, seed=0)
    return model.to(device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=128)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--depths', default='18,34,50,101,152')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('resnet_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    info = card()  # read before the runs, in the same call as the measurement
    crops, k = bench.synthetic(args.batch, 256, seed=0)
    crops, k = crops.to(dev), k.to(dev)
    runs = {}
    for depth in [int(x) for x in args.depths.split(',')]:
        for stride, d in STRIDES:
            for prec in MODES:
                m = build(depth, stride, d, prec, args.joints, dev)
                eng = m.engine(dev)
                out = torch.empty(args.batch, eng.n_out, 3, device=dev)
                for _ in range(args.warmup):  # the second call on these buffers captures the graph
                    eng.forward(crops, k, out=out)
                torch.cuda.synchronize()
                runs[(depth, stride, prec)] = dict(model=m, eng=eng, out=out, ms=[], d=d)
    for _ in range(args.rounds):
        for r in runs.values():
            r['ms'].append(step_ms(r['eng'], crops, k, r['out'], args.steps))
    lines = []
    for (depth, stride, prec), r in runs.items():
        eng = r['eng']
        med = statistics.median(r['ms'])
        # head FLOPs: the 1x1 conv from C to J*(1+D) channels at the feature side
        cout, cin = r['model'].heatmap_heads.conv_final.weight.shape[:2]
        head = 2.0 * (256 // stride) ** 2 * cin * cout
        bb = eng.backbone_flops_per_crop
        whole = (bb + head) * args.batch / (med / 1e3) / 1e12
        lines.append(dict(backbone=f'resnet{depth}', stride=stride, depth=r['d'], precision=prec,
                          ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']),
                          ms_per_step=r['ms'], crops_per_s=args.batch / (med / 1e3),
                          backbone_flops_per_crop=bb, head_flops_per_crop=head,
                          whole_step_tflops=whole, whole_step_tflops_over_989=whole / PEAK_TFLOPS,
                          joints_finite=bool(torch.isfinite(r['out']).all())))
    # per-kernel-class device time: profiler window over plain launches, separate from the timed rounds
    for line, r in zip(lines, runs.values()):
        r['eng'].profile_begin()
        for _ in range(args.steps):
            r['eng'].forward(crops, k, out=r['out'])
        prof = r['eng'].profile_end()
        line['kernel_classes_ms_per_step'] = {name: v['ms'] / args.steps
                                              for name, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}
    res = dict(workload=f'ResNet V1 family @256, {args.batch} crops, J={args.joints}', **info,
               peak_tflops=PEAK_TFLOPS, peak_note='H100 SXM data sheet, dense bf16/fp16 at 700 W; whole-step rate, '
               'not a kernel share of peak', steps=args.steps, rounds=args.rounds, warmup=args.warmup, results=lines)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
