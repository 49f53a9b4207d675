"""Step time of the backbones the reference's builder names last: ResNet-50, -101 and -152 V1.5 at proc_side 256, output
stride 32 (D=8) and 8 (D=32), and the minimalistic MobileNetV3-Small and -Large at stride 32 (D=8), in the 'bf16' and
'fp16' tensor-core modes.  Measured like scripts/resnet_v2_step.py: device buffers, mtb_forward with its captured graph,
medians and spread of alternating rounds (every configuration of one backbone in turn, per round), and per-kernel-class
device times from a separate profiled pass.  The weights are conditioned_random_init_'s; in the ResNets every _3_conv is
damped (x0.3) so that the residual stream stays within the fp16 range.  Prints one JSON line with the card's name,
power limit and max SM clock.

  python scripts/builder_variants_step.py [--batch 128] [--mobilenet-batch 256] [--steps 20] [--rounds 5]
                                          [--backbones resnet50v1_5,...,mobilenetv3-large-mini]"""
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
MODES = ('bf16', 'fp16')
# backbone -> [(stride_test, heatmap depth D)]
BACKBONES = {'resnet50v1_5': ((32, 8), (8, 32)), 'resnet101v1_5': ((32, 8), (8, 32)), 'resnet152v1_5': ((32, 8), (8, 32)),
             'mobilenetv3-small-mini': ((32, 8),), 'mobilenetv3-large-mini': ((32, 8),)}


@torch.no_grad()
def build(backbone, stride, d, precision, joints, device):
    import metrabs_b200
    from metrabs_b200.backbones import mobilenet_v3, resnet
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision=precision, stride_test=stride, depth=d))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    if backbone.startswith('resnet'):
        features = getattr(resnet, backbone)()
    else:
        features = getattr(mobilenet_v3, f'mobilenet_v3_{backbone.split("-")[1]}')(minimalistic=True)
    model = Metrabs(features, ji).eval()
    conditioned_random_init_(model, seed=0)
    for name, m in model.named_modules():
        if name.endswith('_3_conv'):
            m.weight.mul_(0.3)
    model.mark_weights_changed()
    return model.to(device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=128)
    ap.add_argument('--mobilenet-batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--backbones', default=','.join(BACKBONES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('builder_variants_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    info = card()  # read before the runs, in the same call as the measurement
    lines = []
    for backbone in args.backbones.split(','):
        batch = args.batch if backbone.startswith('resnet') else args.mobilenet_batch
        crops, k = bench.synthetic(batch, 256, seed=0)
        crops, k = crops.to(dev), k.to(dev)
        runs = {}
        for stride, d in BACKBONES[backbone]:
            for prec in MODES:
                m = build(backbone, stride, d, prec, args.joints, dev)
                eng = m.engine(dev)
                out = torch.empty(batch, eng.n_out, 3, device=dev)
                for _ in range(args.warmup):  # the second call on these buffers captures the graph
                    eng.forward(crops, k, out=out)
                torch.cuda.synchronize()
                runs[(stride, prec)] = dict(model=m, eng=eng, out=out, ms=[], d=d)
        for _ in range(args.rounds):
            for r in runs.values():
                r['ms'].append(step_ms(r['eng'], crops, k, r['out'], args.steps))
        for (stride, prec), r in runs.items():
            eng = r['eng']
            med = statistics.median(r['ms'])
            cout, cin = r['model'].heatmap_heads.conv_final.weight.shape[:2]
            head = 2.0 * (256 // stride) ** 2 * cin * cout
            bb = eng.backbone_flops_per_crop
            whole = (bb + head) * batch / (med / 1e3) / 1e12
            line = dict(backbone=backbone, stride=stride, depth=r['d'], precision=prec, batch=batch,
                        ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']),
                        ms_per_step=r['ms'], crops_per_s=batch / (med / 1e3), backbone_flops_per_crop=bb,
                        whole_step_tflops=whole, whole_step_tflops_over_989=whole / PEAK_TFLOPS,
                        launches=eng.last_launch_count, joints_finite=bool(torch.isfinite(r['out']).all()))
            eng.profile_begin()
            for _ in range(args.steps):
                eng.forward(crops, k, out=r['out'])
            prof = eng.profile_end()
            line['kernel_classes_ms_per_step'] = {name: v['ms'] / args.steps
                                                  for name, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms']) if v['ms'] > 0}
            lines.append(line)
        del runs
        torch.cuda.empty_cache()
    res = dict(workload=f'ResNet V1.5 and minimalistic MobileNetV3 @256, {args.batch} / {args.mobilenet_batch} crops, '
                        f'J={args.joints}', **info, peak_tflops=PEAK_TFLOPS,
               peak_note='H100 SXM data sheet, dense bf16/fp16 at 700 W; whole-step rate, not a kernel share of peak',
               steps=args.steps, rounds=args.rounds, warmup=args.warmup, results=lines)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
