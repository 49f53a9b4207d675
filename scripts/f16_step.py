"""Cost of the fp16 tensor-core mode: step time of EfficientNetV2-L@256 in 'fp16' against the same model in 'bf16' (same
weights, device buffers, mtb_forward with its captured graph), timed in alternating rounds in one process, plus the
per-kernel-class device time of each mode from the library's CUDA-event profiler in a separate pass (plain launches).
Also reports each mode's feature deviation from fp32 CUDA-core features of the same crops.  Prints one JSON line with the
card's name and power limit.

  python scripts/f16_step.py [--batch 256] [--steps 20] [--rounds 5]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from oracle import port  # noqa: E402
from scripts.latent_step import card, step_ms  # noqa: E402

MODES = ('bf16', 'fp16')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--joints', type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('f16_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    crops, k = bench.synthetic(args.batch, 256, seed=0)
    crops, k = crops.to(dev), k.to(dev)
    runs, sd = {}, None
    for prec in MODES + ('fp32',):
        m = bench.build_model(argparse.Namespace(side=256, precision=prec, joints=args.joints, size='l'), dev)
        if sd is None:
            sd = m.state_dict()
        else:
            m.load_state_dict(sd, strict=True)  # every mode runs the first model's weights
        eng = m.engine(dev)
        feats = eng.backbone(crops[:8]).float()
        out = torch.empty(args.batch, eng.n_out, 3, device=dev)
        if prec != 'fp32':
            for _ in range(3):  # warm-up; the second call on these buffers captures the graph
                eng.forward(crops, k, out=out)
        torch.cuda.synchronize()
        runs[prec] = dict(eng=eng, out=out, ms=[], feats=feats)
    for _ in range(args.rounds):
        for prec in MODES:
            r = runs[prec]
            r['ms'].append(step_ms(r['eng'], crops, k, r['out'], args.steps))
    classes = {}
    for prec in MODES:
        eng = runs[prec]['eng']
        eng.profile_begin()
        for _ in range(args.steps):
            eng.forward(crops, k, out=runs[prec]['out'])
        prof = eng.profile_end()
        classes[prec] = {name: dict(ms_per_step=v['ms'] / args.steps, launches_per_step=v['launches'] / args.steps)
                         for name, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}
    med = {prec: statistics.median(runs[prec]['ms']) for prec in MODES}
    ref = runs['fp32']['feats'].cpu()
    res = dict(workload=f'EfficientNetV2-L@256, {args.batch} crops', **card(),
               bf16_step_ms_median=med['bf16'], fp16_step_ms_median=med['fp16'],
               fp16_over_bf16=med['fp16'] / med['bf16'],
               bf16_step_ms=runs['bf16']['ms'], fp16_step_ms=runs['fp16']['ms'],
               feature_rel_err_vs_fp32={prec: port.relative_error(runs[prec]['feats'].cpu(), ref) for prec in MODES},
               kernel_classes=classes, steps=args.steps, rounds=args.rounds)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
