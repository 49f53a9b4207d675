"""Step time of EfficientNetV2-B0..B3 and EfficientNetV2-XL at proc_side 256, output stride 32, D=8, in the 'bf16' and 'fp16'
tensor-core modes, measured like scripts/effnet_b_step.py (whose Runs class this script drives): device buffers,
mtb_forward with its captured graph, conditioned random weights, --rounds alternating rounds of --steps steps per
configuration, the median and spread (min, max) of the rounds, crops/s, and from a separate profiled pass the device time
per step of each kernel class.  One variant's two modes are resident at a time.

With --baseline-tree DIR (a built checkout of a revision whose fmb_kernel does not take 40- or 56-channel blocks, such as
the parent of the change that admitted them), V2-B2 and V2-B3 are also timed on that revision's library, built from this
tree's tables, in a worker process (effnet_b_step.py --worker) alternating round by round with this tree's models.  Their
identity-shaped FusedMBConv blocks of 56 (B2) and 40 and 56 (B3) channels run there as two tc_conv_kernel launches each,
and every other op runs the same kernels, so the two step times compare the step with and without those fused blocks.
The JSON line then holds both trees' step times, their fmb_kernel and tc_conv_kernel class times, and the ratio.  Prints
one JSON line with the card's name, power limit and max SM clock.

  python scripts/effnet_v2_variants_step.py [--batch 256] [--steps 20] [--rounds 5] [--variants v2-b0,...,xl]
                                            [--baseline-tree DIR]"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MODES = ('bf16', 'fp16')
VARIANTS = ('v2-b0', 'v2-b1', 'v2-b2', 'v2-b3', 'xl')
COMPARED = ('v2-b2', 'v2-b3')  # the variants with 40- or 56-channel fused blocks
CLASSES = ('fmb_kernel', 'tc_conv_kernel')


def tables(variants):
    """variant -> (stages, last_channel, bn_eps), the form effnet_b_step.build takes."""
    from metrabs_b200.backbones import efficientnet as E
    return {v: E.stage_table(v, centered_stride=True) + (1e-3,) for v in variants}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--variants', default=','.join(VARIANTS))
    ap.add_argument('--baseline-tree', default=None, help='a built checkout whose library runs V2-B2 and V2-B3 alongside')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('effnet_v2_variants_step.py measures on the GPU and needs a CUDA device')
    from scripts.effnet_b_step import Runs
    from scripts.latent_step import card
    info = card()  # read before the runs, in the same call as the measurement
    tabs = tables(args.variants.split(','))
    compared = {v: t for v, t in tabs.items() if args.baseline_tree and v in COMPARED}
    results = {}
    for v, t in tabs.items():  # one variant at a time: its two modes alternate round by round
        if v not in compared:
            runs = Runs({v: t}, args)
            for _ in range(args.rounds):
                runs.round()
            results.update(runs.report())
            del runs
            gc.collect()
            torch.cuda.empty_cache()
    base = None
    if compared:
        runs = Runs(compared, args)
        cmd = [sys.executable, os.path.join(ROOT, 'scripts', 'effnet_b_step.py'), '--worker', '--tree',
               os.path.abspath(args.baseline_tree), '--tables', json.dumps(compared)]
        for a in ('batch', 'steps', 'warmup', 'joints'):
            cmd += [f'--{a}', str(getattr(args, a))]
        base = subprocess.Popen(cmd, stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        assert base.stdout.readline().strip() == 'ready'
        for _ in range(args.rounds):  # alternating: this tree's models, then the baseline tree's
            runs.round()
            base.stdin.write('round\n')
            base.stdin.flush()
            assert base.stdout.readline().strip() == 'done'
        results.update(runs.report())
    res = dict(workload=f'EfficientNetV2-B0..B3 / XL @256, stride 32, D=8, {args.batch} crops, J={args.joints}', **info,
               steps=args.steps, rounds=args.rounds, warmup=args.warmup)
    res['results'] = {f'{v}/{p}': results[f'{v}/{p}'] for v in tabs for p in MODES}
    if base:
        base.stdin.write('report\n')
        base.stdin.flush()
        res['baseline_tree'] = os.path.abspath(args.baseline_tree)
        res['baseline_results'] = json.loads(base.stdout.readline())
        base.wait(timeout=120)
        for key, old in res['baseline_results'].items():
            new = res['results'][key]
            tag = key.replace('/', '_')
            res[f'{tag}_unfused_over_fused_step'] = old['ms_per_step_median'] / new['ms_per_step_median']
            res[f'{tag}_class_ms'] = {tree: {c: r['kernel_classes_ms_per_step'].get(c, 0.0) for c in CLASSES}
                                      for tree, r in (('unfused_40_56', old), ('fused', new))}
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
