"""Step time of MobileNetV3-Small and -Large at proc_side 256, output stride 32, D=8, in the 'bf16' and 'fp16' tensor-core
modes: device buffers, mtb_forward with its captured graph, the conditioned random weights bench.py uses (its
`--size mobilenetv3-small` model is the Small one here).  After a warm-up, every configuration is timed for --steps steps
in each of --rounds alternating rounds in one process; the JSON line reports the median and the spread (min, max) of the
rounds, crops/s and, from the library's CUDA-event profiler in a separate pass (plain launches, no graph), the device time
per step of each kernel class.  Depthwise convs of every kernel are in the class `dwconv_kernel`.

With --baseline-tree DIR (a built checkout of another revision of this repository), MobileNetV3-Small is also timed on that
revision's library in the same call: each tree runs in a worker process of its own, both models stay resident, and the
driver alternates the workers round by round.  The JSON line then holds both trees' step times and `dwconv_kernel` class
times.  Prints one JSON line with the card's name, power limit and max SM clock.

  python scripts/mobilenet_step.py [--batch 256] [--steps 20] [--rounds 5] [--baseline-tree DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ('bf16', 'fp16')


def build(variant, precision, joints, device):
    """bench.build_model with the MobileNetV3 `variant`: same config, same conditioned_random_init_."""
    import torch
    import metrabs_b200
    from metrabs_b200.backbones import mobilenet_v3
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision=precision, stride_test=32, depth=8))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    backbone = getattr(mobilenet_v3, f'mobilenet_v3_{variant}')()
    model = Metrabs(backbone, ji).eval()
    conditioned_random_init_(model, seed=0)
    return model.to(torch.device(device))


class Runs:
    """The models of one tree in this process: setup, one timed round, the profiler pass."""

    def __init__(self, variants, args):
        import torch
        import bench
        from scripts.latent_step import step_ms
        self.step_ms, self.args = step_ms, args
        self.dev = torch.device('cuda', 0)
        crops, k = bench.synthetic(args.batch, 256, seed=0)
        self.crops, self.k = crops.to(self.dev), k.to(self.dev)
        self.runs = {}
        for variant in variants:
            for prec in MODES:
                m = build(variant, prec, args.joints, self.dev)
                eng = m.engine(self.dev)
                out = torch.empty(args.batch, eng.n_out, 3, device=self.dev)
                for _ in range(args.warmup):  # the second call on these buffers captures the graph
                    eng.forward(self.crops, self.k, out=out)
                torch.cuda.synchronize()
                self.runs[f'{variant}/{prec}'] = dict(model=m, eng=eng, out=out, ms=[])

    def round(self):
        for r in self.runs.values():
            r['ms'].append(self.step_ms(r['eng'], self.crops, self.k, r['out'], self.args.steps))

    def report(self):
        import torch
        lines = {}
        for key, r in self.runs.items():
            eng = r['eng']
            med = statistics.median(r['ms'])
            line = dict(ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']),
                        ms_per_step=r['ms'], crops_per_s=self.args.batch / (med / 1e3),
                        backbone_flops_per_crop=eng.backbone_flops_per_crop, launches=eng.last_launch_count,
                        joints_finite=bool(torch.isfinite(r['out']).all()))
            eng.profile_begin()
            for _ in range(self.args.steps):
                eng.forward(self.crops, self.k, out=r['out'])
            prof = eng.profile_end()
            line['kernel_classes_ms_per_step'] = {name: v['ms'] / self.args.steps
                                                  for name, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}
            lines[key] = line
        return lines


def worker(args):
    """--worker: the Small models of --tree, driven over stdin / stdout by the main process."""
    sys.path.insert(0, args.tree)
    os.chdir(args.tree)
    runs = Runs(['small'], args)
    print('ready', flush=True)
    for cmd in sys.stdin:
        if cmd.strip() == 'round':
            runs.round()
            print('done', flush=True)
        elif cmd.strip() == 'report':
            print(json.dumps(runs.report()), flush=True)
            return


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--baseline-tree', default=None, help='a built checkout whose MobileNetV3-Small is timed alongside')
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    ap.add_argument('--tree', default=ROOT, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        sys.exit('mobilenet_step.py measures on the GPU and needs a CUDA device')
    from scripts.latent_step import card
    info = card()  # read before the runs, in the same call as the measurement
    runs = Runs(['small', 'large'], args)
    base = None
    if args.baseline_tree:
        cmd = [sys.executable, os.path.abspath(__file__), '--worker', '--tree', os.path.abspath(args.baseline_tree)]
        for a in ('batch', 'steps', 'warmup', 'joints'):
            cmd += [f'--{a}', str(getattr(args, a))]
        base = subprocess.Popen(cmd, stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        assert base.stdout.readline().strip() == 'ready'
    for _ in range(args.rounds):  # alternating: this tree's models, then the baseline tree's
        runs.round()
        if base:
            base.stdin.write('round\n')
            base.stdin.flush()
            assert base.stdout.readline().strip() == 'done'
    res = dict(workload=f'MobileNetV3 @256, stride 32, D=8, {args.batch} crops, J={args.joints}', **info,
               steps=args.steps, rounds=args.rounds, warmup=args.warmup, results=runs.report())
    if base:
        base.stdin.write('report\n')
        base.stdin.flush()
        res['baseline_tree'] = os.path.abspath(args.baseline_tree)
        res['baseline_results'] = json.loads(base.stdout.readline())
        base.wait(timeout=120)
        for prec in MODES:
            new, old = res['results'][f'small/{prec}'], res['baseline_results'][f'small/{prec}']
            res[f'small_{prec}_step_speedup'] = old['ms_per_step_median'] / new['ms_per_step_median']
            res[f'small_{prec}_dwconv_kernel_ms'] = dict(
                baseline=old['kernel_classes_ms_per_step'].get('dwconv_kernel'),
                this_tree=new['kernel_classes_ms_per_step'].get('dwconv_kernel'))
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
