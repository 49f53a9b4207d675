"""Step time of EfficientNet-B0..B7 at proc_side 256, output stride 32, D=8, in the 'bf16' and 'fp16' tensor-core modes:
device buffers, mtb_forward with its captured graph, bench.py's conditioned random weights
(metrabs_b200.init.conditioned_random_init_) on Metrabs(Sequential(PreprocLayer(), efficientnet_bN().features), ji).  After
a warm-up, every configuration is timed for --steps steps in each of --rounds alternating rounds in one process; the JSON
line reports the median and the spread (min, max) of the rounds, crops/s and, from the library's CUDA-event profiler in a
separate pass (plain launches, no graph), the device time per step of each kernel class.  Depthwise convs of every kernel
are in the class `dwconv_kernel`, the separate SE pooling pass in `pool_mean_kernel`.

All sixteen models do not fit in 80 GB at 256 crops together, so one variant's two modes are resident at a time, except for
the variants timed against the baseline.  With --baseline-tree DIR (a built checkout of another revision of this
repository), B0 and B4 are also timed on that revision's library in the same call, built through its
`efficientnet.Features(stages, last_channel)` with this tree's tables (a revision without the B constructors folds BatchNorm with eps 1e-3, which does not change the work; its 5x5 SiLU
ops run dwconv_kernel + pool_mean_kernel).  Each tree runs in a worker process of its own, all models stay resident, and
the driver alternates the workers round by round.  The JSON line then holds both trees' step times and their
`dwconv_kernel` and `pool_mean_kernel` class times.  Prints one JSON line with the card's name, power limit and max SM clock.

  python scripts/effnet_b_step.py [--batch 256] [--steps 20] [--rounds 5] [--variants 0,1,...,7] [--baseline-tree DIR]"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ('bf16', 'fp16')
BASELINE_VARIANTS = ('b0', 'b4')


def tables(variants):
    """variant -> (stages, last_channel, bn_eps) from this tree's metrabs_b200."""
    from metrabs_b200.backbones import efficientnet as E
    return {v: E.b_stage_table(v, centered_stride=True) for v in variants}


def build(table, precision, joints, device):
    """The crop model on efficientnet.Features(stages, last[, eps]) of whichever tree is imported."""
    import torch
    import metrabs_b200
    from metrabs_b200.backbones import efficientnet as E
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    stages, last, eps = table
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision=precision, stride_test=32, depth=8))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    try:
        feats = E.Features(stages, last, eps)
    except TypeError:  # a revision before the B family: eps 1e-3
        feats = E.Features(stages, last)
    model = Metrabs(torch.nn.Sequential(E.PreprocLayer(), feats), ji).eval()
    conditioned_random_init_(model, seed=0)
    return model.to(torch.device(device))


class Runs:
    """The models of one tree in this process: setup, one timed round, the profiler pass."""

    def __init__(self, tabs, args):
        import torch
        import bench
        from scripts.latent_step import step_ms
        self.step_ms, self.args = step_ms, args
        self.dev = torch.device('cuda', 0)
        crops, k = bench.synthetic(args.batch, 256, seed=0)
        self.crops, self.k = crops.to(self.dev), k.to(self.dev)
        self.runs = {}
        for variant, table in tabs.items():
            for prec in MODES:
                m = build(table, prec, args.joints, self.dev)
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
            line['kernel_classes_launches_per_step'] = {name: v['launches'] / self.args.steps for name, v in prof.items()}
            lines[key] = line
        return lines


def worker(args):
    """--worker: the models of --tables on --tree, driven over stdin / stdout by the main process."""
    sys.path.insert(0, args.tree)
    os.chdir(args.tree)
    runs = Runs(json.loads(args.tables), args)
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
    ap.add_argument('--variants', default='0,1,2,3,4,5,6,7')
    ap.add_argument('--baseline-tree', default=None, help='a built checkout whose library runs B0 and B4 alongside')
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    ap.add_argument('--tree', default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument('--tables', default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        sys.exit('effnet_b_step.py measures on the GPU and needs a CUDA device')
    from scripts.latent_step import card
    info = card()  # read before the runs, in the same call as the measurement
    tabs = tables([f'b{v}' for v in args.variants.split(',')])
    compared = {v: t for v, t in tabs.items() if args.baseline_tree and v in BASELINE_VARIANTS}
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
    runs = Runs(compared, args)
    base = None
    if args.baseline_tree:
        cmd = [sys.executable, os.path.abspath(__file__), '--worker', '--tree', os.path.abspath(args.baseline_tree),
               '--tables', json.dumps(tables(BASELINE_VARIANTS))]
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
    res = dict(workload=f'EfficientNet-B @256, stride 32, D=8, {args.batch} crops, J={args.joints}', **info,
               steps=args.steps, rounds=args.rounds, warmup=args.warmup)
    results.update(runs.report())
    res['results'] = {f'{v}/{p}': results[f'{v}/{p}'] for v in tabs for p in MODES}
    if base:
        base.stdin.write('report\n')
        base.stdin.flush()
        res['baseline_tree'] = os.path.abspath(args.baseline_tree)
        res['baseline_results'] = json.loads(base.stdout.readline())
        base.wait(timeout=120)
        for key, old in res['baseline_results'].items():
            new = res['results'].get(key)
            if new is None:
                continue
            tag = key.replace('/', '_')
            res[f'{tag}_step_speedup'] = old['ms_per_step_median'] / new['ms_per_step_median']
            res[f'{tag}_dw_and_pool_ms'] = {
                tree: {c: r['kernel_classes_ms_per_step'].get(c, 0.0) for c in ('dwconv_kernel', 'pool_mean_kernel')}
                for tree, r in (('baseline', old), ('this_tree', new))}
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
