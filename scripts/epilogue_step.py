"""Step time of the workloads whose time goes to the tensor-core epilogues (tc_conv_kernel, tc_conv3x3s1_kernel,
fmb_kernel, tc32_conv_kernel), on this tree's library against a baseline tree's, in one call.

Each tree runs in a worker process of its own (this script with --worker, the tree's package on sys.path), and both load
one configuration at a time: bench.py's model (bench.build_model: conditioned random init, seeded synthetic crops),
or ResNet-50 V2 as scripts/resnet_v2_step.py builds it.  After --warmup steps, the driver alternates --rounds rounds of
--steps steps between the two trees (CUDA events around plain mtb_forward calls on device buffers); then each tree
times every kernel class with the library's CUDA-event profiler in a separate pass, and saves the joints of its last
step.  The JSON line holds per configuration and tree the median and spread (min, max) of the rounds, crops/s, the
per-class device ms per step, the ratio of the medians, and whether the two trees' joints are bit-identical
(np.array_equal), with the card's name, power limit and max SM clock read in the same call.

  python scripts/epilogue_step.py --baseline-tree DIR [--steps 20] [--warmup 3] [--rounds 5] [--configs l/bf16,...]
                                  [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# name -> (size, precision, batch, stride_test, heatmap depth)
CONFIGS = {
    'l/bf16': ('l', 'bf16', 256, 32, 8),          # the flagship workload of bench.py
    'l/fp16': ('l', 'fp16', 256, 32, 8),
    'l/tf32x3': ('l', 'tf32x3', 256, 32, 8),      # bench.py's parity-mode line
    's/bf16': ('s', 'bf16', 256, 32, 8),
    'v2-b3/bf16': ('v2-b3', 'bf16', 256, 32, 8),  # fmb_kernel at 40 and 56 channels
    'resnet50-s8/bf16': ('resnet50', 'bf16', 128, 8, 32),
    'resnet50v2/bf16': ('resnet50v2', 'bf16', 256, 32, 8),  # tc_conv_preact_kernel
}
CLASSES = ('tc_conv_kernel', 'tc_conv3x3s1_kernel', 'fmb_kernel', 'tc32_conv_kernel')


class Worker:
    """One tree's model of the loaded configuration: setup, timed rounds, the profiler pass, the joints."""

    def __init__(self, args):
        self.args, self.run = args, None

    def load(self, name):
        import gc
        import torch
        import bench
        from scripts.latent_step import step_ms
        self.run = None
        gc.collect()
        torch.cuda.empty_cache()
        size, prec, batch, stride, depth = CONFIGS[name]
        dev = torch.device('cuda', 0)
        if size == 'resnet50v2':
            from scripts.resnet_v2_step import build
            model = build(50, stride, depth, prec, self.args.joints, dev)
        else:
            a = types.SimpleNamespace(size=size, side=256, precision=prec, stride=stride, depth=depth, joints=self.args.joints)
            model = bench.build_model(a, dev)
        eng = model.engine(dev)
        crops, k = bench.synthetic(batch, 256, 100)
        crops, k = crops.to(dev), k.to(dev)
        out = torch.empty(batch, eng.n_out, 3, device=dev)
        for _ in range(self.args.warmup):
            eng.forward(crops, k, out=out)
        torch.cuda.synchronize()
        self.run = dict(name=name, batch=batch, model=model, eng=eng, crops=crops, k=k, out=out, ms=[], step_ms=step_ms)

    def round(self):
        r = self.run
        r['ms'].append(r['step_ms'](r['eng'], r['crops'], r['k'], r['out'], self.args.steps))

    def report(self, dump):
        import numpy as np
        import torch
        r = self.run
        np.save(dump, r['out'].float().cpu().numpy())  # the joints of the last timed step
        eng, med = r['eng'], statistics.median(r['ms'])
        eng.profile_begin()
        for _ in range(self.args.steps):
            eng.forward(r['crops'], r['k'], out=r['out'])
        prof = eng.profile_end()
        return dict(ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']), ms_per_step=r['ms'],
                    crops_per_s=r['batch'] / (med / 1e3), joints_finite=bool(torch.isfinite(r['out']).all()),
                    kernel_classes_ms_per_step={n: v['ms'] / self.args.steps
                                                for n, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])})


def worker(args):
    """--worker: serves load / round / report requests on stdin, one reply line each on stdout."""
    sys.path.insert(0, args.tree)
    os.chdir(args.tree)
    w = Worker(args)
    print('ready', flush=True)
    for line in sys.stdin:
        cmd, _, arg = line.strip().partition(' ')
        if cmd == 'load':
            w.load(arg)
            print('loaded', flush=True)
        elif cmd == 'round':
            w.round()
            print('done', flush=True)
        elif cmd == 'report':
            print(json.dumps(w.report(arg)), flush=True)
        elif cmd == 'quit':
            return


class Proc:
    def __init__(self, tree, args):
        cmd = [sys.executable, os.path.abspath(__file__), '--worker', '--tree', os.path.abspath(tree)]
        for a in ('steps', 'warmup', 'joints'):
            cmd += [f'--{a}', str(getattr(args, a))]
        self.p = subprocess.Popen(cmd, stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        self.expect('ready')

    def ask(self, line):
        self.p.stdin.write(line + '\n')
        self.p.stdin.flush()
        return self.p.stdout.readline().strip()

    def expect(self, word, line=None):
        got = self.ask(line) if line else self.p.stdout.readline().strip()
        assert got == word, (word, got)

    def close(self):
        self.p.stdin.write('quit\n')
        self.p.stdin.flush()
        self.p.wait(timeout=120)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-tree', default=None, help='a built checkout of the revision to compare against')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--configs', default=','.join(CONFIGS))
    ap.add_argument('--out', default=None, help='where the joints are saved (default: a new temporary directory)')
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    ap.add_argument('--tree', default=ROOT, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('epilogue_step.py measures on the GPU and needs a CUDA device')
    from scripts.latent_step import card
    info = card()  # read before the runs, in the same call as the measurement
    args.out = os.path.abspath(args.out or tempfile.mkdtemp(prefix='epilogue_step_'))  # the workers run in their trees
    os.makedirs(args.out, exist_ok=True)
    trees = {'this_tree': ROOT}
    if args.baseline_tree:
        trees['baseline'] = args.baseline_tree
    procs = {t: Proc(d, args) for t, d in trees.items()}
    res = dict(**info, steps=args.steps, rounds=args.rounds, warmup=args.warmup, joints=args.joints,
               baseline_tree=os.path.abspath(args.baseline_tree) if args.baseline_tree else None, results={})
    for name in args.configs.split(','):
        for p in procs.values():
            p.expect('loaded', f'load {name}')
        for _ in range(args.rounds):  # alternating: this tree, then the baseline
            for p in procs.values():
                p.expect('done', 'round')
        r = {}
        for t, p in procs.items():
            dump = os.path.join(args.out, f'{name.replace("/", "_")}_{t}.npy')
            r[t] = json.loads(p.ask(f'report {dump}'))
            r[t]['joints'] = dump
        if 'baseline' in r:
            new, old = r['this_tree'], r['baseline']
            r['baseline_over_this_step'] = old['ms_per_step_median'] / new['ms_per_step_median']
            r['class_ms'] = {t: {c: round(r[t]['kernel_classes_ms_per_step'].get(c, 0.0), 3) for c in CLASSES} for t in procs}
            r['joints_bit_identical'] = bool(np.array_equal(np.load(new['joints']), np.load(old['joints'])))
        size, prec, batch, stride, depth = CONFIGS[name]
        res['results'][name] = dict(workload=f'{size}@256, {prec}, {batch} crops, stride {stride}, D={depth}', **r)
        print(json.dumps({name: res['results'][name]}), file=sys.stderr, flush=True)
    for p in procs.values():
        p.close()
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
