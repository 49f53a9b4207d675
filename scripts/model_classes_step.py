"""Step time of the three model classes on one backbone: Metrabs, Metro and Model25D on EfficientNetV2-L@256 with 24 joints
and D = 8, 256 crops, bf16 tensor-core mode, device buffers, mtb_forward with its captured graph.  The three share the
backbone weights and the head's D*J volumetric channels; their steps are timed in alternating rounds in one process with
CUDA events around the steps and a synchronise.  A separate profiled pass gives the head's and the bone-length solve's own
times from the library's CUDA-event profiler.  Prints one JSON line with the card's name and power limit.

  python scripts/model_classes_step.py [--batch 256] [--steps 20] [--rounds 5]"""
import argparse
import json
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import metrabs_b200  # noqa: E402
from oracle import port_model_classes as pm  # noqa: E402
from scripts.latent_step import card, step_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--joints', type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('model_classes_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    j = args.joints
    metrabs = bench.build_model(argparse.Namespace(side=256, precision='bf16', joints=j, size='l'), dev)
    sd = pm.to_volumetric_state_dict(metrabs.state_dict(), j)
    from metrabs_b200.backbones import efficientnet as E
    from metrabs_b200.models.metro import Metro
    from metrabs_b200.models.twofive import Model25D
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision='bf16'))
    edges = pm.tree_edges(j)
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(j)], stick_figure_edges=edges, n_joints=j)
    models = dict(metrabs=metrabs)
    for tag, make in (('metro', lambda bb: Metro(bb, ji)),
                      ('model25d', lambda bb: Model25D(bb, ji, pm.seeded_bone_lengths(len(edges))))):
        m = make(torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet('l').features)).eval()
        m.load_state_dict(sd, strict=True)
        models[tag] = m.to(dev)
    crops, k = bench.synthetic(args.batch, 256, seed=0)
    crops, k = crops.to(dev), k.to(dev)
    runs = {}
    for tag, m in models.items():
        eng = m.engine(dev)
        kk = None if tag == 'metro' else k
        out = torch.empty(args.batch, j, 3, device=dev)
        for _ in range(3):  # warm-up; the second call on these buffers captures the graph
            eng.forward(crops, kk, out=out)
        torch.cuda.synchronize()
        runs[tag] = dict(eng=eng, k=kk, out=out, ms=[])
    for _ in range(args.rounds):
        for r in runs.values():
            r['ms'].append(step_ms(r['eng'], crops, r['k'], r['out'], args.steps))
    kernels = {}
    for tag, r in runs.items():
        r['eng'].profile_begin()
        for _ in range(args.steps):
            r['eng'].forward(crops, r['k'], out=r['out'])
        prof = r['eng'].profile_end()
        kernels[tag] = {name: dict(us_per_step=p['ms'] / args.steps * 1e3, launches_per_step=p['launches'] / args.steps)
                        for name, p in prof.items()
                        if name in ('tc_head_softargmax_kernel', 'recon_pass1+2_kernel', 'bone_solve_kernel')}
    res = dict(workload=f'EfficientNetV2-L@256, {args.batch} crops, {j} joints, D=8, bf16', **card(),
               step_ms_median={tag: statistics.median(r['ms']) for tag, r in runs.items()},
               step_ms={tag: r['ms'] for tag, r in runs.items()},
               crops_per_s_median={tag: args.batch / statistics.median(r['ms']) * 1e3 for tag, r in runs.items()},
               kernels=kernels, steps=args.steps, rounds=args.rounds)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
