"""Cost of the latent-point forward (transform_coords): step time of a plain 48-point model against the same model with
its 48 reconstructed points mapped to 555 joints (combine_points_kernel), plus that kernel's own time from the
library's CUDA-event profiler.  EfficientNetV2-L@256, bf16 tensor-core mode, device buffers, mtb_forward with its
captured graph.  The two models share the backbone and head weights; their steps are timed alternately in the same
process.  Prints one JSON line with the card's name and power limit.

  python scripts/latent_step.py [--batch 256] [--steps 20] [--rounds 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import metrabs_b200  # noqa: E402
from oracle import port, port_latents  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(',')]
        return dict(gpu=name, power_limit=power, sm_clock_max=clock)
    except Exception as e:  # the JSON line still names the device torch sees
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f'unknown ({e})')


def step_ms(eng, crops, k, out, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        eng.forward(crops, k, out=out)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--latents', type=int, default=48)
    ap.add_argument('--joints', type=int, default=555)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('latent_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    margs = argparse.Namespace(side=256, precision='bf16', joints=args.latents, size='l')
    plain = bench.build_model(margs, dev)
    sd = plain.state_dict()
    w1, w2 = port_latents.make_affine_weights(args.joints, args.latents, seed=0)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'affine.npz')
        np.savez(path, w1=w1, w2=w2)
        metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision='bf16', affine_weights=path,
                                                    transform_coords=True))
        from metrabs_b200.backbones import efficientnet as E
        from metrabs_b200.models.metrabs import Metrabs
        ji = types.SimpleNamespace(names=[f'j{i}' for i in range(args.joints)], stick_figure_edges=[(0, 1)],
                                   n_joints=args.joints)
        latent = Metrabs(torch.nn.Sequential(E.PreprocLayer(), E.EfficientNet('l').features), ji).eval()
    latent.load_state_dict(sd, strict=True)
    latent = latent.to(dev)
    crops, k = bench.synthetic(args.batch, 256, seed=0)
    crops, k = crops.to(dev), k.to(dev)
    runs = {}
    for tag, m in (('plain', plain), ('latent', latent)):
        eng = m.engine(dev)
        out = torch.empty(args.batch, eng.n_out, 3, device=dev)
        for _ in range(3):  # warm-up; the second call on these buffers captures the graph
            eng.forward(crops, k, out=out)
        torch.cuda.synchronize()
        runs[tag] = dict(eng=eng, out=out, ms=[])
    for _ in range(args.rounds):
        for tag in ('plain', 'latent'):
            r = runs[tag]
            r['ms'].append(step_ms(r['eng'], crops, k, r['out'], args.steps))
    # the recombination's own time: profiler window (plain launches, no graph) over the same steps
    eng = runs['latent']['eng']
    eng.profile_begin()
    for _ in range(args.steps):
        eng.forward(crops, k, out=runs['latent']['out'])
    prof = eng.profile_end()['combine_points_kernel']
    # the latent model's joints equal the einsum of its own latents (head + reconstruction as the plain model computes)
    lat = runs['plain']['eng'].forward(crops, k)
    ref = torch.einsum('blc,lJ->bJc', lat.double(), torch.from_numpy(w2).to(dev).double())
    err = port.relative_error(runs['latent']['eng'].forward(crops, k).cpu(), ref.cpu())
    res = dict(workload=f'EfficientNetV2-L@256, {args.batch} crops, bf16', **card(),
               plain_points=args.latents, latent_joints=args.joints,
               plain_step_ms_median=statistics.median(runs['plain']['ms']),
               latent_step_ms_median=statistics.median(runs['latent']['ms']),
               plain_step_ms=runs['plain']['ms'], latent_step_ms=runs['latent']['ms'],
               combine_points_kernel_us=prof['ms'] / prof['launches'] * 1e3,
               combine_points_kernel_GBps=prof['bytes'] / (prof['ms'] / 1e3) / 1e9,
               latent_vs_einsum_rel_err=err, steps=args.steps, rounds=args.rounds)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
