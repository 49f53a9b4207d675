"""Step time of the pre-activation ResNets (ResNet-50, -101, -152 V2) at proc_side 256, output stride 32 (D=8) and 8
(D=32), in the 'bf16' and 'fp16' tensor-core modes, measured like scripts/resnet_step.py (device buffers, mtb_forward
with its captured graph, medians and spread of alternating rounds, per-kernel-class device times from a separate
profiled pass), plus the comparison that decides whether a block's _3_conv and the pre-activation behind it run as one
tc_conv_preact_kernel launch: for every distinct fused pair shape of ResNet-50 V2 at strides 32 and 8, the fused launch
(mtb_debug_run_preact_pair) against _3_conv and the pre-activation op run separately (mtb_debug_run_op), kernel time
only (the library's CUDA-event profiler brackets the launches, not the operand conversions), alternating, at the
timed batch.  The weights are conditioned_random_init_'s, with every _3_conv (no BN behind it) damped so that the
residual stream stays finite.  Prints one JSON line with the card's name, power limit and max SM clock.

  python scripts/resnet_v2_step.py [--batch 128] [--steps 20] [--rounds 5] [--depths 50,101,152] [--pair-reps 20]"""
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


@torch.no_grad()
def build(depth, stride, d, precision, joints, device):
    import metrabs_b200
    from metrabs_b200.backbones import resnet
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=256, precision=precision, stride_test=stride, depth=d))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    model = Metrabs(getattr(resnet, f'resnet{depth}v2')(), ji).eval()
    conditioned_random_init_(model, seed=0)
    for name, m in model.named_modules():
        if name.endswith('_3_conv'):
            m.weight.mul_(0.3)
    model.mark_weights_changed()
    return model.to(device)


def kernel_ms(eng, fn, reps):
    """device ms per call of the kernels fn launches (profiler window, every class)"""
    eng.profile_begin()
    for _ in range(reps):
        fn()
    prof = eng.profile_end()
    return sum(v['ms'] for v in prof.values()) / reps


def pair_comparison(batch, reps, rounds, dev):
    """fused vs separate per distinct (H, W, Cin, Cout) of the fused pairs of ResNet-50 V2, bf16 and fp16"""
    out = []
    for stride, d in STRIDES:
        for prec in MODES:
            eng = build(50, stride, d, prec, 24, dev).engine(dev)
            names = eng.op_names()
            seen = {}
            for i in range(len(names) - 1):
                if not eng.op_is_preact_pair(i):
                    continue
                io = eng.op_io(i)
                seen.setdefault((io['in_shape'], io['out_shape']), (i, names[i], names[i + 1]))
            g = torch.Generator().manual_seed(0)
            for (ins, outs), (i, a, b) in seen.items():
                x = torch.randn((batch,) + ins, generator=g).to(dev)
                res = torch.randn((batch,) + outs, generator=g).to(dev)
                fused = lambda: eng.debug_run_preact_pair(i, x, res)  # noqa: E731
                y = eng.debug_run_op(i, x, res)

                def separate():
                    eng.debug_run_op(i, x, res)
                    eng.debug_run_op(i + 1, y)
                fused(), separate()
                torch.cuda.synchronize()
                tf, ts = [], []
                for _ in range(rounds):
                    tf.append(kernel_ms(eng, fused, reps))
                    ts.append(kernel_ms(eng, separate, reps))
                out.append(dict(stride=stride, precision=prec, pair=f'{a} + {b}', in_shape=ins, out_shape=outs,
                                fused_ms=statistics.median(tf), separate_ms=statistics.median(ts),
                                fused_ms_rounds=tf, separate_ms_rounds=ts,
                                speedup=statistics.median(ts) / statistics.median(tf)))
            del eng
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=128)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--joints', type=int, default=24)
    ap.add_argument('--depths', default='50,101,152')
    ap.add_argument('--pair-reps', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('resnet_v2_step.py measures on the GPU and needs a CUDA device')
    dev = torch.device('cuda', 0)
    info = card()  # read before the runs, in the same call as the measurement
    pairs = pair_comparison(args.batch, args.pair_reps, args.rounds, dev)
    crops, k = bench.synthetic(args.batch, 256, seed=0)
    crops, k = crops.to(dev), k.to(dev)
    lines = []
    for depth in [int(x) for x in args.depths.split(',')]:
        runs = {}
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
        for (depth_, stride, prec), r in runs.items():
            eng = r['eng']
            med = statistics.median(r['ms'])
            cout, cin = r['model'].heatmap_heads.conv_final.weight.shape[:2]
            head = 2.0 * (256 // stride) ** 2 * cin * cout
            bb = eng.backbone_flops_per_crop
            whole = (bb + head) * args.batch / (med / 1e3) / 1e12
            line = dict(backbone=f'resnet{depth_}v2', stride=stride, depth=r['d'], precision=prec,
                        ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']),
                        ms_per_step=r['ms'], crops_per_s=args.batch / (med / 1e3), backbone_flops_per_crop=bb,
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
    res = dict(workload=f'ResNet V2 family @256, {args.batch} crops, J={args.joints}', **info, peak_tflops=PEAK_TFLOPS,
               peak_note='H100 SXM data sheet, dense bf16/fp16 at 700 W; whole-step rate, not a kernel share of peak',
               steps=args.steps, rounds=args.rounds, warmup=args.warmup, fused_vs_separate=pairs, results=lines)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
