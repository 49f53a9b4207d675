"""EfficientNetV2-S and -L at proc_side 256 and output stride 32, 16 and 8 (D=8, 24 joints), in the 'bf16' and 'fp16'
tensor-core modes: device buffers, mtb_forward with its captured graph, conditioned random weights
(metrabs_b200.init.conditioned_random_init_).  Per (backbone, output stride) the two modes stay resident and alternate for
--rounds rounds of --steps steps; the JSON line reports the median and spread of the rounds, crops/s and, from the library's
CUDA-event profiler in a separate pass, the device time per step of each kernel class (every depthwise kernel is in
`dwconv_kernel`, the separate SE pooling pass in `pool_mean_kernel`).

The dilated depthwise kernel against the generic path, without a switch: at output stride 8, the per-op profiler times of
the dilated depthwise ops plus their pool ops of a 'bf16' handle (dw3x3s1_dil_tma_kernel, pooling fused) and of a
'bf16_simt' handle (dwconv_kernel + pool_mean_kernel, same storage and shapes), and the achieved GB/s of the dilated ops
next to the undilated TMA-staged ops of the same forward (bytes: input + output in 16 bits, from the shapes).

With --baseline-tree DIR (a built checkout of another revision), the joints of EfficientNetV2-L@256, -S@256, EfficientNet-B0@256
at output stride 32 and ResNet-50@256 at stride 8 ('bf16', seeded weights and crops) are computed on both trees, each in a
process of its own, and compared with np.array_equal; their joints are written to --out (default: a new temporary
directory).

  python scripts/effnet_stride_step.py [--batch 256] [--steps 20] [--rounds 5] [--baseline-tree DIR] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ('bf16', 'fp16')


def build(size, output_stride, precision, joints=24, device='cuda:0', side=256):
    """Crop model on EfficientNet(size[, output_stride]) ('b0' too) or ResNet-50 ('resnet50', output_stride = stride_test)."""
    import torch
    import metrabs_b200
    from metrabs_b200.init import conditioned_random_init_
    from metrabs_b200.models.metrabs import Metrabs
    metrabs_b200.set_config(metrabs_b200.Config(proc_side=side, precision=precision, stride_test=output_stride, depth=8))
    ji = types.SimpleNamespace(names=[f'j{i}' for i in range(joints)], stick_figure_edges=[(0, 1)], n_joints=joints)
    if size == 'resnet50':
        from metrabs_b200.backbones import resnet
        feats = resnet.Features(50)
    else:
        from metrabs_b200.backbones import efficientnet as E
        bb = E.EfficientNet(size, output_stride) if output_stride != 32 else E.EfficientNet(size)
        feats = torch.nn.Sequential(E.PreprocLayer(), bb.features)
    model = Metrabs(feats, ji).eval()
    conditioned_random_init_(model, seed=0)
    return model.to(torch.device(device))


def timing(args):
    import torch
    import bench
    from scripts.latent_step import step_ms
    dev = torch.device('cuda', 0)
    results = {}
    for size in ('s', 'l'):
        for os_ in (32, 16, 8):
            batch = args.batch if (size, os_) != ('l', 8) else args.batch // 2
            crops, k = (t.to(dev) for t in bench.synthetic(batch, 256, seed=0))
            runs = {}
            for prec in MODES:
                m = build(size, os_, prec)
                eng = m.engine(dev)
                out = torch.empty(batch, eng.n_out, 3, device=dev)
                for _ in range(args.warmup):
                    eng.forward(crops, k, out=out)
                torch.cuda.synchronize()
                runs[prec] = dict(m=m, eng=eng, out=out, ms=[])
            for _ in range(args.rounds):
                for r in runs.values():
                    r['ms'].append(step_ms(r['eng'], crops, k, r['out'], args.steps))
            for prec, r in runs.items():
                med = statistics.median(r['ms'])
                line = dict(batch=batch, ms_per_step_median=med, ms_per_step_min=min(r['ms']), ms_per_step_max=max(r['ms']),
                            crops_per_s=batch / (med / 1e3), feature_side=r['eng'].feature_side,
                            backbone_gflop_per_crop=r['eng'].backbone_flops_per_crop / 1e9,
                            joints_finite=bool(torch.isfinite(r['out']).all()))
                r['eng'].profile_begin()
                for _ in range(args.steps):
                    r['eng'].forward(crops, k, out=r['out'])
                prof = r['eng'].profile_end()
                line['kernel_classes_ms_per_step'] = {n: v['ms'] / args.steps for n, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}
                results[f'{size}/os{os_}/{prec}'] = line
            del runs
            torch.cuda.empty_cache()
    return results


def dilated_ab(args):
    """Per-op times at output stride 8: bf16 (dilated TMA kernel, fused pooling) against bf16_simt (dwconv_kernel + pool)."""
    import torch
    import bench
    from metrabs_b200 import _lib
    dev = torch.device('cuda', 0)
    res = {}
    for size in ('s', 'l'):
        batch = args.batch if size == 's' else args.batch // 2
        crops = bench.synthetic(batch, 256, seed=0)[0].to(dev)
        line = {}
        for prec in ('bf16', 'bf16_simt'):
            eng = build(size, 8, prec).engine(dev)
            dil = [i for i in range(len(eng.op_names())) if eng.op_names()[i].endswith('.block.1') or
                   eng.op_names()[i].endswith('.block.0')]
            dw = [i for i in dil if _is_dw(eng, i)]
            for _ in range(args.warmup):
                eng.backbone(crops)
            eng.profile_begin()
            for _ in range(args.steps):
                eng.backbone(crops)
            eng.profile_end()
            ops = eng.profile_op_times()
            names = eng.op_names()
            kinds = {i: eng.op_dw_kernel(i) for i in dw}
            dil_ops = [i for i in dw if _dilation(eng, i, size) > 1]
            und_tma = [i for i in dw if kinds[i] == _lib.DW_TMA]
            ms = lambda idx: sum(ops[i][2] for i in idx) / args.steps  # noqa: E731
            gb = lambda idx: sum(batch * ops[i][4] for i in idx) / 1e9  # noqa: E731  activation bytes per forward
            pools = [i + 1 for i in dil_ops if names[i + 1].endswith('.avgpool')]
            line[prec] = dict(dilated_ops=len(dil_ops), kernels=sorted({kinds[i] for i in dil_ops}),
                              dilated_dw_ms=ms(dil_ops), their_pool_ms=ms(pools), dilated_total_ms=ms(dil_ops) + ms(pools),
                              dilated_dw_gb_per_s=gb(dil_ops) / (ms(dil_ops) / 1e3) if ms(dil_ops) else None,
                              undilated_tma_ops=len(und_tma),
                              undilated_tma_gb_per_s=gb(und_tma) / (ms(und_tma) / 1e3) if und_tma and ms(und_tma) else None)
            del eng
            torch.cuda.empty_cache()
        res[f'{size}/os8/batch{batch}'] = line
    return res


def _is_dw(eng, i):
    try:
        eng.op_dw_kernel(i)
        return True
    except Exception:
        return False


def _dilation(eng, i, size):
    """Dilation of depthwise op i, from the stage table (first block din, later blocks dout)."""
    from metrabs_b200.backbones import efficientnet as E
    stages, _ = E.stage_table(size, True, output_stride=8)
    si, bi = (int(v) for v in eng.op_names()[i].split('.')[2:4])
    st = stages[si - 1]
    return st['dilation_in'] if bi == 0 else st['dilation_out']


WORKLOADS = (('l', 32), ('s', 32), ('b0', 32), ('resnet50', 8))


def outputs(args):
    """--outputs: joints of WORKLOADS on the tree this process imports, written to --npz."""
    import numpy as np
    import torch
    import bench
    crops, k = (t.cuda() for t in bench.synthetic(16, 256, seed=0))
    data = {}
    for size, s in WORKLOADS:
        m = build(size, s, 'bf16')
        with torch.inference_mode():
            data[f'{size}@{s}'] = m((crops, k)).cpu().numpy()
        del m
        torch.cuda.empty_cache()
    np.savez(args.npz, **data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--baseline-tree', default=None)
    ap.add_argument('--out', default=None, help='directory for the joints compared with --baseline-tree')
    ap.add_argument('--outputs', action='store_true', help=argparse.SUPPRESS)
    ap.add_argument('--npz', default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.outputs:
        return outputs(args)
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        sys.exit('effnet_stride_step.py measures on the GPU and needs a CUDA device')
    from scripts.latent_step import card
    line = dict(card())
    if args.baseline_tree:
        import numpy as np
        args.out = args.out or tempfile.mkdtemp(prefix='effnet_stride_step_')
        os.makedirs(args.out, exist_ok=True)
        got = {}
        for tag, tree in (('this', ROOT), ('baseline', os.path.abspath(args.baseline_tree))):
            npz = os.path.join(args.out, f'stride32_outputs_{tag}.npz')
            subprocess.run([sys.executable, os.path.abspath(__file__), '--outputs', '--npz', npz], cwd=tree, check=True,
                           env=dict(os.environ, PYTHONPATH=tree))
            got[tag] = np.load(npz)
        line['equal_to_baseline'] = {k: bool(np.array_equal(got['this'][k], got['baseline'][k])) for k in got['this'].files}
    line['dilated_vs_generic'] = dilated_ab(args)
    line['steps'] = timing(args)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
