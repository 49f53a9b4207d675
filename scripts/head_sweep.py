"""Config c5 (head-only isolation, BASELINE.md section 2): roofline sweep of
  (1) the standalone soft-argmax over materialised logits (reference layout [B,D,J,H,W], ptu.soft_argmax) - HBM-bound,
      algorithmic bytes = B*J*D*H*W*sizeof(elt) + 12*B*J  (SURVEY.md 8d);
  (2) the fused head (1x1-conv GEMM on wgmma + soft-argmax epilogue, logits never stored), readings 5a (8x8, D=8) and
      5b (32x32, D=32) of the inconsistent BASELINE.json c5 line: FLOPs 2*B*H*W*C*N, bytes 2*B*H*W*C + 2*C*N + 20*B*J.
Prints one JSON line per point; peaks from MEASURED_PEAKS.json."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
import metrabs_b200  # noqa: E402
from metrabs_b200 import _lib, ptu  # noqa: E402
from metrabs_b200.engine import Engine, make_config  # noqa: E402


def timed(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters / 1e3


def main():
    pk = bench.peaks()
    dev = torch.device('cuda', 0)
    J = 24
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for B in (64, 128, 256, 512, 1024):
            D = H = W = 32
            if B * J * D * H * W * (4 if dtype == torch.float32 else 2) > 8e9:
                continue
            x = (torch.randn(B, D, J, H, W, device=dev) * 4).to(dtype)
            sec = timed(lambda: ptu.soft_argmax(x, dim=(4, 3, 1)))
            nbytes = x.numel() * x.element_size() + 12 * B * J
            print(json.dumps(dict(kernel='softargmax_bdjhw_kernel', dtype=str(dtype).split('.')[-1], B=B, volume='32x32x32',
                                  us=sec * 1e6, GBps=nbytes / sec / 1e9, frac_of_hbm_peak=nbytes / sec / 1e9 / pk['hbm_gbs'],
                                  inputs_mb=nbytes / 1e6)), flush=True)
            del x
    for (hw, D, tag) in ((8, 8, '5a'), (32, 32, '5b')):
        C = 2048
        N = J * (1 + D)
        cfg = metrabs_b200.Config(proc_side=hw * 8, stride_test=8, depth=D, precision='bf16')
        eng = Engine(make_config(cfg, J, arch=_lib.ARCH_HEAD_ONLY, feature_channels=C))
        g = torch.Generator().manual_seed(0)
        eng.load_state_dict({'heatmap_heads.conv_final.weight': torch.randn(N, C, 1, 1, generator=g) * (8 / C ** 0.5),
                             'heatmap_heads.conv_final.bias': torch.zeros(N)})
        for B in (64, 128, 256, 512, 1024):
            if B * hw * hw * C * 2 > 6e9:
                continue
            f = torch.randn(B, hw, hw, C, device=dev).bfloat16()
            sec = timed(lambda: eng.head_decode(f))
            flops = 2.0 * B * hw * hw * C * N
            nbytes = 2.0 * B * hw * hw * C + 2.0 * C * N + 20.0 * B * J
            print(json.dumps(dict(kernel='tc_head_kernel+head_finalize_kernel', reading=tag, B=B, hw=hw, D=D, N=N,
                                  us=sec * 1e6, TFLOPs=flops / sec / 1e12, frac_of_tensor_peak=flops / sec / 1e12 / pk['tflops_burst'],
                                  GBps=nbytes / sec / 1e9, frac_of_hbm_peak=nbytes / sec / 1e9 / pk['hbm_gbs'],
                                  logits_bytes_avoided_mb=B * hw * hw * N * 4 / 1e6)), flush=True)
            del f
        eng.close()


if __name__ == '__main__':
    main()
