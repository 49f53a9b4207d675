"""TEST INFRASTRUCTURE (like oracle/port.py; never imported by metrabs_b200/).

fp16-storage restatement of the EfficientNetV2 crop-model path: oracle/port_bf16.py with its rounding `_q` to
torch.float16 instead of torch.bfloat16, i.e. the roundings of the device's fp16 tensor-core mode (MTB_PRECISION_F16_TC)
at the points where libmetrabs_b200 rounds: fp16-rounded GEMM weights and head weights, fp16 activation storage, fp32
accumulation, SE FCs, logits and decode.  This is the arithmetic the reference deploys under
torch.autocast(dtype=torch.float16) (metrabs_pytorch/multiperson/multiperson_model.py:240-242), to the extent that its
autocast keeps the same tensors in fp16.  Overflow gives inf, as under autocast.

The code is port_bf16's, not a copy: this module loads a private instance of that module and swaps its `_q`, so
oracle/port_bf16 itself (and the tests that monkeypatch it) are untouched."""
import importlib.util

import torch

from oracle import port_bf16 as _bf16_module


def _q(x):
    return x.to(torch.float16).to(torch.float32)


def _load_instance():
    spec = importlib.util.find_spec(_bf16_module.__name__)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod._q = _q
    return mod


_impl = _load_instance()


def effnet_features_f16(sd, spec, image, prefix='backbone.1'):
    return _impl.effnet_features_bf16(sd, spec, image, prefix)


def metrabs_forward_f16(sd, spec, cfg, n_joints, image, intrinsics, stages=None):
    """oracle/port.metrabs_forward with fp16 storage emulated (features fp16, head weights fp16, decode fp32).  With
    `stages`, also records stages['max_abs']: the largest |value| rounded to fp16 anywhere on the path (weights and
    activations), to show how far the fixtures stay from the fp16 limit of 65504."""
    if stages is None:
        return _impl.metrabs_forward_bf16(sd, spec, cfg, n_joints, image, intrinsics)
    peak = [0.0]

    def q_tracked(x):
        peak[0] = max(peak[0], float(x.abs().max()))
        return _q(x)

    _impl._q = q_tracked
    try:
        out = _impl.metrabs_forward_bf16(sd, spec, cfg, n_joints, image, intrinsics, stages=stages)
    finally:
        _impl._q = _q
    stages['max_abs'] = peak[0]
    return out
