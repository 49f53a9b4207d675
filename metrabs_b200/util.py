"""Config of the crop-model path.  Mirrors the attribute names the reference reads from its hydra ``get_config()``
singleton (/root/reference/metrabs_pytorch/util.py:41-57, config/config_l.yaml:1-21) with a plain dataclass."""
import dataclasses
from typing import Optional


@dataclasses.dataclass
class Config:
    proc_side: int = 256
    stride_train: int = 32
    stride_test: int = 32
    centered_stride: bool = True
    legacy_centered_stride_bug: bool = False
    backbone: str = 'efficientnetv2-s'
    efficientnet_size: str = 's'
    depth: int = 8
    box_size_mm: float = 2200.0
    weak_perspective: bool = False
    mix_3d_inside_fov: Optional[float] = 0.5
    affine_weights: Optional[str] = None
    transform_coords: bool = False
    predict_all_and_latents: bool = False
    regularize_to_manifold: bool = False
    # build-specific: arithmetic of the conv kernels: 'fp32' and 'tf32x3' (parity modes), 'bf16' (tensor-core throughput
    # mode), 'fp16' (tensor cores, the reference's fp16-autocast arithmetic); 'bf16_simt' / 'fp16_simt' are their CUDA-core
    # verification twins
    precision: str = 'fp32'


_cfg = Config()


def get_config(config_name=None):
    """Same call shape as the reference's get_config(); ``config_name`` may be a YAML path with the reference keys."""
    global _cfg
    if config_name is not None:
        import yaml
        with open(config_name) as f:
            d = yaml.safe_load(f) or {}
        known = {f.name for f in dataclasses.fields(Config)}
        _cfg = Config(**{k: v for k, v in d.items() if k in known})
    return _cfg


def set_config(cfg=None, **kwargs):
    global _cfg
    _cfg = cfg if cfg is not None else dataclasses.replace(_cfg, **kwargs)
    return _cfg
