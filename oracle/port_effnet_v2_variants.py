"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of EfficientNetV2-B0..B3 and EfficientNetV2-XL, the TF reference's
``efficientnetv2-b0`` .. ``-b3`` and ``efficientnetv2-xl`` (``metrabs_tf/backbones/efficientnet/effnetv2_configs.py``
:145-152, :240-248, :249-282, built by ``effnetv2_model.py``).

* Tables: ``v2_base_block`` scaled by the variant's (width, depth) and ``v2_xl_block`` at (1.0, 1.0), with TF's rules
  (effnetv2_model.py:76-94): channels ``round_filters`` (nearest multiple of 8, at least 8, without torchvision's 0.9
  rule), layers ``round_repeats`` (ceil), stem ``round_filters(32)`` (:446, the first row's cin), head
  ``round_filters(1280)`` (:479).  The ``_br`` row (the last strided stage) takes the bottom-right shift under
  ``centered_stride``.
* Blocks: the V2 grammar of ``oracle/port.py`` (FusedMBConv rows, MBConv rows with SE width ``cin // 4``, BatchNorm eps
  1e-3), so the spec is a ``port.EffNetSpec`` and ``port.effnet_features``, ``port.make_effnet_state_dict`` and
  ``port_ops.effnet_op_table`` / ``layer_bound`` apply as they are.

Parity pin: the TF model cannot run without TensorFlow, so ``oracle/gen_golden_effnet_v2_variants.py`` builds the
reference's PyTorch ``EfficientNet`` (``metrabs_pytorch/backbones/efficientnet.py`` :238-330) from ``FusedMBConvConfig`` /
``MBConvConfig`` rows with these channels and ``last_channel``, and commits its outputs under
``tests/golden/effnetv2{b0,b3,xl}_*.npz``; ``tests/test_oracle_effnet_v2_variants.py`` checks this restatement against
those files and the tables against the TF block strings.
"""
import math

from oracle import port

# (block, expand, kernel, stride, cin, cout, layers, bottom-right shift on this row under centered_stride)
V2_BASE = [('fused', 1, 3, 1, 32, 16, 1, False), ('fused', 4, 3, 2, 16, 32, 2, False),
           ('fused', 4, 3, 2, 32, 48, 2, False), ('mb', 4, 3, 2, 48, 96, 3, False), ('mb', 6, 3, 1, 96, 112, 5, False),
           ('mb', 6, 3, 2, 112, 192, 8, True)]
V2_XL = [('fused', 1, 3, 1, 32, 32, 4, False), ('fused', 4, 3, 2, 32, 64, 8, False), ('fused', 4, 3, 2, 64, 96, 8, False),
         ('mb', 4, 3, 2, 96, 192, 16, False), ('mb', 6, 3, 1, 192, 256, 24, False), ('mb', 6, 3, 2, 256, 512, 32, True),
         ('mb', 6, 3, 1, 512, 640, 8, False)]
# name -> (base rows, width, depth)  (effnetv2_configs.py:266-281)
VARIANTS = {'efficientnetv2-b0': (V2_BASE, 1.0, 1.0), 'efficientnetv2-b1': (V2_BASE, 1.0, 1.1),
            'efficientnetv2-b2': (V2_BASE, 1.1, 1.2), 'efficientnetv2-b3': (V2_BASE, 1.2, 1.4),
            'efficientnetv2-xl': (V2_XL, 1.0, 1.0)}


def round_filters(filters, width, divisor=8):
    """effnetv2_model.py:76-87 (min_depth = divisor)."""
    return max(divisor, int(filters * width + divisor / 2) // divisor * divisor)


def round_repeats(repeats, depth):
    """effnetv2_model.py:90-94."""
    return int(math.ceil(depth * repeats))


def effnet_spec(name, centered_stride=True):
    """'efficientnetv2-b0' .. 'efficientnetv2-b3', 'efficientnetv2-xl' -> port.EffNetSpec."""
    rows, width, depth = VARIANTS[name]
    stages = [port.StageSpec(b, e, k, s, round_filters(ci, width), round_filters(co, width), round_repeats(n, depth),
                             bool(br and centered_stride))
              for b, e, k, s, ci, co, n, br in rows]
    return port.EffNetSpec(name, stages, round_filters(1280, width))


def identity_fused_blocks(spec):
    """(Cin, Cexp) of the stride-1 FusedMBConv blocks with Cin = Cout and an expand conv: the blocks fmb_kernel runs."""
    return sorted({(b['cin'], b['cin'] * b['expand']) for b in port.effnet_block_list(spec)
                   if b['block'] == 'fused' and b['expand'] != 1 and b['stride'] == 1 and b['cin'] == b['cout']})
