"""CPU: host-side tiling logic of the CUDA kernels (no device needed)."""
import ctypes as C
import os

import pytest

from metrabs_b200 import _lib


def _plan(h, w):
    g, bh, nrb, sb = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    rc = _lib.lib().mtb_debug_dw_plan(h, w, C.byref(g), C.byref(bh), C.byref(nrb), C.byref(sb))
    assert rc == 0
    return g.value, bh.value, nrb.value, sb.value


@pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason='libmetrabs_b200.so not built')
def test_depthwise_tma_plan_covers_the_map_within_the_shared_memory_budget():
    """dw3x3s1_tma_kernel (csrc/dw_tma.cuh): every HxW map either gets a plan whose row bands cover all rows, whose stage
    fits the 52 KB budget (2 stages x 2 CTAs per SM) and whose pooling slices fit the engine's 8 slots, or no plan."""
    for h in list(range(1, 40)) + [48, 56, 64, 96, 112, 128, 192]:
        for w in sorted({h, max(1, h // 2), h + 3, 2 * h}):
            g, bh, nrb, sb = _plan(h, w)
            if g == 0:
                assert (w + 2) * 128 * (4 + 2) > 52 * 1024 or w + 2 > 256, (h, w)  # only maps too wide for one 4-row band
                continue
            assert 1 <= g <= 8 and 1 <= bh <= h
            assert nrb * bh >= h and (nrb - 1) * bh < h          # bands tile the rows exactly once
            assert sb == 128 * (w + 2) * (bh + 2) * g and sb <= 52 * 1024
            assert g == 1 or nrb == 1                              # crops are grouped only when an item holds whole crops
    # the shapes of the benchmark configs: EfficientNetV2 @256 (16x16, 8x8) and @384 (24x24, 12x12)
    assert _plan(16, 16)[:3] == (1, 16, 1)
    assert _plan(8, 8)[:3] == (4, 8, 1)
    assert _plan(12, 12)[1:3] == (12, 1)
    g, bh, nrb, _ = _plan(24, 24)
    assert g == 1 and nrb * bh >= 24 and nrb <= 8
