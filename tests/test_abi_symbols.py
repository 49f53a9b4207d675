"""CPU: libmetrabs_b200.so loads (no GPU needed) and exports every function include/metrabs_b200.h declares; the ctypes
binding covers the same set; compute entry points fail loudly without a device instead of falling back."""
import ctypes
import os
import re

import pytest
import torch

from metrabs_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(mtb_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libmetrabs_b200.so not built (run __graft_entry__.build())')
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = declared_functions()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert set(_lib.EXPORTED_SYMBOLS) == set(names)
    assert lib.mtb_version is not None


def test_kernel_values_match_the_header():
    """every value of the header's mtb_kernel enum has its _lib twin of the same name, numbered 0, 1, ... in order"""
    src = open(os.path.join(ROOT, 'include', 'metrabs_b200.h')).read()
    body = re.sub(r'/\*.*?\*/', '', re.search(r'typedef enum \{([^}]*)\} mtb_kernel;', src, re.S).group(1), flags=re.S)
    values = {}
    for name, expr in re.findall(r'MTB_([A-Z0-9_]+) = ([^,]+)', body):
        values[name] = eval(re.sub(r'MTB_([A-Z0-9_]+)', lambda m: str(values[m.group(1)]), expr.strip()))
    assert list(values.values()) == list(range(23)), values
    assert {k: getattr(_lib, k, None) for k in values} == values


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU behaviour')
def test_no_cpu_fallback():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libmetrabs_b200.so not built')
    import metrabs_b200
    from metrabs_b200.engine import Engine, make_config
    from metrabs_b200.backbones.efficientnet import stage_table
    stages, last = stage_table('tiny', True)
    with pytest.raises(_lib.MetrabsB200Error, match='no CUDA device'):
        Engine(make_config(metrabs_b200.Config(proc_side=64), 8, stages=stages, last_channel=last))
    from metrabs_b200 import ptu
    with pytest.raises(_lib.MetrabsB200Error):
        ptu.soft_argmax(torch.zeros(1, 2, 3, 4, 4), dim=(4, 3, 1))
