"""CPU: the tensor-core epilogues of the built library issue their global loads in batches, not one behind each store.

Read from the SASS of libmetrabs_b200.so (cuobjdump, no GPU needed):
- tc_conv_kernel<bf16, SiLU, 0, 128> (the MBConv expand GEMMs) and <bf16, NONE, 1, 128> (the projections with a
  residual) write their staging tile with shared-memory stores, never generic ST.E stores (a generic store may alias
  global memory, so no later load can be issued ahead of it).
- The expand GEMM loads each bias pair once per tile: at most BN / 8 = 16 LDG.E.64.CONSTANT per thread, not one per row
  group and column (64).  (At BN = 128 with a residual the bias pairs are loaded at their use, see tc_tile_epilogue.)
- fmb_kernel's epilogue-2 issues every bias and residual load before its first global store (BN2 = 32, 64: the widths
  of every EfficientNetV2 FusedMBConv block up to 64 channels)."""
import os
import re
import shutil
import subprocess

import pytest

from metrabs_b200 import _lib

CUDA_BIN = '/usr/local/cuda/bin'
TC = '_ZN3mtb14tc_conv_kernelI13__nv_bfloat16Li{act}ELi{res}ELi128ELb0EEEv14CUtensorMap_stS2_S2_NS_12TcConvParamsEPKf'
FMB = '_ZN3mtb10fmb_kernelI{t}Li{bn}EEEv14CUtensorMap_stS2_S2_NS_9FmbParamsE'


def cuobjdump():
    exe = shutil.which('cuobjdump') or os.path.join(CUDA_BIN, 'cuobjdump')
    return exe if os.access(exe, os.X_OK) else None


def sass(fun):
    """-> the SASS instructions of kernel `fun` (mangled name), one per list item"""
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libmetrabs_b200.so not built (run __graft_entry__.build())')
    exe = cuobjdump()
    if exe is None:
        pytest.skip('cuobjdump not found')
    out = subprocess.run([exe, '-sass', '-fun', fun, _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    ins = re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', out)
    assert ins, f'no SASS for {fun}'
    return ins


def opcode(i):
    """'@!P0 LDG.E.64.CONSTANT R2, desc[..]' -> 'LDG.E.64.CONSTANT'"""
    return re.sub(r'^@!?U?P\w+\s+', '', i).split()[0]


@pytest.mark.parametrize('act,res', [(1, 0), (0, 1)], ids=['silu_expand', 'residual_projection'])
def test_tc_conv_epilogue_stages_through_shared_memory(act, res):
    ops = [opcode(i) for i in sass(TC.format(act=act, res=res))]
    generic = [o for o in ops if re.fullmatch(r'ST(\.E)?(\.\w+)*', o)]
    assert not generic, f'{len(generic)} generic stores: {sorted(set(generic))}'
    assert sum(o.startswith('STS') for o in ops) >= 16
    if res == 0:
        bias = sum(o == 'LDG.E.64.CONSTANT' for o in ops)
        assert 0 < bias <= 128 // 8, f'{bias} bias loads per thread'


@pytest.mark.parametrize('t,bn', [('13__nv_bfloat16', 64), ('13__nv_bfloat16', 32), ('6__half', 64)])
def test_fmb_epilogue2_loads_before_its_first_store(t, bn):
    ops = [opcode(i) for i in sass(FMB.format(t=t, bn=bn))]
    first = next(k for k, o in enumerate(ops) if o.startswith('STG'))
    late = [o for o in ops[first:] if o.startswith('LDG')]
    assert not late, f'{len(late)} global loads after the first global store: {sorted(set(late))}'
