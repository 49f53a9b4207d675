"""CPU: fmb_kernel's per-chunk path in the built library's SASS (cuobjdump, no GPU needed), for both 16-bit types and
every output width BN2 (32: Cin 16-32, 64: Cin 40-64, 128: Cin 72-96).
- Epilogue-1 writes A2 with shared-memory stores, never generic ST / ST.E stores (a generic store may alias global
  memory, so no global load could be issued ahead of it), and all 16 of its bias1 loads come before its first store.
- GEMM-1 leaves out the k16 steps of the last 64-channel k-chunk that hold only TMA zero fill (Cin 96: 6 of every 8 per
  tap).  Its k-blocks are whole committed groups: one WARPGROUP.ARRIVE, the HGMMAs, one DEPBAR, with no branch between two
  HGMMAs of a group and no HGMMA of ptxas' own.  The short and the full last k-block are two such groups, selected by one
  branch.
- Epilogue-2 issues every bias and residual load before its first global store, at BN2 = 128 too."""
import re

import pytest

from tests.test_sass_epilogue import FMB, opcode, sass

INSTANCES = [(t, bn) for t in ('13__nv_bfloat16', '6__half') for bn in (32, 64, 128)]
IDS = [f'{"bf16" if t.endswith("bfloat16") else "fp16"}_bn{bn}' for t, bn in INSTANCES]
GEMM1 = 'HGMMA.64x128x16'  # GEMM-1's N is always the 128-channel chunk


def kblock_groups(ins):
    """-> one (HGMMA opcodes, branched inside) entry per WARPGROUP.ARRIVE: the wgmmas of one committed group"""
    groups, branch = [], False
    for i in ins:
        o = opcode(i)
        if o == 'WARPGROUP.ARRIVE':
            groups.append([[], False])
            branch = False
        elif groups and o.startswith('HGMMA'):
            groups[-1][0].append(o)
            groups[-1][1] |= branch and len(groups[-1][0]) > 1
            branch = False
        elif o == 'BRA':
            branch = True
    return [(h, b) for h, b in groups if h]


@pytest.mark.parametrize('t,bn', INSTANCES, ids=IDS)
def test_fmb_epilogue1_stores_to_shared_memory_after_its_bias_loads(t, bn):
    ops = [opcode(i) for i in sass(FMB.format(t=t, bn=bn))]
    generic = [o for o in ops if re.fullmatch(r'ST(\.E)?(\.\w+)*', o)]
    assert not generic, f'{len(generic)} generic stores: {sorted(set(generic))}'
    assert sum(o.startswith('STS') for o in ops) >= 16
    first = next(k for k, o in enumerate(ops) if o.startswith('STS'))
    bias1 = sum(o == 'LDG.E.64.CONSTANT' for o in ops[:first])
    assert bias1 == 128 // 8, f'{bias1} of the 16 bias1 loads before the first A2 store'


@pytest.mark.parametrize('t,bn', INSTANCES, ids=IDS)
def test_fmb_gemm1_skips_zero_fill_steps_in_whole_groups(t, bn):
    ins = sass(FMB.format(t=t, bn=bn))
    ops = [opcode(i) for i in ins]
    assert not [o for o in ops if o.startswith('HGMMA') and not o.startswith(('HGMMA.64x128x16', f'HGMMA.64x{bn}x16'))], \
        'an HGMMA of a shape the kernel does not issue (ptxas closing a group of its own)'
    groups = kblock_groups(ins)
    split = [h for h, b in groups if b]
    assert not split, f'{len(split)} groups with a branch between their HGMMAs'
    sizes = sorted({len(h) for h, _ in groups if all(o.startswith(GEMM1) for o in h) and len(h) <= 4})
    # the last k-chunk's k-block in both forms (BN2 = 32: 1 / 2 steps, 64: 3 / 4, 128: 1 / 2), and at BN2 = 128 the full
    # first k-chunk's 4
    want = {32: [1, 2], 64: [3, 4], 128: [1, 2, 4]}[bn]
    assert sizes == want, f'GEMM-1 groups of {sizes} HGMMAs, want {want}'
    waits = [i for i in ins if opcode(i) == 'WARPGROUP.DEPBAR.LE']
    assert any(re.search(r'gsb0,\s*0x1\b', i) for i in waits), 'no k-block waits with one group in flight'


@pytest.mark.parametrize('t', ['13__nv_bfloat16', '6__half'], ids=['bf16', 'fp16'])
def test_fmb_epilogue2_loads_before_its_first_store_at_bn128(t):
    ops = [opcode(i) for i in sass(FMB.format(t=t, bn=128))]
    first = next(k for k, o in enumerate(ops) if o.startswith('STG'))
    late = [o for o in ops[first:] if o.startswith('LDG')]
    assert not late, f'{len(late)} global loads after the first global store: {sorted(set(late))}'
