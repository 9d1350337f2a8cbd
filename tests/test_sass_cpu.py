"""CPU: static check of the built library's machine code (cuobjdump -sass, tools/sass_histogram.py) - the hot kernels are written
for Hopper's tensor cores and copy engines, not recompiled legacy paths: warpgroup MMAs (HGMMA), bulk copies (UBLKCP), mbarrier
operations, no mma.sync (HMMA) anywhere; and the fused kernel's issue block of one staged k-block holds exactly its eight
bf16 MMAs, separated only by uniform predicate / descriptor moves, the skip of an empty slot and the register fence before
each MMA - no wgmma wait, barrier or memory access inside the block."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))


@pytest.fixture(scope='module')
def table(built_lib):
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    import sass_histogram as sh
    lib = os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')
    return {name: (dict(zip(sh.COLS, counts)), block, var) for name, _, counts, block, var in sh.rows(lib)}


def test_no_legacy_tensor_core_instructions(table):
    assert table and all(c['HMMA'] == 0 for c, _, _ in table.values())


def test_fused_kernel_is_wgmma_native(table):
    counts, block, var = next(v for k, v in table.items() if 'fused_conv_kernel' in k)
    assert counts['HGMMA'] >= 8 and counts['UBLKCP'] > 0 and counts['SYNCS'] > 0 and counts['REDG'] > 0
    assert block == 8, block                          # the eight MMA slots of one staged k-block, nothing more


def test_streaming_and_gemm_kernels_use_bulk_copies(table):
    tp = next(v for k, v in table.items() if 'tpconv_accumulate_kernel' in k)
    assert tp[0]['UBLKCP'] > 0 and tp[0]['REDG'] > 0 and tp[0]['HGMMA'] == 0        # HBM-bound: no tensor cores by design
    gemm = [v for k, v in table.items() if 'radial_gemm_kernel' in k]
    assert gemm and all(c['HGMMA'] > 0 and c['UBLKCP'] > 0 for c, _, _ in gemm)
