"""The wgmma GEMM writes its 16-bit output through a shared-memory staging tile.

The epilogue of `gemm_kernel` stages the output tile in shared memory.  Row output (over the residual the producer warp
prefetched into it) is written out by the producer with `cp.async.bulk.tensor` stores, head-split output by the consumers
in 16-byte chunks.  Without this the consumer warps store to
global memory straight from registers, each residual load waiting for the store before it (the two may alias), which
is correct but slow, so only the SASS shows the difference.  Companion of test_sass_wgmma.py.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_abi import _build
from test_sass_wgmma import _functions


def _gemm_kernels():
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([cuobjdump, '-sass', _build()], capture_output=True, text=True, check=True).stdout
    kernels = {n: ls for n, ls in _functions(sass).items() if re.search(r'\d+gemm_kernelI', n)}
    assert len(kernels) == 4, sorted(kernels)       # {bf16, fp16} x {plain, LoRA}
    return kernels


def test_every_gemm_kernel_issues_tma_stores():
    missing = [n for n, ls in _gemm_kernels().items() if not any('UTMASTG' in line for line in ls)]
    assert not missing, f'no TMA store (UTMASTG) in: {missing}'


def test_16bit_output_is_not_stored_element_by_element():
    # head-split output (Q/K rows and V^T) is copied out of the staging tile in 16-byte chunks; the one 2-byte store
    # left is the element-wise copy of a chunk whose destination is not contiguous (V^T tokens across a batch boundary
    # at a token count that is not a multiple of 8, or unaligned row output).  The register epilogue had 80.
    for n, ls in _gemm_kernels().items():
        u16 = sum('STG.E.U16' in line for line in ls)
        v128 = sum('STG.E.128' in line for line in ls)
        assert u16 <= 1 and v128 >= 1, f'{n}: {u16} STG.E.U16, {v128} STG.E.128'


def test_epilogue_operands_are_loaded_once_per_tile():
    # bias, per-batch bias and the LoRA up rows are staged in shared memory before the tile's first store, so the
    # epilogue loads them with a handful of instructions per tile instead of one load per output column pair.  What is
    # left: the producer's L2 prefetch, the split-K finalize, and the residual pairs of row output whose residual TMA
    # cannot address (40 loads).  The register epilogue had 415 (560 with LoRA).
    for n, ls in _gemm_kernels().items():
        ldg = sum(bool(re.search(r'\bLDG\.', line)) for line in ls)
        assert ldg <= 128, f'{n}: {ldg} global loads'
