"""The GEMM epilogue is compiled once per output path, so a tile runs only the code of its path.

Each 16-bit output path of `gemm_kernel` (rows with or without residual, head-split with V^T groups) and the fp32 path
store a column group through their own compile-time instantiation of `epi_store()`, with constant staging offsets, after
one shared piece of code that adds the bias and LoRA terms.  When every path was a runtime branch inside one unrolled loop
over the 20 column groups, each group recomputed its swizzled staging address and tested every path: the variants held
10,248-13,064 SASS instructions, and writing a tile into the staging tile took 7-12 us on an H100.  The count is only a
proxy: the instructions one tile executes are what matter, and the timeline of tools/gemm_shape_bench.py measures those.
Companion of test_sass_gemm_epilogue.py.
"""
import re

from test_sass_gemm_epilogue import _gemm_kernels

# instruction lines of cuobjdump -sass: "/*0a30*/   HGMMA.64x160x16.F32 ... ;"
_INSN = re.compile(r'/\*[0-9a-f]{4,}\*/\s+\S')

MAX_INSNS = {False: 8_400,      # gemm_kernel<F16, false>
             True: 10_000}      # gemm_kernel<F16, true> (LoRA)


def test_gemm_kernel_size():
    for name, lines in _gemm_kernels().items():
        lora = re.search(r'gemm_kernelILb[01]ELb([01])E', name).group(1) == '1'
        n = sum(bool(_INSN.search(line)) for line in lines)
        assert n <= MAX_INSNS[lora], f'{name}: {n} SASS instructions (bound {MAX_INSNS[lora]})'
