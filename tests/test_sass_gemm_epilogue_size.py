"""In the denoise step every GEMM launch follows other kernels and starts from a cold instruction cache, so the kernel's
code size costs time.  The thread's two tile rows share one copy of the epilogue (a rolled row loop, accumulator registers
picked by selects), which keeps every gemm_kernel variant under 7,000 SASS instructions; with the row loop unrolled the
variants held 7,744-9,432 and the step's GEMM launches took 5.0 ms instead of 4.65 ms on an H100 (700 W).  Companion of
test_sass_gemm_size.py.
"""
import re

from test_sass_gemm_epilogue import _gemm_kernels

_INSN = re.compile(r'/\*[0-9a-f]{4,}\*/\s+\S')
_LOCAL = re.compile(r'\b(LDL|STL)\b')


def test_gemm_kernel_epilogue_rolled():
    for name, lines in _gemm_kernels().items():
        n = sum(bool(_INSN.search(line)) for line in lines)
        assert n <= 7_000, f'{name}: {n} SASS instructions (bound 7,000)'
        assert not any(_LOCAL.search(line) for line in lines), f'{name}: local-memory access'
