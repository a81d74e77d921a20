"""The wgmma GEMM and forward-attention kernels issue their warpgroup MMAs back to back.

ptxas silently serialises every wgmma of a kernel (a `WARPGROUP.DEPBAR` wait after each `HGMMA`) when the kernel holds a
function call (printf, even in a cold path) or a wgmma under a runtime branch.  The kernels then run far below the tensor
core rate while staying correct, so only the SASS shows it.  Companion of test_abi.py::test_sass_is_hopper_native.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_abi import _build


def _functions(sass):
    """cuobjdump -sass text -> {mangled function name: its SASS lines}"""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None:
            out[name].append(line)
    return out


def _longest_hgmma_run(lines):
    """Most HGMMAs issued one after another with no WARPGROUP.DEPBAR (wait) between them."""
    best = run = 0
    for line in lines:
        if 'HGMMA.' in line:
            run += 1
            best = max(best, run)
        elif 'WARPGROUP.DEPBAR' in line:
            run = 0
    return best


def test_wgmma_kernels_are_not_serialised():
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    lib_path = _build()
    sass = subprocess.run([cuobjdump, '-sass', lib_path], capture_output=True, text=True, check=True).stdout
    funcs = _functions(sass)
    # mangled names: mos::gemm_kernel<...> and mos::attn_kernel<...> (not the attn_bwd_* kernels)
    checked = {n: ls for n, ls in funcs.items() if re.search(r'\d+(gemm_kernel|attn_kernel)I', n)}
    assert sum('gemm_kernel' in n for n in checked) >= 2, sorted(funcs)
    assert sum('attn_kernel' in n for n in checked) >= 6, sorted(funcs)
    serialised = [n for n, ls in checked.items() if _longest_hgmma_run(ls) < 2]
    assert not serialised, f'every HGMMA is followed by a WARPGROUP.DEPBAR in: {serialised}'
