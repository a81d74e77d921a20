"""SASS of the forward attention kernels (csrc/attention.cu): register-resident and software-pipelined.

Every attn_kernel instantiation keeps its S / O / P fragments in registers (no local-memory traffic, no stack frame).
In the multi-tile d = 40 kernel, the KV-tile loop runs a tile's exponentials while the previous tile's P V is still on
the tensor cores.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_abi import _build
from test_sass_wgmma import _functions


def _dump(flag):
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    return subprocess.run([cuobjdump, flag, _build()], capture_output=True, text=True, check=True).stdout


def _attn(names):
    return [n for n in names if re.search(r'\d+attn_kernelI', n)]


def test_attention_kernels_have_no_local_memory():
    funcs = _functions(_dump('-sass'))
    kernels = _attn(funcs)
    assert len(kernels) >= 6, sorted(funcs)
    spilling = [n for n in kernels if any(re.search(r'\b(LDL|STL)\b', line) for line in funcs[n])]
    assert not spilling, spilling
    usage = {}
    name = None
    for line in _dump('-res-usage').splitlines():
        m = re.match(r'\s*Function (\S+?):?$', line)
        if m:
            name = m.group(1)
        elif name is not None and 'STACK:' in line:
            usage[name] = int(re.search(r'STACK:(\d+)', line).group(1))
    assert set(kernels) <= set(usage), sorted(usage)
    assert all(usage[n] == 0 for n in kernels), {n: usage[n] for n in kernels}


def test_d40_multi_tile_exponentials_run_under_pv():
    """The KV-tile loop issues the previous tile's P V and runs exponentials before waiting for it: some MUFU.EX2
    follows a P V HGMMA (64x48, A from registers) with no WARPGROUP.DEPBAR between them.  A loop that waits for each
    product before the softmax has none."""
    funcs = _functions(_dump('-sass'))
    d40 = [n for n in _attn(funcs) if 'attn_kernelILi40ELb0E' in n]
    assert len(d40) == 2, sorted(funcs)
    for n in d40:
        pv_in_flight, under = False, 0
        for line in funcs[n]:
            if 'HGMMA.64x48x16' in line:
                pv_in_flight = True
            elif 'WARPGROUP.DEPBAR' in line:
                pv_in_flight = False
            elif 'MUFU.EX2' in line and pv_in_flight:
                under += 1
        assert under >= 16, f'{n}: {under} exponentials issued while a P V wgmma is in flight'
