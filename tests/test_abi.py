"""The C-ABI shared library loads on a CPU-only box and exports every symbol include/mos_sm100.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    import __graft_entry__ as g
    return g.build()


def test_library_builds_loads_and_exports_header_symbols():
    lib_path = _build()
    lib = ctypes.CDLL(lib_path)
    header = open(os.path.join(ROOT, 'include', 'mos_sm100.h')).read()
    header = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
    names = set(re.findall(r'\b(mos_[a-z0-9_]+)\s*\(', header))
    assert len(names) >= 15
    for n in sorted(names):
        assert hasattr(lib, n), f'{n} declared in include/mos_sm100.h but not exported'
    lib.mos_version.restype = ctypes.c_int
    assert lib.mos_version() >= 100
    lib.mos_last_error.restype = ctypes.c_char_p
    assert isinstance(lib.mos_last_error(), bytes)


def test_argument_validation_without_gpu():
    """Validation happens before any CUDA call, so the error channel can be exercised on CPU."""
    from mos_b200 import _lib
    lib = _lib.lib()
    a = _lib.GemmArgs()
    rc = lib.mos_gemm_bf16(ctypes.byref(a), None)
    assert rc == -1 and b'NULL' in lib.mos_last_error()
    rc = lib.mos_attention_fwd(None, None, None, None, ctypes.c_int64(0), None, 1, 8, 40, 1, 1, 8, ctypes.c_float(1), 0, None)
    assert rc == -1
    # the activation dtype is validated too (MOS_DT_BF16 = 0 / MOS_DT_F16 = 1)
    rc = lib.mos_layernorm_fwd(ctypes.c_void_p(16), ctypes.c_int64(8), ctypes.c_int64(1), 8, ctypes.c_void_p(16), ctypes.c_void_p(16),
                               ctypes.c_float(1e-5), ctypes.c_void_p(16), ctypes.c_int64(8), 7, None)
    assert rc == -1 and b'act_dtype' in lib.mos_last_error()


def test_sass_is_hopper_native():
    """SASS of the built library must contain sm_90a warpgroup MMAs (HGMMA) and TMA (UTMALDG)."""
    import shutil
    import subprocess
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip('cuobjdump not available')
    lib_path = _build()
    sass = subprocess.run([cuobjdump, '-sass', lib_path], capture_output=True, text=True).stdout
    assert 'arch = sm_90a' in sass and 'HGMMA' in sass and 'UTMALDG' in sass
    assert 'HMMA.' not in sass, 'legacy mma.sync path found'
