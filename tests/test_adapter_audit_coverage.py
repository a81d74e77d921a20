"""Every library entry point that mos_b200/adapter_ops.py calls is audited by tests/adapter_audit.py, and by no other launch
audit, and no module of mos_b200 besides ops.py (kept in step by test_launch_audit_coverage.py) and adapter_ops.py calls
the library directly, so a kernel added later cannot go unaudited without anyone noticing."""
import pathlib
import re

import adapter_audit
import attention_audit
import gemm_audit
import norm_audit

PKG = pathlib.Path(__file__).resolve().parents[1] / 'mix-of-show_b200' / 'mos_b200'
CALL = re.compile(r'_lib\.lib\(\)\.(mos_\w+)\(')


def symbols(name):
    return set(CALL.findall((PKG / name).read_text()))


def test_adapter_ops_symbols_are_exactly_the_adapter_audit():
    syms = symbols('adapter_ops.py')
    assert {'mos_pixel_unshuffle', 'mos_relu_rows', 'mos_avgpool2x'} <= syms, syms
    assert syms == set(adapter_audit.ENTRY_POINTS)
    from mos_b200 import adapter_ops
    assert all(callable(getattr(adapter_ops, n)) for n in adapter_audit.OPS)


def test_adapter_entry_points_owned_by_one_audit_only():
    others = set(gemm_audit.Recorder.ENTRY_POINTS) | set(attention_audit.ENTRY_POINTS) | set(norm_audit.ENTRY_POINTS)
    assert not set(adapter_audit.ENTRY_POINTS) & others
    assert not set(adapter_audit.ENTRY_POINTS) & symbols('ops.py')


def test_no_other_module_calls_the_library():
    stray = {p.name: CALL.findall(p.read_text()) for p in PKG.glob('*.py') if p.name not in ('ops.py', 'adapter_ops.py')}
    assert not {k: v for k, v in stray.items() if v}, stray
