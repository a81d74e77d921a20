"""Every library entry point that mos_b200/ops.py calls is audited by exactly one launch audit (gemm_audit,
attention_audit, norm_audit, solver_audit) or listed below with the reason it is not, so a kernel added to ops.py later
cannot go unaudited without anyone noticing."""
import pathlib
import re

import attention_audit
import gemm_audit
import norm_audit
import solver_audit

OPS_PY = pathlib.Path(__file__).resolve().parents[1] / 'mix-of-show_b200' / 'mos_b200' / 'ops.py'

EXCLUDED = {}
AUDITS = {'gemm_audit': gemm_audit.Recorder.ENTRY_POINTS, 'attention_audit': attention_audit.ENTRY_POINTS,
          'norm_audit': norm_audit.ENTRY_POINTS, 'solver_audit': solver_audit.ENTRY_POINTS}


def ops_symbols():
    return set(re.findall(r'_lib\.lib\(\)\.(mos_\w+)\(', OPS_PY.read_text()))


def test_ops_symbols_found():
    syms = ops_symbols()
    assert {'mos_gemm_bf16', 'mos_groupnorm_fwd', 'mos_attention_bwd', 'mos_lbfgs_solve_batch'} <= syms, syms


def test_every_ops_symbol_audited_once_or_excluded():
    problems = []
    for s in sorted(ops_symbols()):
        owners = [name for name, eps in AUDITS.items() if s in eps]
        if len(owners) + (s in EXCLUDED) != 1:
            problems.append(f'{s}: audited by {owners or "none"}' + (', and excluded' if s in EXCLUDED else ''))
    assert not problems, '\n'.join(problems)


def test_audits_name_only_real_symbols():
    syms = ops_symbols()
    stale = sorted(set(EXCLUDED).union(*AUDITS.values()) - syms)
    assert not stale, stale
    assert all(EXCLUDED.values())
