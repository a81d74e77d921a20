"""Every library entry point that mos_b200/ops.py calls is audited by exactly one launch audit (gemm_audit,
attention_audit, norm_audit) or listed below with the reason it is not, so a kernel added to ops.py later cannot go
unaudited without anyone noticing."""
import pathlib
import re

import attention_audit
import gemm_audit
import norm_audit

OPS_PY = pathlib.Path(__file__).resolve().parents[1] / 'mix-of-show_b200' / 'mos_b200' / 'ops.py'

_SOLVER = 'gradient-fusion solver (fusion.cu / lbfgs.cu): fp32 / fp64 solver arithmetic, audited on its own'
EXCLUDED = {
    'mos_transpose_bf16': _SOLVER,
    'mos_gram_small': _SOLVER,
    'mos_atb_small': _SOLVER,
    'mos_sgemm_nn': _SOLVER,
    'mos_dgemm_mixed': _SOLVER,
    'mos_ls_grad_loss': _SOLVER,
    'mos_vec_dot': _SOLVER,
    'mos_vec_asum': _SOLVER,
    'mos_vec_absmax': _SOLVER,
    'mos_vec_axpby': _SOLVER,
    'mos_lbfgs_direction': _SOLVER,
    'mos_lbfgs_solve_batch': _SOLVER,
    'mos_lora_merge': _SOLVER,
}
AUDITS = {'gemm_audit': gemm_audit.Recorder.ENTRY_POINTS, 'attention_audit': attention_audit.ENTRY_POINTS,
          'norm_audit': norm_audit.ENTRY_POINTS}


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
