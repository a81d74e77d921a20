"""Launch audit of the gradient-fusion solver kernels (csrc/fusion.cu, csrc/lbfgs.cu): every call of an entry point in
ENTRY_POINTS made through its `ops.*` wrapper in a real fusion walk, checked on its own.

These kernels produce what gradient fusion writes to disk: the fused weights.  A wrong one fails silently (sampling
still makes images, just worse ones), so each launch is compared with a float64 reference of the same operation.

Records are built as in norm_audit.py from the arguments that reach the `mos_*` entry point: every pointer is mapped
into the storage of a tensor argument of the `ops.*` call (the history vectors of lbfgs_direction and the problems of
lbfgs_solve_batch are tensor arguments too), and each operand window is read there at the layout the kernel uses.  The
rows of the lora_merge table point into tensors that only the caller holds (the state-dict copies and the `_merged`
temporaries): they are resolved against the tensors registered with the recorder.

Element bounds (a).  u = 2^-24 (fp32), u64 = 2^-53.  An fp32 (fp64) sum of n terms in any order errs by at most
(n - 1) u sum |terms|; the constants below add the products and the final roundings.  For the fp64 kernels the float64
reference rounds as well, so their bounds cover both sides (2 gamma).
- transpose_bf16: bit-exact, out[c, r] = x[r, c] for c < C, r < rows at pitch ldo; the pad columns [rows, ldo) are
  outside the window and must stay unchanged (c).  Preconditions: ldx >= C, ldo >= rows.
- gram_small, atb_small: n products summed per element: (n + 2) u sum_r |x_ri| |y_rj|, plus u |result| when accumulating.
- sgemm_nn: (K + 2) u |alpha| sum_k |a_ik| |b_kj| + 2u |beta c|.  With beta = 0 the kernel must not read C: the recorder
  fills C with NaN before such a launch, so a read shows up as NaN in (a).
- dgemm_mixed: fp32 -> fp64 is exact, so 2 (K + 2) u64 sum |a| |b|.  A product accumulated in fp32 errs by ~K u and
  breaks it by nine orders of magnitude.
- ls_grad_loss: grad = 2 s (y - c) in fp64, then one fp32 rounding: u |grad| + 4 u64 2s (|y| + |c|); loss = s sum w (y -
  2c) + f0 over n fp64 terms: 2 (n + 4) u64 s sum |w| |y - 2c| + u64 |f0|.
- vec_dot, vec_asum: 256 x 256 threads; each sums ceil(n / 65536) terms, then 5 + 3 tree levels in the block and 8 over
  the 256 partials: (ceil(n / 65536) + 16) u sum |terms| (the product's own rounding included).
- vec_absmax: max |fl(scale a)|: u |result|; NaN exactly where the reference is NaN (torch's abs().max() propagates it).
- vec_axpby: alpha x + beta y, two products and an add: 2u (|alpha x| + |beta y|).  With beta = 0, y is poisoned with NaN
  first (unless x aliases y), as for sgemm.
- lbfgs_direction: a float64 two-loop recursion from the same S, Y, rho (as passed) and h_diag (fp32, as passed), with a
  first-order error bound e (per element of v) carried alongside it through the 2k + 1 steps: each dot <h, v> errs by
  sum |h| e + gamma_dot sum |h| |v| (gamma_dot the vec_dot constant above); its coefficient (al = dot rho, then -al or
  al - be, cast to fp32) by |rho| times that plus 2u |coefficient| (the kernel and the reference round two different
  float64 values to fp32, one u each); each update v + c h (one fma) adds |h| e_c + u |v + c h| to e; the h_diag scaling multiplies e by |h_diag| and adds u |h_diag v|.  gtd is the last dot.  No fixed
  tolerance.  Being worst case in every dot, the bound grows geometrically with k (each step multiplies it by about
  1 + rho sum |s| |y|, ~1.6 for random pairs): 3e-6 |d| at k = 1, 2e-5 at k = 3, 1e-3 at k = 7, and at k = 25 it only
  guards against gross faults; test_fusion_gpu.py holds deep histories to the host-driven recursion bit for bit.
  Window: d, work[0..k] and partial[0..255] as scratch, gtd[0]; partial[256] (the block counter) is zero on entry (p)
  and, being outside the window, must be zero again on exit (c).
- lora_merge: W + alpha up @ down per table row: (rank + 2) u |alpha| sum_r |up_or| |down_ri| + u |W'|.  A 4-D 1x1-conv
  weight is the same [out, in] rows.
- lbfgs_solve_batch: the solve level.  (i) each best_D is bit-identical to gradient_fusion.lbfgs_minimize (the Python
  driver, whose launches this audit checks one by one) run through the same library on the snapshotted G, R, s, f0;
  (ii) the returned best_loss equals f(best_D) = s <D, D G - 2 R> + f0 recomputed in float64 within 2 (in + out in +
  8) u64 s sum |D| (|D| |G| + 2 |R|) + 2 u64 |f0|; (iii) f(best_D) <= f0 within that bound.  Only each problem's best_D
  is written (c), G and R stay unchanged (d), and a relaunch is bit-identical with the walk's worker count (e) and with
  one worker.
The bounds grow with magnitudes, not with the values; a ratio above 1 is a finding, not a reason to widen them.

Checks of every launch (`check_launch`): (p) the preconditions above; (a) the element bound, the bit-exact outputs bit for
bit; (b) the rel-L2 of each output against its reference is reported (the table's worst rel-L2); (c) every element of a
written storage outside the launch's window is bitwise unchanged.  The recorder (gemm_audit.LaunchRecorder) adds (d)
unchanged operands and (e) a bit-identical relaunch.
"""
import contextlib
import ctypes
import os
import re

import torch

import gemm_audit as ga
from gemm_audit import Stats, _Storages  # noqa: F401  (the table and storage map of every audit)

U32 = 2.0 ** -24
U64 = 2.0 ** -53
F32, F64, BF = torch.float32, torch.float64, torch.bfloat16
RED_THREADS = 256 * 256                 # RED_BLOCKS x 256 threads of the fusion.cu reductions
RED_LEVELS = 16                         # 5 + 3 tree levels in a block, 8 over the 256 partials
_BITS = ga._BITS

# --------------------------------------------------------------------------------------------------- ABI tables
_ARGS = {
    'mos_transpose_bf16': ('x', 'ldx', 'rows', 'C', 'out', 'ldo'),
    'mos_gram_small': ('X', 'n', 'd', 'G', 'accumulate'),
    'mos_atb_small': ('X', 'Y', 'n', 'dx', 'dy', 'out', 'accumulate'),
    'mos_sgemm_nn': ('A', 'B', 'C', 'M', 'N', 'K', 'alpha', 'beta'),
    'mos_dgemm_mixed': ('A', 'B', 'C', 'M', 'N', 'K'),
    'mos_ls_grad_loss': ('W', 'Y', 'Cm', 'n', 's', 'f0', 'grad', 'loss', 'scratch'),
    'mos_vec_dot': ('a', 'b', 'n', 'out', 'scratch'),
    'mos_vec_asum': ('a', 'n', 'out', 'scratch'),
    'mos_vec_absmax': ('a', 'n', 'scale', 'out', 'scratch'),
    'mos_vec_axpby': ('y', 'x', 'alpha', 'beta', 'n'),
    'mos_lbfgs_direction': ('S', 'Y', 'rho', 'k', 'g', 'h_diag', 'n', 'd', 'work', 'partial', 'gtd'),
    'mos_lbfgs_solve_batch': ('probs', 'n_probs', 'workers'),
    'mos_lora_merge': ('table', 'n_layers', 'alpha'),
}
ENTRY_POINTS = tuple(_ARGS)
_FLOATS = ('alpha', 'beta', 's', 'f0', 'scale', 'h_diag')
_PROBLEM = ('G', 'R', 'out_f', 'in_f', 's', 'f0', 'max_iter', 'history', 'best_D')


def abi_of(entry, args):
    """the ctypes arguments of an entry point -> plain dict (pointers as ints, 0 for NULL; floats as passed; the host
    arrays of lbfgs_direction as lists; the problems of lbfgs_solve_batch as dicts, with `_ct` the ctypes array)"""
    a = {}
    for n, v in zip(_ARGS[entry], args):
        if n == 'probs':
            continue
        if hasattr(v, '_length_'):
            a[n] = [float(e) if n == 'rho' else int(e or 0) for e in v]
            continue
        v = getattr(v, 'value', v)
        a[n] = float(v) if n in _FLOATS else (0 if v is None else int(v))
    if entry == 'mos_lbfgs_direction':
        a['S'], a['Y'], a['rho'] = a['S'][:a['k']], a['Y'][:a['k']], a['rho'][:a['k']]
    if entry == 'mos_lbfgs_solve_batch':
        a['probs'] = [{f: (getattr(p, f) or 0) if f in ('G', 'R', 'best_D') else getattr(p, f) for f in _PROBLEM}
                      for p in list(args[0])[:a['n_probs']]]
        a['_ct'] = args[0]
    return a


# --------------------------------------------------------------------------------------------------- host rules
def dgemm_tile(env=None):
    """the CTA tile of a mos_dgemm_mixed launch: a copy of the host rule in csrc/fusion.cu (MOS_DGEMM_TILE, read once per
    process with atoi: unset or 0 = 64 x 64, 1 = 32 x 64, 2 = 64 x 64, any other value 64 x 128); keep the two in step"""
    e = os.environ.get('MOS_DGEMM_TILE') if env is None else env
    m = re.match(r'\s*[+-]?\d+', e or '')
    v = int(m.group()) if m else 0
    return {0: '64x64', 1: '32x64', 2: '64x64'}.get(v, '64x128')


def solver_path(rec):
    """Path key of a launch: the features that select code or a loop tail in csrc/fusion.cu / lbfgs.cu"""
    e, a = rec['op'], rec['abi']
    if e == 'mos_transpose_bf16':
        return 'transpose_bf16' + ('|rtail' if a['rows'] % 32 else '') + ('|ctail' if a['C'] % 32 else '') + \
            ('|strided' if a['ldx'] != a['C'] else '')
    if e in ('mos_gram_small', 'mos_atb_small'):
        return e[4:] + ('|ntail' if a['n'] % 16 else '') + ('|acc' if a['accumulate'] else '')
    if e == 'mos_sgemm_nn':
        return 'sgemm_nn' + ('|beta0' if a['beta'] == 0 else '|beta')
    if e == 'mos_dgemm_mixed':
        return f'dgemm_mixed|{dgemm_tile()}'
    if e == 'mos_vec_absmax':
        return 'vec_absmax' + ('|scaled' if a['scale'] != 1.0 else '')
    if e == 'mos_vec_axpby':
        return 'vec_axpby|' + ('beta0' if a['beta'] == 0 else 'beta1' if a['beta'] == 1 else 'beta')
    if e == 'mos_lbfgs_direction':
        k = a['k']
        return 'lbfgs_direction|' + ('k=0' if k == 0 else 'k=25' if k == 25 else 'k<25')
    if e == 'mos_lbfgs_solve_batch':
        return f"lbfgs_solve_batch|workers={min(a['workers'], a['n_probs'])}"
    return e[4:]


# --------------------------------------------------------------------------------------------------- records
def _overlap(S, p0, n0, p1, n1):
    return S.find(p0, 'a')[0] == S.find(p1, 'b')[0] and p0 < p1 + n1 and p1 < p0 + n0


def record(entry, a, S):
    """the launch record of one entry-point call (operand windows and written storages still live).  rec['poison']:
    output windows the recorder fills with NaN before the launch (outputs the kernel must not read)"""
    x, targets, pre, inplace, poison = {}, [], [], [], []

    def win(name, dtype, size, stride, p=None, table=False):
        x[name] = S.window(a[name] if p is None else p, name, dtype, size, stride, table=table)
        return x[name]

    def target(name, dtype, size, stride, p=None, scratch=False, table=False):
        base, off = S.find(a[name] if p is None else p, name, table=table)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{name}: pointer not aligned to its element size'
        t = dict(name=name, mem=(base, dtype), off=off // es, size=tuple(size), stride=tuple(stride), scratch=scratch)
        S.flat(base, dtype).as_strided(t['size'], t['stride'], t['off'])     # raises if it runs past its storage
        targets.append(t)
        return t

    if entry == 'mos_transpose_bf16':
        rows, C = a['rows'], a['C']
        if a['ldx'] < C:
            pre.append(f"(p) ldx {a['ldx']} < C {C}")
        if a['ldo'] < rows:
            pre.append(f"(p) ldo {a['ldo']} < rows {rows}")
        win('x', BF, (rows, C), (a['ldx'], 1))
        target('out', BF, (C, rows), (a['ldo'], 1))
    elif entry in ('mos_gram_small', 'mos_atb_small'):
        n = a['n']
        if entry == 'mos_gram_small':
            dx = dy = a['d']
            win('X', F32, (n, dx), (dx, 1))
            x['Y'] = x['X']
            out = 'G'
        else:
            dx, dy = a['dx'], a['dy']
            win('X', F32, (n, dx), (dx, 1))
            win('Y', F32, (n, dy), (dy, 1))
            out = 'out'
        target(out, F32, (dx, dy), (dy, 1))
        if a['accumulate']:
            win(out, F32, (dx, dy), (dy, 1))
            inplace.append(out)
    elif entry == 'mos_sgemm_nn':
        M, N, K = a['M'], a['N'], a['K']
        win('A', F32, (M, K), (K, 1))
        win('B', F32, (K, N), (N, 1))
        t = target('C', F32, (M, N), (N, 1))
        if a['beta'] != 0:
            win('C', F32, (M, N), (N, 1))
            inplace.append('C')
        else:
            poison.append(t)
    elif entry == 'mos_dgemm_mixed':
        M, N, K = a['M'], a['N'], a['K']
        win('A', F32, (M, K), (K, 1))
        win('B', F64, (K, N), (N, 1))
        target('C', F64, (M, N), (N, 1))
    elif entry == 'mos_ls_grad_loss':
        n = a['n']
        win('W', F32, (n,), (1,))
        win('Y', F64, (n,), (1,))
        win('Cm', F64, (n,), (1,))
        target('grad', F32, (n,), (1,))
        target('loss', F64, (1,), (1,))
        target('scratch', F64, (256,), (1,), scratch=True)
    elif entry in ('mos_vec_dot', 'mos_vec_asum', 'mos_vec_absmax'):
        n = a['n']
        win('a', F32, (n,), (1,))
        if entry == 'mos_vec_dot':
            win('b', F32, (n,), (1,))
        target('out', F32, (1,), (1,))
        target('scratch', F32, (256,), (1,), scratch=True)
    elif entry == 'mos_vec_axpby':
        n = a['n']
        win('x', F32, (n,), (1,))
        t = target('y', F32, (n,), (1,))
        if a['beta'] != 0:
            win('y', F32, (n,), (1,))
            inplace.append('y')
        elif not _overlap(S, a['x'], 4 * n, a['y'], 4 * n):
            poison.append(t)
    elif entry == 'mos_lbfgs_direction':
        n, k = a['n'], a['k']
        win('g', F32, (n,), (1,))
        for i in range(k):
            win(f'S{i}', F32, (n,), (1,), p=a['S'][i])
            win(f'Y{i}', F32, (n,), (1,), p=a['Y'][i])
        target('d', F32, (n,), (1,))
        target('work', F64, (k + 1,), (1,), scratch=True)
        target('partial', F32, (256,), (1,), scratch=True)
        target('gtd', F32, (1,), (1,))
        counter = S.window(a['partial'] + 4 * 256, 'partial[256]', F32, (1,), (1,))
        if counter.view(torch.int32).item() != 0:
            pre.append('(p) partial[256] (the block counter) is not zero on entry')
    elif entry == 'mos_lbfgs_solve_batch':
        for i, p in enumerate(a['probs']):
            o, n = p['out_f'], p['in_f']
            win(f'G{i}', F64, (n, n), (n, 1), p=p['G'])
            win(f'R{i}', F64, (o, n), (n, 1), p=p['R'])
            target(f'best_D{i}', F32, (o * n,), (1,), p=p['best_D'])
    elif entry == 'mos_lora_merge':
        table = win('table', torch.int64, (a['n_layers'], 6), (6, 1))
        for i, (pw, pd, pu, o, n, r) in enumerate(table.tolist()):
            try:
                win(f'down{i}', F32, (r, n), (n, 1), p=pd, table=True)
                win(f'up{i}', F32, (o, r), (r, 1), p=pu, table=True)
                win(f'W{i}', F32, (o, n), (n, 1), p=pw, table=True)
                target(f'W{i}', F32, (o, n), (n, 1), p=pw, table=True)
                inplace.append(f'W{i}')
            except AssertionError as e:
                pre.append(f'(p) table row {i}: {e}')
    return {'op': entry, 'abi': a, 'in': x, 'targets': targets, 'pre': pre, 'inplace': tuple(inplace),
            'poison': poison}


# --------------------------------------------------------------------------------------------------- references
def red_gamma(n):
    """the relative constant of the fusion.cu reductions over n terms"""
    return (-(-n // RED_THREADS) + RED_LEVELS) * U32


def _d(t):
    return t.double()


def lbfgs_reference(g, S, Y, rho, h_diag):
    """float64 two-loop recursion with a first-order error bound carried alongside (module docstring) -> (d, e_d,
    gtd, e_gtd); S, Y oldest first, rho as passed, h_diag the fp32 value passed"""
    n = g.numel()
    gam = red_gamma(n)
    k = len(S)
    v = -_d(g)
    e = torch.zeros_like(v)

    def dot(h):
        h = _d(h)
        return float(h @ v), float(h.abs() @ e + gam * (h.abs() @ v.abs()))

    def update(h, c, e_c):
        nonlocal v, e
        h = _d(h)
        v = v + c * h
        e = e + h.abs() * e_c + U32 * v.abs()

    al, e_al = [0.0] * k, [0.0] * k
    for i in range(k - 1, -1, -1):
        dt, ed = dot(S[i])
        al[i], e_al[i] = dt * rho[i], abs(rho[i]) * ed
        c = float(torch.tensor(-al[i], dtype=F64).float())           # the coefficient is applied as fp32
        update(Y[i], c, e_al[i] + 2 * U32 * abs(al[i]) + 2 * U64 * abs(al[i]))
    h = float(torch.tensor(h_diag, dtype=F32))
    v = h * v
    e = abs(h) * e + U32 * v.abs()
    for i in range(k):
        dt, ed = dot(Y[i])
        be = dt * rho[i]
        c64 = al[i] - be
        c = float(torch.tensor(c64, dtype=F64).float())
        update(S[i], c, e_al[i] + abs(rho[i]) * ed + 2 * U32 * abs(c64) + 2 * U64 * (abs(al[i]) + abs(be)))
    gtd, e_gtd = dot(g)
    return v, e, gtd, e_gtd + U32 * abs(gtd)


def reference(rec):
    """float64 reference of a launch: {target name: (value, bound)}; bound None = bit-exact.  Pure function of rec."""
    e, a, x = rec['op'], rec['abi'], rec['in']
    if e == 'mos_transpose_bf16':
        return {'out': (_d(x['x']).t(), None)}
    if e in ('mos_gram_small', 'mos_atb_small'):
        out = 'G' if e == 'mos_gram_small' else 'out'
        X, Y = _d(x['X']), _d(x['Y'])
        r = X.t() @ Y
        b = (a['n'] + 2) * U32 * (X.abs().t() @ Y.abs())
        if a['accumulate']:
            r = r + _d(x[out])
            b = b + U32 * r.abs()
        return {out: (r, b)}
    if e == 'mos_sgemm_nn':
        A, B, al, be = _d(x['A']), _d(x['B']), a['alpha'], a['beta']
        r = al * (A @ B)
        b = (a['K'] + 2) * U32 * abs(al) * (A.abs() @ B.abs())
        if be != 0:
            bc = be * _d(x['C'])
            r, b = r + bc, b + 2 * U32 * bc.abs()
        return {'C': (r, b)}
    if e == 'mos_dgemm_mixed':
        A, B = _d(x['A']), x['B'].double()
        return {'C': (A @ B, 2 * (a['K'] + 2) * U64 * (A.abs() @ B.abs()))}
    if e == 'mos_ls_grad_loss':
        W, Y, C, s, f0 = _d(x['W']), x['Y'].double(), x['Cm'].double(), a['s'], a['f0']
        g = 2.0 * s * (Y - C)
        gb = U32 * g.abs() + 4 * U64 * 2 * abs(s) * (Y.abs() + C.abs())
        t = Y - 2.0 * C
        loss = s * float(W @ t) + f0
        lb = 2 * (a['n'] + 4) * U64 * abs(s) * float(W.abs() @ t.abs()) + U64 * abs(f0)
        return {'grad': (g, gb), 'loss': (torch.tensor([loss], dtype=F64), torch.tensor([lb], dtype=F64))}
    if e == 'mos_vec_dot':
        p = _d(x['a']) * _d(x['b'])
        return {'out': (p.sum().reshape(1), (red_gamma(a['n']) * p.abs().sum()).reshape(1))}
    if e == 'mos_vec_asum':
        p = _d(x['a']).abs()
        return {'out': (p.sum().reshape(1), (red_gamma(a['n']) * p.sum()).reshape(1))}
    if e == 'mos_vec_absmax':
        v = (_d(x['a']) * a['scale']).abs()
        r = v.max() if not torch.isnan(v).any() else torch.tensor(float('nan'), dtype=F64)
        return {'out': (r.reshape(1), (U32 * r.abs()).reshape(1))}
    if e == 'mos_vec_axpby':
        ax = a['alpha'] * _d(x['x'])
        by = a['beta'] * _d(x['y']) if a['beta'] != 0 else torch.zeros_like(ax)
        return {'y': (ax + by, 2 * U32 * (ax.abs() + by.abs()))}
    if e == 'mos_lbfgs_direction':
        k = a['k']
        d, ed, gtd, eg = lbfgs_reference(x['g'], [x[f'S{i}'] for i in range(k)], [x[f'Y{i}'] for i in range(k)],
                                         a['rho'], a['h_diag'])
        return {'d': (d, ed), 'gtd': (torch.tensor([gtd], dtype=F64), torch.tensor([eg], dtype=F64))}
    if e == 'mos_lora_merge':
        out = {}
        al = a['alpha']
        for i in range(a['n_layers']):
            if f'W{i}' not in x:
                continue
            up, dn = _d(x[f'up{i}']), _d(x[f'down{i}'])
            r = _d(x[f'W{i}']) + al * (up @ dn)
            out[f'W{i}'] = (r, (up.shape[1] + 2) * U32 * abs(al) * (up.abs() @ dn.abs()) + U32 * r.abs())
        return out
    return {}


def gram_loss(D, G, R, s, f0):
    """f(D) = s <D, D G - 2 R> + f0 in float64 and the bound of (ii) (module docstring); D [out, in]"""
    D, G, R = D.double(), G.double(), R.double()
    val = s * float((D * (D @ G - 2.0 * R)).sum()) + f0
    n_in = G.shape[0]
    mag = abs(s) * float((D.abs() * (D.abs() @ G.abs() + 2.0 * R.abs())).sum())
    return val, 2 * (n_in + D.numel() + 8) * U64 * mag + 2 * U64 * abs(f0)


# --------------------------------------------------------------------------------------------------- checks
def _view(rec, t, which):
    return rec['mem'][t['mem']][which].as_strided(t['size'], t['stride'], t['off'])


def check_window(rec, errors):
    """(c): every element of a written storage outside the launch's targets is bitwise unchanged"""
    for key, m in rec['mem'].items():
        before, after = m['before'], m['after']
        mask = torch.zeros(before.numel(), dtype=torch.bool, device=before.device)
        for t in rec['targets']:
            if t['mem'] == key:
                mask.as_strided(t['size'], t['stride'], t['off']).fill_(True)
        bits = _BITS[before.element_size()]
        diff = (before.view(bits) != after.view(bits)) & ~mask
        if diff.any():
            i = int(diff.nonzero()[0])
            errors.append(f'(c) {int(diff.sum())} element(s) outside the window changed (first at element {i} of '
                          f'the storage)')


def check_launch(rec):
    """(p), (a), (b), (c) of one launch (not lbfgs_solve_batch, whose checks need the library: SolverRecorder)"""
    errors, ratio, rel = list(rec['pre']), 0.0, 0.0
    refs = reference(rec)
    for t in rec['targets']:
        if t['scratch'] or t['name'] not in refs:
            continue
        got = _view(rec, t, 'after')
        r, b = refs[t['name']]
        r, b = r.to(got.device), (None if b is None else b.to(got.device))
        if b is None:
            bits = _BITS[got.element_size()]
            want = r.to(got.dtype)
            if not torch.equal(got.view(bits), want.view(bits)):
                errors.append(f"(a) {t['name']}: {int((got.view(bits) != want.view(bits)).sum())} element(s) differ "
                              f'from the bit-exact reference')
            continue
        g = got.double()
        nan_r, nan_g = torch.isnan(r), torch.isnan(g)
        if not torch.equal(nan_r, nan_g):
            errors.append(f"(a) {t['name']}: NaN at {int((nan_r != nan_g).sum())} element(s) where the reference "
                          f"{'is' if nan_r.any() else 'is not'} NaN")
        ok = ~(nan_r | nan_g)
        err = (g - r).abs()[ok]
        bound = b.to(r.device)[ok]
        if err.numel():
            bad = err > bound
            q = err / bound.clamp_min(1e-300)
            q = torch.where(err == 0, torch.zeros_like(q), q)
            ratio = max(ratio, float(q.max()))
            if bad.any():
                i = int(bad.nonzero()[0])
                errors.append(f"(a) {t['name']}: {int(bad.sum())} element(s) out of bound, first: got {float(err[i]):.3e} "
                              f'error, bound {float(bound[i]):.3e}')
            rn = float(r[ok].norm())
            rel = max(rel, float((g[ok] - r[ok]).norm()) / rn if rn > 0 else float(err.max() > 0))
    check_window(rec, errors)
    return {'ratio': ratio, 'tile_rel': rel, 'tile': 0.0, 'errors': errors}


def check_solve(rec, python_solve, relaunch_one_worker):
    """(i)-(iii) and the one-worker relaunch of an lbfgs_solve_batch launch (module docstring).  python_solve(G, R, s,
    f0, iters, history) -> best_D of the Python driver (None: it found no finite loss); relaunch_one_worker() -> the
    best_D of each problem after a relaunch with one worker from the same bytes"""
    a, x = rec['abi'], rec['in']
    errors, ratio, rel = list(rec['pre']), 0.0, 0.0
    ct = a['_ct']
    for i, p in enumerate(a['probs']):
        t = next(t for t in rec['targets'] if t['name'] == f'best_D{i}')
        got = _view(rec, t, 'after')
        want = python_solve(x[f'G{i}'], x[f'R{i}'], p['s'], p['f0'], p['max_iter'], p['history'])
        if want is None or not torch.equal(got.view(torch.int32), want.reshape(-1).view(torch.int32)):
            errors.append(f'(i) problem {i}: best_D is not bit-identical to the Python driver\'s')
        D = got.reshape(p['out_f'], p['in_f'])
        f, b = gram_loss(D, x[f'G{i}'], x[f'R{i}'], p['s'], p['f0'])
        best = ct[i].best_loss[0] if ct[i].best_loss else float('nan')
        q = abs(best - f) / b if b > 0 else float(best != f)
        ratio = max(ratio, q)
        if not abs(best - f) <= b:
            errors.append(f'(ii) problem {i}: returned best_loss {best!r} but f(best_D) = {f!r} (bound {b:.3e})')
        if not f <= p['f0'] + b:
            errors.append(f"(iii) problem {i}: f(best_D) = {f!r} above the starting loss f0 = {p['f0']!r}")
        rel = max(rel, abs(best - f) / max(abs(f), 1e-300))
    check_window(rec, errors)
    again = relaunch_one_worker()
    for i, d1 in enumerate(again):
        t = next(t for t in rec['targets'] if t['name'] == f'best_D{i}')
        if not torch.equal(d1.view(torch.int32), _view(rec, t, 'after').view(torch.int32)):
            errors.append(f'(e) problem {i}: a relaunch with one worker is not bit-identical')
    return {'ratio': ratio, 'tile_rel': rel, 'tile': 0.0, 'errors': errors}


# --------------------------------------------------------------------------------------------------- recorder
class Recorder(ga.LaunchRecorder):
    """audits every gradient-fusion solver launch made inside it.  The tensors that `.contiguous()` returns inside
    gradient_fusion.merge_lora_into_weight and gradient_fusion._merged are registered (the lora_merge table points into
    them).  The solve-level checks run the Python driver through the same library with the audit suspended."""
    OPS = ('transpose_bf16', 'gram_small', 'atb_small', 'sgemm_nn', 'dgemm_mixed', 'ls_grad_loss', 'vec_dot', 'vec_asum',
           'vec_absmax', 'vec_axpby', 'lbfgs_direction', 'lbfgs_solve_batch', 'lora_merge')
    ENTRY_POINTS = ENTRY_POINTS
    _MERGE_FNS = ('merge_lora_into_weight', '_merged')

    def __init__(self, stats=None, determinism='all'):
        super().__init__(stats, determinism)
        self._inner = False

    def __enter__(self):
        super().__enter__()
        import gradient_fusion as gf
        self._gf = gf
        self._orig_gf = {n: getattr(gf, n) for n in self._MERGE_FNS}
        rec = self

        def registering(fn):
            def _registering(*args, **kwargs):
                orig = torch.Tensor.contiguous

                def contiguous(t, *a, **k):
                    out = orig(t, *a, **k)
                    rec.register(out)
                    return out
                torch.Tensor.contiguous = contiguous
                try:
                    return fn(*args, **kwargs)
                finally:
                    torch.Tensor.contiguous = orig
            return _registering
        for n, fn in self._orig_gf.items():
            setattr(gf, n, registering(fn))
        return self

    def __exit__(self, *exc):
        for n, fn in self._orig_gf.items():
            setattr(self._gf, n, fn)
        return super().__exit__(*exc)

    @contextlib.contextmanager
    def unaudited(self):
        """run library calls without auditing them (the Python driver of a solve-level check)"""
        saved = {n: getattr(self._ops, n) for n in self._orig_ops}
        for n, fn in self._orig_ops.items():
            setattr(self._ops, n, fn)
        self._inner = True
        try:
            yield
        finally:
            for n, fn in saved.items():
                setattr(self._ops, n, fn)
            self._inner = False

    def _audit(self, entry, launch, args):
        if self._inner:
            return launch()
        self._args = args
        return super()._audit(entry, launch, args)

    def record(self, entry, args, S):
        self._storages = S
        rec = record(entry, abi_of(entry, args[:len(_ARGS[entry])]), S)
        for t in rec['poison']:
            w = S.flat(*t['mem']).as_strided(t['size'], t['stride'], t['off'])
            w.fill_(float('nan'))
        return rec

    def key(self, rec):
        return solver_path(rec)

    def check(self, rec):
        if rec['op'] != 'mos_lbfgs_solve_batch':
            return check_launch(rec)
        gf = self._gf
        real = self._orig_lib()

        def python_solve(G, R, s, f0, iters, history):
            with self.unaudited():
                P = gf._GramProblem(G.clone(), R.clone(), s, f0, None)
                gf.lbfgs_minimize(P, torch.zeros(R.numel(), device=R.device, dtype=F32), iters, history=history)
                if R.is_cuda:
                    torch.cuda.synchronize()
            return P.best_D

        def relaunch_one_worker():
            flats = {k: self._storages.flat(*k) for k in rec['mem']}
            for k, f in flats.items():
                f.copy_(rec['mem'][k]['before'])
            args = self._args
            with self.unaudited():
                rc = real.mos_lbfgs_solve_batch(args[0], args[1], ctypes.c_int32(1))
            if any(v.is_cuda for v in rec['in'].values()):
                torch.cuda.synchronize()
            assert rc == 0, rc
            outs = [_view({'mem': {k: {'x': f}}}, t, 'x').clone() for t in rec['targets'] for k, f in flats.items()
                    if t['mem'] == k]
            for k, f in flats.items():
                f.copy_(rec['mem'][k]['after'])
            return outs
        return check_solve(rec, python_solve, relaunch_one_worker)
