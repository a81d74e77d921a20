"""The L-BFGS statement of gradient fusion (gradient_fusion.lbfgs_minimize / _strong_wolfe, which csrc/lbfgs.cu follows
launch for launch) against torch.optim.LBFGS, the optimiser the reference calls (gradient_fusion.py:76-85): lr 1,
history 25, strong-Wolfe line search, tolerances 1e-16, one .step of max_iter iterations.

Both run in float64 on the CPU on the same objective: gradient_fusion's `ops` is replaced by float64 stand-ins of the
vector primitives it calls, and the problem object evaluates the objective in float64.  They must agree on the number of
closure evaluations, on the number of iterations and on the iterate.  Beside Gram-form quadratics (the only objective
lbfgs.cu solves, where the cubic step is exact and most branches of the line search never run) the cases include
non-quadratic objectives, and a line tracer counts the branches of the driver each case takes: every branch listed in
BRANCHES must be taken by at least one case, so none of them is compared vacuously.  The GPU tests that hold the
native driver bit-identical to the Python one (test_fusion_gpu.py, test_fusion_wholeblock_gpu.py) carry this result over
to lbfgs.cu.
"""
import inspect
import sys
import types

import pytest
import torch

import gradient_fusion as gf

F64 = torch.float64

# branch -> a statement of gradient_fusion.py that only that branch executes
BRANCHES = {
    'zoom phase': 't = _cubic_min(br[0][0], br[0][1], br[0][3], br[1][0], br[1][1], br[1][3])',
    'insufficient progress': 'stalled = True',
    'max_ls exit': 'br = [[0.0, f, g, gtd], [t, f_new, g_new, gtd_new]]',
    'more than 25 pairs': 'S.pop(0), Y.pop(0), rho.pop(0)',
}
# counted statements: the curvature test, the pair it stores, the iteration counter, the two stopping tests' breaks
_COUNTED = {
    'ys test': 'if ys > 1e-10:',
    'pair stored': 'S.append(s), Y.append(y), rho.append(1.0 / ys)',
    'iteration': 'n_iter += 1',
    'stop test': 'if g_max <= tol_grad or step_max <= tol_change or abs(loss - prev_loss) < tol_change:',
    'eval test': 'if n_iter == max_iter or evals >= max_eval:',
}


def _lines():
    src = inspect.getsource(gf).splitlines()
    out = {}
    for name, stmt in {**BRANCHES, **_COUNTED}.items():
        hits = [i for i, line in enumerate(src, start=1) if line.strip() == stmt]
        assert len(hits) == 1, (name, hits)
        out[name] = hits[0]
    return out


LINES = _lines()


class Ops:
    """float64 stand-ins of the primitives lbfgs_minimize calls (the algorithm, not the kernels, is under test)"""

    @staticmethod
    def vec_axpby(y, x, alpha, beta=1.0):
        if beta == 1.0:
            return y.add_(x, alpha=alpha)          # as torch.optim.LBFGS._add_grad and Tensor.sub
        assert beta == 0.0
        return y.copy_(x.mul(alpha))

    @staticmethod
    def vec_asum(a, out, scratch):
        out[0] = a.abs().sum()

    @staticmethod
    def lbfgs_direction(S, Y, rho, g, h_diag, d, work, partial, gtd):
        k = len(S)
        q = g.neg()
        al = [0.0] * k
        for i in range(k - 1, -1, -1):
            al[i] = float(S[i].dot(q)) * rho[i]
            q.add_(Y[i], alpha=-al[i])
        r = q * h_diag
        for i in range(k):
            be = float(Y[i].dot(r)) * rho[i]
            r.add_(S[i], alpha=al[i] - be)
        d.copy_(r)
        gtd[0] = g.dot(d)
        return d


class Problem:
    """the interface of gradient_fusion._GramProblem over a float64 objective fn(x) -> (loss, grad)"""

    def __init__(self, fn):
        self.fn = fn
        self.scal, self.scratch, self.gtd = torch.zeros(1, dtype=F64), None, torch.zeros(1, dtype=F64)
        self.work = self.partial = None
        self.evals = 0

    def dot(self, a, b):
        return float(a.dot(b))

    def dot2(self, a, b, c, d):
        return float(a.dot(b)), float(c.dot(d))

    def absmax(self, a, scale=1.0):
        return float((a * scale).abs().max())

    def absmax2(self, a, b, scale_b):
        self.last_max = self.absmax(a), self.absmax(b, scale_b)
        return self.last_max

    def closure(self, x):
        self.evals += 1
        return self.fn(x)


def run_ours(fn, x0, max_iter, monkeypatch):
    monkeypatch.setattr(gf, 'ops', types.SimpleNamespace(**{n: getattr(Ops, n) for n in
                                                            ('vec_axpby', 'vec_asum', 'lbfgs_direction')}))
    P = Problem(fn)
    hits = dict.fromkeys(LINES, 0)
    where = {v: k for k, v in LINES.items()}
    fname = gf.__file__

    def tracer(frame, event, arg):
        if frame.f_code.co_filename != fname:
            return None
        if event == 'line' and frame.f_lineno in where:
            hits[where[frame.f_lineno]] += 1
        return tracer
    sys.settrace(tracer)
    try:
        x = gf.lbfgs_minimize(P, x0.clone(), max_iter)
    finally:
        sys.settrace(None)
    return x, P.evals, hits, getattr(P, 'last_max', None)


def run_torch(fn, x0, max_iter, monkeypatch):
    """torch.optim.LBFGS.step; recent torch calls its line search with max_ls = max_eval - evals (the remaining budget),
    the torch the reference was written against with the default max_ls = 25, which gradient fusion keeps: the line
    search is called with max_ls = 25 here"""
    import torch.optim.lbfgs as tl
    orig = tl._strong_wolfe
    monkeypatch.setattr(tl, '_strong_wolfe', lambda *a, **k: orig(*a, **dict(k, max_ls=25)))
    p = torch.nn.Parameter(x0.clone())
    opt = torch.optim.LBFGS([p], lr=1, max_iter=max_iter, history_size=25, line_search_fn='strong_wolfe',
                            tolerance_grad=1e-16, tolerance_change=1e-16)

    def closure():
        opt.zero_grad()
        loss, g = fn(p.detach())
        p.grad = g.clone()
        return torch.tensor(loss, dtype=F64)
    opt.step(closure)
    st = opt.state[p]
    return p.detach(), st['func_evals'], st['n_iter']


# ---------------------------------------------------------------------------------------------------- objectives
def gram(out_f, in_f, n_rows, seed, cond=1.0):
    """f(D) = s <D, D G - 2 R> + f0 with an exactly solvable right-hand side (lbfgs.cu's objective)"""
    g = torch.Generator().manual_seed(seed)
    K = torch.randn(n_rows, in_f, generator=g, dtype=F64) * torch.logspace(0, cond, in_f, dtype=F64)
    G = K.t() @ K
    Dt = torch.randn(out_f, in_f, generator=g, dtype=F64) * 0.05
    R = Dt @ G
    s = 1.0 / (n_rows * out_f)
    f0 = s * float((Dt * (Dt @ G)).sum())

    def fn(x):
        D = x.view(out_f, in_f)
        DG = D @ G
        return s * float((D * (DG - 2.0 * R)).sum()) + f0, (2.0 * s * (DG - R)).reshape(-1)
    return fn, torch.zeros(out_f * in_f, dtype=F64)


def rosenbrock(n):
    def fn(x):
        a, b = x[:-1], x[1:]
        f = float((100.0 * (b - a * a) ** 2 + (1.0 - a) ** 2).sum())
        g = torch.zeros_like(x)
        g[:-1] += -400.0 * a * (b - a * a) - 2.0 * (1.0 - a)
        g[1:] += 200.0 * (b - a * a)
        return f, g
    x0 = torch.tensor([-1.2, 1.0] * (n // 2), dtype=F64)
    return fn, x0


def log_sum_exp(n, seed):
    """log sum exp(A x) + |x|^2 / 200"""
    A = torch.randn(3 * n, n, generator=torch.Generator().manual_seed(seed), dtype=F64)

    def fn(x):
        z = A @ x
        m = z.max()
        e = torch.exp(z - m)
        f = float(m + torch.log(e.sum()) + 0.005 * x.dot(x))
        return f, A.t() @ (e / e.sum()) + 0.01 * x
    return fn, torch.full((n,), 0.5, dtype=F64)


def stiff(n):
    """50 |x|^2 from a point where |g|_1 < 1: the first step (t = 1) overshoots the minimiser along d 100-fold, so the
    zoom's cubic step lands within 10 % of the bracket's end (insufficient progress)"""
    def fn(x):
        return float(50.0 * x.dot(x)), 100.0 * x
    return fn, torch.linspace(1e-3, 2e-3, n, dtype=F64)


def quartic_descent(n):
    """-sum x^4 / 4 from linspace(0.5, 1): the slope steepens along the direction, so the curvature condition never holds
    and the bracketing phase extrapolates until it runs out of max_ls.  (A concave quadratic would do the same, but on an
    exactly quadratic line the cubic's denominator g2 - g1 + 2 d2 cancels to zero and the step goes to either bound by
    the sign of a rounding error.)"""
    def fn(x):
        return float(-(x ** 4).sum() / 4.0), -(x ** 3)
    return fn, torch.linspace(0.5, 1.0, n, dtype=F64)


def double_well(n):
    """sum (x^2 - 1)^2 started inside the concave region: a step there gives <y, s> <= 0 and the pair is skipped"""
    def fn(x):
        return float(((x * x - 1.0) ** 2).sum()), 4.0 * x * (x * x - 1.0)
    return fn, torch.linspace(0.05, 0.3, n, dtype=F64)


CASES = {
    'gram 12x20 (over-determined)': (lambda: gram(12, 20, 40, 1), 50),
    'gram 8x60 (under-determined, 40 rows)': (lambda: gram(8, 60, 40, 2), 60),
    'gram 4x200 ill-conditioned': (lambda: gram(4, 200, 300, 3, cond=1.5), 80),
    'rosenbrock 10': (lambda: rosenbrock(10), 100),
    'rosenbrock 2 (max_eval)': (lambda: rosenbrock(2), 20),
    'stiff quadratic': (lambda: stiff(5), 5),
    'log-sum-exp 30': (lambda: log_sum_exp(30, 4), 60),
    'quartic descent (max_ls)': (lambda: quartic_descent(5), 1),
    'double well': (lambda: double_well(6), 40),
}
TAKEN = {}


@pytest.mark.parametrize('case', list(CASES))
def test_lbfgs_minimize_matches_torch_lbfgs(case, monkeypatch):
    """evaluations and iterations exactly; the iterate to float64 rounding.  The stand-ins issue the tensor operations
    torch.optim.LBFGS issues (dot, add_ with alpha, mul), so the iterates come out bit-identical (measured on every
    case); the bound of 1e-12 of max |x| only leaves room for a different vectorisation of those operations, while any
    algorithmic difference (another step, pair or line-search point) moves the iterate by far more"""
    make, max_iter = CASES[case]
    fn, x0 = make()
    x, evals, hits, last_max = run_ours(fn, x0, max_iter, monkeypatch)
    xt, evals_t, n_iter_t = run_torch(fn, x0, max_iter, monkeypatch)
    assert (evals, hits['iteration']) == (evals_t, n_iter_t), (case, evals, hits['iteration'], evals_t, n_iter_t)
    err = float((x - xt).abs().max()) / max(float(xt.abs().max()), 1e-300)
    assert err <= 1e-12, (case, err)
    taken = {b for b in BRANCHES if hits[b]}
    if hits['ys test'] > hits['pair stored']:
        taken.add('skipped pair')
    # how the run ended: the step / gradient / loss-change test or the evaluation budget
    if evals >= max_iter * 5 // 4 and hits['iteration'] < max_iter:
        taken.add('stop on max_eval')
    if hits['stop test'] == hits['iteration'] and min(last_max) > 1e-16:
        taken.add('stop on |d loss| < tol')     # the last stopping test broke the loop, by neither |g| nor the step
    TAKEN[case] = taken
    print(f'{case}: {evals} evaluations, {hits["iteration"]} iterations, iterate rel diff {err:.1e}, '
          f'branches {sorted(taken)}')



def test_every_branch_taken():
    """runs after the cases above: each listed branch of the driver was taken by at least one case"""
    if len(TAKEN) < len(CASES):
        pytest.skip('needs the cases of test_lbfgs_minimize_matches_torch_lbfgs in the same session')
    union = set().union(*TAKEN.values())
    want = set(BRANCHES) | {'skipped pair', 'stop on max_eval', 'stop on |d loss| < tol'}
    print('branches taken: ' + ', '.join(f'{b}: {[c for c, t in TAKEN.items() if b in t]}' for b in sorted(want)))
    assert union >= want, f'never taken: {sorted(want - union)}'
