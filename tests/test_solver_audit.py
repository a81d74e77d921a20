"""The gradient-fusion solver launch audit (tests/solver_audit.py) on the CPU: its float64 references against independent
torch statements of the same operations, and its checks against a stand-in library.

Launches are made by the real `ops.*` wrappers with CPU tensors through the audit's own Recorder, so the records come
from the ABI arguments exactly as on the GPU.  The stand-in is a library over host memory: it reads its operands through
the raw pointers it is passed and writes the rounded float64 result of each entry point (its lbfgs_solve_batch runs the
Python driver, gradient_fusion.lbfgs_minimize, through the stand-in itself).  Every mutation case breaks it the way a
faulty kernel would, and the check it targets must flag it while the unbroken stand-in passes every check.
"""
import contextlib
import ctypes

import pytest
import torch

import solver_audit as sa

F32, F64, BF = torch.float32, torch.float64, torch.bfloat16


def rnd(shape, seed, scale=1.0, dtype=F32):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dtype)


def host(p, dtype, n):
    """n elements of `dtype` at host address p, as a tensor sharing that memory"""
    es = torch.empty(0, dtype=dtype).element_size()
    return torch.frombuffer((ctypes.c_char * (n * es)).from_address(p), dtype=dtype)


def val(v):
    return getattr(v, 'value', v)


class StandIn:
    """the entry points of ENTRY_POINTS over host memory; `mut` names one defect to inject"""

    def __init__(self, mut=None):
        self.mut, self.recorder, self.err = mut, None, b''

    def mos_last_error(self):
        return self.err

    def __getattr__(self, name):
        if name not in sa.ENTRY_POINTS:
            raise AttributeError(name)
        return lambda *args: getattr(self, '_' + name[4:])(*[val(a) if not hasattr(a, '_length_') else a for a in args])

    def _transpose_bf16(self, x, ldx, rows, C, out, ldo, _s):
        X = host(x, BF, (rows - 1) * ldx + C).as_strided((rows, C), (ldx, 1))
        O = host(out, BF, (C - 1) * ldo + rows).as_strided((C, rows), (ldo, 1))
        r1 = rows // 32 * 32 if self.mut == 'transpose_tail' and rows % 32 else rows
        O[:, :r1] = X[:r1].t()
        return 0

    def _atb(self, X, Y, n, dx, dy, out, acc):
        A = host(X, F32, n * dx).view(n, dx).double()
        B = host(Y, F32, n * dy).view(n, dy).double()
        if self.mut == 'atb_ktile' and n % 16:
            A, B = A[:n // 16 * 16], B[:n // 16 * 16]
        O = host(out, F32, dx * dy).view(dx, dy)
        O.copy_((A.t() @ B + (O.double() if acc else 0)).float())
        return 0

    def _gram_small(self, X, n, d, G, acc, _s):
        return self._atb(X, X, n, d, d, G, acc)

    def _atb_small(self, X, Y, n, dx, dy, out, acc, _s):
        return self._atb(X, Y, n, dx, dy, out, acc)

    def _sgemm_nn(self, A, B, C, M, N, K, alpha, beta, _s):
        a, b = host(A, F32, M * K).view(M, K).double(), host(B, F32, K * N).view(K, N).double()
        c = host(C, F32, M * N).view(M, N)
        reads = beta != 0 or self.mut == 'sgemm_reads_c'
        c.copy_((alpha * (a @ b) + (beta * c.double() if reads else 0)).float())
        return 0

    def _dgemm_mixed(self, A, B, C, M, N, K, _s):
        a, b = host(A, F32, M * K).view(M, K), host(B, F64, K * N).view(K, N)
        c = host(C, F64, M * N).view(M, N)
        c.copy_(a.double() @ b if self.mut != 'dgemm_fp32' else (a @ b.float()).double())
        return 0

    def _ls_grad_loss(self, W, Y, Cm, n, s, f0, grad, loss, scratch, _s):
        w, y, c = host(W, F32, n).double(), host(Y, F64, n), host(Cm, F64, n)
        host(grad, F32, n).copy_((2.0 * s * (y - c)).float())
        host(loss, F64, 1)[0] = s * float(w @ (y - 2.0 * c)) + (0.0 if self.mut == 'loss_no_f0' else f0)
        host(scratch, F64, 256).fill_(1.0)
        return 0

    def _vec_dot(self, a, b, n, out, scratch, _s):
        p = host(a, F32, n).double() * host(b, F32, n).double()
        if self.mut == 'dot_drop_partial':
            p = p[(torch.arange(n) // 256) % 256 != 255]             # block 255's partial is lost
        host(out, F32, 1)[0] = float(p.sum())
        host(scratch, F32, 256).fill_(1.0)
        return 0

    def _vec_asum(self, a, n, out, scratch, _s):
        host(out, F32, 1)[0] = float(host(a, F32, n).double().abs().sum())
        host(scratch, F32, 256).fill_(1.0)
        return 0

    def _vec_absmax(self, a, n, scale, out, scratch, _s):
        v = (host(a, F32, n) * scale).abs()
        host(out, F32, 1)[0] = float(v.nan_to_num(0.0).max() if self.mut == 'absmax_nan' else v.max())
        host(scratch, F32, 256).fill_(1.0)
        return 0

    def _vec_axpby(self, y, x, alpha, beta, n, _s):
        Y, X = host(y, F32, n), host(x, F32, n)
        reads = beta != 0 or self.mut == 'axpby_reads_y'
        Y.copy_((alpha * X.double() + (beta * Y.double() if reads else 0)).float())
        return 0

    def _lbfgs_direction(self, S, Y, rho, k, g, h_diag, n, d, work, partial, gtd, _s):
        Sv = [host(S[i], F32, n) for i in range(k)]
        Yv = [host(Y[i], F32, n) for i in range(k)]
        rh = [rho[i] for i in range(k)]
        if self.mut == 'dir_prev_coef' and k >= 2:
            rh = rh[1:] + rh[:1]                                     # each pair scaled with its neighbour's rho
        hd = 1.0 if self.mut == 'dir_no_hdiag' else h_diag
        v, _, gd, _ = sa.lbfgs_reference(host(g, F32, n), Sv, Yv, rh, hd)
        host(d, F32, n).copy_(v.float())
        host(gtd, F32, 1)[0] = gd
        host(work, F64, k + 1).fill_(3.0)
        host(partial, F32, 256).fill_(2.0)
        if self.mut == 'dir_counter':
            host(partial + 4 * 256, torch.int32, 1)[0] = 256
        return 0

    def _lora_merge(self, table, n_layers, alpha, _s):
        for pw, pd, pu, o, i, r in host(table, torch.int64, 6 * n_layers).view(n_layers, 6).tolist():
            W = host(pw, F32, o * i).view(o, i)
            dn, up = host(pd, F32, r * i).view(r, i).double(), host(pu, F32, o * r).view(o, r).double()
            if self.mut == 'lora_drop_rank':
                dn, up = dn[:-1], up[:, :-1]
            W.copy_((W.double() + alpha * (up @ dn)).float())
        return 0

    def _lbfgs_solve_batch(self, probs, n, workers):
        import gradient_fusion as gf
        rec = self.recorder
        for j in range(n):
            p = probs[j]
            o, i = p.out_f, p.in_f
            G, R = host(p.G, F64, i * i).view(i, i), host(p.R, F64, o * i).view(o, i)
            with rec.unaudited() if rec is not None and rec._ctx else contextlib.nullcontext():
                P = gf._GramProblem(G, R, p.s, p.f0, None)
                closure = P.closure

                def closure_last(D, closure=closure, P=P):
                    P.last_loss, g = closure(D)
                    return P.last_loss, g
                P.closure = closure_last
                gf.lbfgs_minimize(P, torch.zeros(o * i), p.max_iter, history=p.history)
            if P.best_D is None:
                self.err = f'mos_lbfgs_solve_batch: problem {j}: no finite loss'.encode()
                return -1
            host(p.best_D, F32, o * i).copy_(P.best_D)
            if self.mut == 'solve_write_past':
                host(p.best_D + 4 * o * i, F32, 1)[0] = 1.0
            p.best_loss[0] = P.last_loss if self.mut == 'solve_last_loss' else P.best_loss
            p.n_evals[0] = P.evals
        if self.mut == 'solve_swapped_loss' and n > 1:               # each loss lands in the next problem's slot
            losses = [probs[j].best_loss[0] for j in range(n)]
            for j in range(n):
                probs[j].best_loss[0] = losses[j - 1]
        return 0


@pytest.fixture
def audit(monkeypatch):
    """audit(mut=None) -> a Recorder over the stand-in library (CPU tensors)"""
    from mos_b200 import _lib, ops
    monkeypatch.setattr(ops, 'current_stream', lambda: None)

    def make(mut=None):
        lib = StandIn(mut)
        monkeypatch.setattr(_lib, 'lib', lambda: lib)
        r = sa.Recorder()
        lib.recorder = r
        return r
    return make


def ok(r):
    assert not r.stats.failures, '\n'.join(r.stats.failures)
    assert r.stats.rows
    return r


def flagged(r, letter):
    assert any(f'({letter})' in e for e in r.stats.failures), r.stats.failures


# ---------------------------------------------------------------------------------------------------- launches
def run_transpose(audit, mut=None, rows=75, C=45, ldx=64, pad=7):
    from mos_b200 import ops
    buf = rnd((rows, ldx), 1, dtype=BF)
    out = torch.full((C, rows + pad), 5.0, dtype=BF)
    with audit(mut) as r:
        ops.transpose_bf16(buf[:, :C], out, rows=rows, C=C, ldx=ldx)
    return r


def run_atb(audit, mut=None, n=45, dx=100, dy=37, acc=True, gram=False):
    from mos_b200 import ops
    X, Y = rnd((n, dx), 2), rnd((n, dy), 3)
    with audit(mut) as r:
        if gram:
            ops.gram_small(X, rnd((dx, dx), 4), accumulate=acc)
        else:
            ops.atb_small(X, Y, rnd((dx, dy), 4), accumulate=acc)
    return r


def run_sgemm(audit, mut=None, beta=0.0):
    from mos_b200 import ops
    C = torch.full((65, 130), float('nan')) if beta == 0 else rnd((65, 130), 7)
    with audit(mut) as r:
        ops.sgemm_nn(rnd((65, 4 * 33), 5), rnd((4 * 33, 130), 6), C, alpha=-1.0 if beta else 1.0, beta=beta)
    return r


def run_dgemm(audit, mut=None, M=100, K=70, N=130):
    from mos_b200 import ops
    with audit(mut) as r:
        ops.dgemm_mixed(rnd((M, K), 8), rnd((K, N), 9, dtype=F64), torch.empty(M, N, dtype=F64))
    return r


def run_loss(audit, mut=None, n=1000):
    from mos_b200 import ops
    loss, scratch = torch.zeros(1, dtype=F64), torch.zeros(300, dtype=F64)
    with audit(mut) as r:
        ops.ls_grad_loss(rnd((n,), 10), rnd((n,), 11, dtype=F64), rnd((n,), 12, dtype=F64), 1e-3, 2.5,
                         torch.empty(n), loss, scratch)
    return r


def run_reductions(audit, mut=None, n=100003, nan=False):
    from mos_b200 import ops
    a, b = rnd((n,), 13), rnd((n,), 14)
    if nan:
        a[n // 2] = float('nan')
    out, scratch = torch.zeros(4), torch.zeros(300)
    with audit(mut) as r:
        ops.vec_dot(a, b, out[0:1], scratch)
        ops.vec_asum(a, out[1:2], scratch)
        ops.vec_absmax(a, out[2:3], scratch, 2.0)
        ops.vec_absmax(b, out[3:4], scratch)
    return r


def run_axpby(audit, mut=None, n=3000):
    from mos_b200 import ops
    x = rnd((n,), 15)
    with audit(mut) as r:
        ops.vec_axpby(torch.full((n,), float('nan')), x, -1.0, 0.0)
        ops.vec_axpby(rnd((n,), 16), x, 0.25, 1.0)
        ops.vec_axpby(rnd((n,), 16), x, 0.25, -0.5)
    return r


def history(n, k, seed=20):
    g = rnd((n,), seed)
    S = [rnd((n,), seed + 1 + i, 0.1) for i in range(k)]
    Y = [S[i] * (1.0 + 0.1 * i) + rnd((n,), seed + 100 + i, 0.05) for i in range(k)]
    rho = [1.0 / float(Y[i].double() @ S[i].double()) for i in range(k)]
    h = float(Y[-1].double() @ S[-1].double() / (Y[-1].double() @ Y[-1].double())) if k else 0.37
    return g, S, Y, rho, h


def run_direction(audit, mut=None, n=1001, k=3):
    from mos_b200 import ops
    g, S, Y, rho, h = history(n, k)
    if k == 25:                                      # a wrapped ring: pairs live at rotated offsets of one buffer
        ring = torch.stack(S[3:] + S[:3])
        S = [ring[(i + 22) % 25] for i in range(25)]
    work, partial, gtd = torch.zeros(64, dtype=F64), torch.zeros(260), torch.zeros(1)
    with audit(mut) as r:
        ops.lbfgs_direction(S, Y, rho, g, h, torch.full((n,), float('nan')), work, partial, gtd)
    return r


def run_lora(audit, mut=None, rank=4, conv=False):
    from mos_b200 import ops
    W1 = rnd((64, 96, 1, 1) if conv else (64, 96), 30)
    W2 = rnd((40, 33), 31)
    d1, u1 = rnd((rank, 96), 32, 0.1), rnd((64, rank), 33, 0.1)
    d2, u2 = rnd((rank, 33), 34, 0.1), rnd((40, rank), 35, 0.1)
    table = torch.tensor([[W1.data_ptr(), d1.data_ptr(), u1.data_ptr(), 64, 96, rank],
                          [W2.data_ptr(), d2.data_ptr(), u2.data_ptr(), 40, 33, rank]], dtype=torch.int64)
    with audit(mut) as r:
        r.register(W1, W2, d1, u1, d2, u2)
        ops.lora_merge(table, 2, 0.7)
    return r


def gram_problem(out_f, in_f, n_rows, seed, scale=1.0):
    K = rnd((n_rows, in_f), seed, dtype=F64)
    G = (K.t() @ K) * scale
    W0 = rnd((out_f, in_f), seed + 1, in_f ** -0.5, dtype=F64)
    Wt = W0 + 0.05 * rnd((out_f, in_f), seed + 2, dtype=F64)
    R = Wt @ G - W0 @ G
    s = 1.0 / (n_rows * out_f)
    f0 = s * float((Wt - W0).mul((Wt - W0) @ G).sum())
    return G.contiguous(), R.contiguous(), s, f0


def overshoot_problem():
    """a solve whose last evaluation is not its best: the gradient is flat and tiny (|g| = 5e-10 in each of 2e4
    elements, so |g|_1 < 1 and the first trial step is t = 1) while G = 1e4 I puts the minimiser along d at t = 2.5e-3.
    The trial point is worse than the start, and the zoom stops at once (|1 - 0| max |d| < 1e-9): the line search keeps
    t = 0, so the best loss is f0 = 0 and the last evaluation's is 1e-12"""
    o, i = 100, 200
    G = torch.eye(i, dtype=F64) * 1e4
    R = rnd((o, i), 42, dtype=F64).sign() * 1.25e-8
    return G, R.contiguous(), 0.02, 0.0


def run_solve(audit, mut=None, iters=6):
    from mos_b200 import ops
    G, R, s, f0 = gram_problem(12, 20, 30, 40)
    G2, R2, s2, f02 = gram_problem(5, 9, 50, 41)
    G3, R3, s3, f03 = overshoot_problem()
    buf = torch.full((12 * 20 + 8,), 9.0)
    b2, b3 = torch.zeros(45), torch.zeros(R3.numel())
    with audit(mut) as r:
        res = ops.lbfgs_solve_batch([(G, R, s, f0, buf[:240]), (G2, R2, s2, f02, b2), (G3, R3, s3, f03, b3)], iters,
                                    workers=2)
    return r, res


# ---------------------------------------------------------------------------------------------------- the unbroken stand-in
def test_unbroken_standin_passes_every_check(audit):
    ok(run_transpose(audit))
    ok(run_transpose(audit, rows=64, C=64, ldx=64, pad=0))
    for acc in (False, True):
        ok(run_atb(audit, acc=acc))
        ok(run_atb(audit, n=33, dx=3072, dy=5, acc=acc, gram=False))
    ok(run_atb(audit, n=300, dx=3072, acc=True, gram=True))
    ok(run_sgemm(audit, beta=0.0))
    ok(run_sgemm(audit, beta=1.0))
    ok(run_dgemm(audit))
    ok(run_loss(audit))
    for n in (1, 100003):
        ok(run_reductions(audit, n=n))
    r = ok(run_reductions(audit, nan=True))                       # NaN in: NaN out of dot, asum and absmax
    ok(run_axpby(audit))
    for k in (0, 1, 25):
        ok(run_direction(audit, k=k))
    for rank, conv in ((1, False), (128, False), (4, True)):
        ok(run_lora(audit, rank=rank, conv=conv))
    r, res = run_solve(audit)
    ok(r)
    assert set(r.stats.rows) == {'lbfgs_solve_batch|workers=2'}
    assert all(e > 1 for _, e in res)


def test_path_keys():
    rec = {'op': 'mos_transpose_bf16', 'abi': dict(rows=75, C=45, ldx=64)}
    assert sa.solver_path(rec) == 'transpose_bf16|rtail|ctail|strided'
    assert [sa.dgemm_tile(e) for e in (None, '', '0', '1', '2', '3', '7', 'x')] == \
        [sa.dgemm_tile(), '64x64', '64x64', '32x64', '64x64', '64x128', '64x128', '64x64']


def test_reductions_at_the_ff_proj_size():
    """13.1 M elements ([10240, 1280], ff.net.0.proj) through the references of the grid-stride reductions: the bound of
    vec_dot covers an fp32 sum in the kernel's order (per thread, then the trees), and vec_absmax keeps NaN"""
    n = 10240 * 1280
    a, b = rnd((n,), 50), rnd((n,), 51)
    p = a * b                                  # the kernel's fp32 products; thread j sums p[j], p[j + 65536], ... in order
    part = p.view(-1, sa.RED_THREADS)          # n = 200 x 65536: no tail
    t = part[0].clone()
    for row in part[1:]:
        t += row
    got = float(t.view(256, 256).sum(1).sum())
    rec = {'op': 'mos_vec_dot', 'abi': {'n': n}, 'in': {'a': a, 'b': b}}
    r, bnd = sa.reference(rec)['out']
    assert abs(got - float(r)) <= float(bnd)
    assert float(bnd) < 1e-4 * float(p.double().abs().sum())
    a[n - 1] = float('nan')
    r, _ = sa.reference({'op': 'mos_vec_absmax', 'abi': {'n': n, 'scale': 1.0}, 'in': {'a': a}})['out']
    assert torch.isnan(r).all()


# ---------------------------------------------------------------------------------------------------- references
def test_references_vs_torch():
    X, Y = rnd((45, 100), 60), rnd((45, 37), 61)
    ref = sa.reference({'op': 'mos_atb_small', 'abi': dict(n=45, accumulate=0), 'in': {'X': X, 'Y': Y}})['out'][0]
    assert torch.allclose(ref, torch.einsum('ri,rj->ij', X.double(), Y.double()), rtol=0, atol=1e-12)
    A, B = rnd((30, 20), 62), rnd((20, 10), 63, dtype=F64)
    ref = sa.reference({'op': 'mos_dgemm_mixed', 'abi': dict(K=20), 'in': {'A': A, 'B': B}})['C'][0]
    assert torch.allclose(ref, torch.matmul(A.to(F64), B), rtol=0, atol=1e-12)
    W, d, u = rnd((8, 6), 64), rnd((2, 6), 65), rnd((8, 2), 66)
    ref = sa.reference({'op': 'mos_lora_merge', 'abi': dict(n_layers=1, alpha=0.5),
                        'in': {'W0': W, 'down0': d, 'up0': u}})['W0'][0]
    want = W.double() + 0.5 * sum(torch.outer(u[:, r].double(), d[r].double()) for r in range(2))
    assert torch.allclose(ref, want, rtol=0, atol=1e-12)
    x = torch.tensor([1.0, -3.0, float('nan')])
    assert torch.isnan(sa.reference({'op': 'mos_vec_absmax', 'abi': dict(n=3, scale=1.0), 'in': {'a': x}})['out'][0]).all()


@pytest.mark.parametrize('k', [0, 1, 7, 25])
def test_lbfgs_reference_vs_explicit_two_loop_recursion(k):
    """the audit's recursion (with its fp32 coefficients) against torch's own float64 statement (torch.optim.lbfgs:
    q = -g; al_i = rho_i <s_i, q>; q -= al_i y_i; r = h q; be_i = rho_i <y_i, r>; r += (al_i - be_i) s_i)"""
    n = 2000
    g, S, Y, rho, h = history(n, k, seed=70)
    d, e, gtd, eg = sa.lbfgs_reference(g, S, Y, rho, h)
    q = -g.double()
    al = [0.0] * k
    for i in range(k - 1, -1, -1):
        al[i] = float(S[i].double().dot(q)) * rho[i]
        q = q.add(Y[i].double(), alpha=-al[i])
    r = q * float(torch.tensor(h, dtype=F32))
    for i in range(k):
        be = float(Y[i].double().dot(r)) * rho[i]
        r = r.add(S[i].double(), alpha=al[i] - be)
    # the only difference: the audit applies each coefficient rounded to fp32, as the kernel does
    assert ((d - r).abs() <= e).all()
    assert abs(gtd - float(g.double().dot(r))) <= eg
    if k <= 3:                  # the worst-case bound grows geometrically with k (solver_audit.py): tight for short histories
        assert float(e.max()) < 1e-4 * float(r.abs().max())


# ---------------------------------------------------------------------------------------------------- mutations
MUTATIONS = [
    ('transpose_tail', lambda a: run_transpose(a, 'transpose_tail'), 'a'),
    ('atb_ktile', lambda a: run_atb(a, 'atb_ktile'), 'a'),
    ('sgemm_reads_c', lambda a: run_sgemm(a, 'sgemm_reads_c'), 'a'),
    ('dgemm_fp32', lambda a: run_dgemm(a, 'dgemm_fp32'), 'a'),
    ('loss_no_f0', lambda a: run_loss(a, 'loss_no_f0'), 'a'),
    ('dot_drop_partial', lambda a: run_reductions(a, 'dot_drop_partial'), 'a'),
    ('absmax_nan', lambda a: run_reductions(a, 'absmax_nan', nan=True), 'a'),
    ('axpby_reads_y', lambda a: run_axpby(a, 'axpby_reads_y'), 'a'),
    ('dir_prev_coef', lambda a: run_direction(a, 'dir_prev_coef'), 'a'),
    ('dir_no_hdiag', lambda a: run_direction(a, 'dir_no_hdiag'), 'a'),
    ('dir_counter', lambda a: run_direction(a, 'dir_counter'), 'c'),
    ('lora_drop_rank', lambda a: run_lora(a, 'lora_drop_rank'), 'a'),
    ('solve_write_past', lambda a: run_solve(a, 'solve_write_past')[0], 'c'),
    ('solve_swapped_loss', lambda a: run_solve(a, 'solve_swapped_loss')[0], 'ii'),
    ('solve_last_loss', lambda a: run_solve(a, 'solve_last_loss')[0], 'ii'),
]


@pytest.mark.parametrize('mut,run,letter', MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_mutation_flagged_by_its_check(audit, mut, run, letter):
    flagged(run(audit), letter)


def test_preconditions_flagged(audit):
    from mos_b200 import ops
    partial = torch.zeros(260)
    partial.view(torch.int32)[256] = 3
    g, S, Y, rho, h = history(100, 2)
    with audit() as r:
        ops.lbfgs_direction(S, Y, rho, g, h, torch.empty(100), torch.zeros(8, dtype=F64), partial, torch.zeros(1))
    flagged(r, 'p')
    with audit() as r:
        ops.transpose_bf16(rnd((40, 64), 1, dtype=BF), torch.zeros(64, 48, dtype=BF), rows=40, C=64, ldx=32)
    flagged(r, 'p')
