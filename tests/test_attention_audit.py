"""The attention launch audit (tests/attention_audit.py) on the CPU: its float64 reference against
F.scaled_dot_product_attention and autograd, and its checks against a stand-in library that computes the ops with torch.

Launches are made by the real `ops.attention*` / `ops.attn_delta` / `ops.heads_transpose` with CPU tensors, through the
audit's own Recorder, so the records come from the ABI arguments exactly as on the GPU.  The stand-in reads its operands
at the kernels' layouts from those arguments; every mutation case breaks it (or its inputs) the way a faulty kernel or
engine would, and the check it targets must flag it while the unbroken stand-in passes every check.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import attention_audit as aa

F16, BF16 = torch.float16, torch.bfloat16


def rnd(shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dtype)


def _live(S, t):
    base, dtype = t['mem']
    return S.flat(base, dtype).as_strided(t['size'], t['stride'], t['off'])


class StandIn:
    """torch restatement of the six entry points; `mut` names one defect to inject"""

    def __init__(self, mut=None):
        self.mut, self.calls, self.recorder = mut, 0, None

    def _rec(self, entry, args):
        S = aa._Storages(self.recorder._ctx[0])
        return aa.record(entry, aa.abi_of(entry, args[:len(aa._ARGS[entry])]), S), S

    def _fwd(self, entry, args):
        rec, S = self._rec(entry, args)
        a, x = rec['abi'], rec['in']
        d, nq, nk = a['head_dim'], a['nq'], a['nk']
        ext = 1 if self.mut == 'mask+1' else 0                    # reads key nk: K beyond the window is zero-filled
        Q = x['Q'][:, :, :d].double()
        K = F.pad(x['K'][:, :, :d].double(), (0, 0, 0, ext))
        V = x['Vt'][:, :d, :nk + ext].double().transpose(1, 2)
        Sx = (Q @ K.transpose(1, 2)) * a['scale']
        if a['causal']:
            q = torch.arange(nq)[:, None]
            k = torch.arange(nk)[None, :]
            Sx = Sx.masked_fill(k >= q if self.mut == 'causal_diag' else k > q, -math.inf)
        P = torch.softmax(Sx, -1)
        out = P.to(a['dt']).double() @ V
        if self.mut == 'tile':
            out[1, 128:256] *= 1.1
        t = {tt['name']: tt for tt in rec['targets']}
        B, H = a['batch'], a['heads']
        _live(S, t['out']).copy_(out.view(B, H, nq, d))
        if self.mut == 'nondet' and self.calls % 2:                 # the relaunch differs in one last bit
            S.flat(t['out']['mem'][0], torch.int16)[t['out']['off']] ^= 1
        if self.mut == 'write_past':
            S.flat(*t['out']['mem'])[t['out']['off'] + H * d] = 1.0
        if a['lse2']:
            lse = torch.logsumexp(Sx, -1)
            _live(S, t['lse2']).copy_(lse if self.mut == 'lse_ln' else lse / math.log(2))
        if a['probs']:
            _live(S, t['probs']).copy_(P[:, :, :nk])
        if a['pcols']:
            pos = (x['pos'].long().repeat_interleave(H, 0) + (1 if self.mut == 'pcols+1' else 0)).clamp(0, nk - 1)
            _live(S, t['pcols']).copy_(P.gather(2, pos[:, None, :].expand(-1, nq, -1)))
        self.calls += 1
        return 0

    def mos_attention_fwd(self, *args):
        return self._fwd('mos_attention_fwd', args)

    def mos_attention_fwd_train(self, *args):
        return self._fwd('mos_attention_fwd_train', args)

    def mos_attention_fwd_causal(self, *args):
        return self._fwd('mos_attention_fwd_causal', args)

    def mos_attention_bwd(self, *args):
        rec, S = self._rec('mos_attention_bwd', args)
        a, x = rec['abi'], rec['in']
        d, nq, nk, H = a['head_dim'], a['nq'], a['nk'], a['heads']
        Q, dO = x['Qt'][:, :d, :nq].double().transpose(1, 2), x['dOt'][:, :d, :nq].double().transpose(1, 2)
        K, V = x['K'][:, :, :d].double(), x['V'][:, :, :d].double()
        Kt = x['Kt'][:, :d, :nk].double().transpose(1, 2)
        Sx = x['Q'][:, :, :d].double() @ K.transpose(1, 2) * a['scale']
        P = torch.exp(Sx - x['lse2'].double()[:, :, None] * math.log(2))
        if a['causal']:
            P = P.masked_fill(torch.arange(nk)[None, :] > torch.arange(nq)[:, None], 0)
        dP = x['dO'][:, :, :d].double() @ V.transpose(1, 2)
        if a['gcols']:
            pos = x['pos'].long().repeat_interleave(H, 0)
            dP.scatter_add_(2, pos[:, None, :].expand(-1, nq, -1), x['gcols'].double().repeat_interleave(H, 0))
        dS = P * (dP - x['delta'].double()[:, :, None]) * a['scale']
        dq, dk, dv = dS.to(BF16).double() @ Kt, dS.transpose(1, 2).to(BF16).double() @ Q, P.transpose(1, 2).to(BF16).double() @ dO
        B = a['batch']
        if self.mut == 'dv_swap':
            dv = dv.view(B, H, nk, d)[:, [1, 0] + list(range(2, H))].reshape(B * H, nk, d)
        t = {tt['name']: tt for tt in rec['targets']}
        for n, v in (('dq', dq), ('dk', dk), ('dv', dv)):
            _live(S, t[n]).copy_(v.view(B, H, -1, d))
        return 0

    def mos_attn_delta(self, *args):
        rec, S = self._rec('mos_attn_delta', args)
        a, x = rec['abi'], rec['in']
        B, H, d, N = a['batch'], a['heads'], a['head_dim'], a['N']
        O = x['O'].double().reshape(B * H, N, d)
        val = (x['dO'][:, :, :d].double() * O).sum(-1)
        if a['pcols']:
            val += (x['pcols'].double() * x['gcols'].double().repeat_interleave(H, 0)).sum(-1)
        _live(S, rec['targets'][0]).copy_(val)
        return 0

    def mos_heads_transpose(self, *args):
        rec, S = self._rec('mos_heads_transpose', args)
        a = rec['abi']
        _live(S, rec['targets'][0]).copy_(rec['in']['src'][:, :a['R'], :a['DV']].transpose(1, 2))
        return 0


@pytest.fixture
def audit(monkeypatch):
    """audit(mut=None) -> a Recorder over the stand-in library (CPU tensors)"""
    from mos_b200 import _lib, ops
    monkeypatch.setattr(ops, 'current_stream', lambda: None)

    def make(mut=None):
        lib = StandIn(mut)
        monkeypatch.setattr(_lib, 'lib', lambda: lib)
        r = aa.Recorder()
        lib.recorder = r
        return r
    return make


def _only(r):
    """the one launch recorded: its key, its row and the audit's failures"""
    assert len(r.stats.rows) == 1, r.stats.rows
    return next(iter(r.stats.rows)), r.stats.failures


def ok(r):
    assert not r.stats.failures, '\n'.join(r.stats.failures)
    return r


def flagged(r, letter):
    assert any(f'({letter})' in e for e in r.stats.failures), r.stats.failures


# ---------------------------------------------------------------------------------------------------- operands
def heads_rows(B, H, n, d, seed, dtype, scale=1.0, live=None):
    """[B*H, n, DP] rows with zero pad columns (live: columns beyond it are zero too)"""
    t = torch.zeros(B * H, n, aa._r(d, 64), dtype=dtype)
    t[:, :, :live or d] = rnd((B * H, n, live or d), seed, scale, dtype)
    return t


def transposed(rows, d, n8):
    BH, n, _ = rows.shape
    t = torch.zeros(BH, aa._r(d, 16), n8, dtype=rows.dtype)
    t[:, :d, :n] = rows[:, :, :d].transpose(1, 2)
    return t


def fwd_operands(B, H, nq, nk, d, dtype, seed=0, live=None):
    Q = heads_rows(B, H, nq, d, seed, dtype, live=live)
    K = heads_rows(B, H, nk, d, seed + 1, dtype, live=live)
    V = heads_rows(B, H, nk, d, seed + 2, dtype, live=live)
    return Q, K, V, transposed(V, d, aa._r(nk, 8))


def run_fwd(audit, mut=None, B=2, H=2, nq=300, nk=300, d=40, dtype=F16, probs=False, ldo=None):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(B, H, nq, nk, d, dtype)
    ldo = ldo or H * d
    out = torch.zeros(B, nq, ldo, dtype=dtype)
    pr = torch.zeros(B * H, nq, nk) if probs else None
    with audit(mut) as r:
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, probs=pr, ldo=ldo)
    return r


def run_train_fwd(audit, mut=None, B=2, H=2, nq=256, nk=77, d=40, pcols=True):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(B, H, nq, nk, d, BF16, seed=3)
    out = torch.zeros(B, nq, H * d, dtype=BF16)
    lse = torch.zeros(B * H, nq)
    pc = torch.zeros(B * H, nq, 2) if pcols else None
    pos = torch.tensor([[4, 5], [7, 9]], dtype=torch.int32)[:B] if pcols else None
    with audit(mut) as r:
        ops.attention_train(Q, K, Vt, out, lse, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, pcols=pc, pos=pos)
    return r


def run_causal(audit, mut=None, B=2, H=2, n=77):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(B, H, n, n, 80, BF16, seed=5, live=64)
    out = torch.zeros(B, n, H * 80, dtype=BF16)
    lse = torch.zeros(B * H, n)
    with audit(mut) as r:
        ops.attention_causal(Q, K, Vt, out, batch=B, heads=H, head_dim=80, n=n, scale=64 ** -0.5, lse2=lse)
    return r


def bwd_operands(B, H, nq, nk, d, causal=False, gcols=False, seed=10, live=None):
    """Q, K, V, dO rows with the float64 lse2 and delta of the forward they belong to (rounded to fp32)"""
    Q, K, V, _ = fwd_operands(B, H, nq, nk, d, BF16, seed, live=live)
    dO = heads_rows(B, H, nq, d, seed + 3, BF16, 0.5, live=live)
    scale = d ** -0.5 if live is None else live ** -0.5
    Sx = Q[:, :, :d].double() @ K[:, :, :d].double().transpose(1, 2) * scale
    if causal:
        Sx = Sx.masked_fill(torch.arange(nk)[None, :] > torch.arange(nq)[:, None], -math.inf)
    P = torch.softmax(Sx, -1)
    O = P @ V[:, :, :d].double()
    lse2 = (torch.logsumexp(Sx, -1) / math.log(2)).float()
    g = pos = None
    delta = (dO[:, :, :d].double() * O).sum(-1)
    if gcols:
        pos = torch.tensor([[3, 1], [0, 2]], dtype=torch.int32)[:B]
        g = rnd((B, nq, 2), seed + 4, 0.3)
        pc = P.gather(2, pos.long().repeat_interleave(H, 0)[:, None, :].expand(-1, nq, -1))
        delta += (pc * g.double().repeat_interleave(H, 0)).sum(-1)
    return dict(Q=Q, K=K, V=V, dO=dO, O=O, lse2=lse2, delta=delta.float(), gcols=g, pos=pos, scale=scale, P=P)


def run_bwd(audit, mut=None, B=2, H=2, nq=16, nk=16, d=40, causal=False, gcols=False, live=None, ops_=None):
    """the engines' sequence: three heads_transpose launches and the backward writing dq | dk | dv thirds of one
    storage at pitch 3 * H * d; -> (recorder, operands, dqkv)"""
    from mos_b200 import ops
    o = bwd_operands(B, H, nq, nk, d, causal, gcols, live=live)
    C = H * d
    DV = aa._r(d, 16)
    Qt, dOt = (torch.zeros(B * H, DV, aa._r(nq, 8), dtype=BF16) for _ in range(2))
    Kt = torch.zeros(B * H, DV, aa._r(nk, 8), dtype=BF16)
    dqkv = torch.zeros(B * max(nq, nk), 3 * C, dtype=BF16)
    with audit(mut) as r:
        ops.heads_transpose(o['Q'], Qt)
        ops.heads_transpose(o['dO'], dOt)
        ops.heads_transpose(o['K'], Kt)
        if ops_ is not None:
            ops_(o, Qt, Kt, dOt)
        ops.attention_bwd(o['Q'], o['K'], o['V'], o['dO'], Qt, Kt, dOt, o['lse2'], o['delta'], dqkv[:B * nq, :C],
                          dqkv[:B * nk, C:2 * C], dqkv[:B * nk, 2 * C:], batch=B, heads=H, head_dim=d, nq=nq, nk=nk,
                          scale=o['scale'], gcols=o['gcols'], pos=o['pos'], lddq=3 * C, lddk=3 * C, lddv=3 * C,
                          causal=causal)
    return r, o, dqkv


# ------------------------------------------------------------------------------------- reference vs restatements
def _sdpa_check(rec, Q, K, V, d, scale, causal=False):
    assert abs(rec['abi']['scale'] - scale) <= 2 ** -24 * scale
    scale = rec['abi']['scale']                                    # the fp32 value the kernel is given
    want = F.scaled_dot_product_attention(Q[:, :, :d].double(), K[:, :, :d].double(), V[:, :, :d].double(),
                                          is_causal=causal, scale=scale)
    ref = aa.reference(rec)
    assert torch.allclose(ref['out'][0][..., :d], want, rtol=1e-10, atol=1e-12)
    assert not ref['out'][0][..., d:].any()                        # zero columns past the live ones
    return ref


@pytest.mark.parametrize('d', [40, 80, 160])
@pytest.mark.parametrize('nq,nk', [(77, 77), (4, 77), (300, 4)], ids=['T77', 'nq4', 'nk4'])
def test_forward_reference_vs_sdpa(audit, d, nq, nk):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(2, 2, nq, nk, d, F16)
    out = torch.zeros(2, nq, 2 * d, dtype=F16)
    probs = torch.zeros(4, nq, nk) if nk <= 128 else None
    with audit() as r:
        ops.attention(Q, K, Vt, out, batch=2, heads=2, head_dim=d, nq=nq, nk=nk, probs=probs)
    ok(r)
    ref = _sdpa_check(r.last, Q, K, V, d, d ** -0.5)
    if probs is not None:
        S = Q[:, :, :d].double() @ K[:, :, :d].double().transpose(1, 2) * r.last['abi']['scale']
        assert torch.allclose(ref['probs'][0], torch.softmax(S, -1), rtol=1e-12, atol=1e-15)


def test_causal_reference_64_live_columns(audit):
    """CLIP: 64-dim heads run as head_dim 80 (zero columns 64..79), scale 64^-0.5, causal at n = 77, lse2 in log2"""
    r = ok(run_causal(audit))
    rec = r.last
    Q, K, Vt = rec['in']['Q'], rec['in']['K'], rec['in']['Vt']
    V = Vt[:, :80, :77].transpose(1, 2)
    ref = _sdpa_check(rec, Q[:, :, :64], K[:, :, :64], V[:, :, :64].contiguous(), 64, 64 ** -0.5, causal=True)
    S = (Q[:, :, :64].double() @ K[:, :, :64].double().transpose(1, 2)) * 64 ** -0.5
    S = S.masked_fill(torch.arange(77)[None, :] > torch.arange(77)[:, None], -math.inf)
    assert torch.allclose(ref['lse2'][0], torch.logsumexp(S, -1) / math.log(2), rtol=1e-12, atol=1e-12)
    assert _only(r)[0] == 'fwd|bf16|D=80|one|causal|lse2|qtail|ktail'


@pytest.mark.parametrize('d,live,causal', [(40, None, False), (80, None, False), (160, None, False), (80, 64, True)])
@pytest.mark.parametrize('nq,nk', [(77, 77), (4, 4), (16, 77)], ids=['T77', 'n4', 'cross16'])
def test_backward_reference_vs_autograd(audit, d, live, causal, nq, nk):
    """dQ, dK, dV and delta against autograd of  sum(out * dO) + sum(P[:, :, pos] * gcols)  in float64"""
    if causal and nq != nk:
        pytest.skip('causal attention is self-attention')
    from mos_b200 import ops

    def add_delta(o, Qt, Kt, dOt):
        delta = torch.zeros_like(o['delta'])
        B, H = 2, 2
        O = o['O'].view(B, H, nq, d).permute(0, 2, 1, 3).reshape(B, nq, H * d).to(BF16).contiguous()
        pc = o['P'].gather(2, o['pos'].long().repeat_interleave(H, 0)[:, None, :].expand(-1, nq, -1)).float()
        ops.attn_delta(o['dO'], O, delta, batch=B, heads=H, head_dim=d, N=nq, pcols=pc, gcols=o['gcols'])
        Ob = O.double().view(B, nq, H, d).permute(0, 2, 1, 3).reshape(B * H, nq, d)
        o['delta_want'] = (o['dO'][:, :, :d].double() * Ob).sum(-1) + (pc.double() * o['gcols'].double()
                                                                        .repeat_interleave(H, 0)).sum(-1)
        o['delta_rec'] = delta
    gcols = not causal
    r, o, dqkv = run_bwd(audit, nq=nq, nk=nk, d=d, causal=causal, gcols=gcols, live=live,
                         ops_=add_delta if gcols else None)
    ok(r)
    B, H = 2, 2
    q, k, v = (o[n][:, :, :d].double().requires_grad_() for n in ('Q', 'K', 'V'))
    S = q @ k.transpose(1, 2) * o['scale']
    if causal:
        S = S.masked_fill(torch.arange(nk)[None, :] > torch.arange(nq)[:, None], -math.inf)
    P = torch.softmax(S, -1)
    loss = ((P @ v) * o['dO'][:, :, :d].double()).sum()
    if gcols:
        pos = o['pos'].long().repeat_interleave(H, 0)[:, None, :].expand(-1, nq, -1)
        loss = loss + (P.gather(2, pos) * o['gcols'].double().repeat_interleave(H, 0)).sum()
    loss.backward()
    rec = r.last
    ref = aa.reference(rec)
    for n, g in (('dq', q.grad), ('dk', k.grad), ('dv', v.grad)):
        assert torch.allclose(ref[n][0], g, rtol=1e-5, atol=1e-6 * g.abs().max().item()), n
    if gcols:
        assert torch.allclose(o['delta_rec'].double(), o['delta_want'], rtol=1e-6, atol=1e-7)


def test_transpose_and_delta_keys(audit):
    r, o, _ = run_bwd(audit, nq=4, nk=77, d=160)
    ok(r)
    assert set(r.stats.rows) == {'transpose|DP=192|DV=160|rtail', 'transpose|DP=192|DV=160|rtail',
                                 'bwd|bf16|D=160|multi|qtail|ktail'}


def test_path_keys(audit):
    assert _only(ok(run_fwd(audit)))[0] == 'fwd|fp16|D=40|multi|qtail|ktail'
    assert _only(ok(run_fwd(audit, nq=256, nk=77, probs=True)))[0] == 'fwd|fp16|D=40|one|probs|ktail'
    assert _only(ok(run_fwd(audit, nq=256, nk=77, d=80)))[0] == 'fwd|fp16|D=80|multi|ktail'
    assert _only(ok(run_fwd(audit, nq=288, nk=288, d=160)))[0] == 'fwd|fp16|D=160|multi|qtail|ktail'
    assert _only(ok(run_train_fwd(audit)))[0] == 'fwd|bf16|D=40|one|lse2|pcols|ktail'


def test_stand_in_passes_every_check(audit):
    """the unbroken stand-in: pitched output, 288-token tails, training forward with pcols, a 16-token backward with gcols"""
    ok(run_fwd(audit, ldo=2 * 40 + 16))
    ok(run_fwd(audit, nq=288, nk=288, d=160, dtype=BF16))
    ok(run_train_fwd(audit))
    r, _, _ = run_bwd(audit, gcols=True)
    ok(r)


# -------------------------------------------------------------------------------------------------- mutation cases
def test_mutation_one_tile_scaled(audit):
    r = run_fwd(audit, 'tile')
    flagged(r, 'a')
    flagged(r, 'b')


def test_mutation_key_mask_off_by_one(audit):
    flagged(run_fwd(audit, 'mask+1', nq=128, nk=77), 'a')


def test_mutation_causal_diagonal_excluded(audit):
    flagged(run_causal(audit, 'causal_diag'), 'a')


def test_mutation_pcols_one_column_late(audit):
    flagged(run_train_fwd(audit, 'pcols+1'), 'a')


def test_mutation_lse2_natural_log(audit):
    flagged(run_train_fwd(audit, 'lse_ln'), 'a')


def test_mutation_dv_heads_swapped(audit):
    flagged(run_bwd(audit, 'dv_swap')[0], 'a')


def test_mutation_write_past_heads_columns(audit):
    r = run_fwd(audit, 'write_past', ldo=2 * 40 + 16)
    flagged(r, 'c')


def test_mutation_nonzero_q_pad_column(audit):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(2, 2, 128, 77, 40, F16)
    Q[3, 17, 41] = 0.5
    with audit() as r:
        ops.attention(Q, K, Vt, torch.zeros(2, 128, 80, dtype=F16), batch=2, heads=2, head_dim=40, nq=128, nk=77)
    flagged(r, 'p')


def test_mutation_vt_pad_token_nan(audit):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(2, 2, 128, 77, 40, F16)
    Vt[1, 5, 78] = math.nan
    with audit() as r:
        ops.attention(Q, K, Vt, torch.zeros(2, 128, 80, dtype=F16), batch=2, heads=2, head_dim=40, nq=128, nk=77)
    flagged(r, 'p')


def test_mutation_stale_qt(audit):
    """Qt transposed from another layer's Q: the backward's precondition fails"""
    def stale(o, Qt, Kt, dOt):
        Qt.copy_(transposed(heads_rows(2, 2, 16, 40, 99, BF16), 40, Qt.shape[2]))
    flagged(run_bwd(audit, ops_=stale)[0], 'p')


def test_mutation_nondeterministic_relaunch(audit):
    flagged(run_fwd(audit, 'nondet'), 'e')


def test_pos_out_of_range(audit):
    from mos_b200 import ops
    Q, K, V, Vt = fwd_operands(1, 2, 64, 77, 40, BF16)
    with audit() as r:
        ops.attention_train(Q, K, Vt, torch.zeros(1, 64, 80, dtype=BF16), torch.zeros(2, 64), batch=1, heads=2,
                            head_dim=40, nq=64, nk=77, pcols=torch.zeros(2, 64, 2),
                            pos=torch.tensor([[3, 77]], dtype=torch.int32))
    flagged(r, 'p')
