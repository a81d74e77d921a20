"""Launch audit of the attention family: every `ops.attention` / `ops.attention_train` / `ops.attention_causal` /
`ops.attention_bwd` / `ops.attn_delta` / `ops.heads_transpose` call of a real engine walk, checked on its own.

A launch record is built from the arguments that reach the `mos_*` entry point (pointers, `ldo` / `ldd*`, `nk8` / `nq8`,
`head_dim`, `scale`, `act_dtype`), not from the Python views the engine passed: every pointer is mapped into the storage of
a tensor argument and the windows are read there at the kernels' layouts (DP = roundup(d, 64), DV = roundup(d, 16)):

    Q, K (and V, dO in the backward)  [B*H, n, DP]          rows, pad columns [d, DP) zero
    Vt, Qt, Kt, dOt                   [B*H, DV, n8]         transposed, pad rows [d, DV) and pad tokens [n, n8) zero
    out, dq, dk, dv                   [B, n, ld]            head h at columns [h*d, (h+1)*d)
    lse2, delta [B*H, nq]; probs [B*H, nq, nk]; pcols [B*H, nq, 2]; gcols [B, nq, 2]; pos int32 [B, 2]

Record layout: {'op': 'fwd' | 'bwd' | 'delta' | 'transpose', 'abi': {...}, 'in': {operand windows},
'targets': [{'name', 'mem', 'off', 'size', 'stride'}], 'pre': [(p) messages], 'mem': {storage: {'before', 'after'}}}.
`reference` and `check_launch` are pure functions of a record (they run on CPU tensors too).

Float64 reference (the launch's own inputs, so each launch is checked in isolation), c = scale * log2(e):
- forward: X = c Q_d K_d^T over the first d columns (causal: keys > query masked), P = softmax, out = P V,
  lse2 = log2 sum_k 2^X_k, probs = P, pcols[bh, q, i] = P[bh, q, pos[b][i]];
- backward: P = 2^(X - lse2) with the lse2 the launch was given, dP = dO V^T + G (G: gcols at the pos columns),
  dS = P o (dP - delta), dQ = scale dS K, dK = scale dS^T Q, dV = P^T dO;
- attn_delta: sum_j dO O + sum_i pcols gcols;  heads_transpose: dst[bh, j, r] = src[bh, r, j] for j < DV, r < R (exact).

Element bound (a), derived from the kernels' roundings (u = 2^-24 fp32, u16 = 2^-8 bf16 / 2^-11 fp16, u_ex2 = 2^-22 the
relative error of ex2.approx.ftz.f32, T the number of key tiles of the launch):
- logits: the fp32 QK^T has d exact products (16-bit x 16-bit fits fp32) and d - 1 additions; the fp32 c costs two more
  roundings and the scaling one: |dX_k| <= e_k = (d + 4) u |c| sum_i |Q_i K_ki|.
- p_k = ex2(X_k - m): the subtraction rounds (u |X_k - m|), ex2 adds u_ex2, and the online rescales multiply tile j's terms
  by at most T factors ex2(m_old - m_new) (u_ex2 + 2u each).  A common factor of a tile's terms in O and in l cancels
  except for its spread, so every error is a relative error of p_k:
      delta_k = ln2 (e_k + u |X_k - m|) + u_ex2 + T (u_ex2 + 2u).
  ex2 flushes results below 2^-126 and P is rounded to the activation type before PV (relative u16, absolute t16 =
  2^-25 fp16 subnormal half-step / 2^-126 bf16); p_k <= 1 relative to the running max and l >= 1, so these stay absolute.
- out_j = sum_k p_k V_kj / sum_k p_k: with A_j = sum_k P_k |V_kj|, D = sum_k P_k delta_k and nk + 2T + 8 fp32 roundings in
  each sum and the normalisation,
      |out - ref| <= u16 |ref| + (1 + u16) [u16 A_j + sum_k P_k delta_k |V_kj| + D |ref| + (nk + 2T + 8) u (A_j + |ref|)
                                             + t16 sum_k |V_kj|]
  (the first u16 is the output rounding).
- lse2 = m + log2f(l): (D + (nk + 2T + 8) u) / ln2 + 2u (|lse2| + |log2 l|) (log2f: 1 ulp, the final add: 1 ulp).
- probs / pcols (fp32, one key tile): P_k (delta_k + D + (nk + 10) u) + 2^-126.
- backward: P_k = ex2(fma(S, c, -lse2)) has delta_k = ln2 (e_k + u |X_k - lse2|) + u_ex2, plus 2^-126 absolute; dP has
  (d + 1) u sum_i |dO_i V_ki|, the + G and - delta one u each; dS = P (dP + G - delta) scale two more.  dS (dQ, dK) and P
  (dV) are rounded to bf16 before their wgmma (u16 of the value), the products accumulate in fp32 over nk (dQ) or
  nq (dK, dV) terms, and the output is rounded to bf16:
      |dQ - ref| <= u16 |ref| + (1 + u16) sum_k (E_k + (nk + 8) u (|dS_k| + E_k)) |K_k|,
      E_k = (1 + u16) e(dS_k) + u16 |dS_k|,  and likewise dK (over queries, |Q|) and dV (P for dS, |dO|).
- attn_delta: (d + 4) u (sum_j |dO O| + sum_i |pcols gcols|).
The bound grows with the magnitude sums, not with the values; a ratio above 1 is a finding, not a reason to widen it.

Checks of every launch (`check_launch`):
  p. the bytes the kernel is about to read: every pad above is zero (bitwise: -0.0 and NaN are not), pos lies in [0, nk),
     and in the backward Qt / Kt / dOt equal the transposes of the Q / K / dO windows bit for bit (with zero pads); the
     heads_transpose destination's pad tokens are zero before the launch (the kernel leaves them);
  a. the element bound above for out, lse2, probs, pcols, delta, dQ, dK, dV; heads_transpose bit-exact;
  b. rel-L2 per (bh, 128-query tile) (dK, dV: per 128-key tile) within the existing tests' limits: out 8e-3 (bf16) /
     1e-3 (fp16), probs and pcols 1e-4, lse2 2e-3 absolute (RMS), backward and delta 2e-2;
  c. every byte of a written storage outside the launch's window is bitwise unchanged.
The recorder adds (d) the operand windows are unchanged by the launch and (e) one more launch from the same bytes is
bit-identical (the backward uses no atomics).
"""
import math

import torch

import gemm_audit as ga
from gemm_audit import Stats, _Storages  # noqa: F401  (Stats is the table of both audits)

U32 = 2.0 ** -24
U_EX2 = 2.0 ** -22
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
FTZ = 2.0 ** -126
U16 = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
T16 = {torch.bfloat16: FTZ, torch.float16: 2.0 ** -25}
TINY_OUT = ga.TINY_OUT
DT16 = ga.DT16
QT = 128                       # query tile of the forward kernel and of the dQ kernel; key tile of the dK / dV kernel
BT_BWD = 64                    # inner tile of both backward kernels
TILE_TOL = {'out': {torch.bfloat16: 8e-3, torch.float16: 1e-3}, 'probs': 1e-4, 'pcols': 1e-4, 'lse2': 2e-3,
            'dq': 2e-2, 'dk': 2e-2, 'dv': 2e-2, 'delta': 2e-2}
CHUNK_ELEMS = 1 << 26          # float64 elements of one [B*H, queries, keys] block of the reference
_BITS = ga._BITS


def _r(x, m):
    return (x + m - 1) // m * m


# --------------------------------------------------------------------------------------------------- path keys
def fwd_one(a):
    """launch_attn's ONE (one 128-key tile, probabilities in registers): d = 40 / 160 with nk <= 128, and causal"""
    return a['causal'] or (a['head_dim'] != 80 and a['nk'] <= 128)


def fwd_bkv(a):
    """the forward kernel's key tile (AttnCfg::BKV)"""
    return 128 if fwd_one(a) or a['head_dim'] <= 80 else 64


def attn_path(rec):
    """Path key of a launch: the features that select code in csrc/attention.cu, attention_bwd.cu and backward.cu
    (a copy of their host rules; keep them in step)."""
    a = rec['abi']
    if rec['op'] == 'transpose':
        return f"transpose|DP={a['DP']}|DV={a['DV']}" + ('|rtail' if a['R'] % 8 else '')
    if rec['op'] == 'delta':
        return f"delta|D={a['head_dim']}" + ('|pcols' if a['pcols'] else '')
    dt = 'fp16' if a['dt'] == torch.float16 else 'bf16'
    if rec['op'] == 'fwd':
        key = ['fwd', dt, f"D={a['head_dim']}", 'one' if fwd_one(a) else 'multi']
        bkv = fwd_bkv(a)
        flags = ['causal'] * a['causal'] + ['probs'] * bool(a['probs']) + ['lse2'] * bool(a['lse2']) + \
            ['pcols'] * bool(a['pcols'])
    else:
        key = ['bwd', dt, f"D={a['head_dim']}", 'one' if a['nk'] <= BT_BWD else 'multi']
        bkv = BT_BWD
        flags = ['causal'] * a['causal'] + ['gcols'] * bool(a['gcols'])
    flags += ['qtail'] * (a['nq'] % QT != 0) + ['ktail'] * (a['nk'] % bkv != 0)
    return '|'.join(key + flags)


# --------------------------------------------------------------------------------------------------- reference
def _bh_rows(t, heads):
    """[B, ...] per-batch operand -> [B*H, ...]"""
    return t.repeat_interleave(heads, 0)


def _gcols_dense(rec, q0, q1, nk, dev):
    """G [BH, q1 - q0, nk]: gcols[b, q, i] at key column pos[b][i]"""
    a, x = rec['abi'], rec['in']
    BH = a['batch'] * a['heads']
    G = torch.zeros(BH, q1 - q0, nk, dtype=torch.float64, device=dev)
    if x.get('gcols') is None:
        return G
    g = _bh_rows(x['gcols'][:, q0:q1].double(), a['heads'])               # [BH, qc, 2]
    pos = _bh_rows(x['pos'].long().clamp(0, nk - 1), a['heads'])           # [BH, 2]
    G.scatter_add_(2, pos[:, None, :].expand(-1, q1 - q0, -1), g)
    return G


def _q_chunk(rec, nk):
    a = rec['abi']
    BH = a['batch'] * a['heads']
    return max(QT, CHUNK_ELEMS // max(BH * nk, 1) // QT * QT)


def _causal_mask(q0, q1, nk, dev):
    q = torch.arange(q0, q1, device=dev)[:, None]
    return torch.arange(nk, device=dev)[None, :] > q                       # True: masked


def _fwd_reference(rec):
    a, x = rec['abi'], rec['in']
    d, nq, nk, dt = a['head_dim'], a['nq'], a['nk'], a['dt']
    u16, t16 = U16[dt], T16[dt]
    c = a['scale'] * LOG2E
    T = 1 if fwd_one(a) else -(-nk // fwd_bkv(a))
    K = x['K'][:, :, :d].double()
    V = x['Vt'][:, :d, :nk].double().transpose(1, 2)                       # [BH, nk, d]
    Va = V.abs()
    Vsum = Va.sum(1, keepdim=True)                                          # [BH, 1, d]
    nacc = nk + 2 * T + 8
    res = {k: [] for k in ('out', 'lse2', 'probs', 'pcols')}
    step = _q_chunk(rec, nk)
    for q0 in range(0, nq, step):
        q1 = min(nq, q0 + step)
        Qc = x['Q'][:, q0:q1, :d].double()
        X = c * (Qc @ K.transpose(1, 2))
        MS = abs(c) * (Qc.abs() @ K.abs().transpose(1, 2))
        live = torch.ones_like(X, dtype=torch.bool)
        if a['causal']:
            live = ~_causal_mask(q0, q1, nk, X.device).expand_as(X)
            X.masked_fill_(~live, -math.inf)
        m = X.amax(-1, keepdim=True)
        E = torch.exp2(X - m)
        l = E.sum(-1, keepdim=True)
        P = E / l
        dlt = LN2 * ((d + 4) * U32 * MS + U32 * (X - m).abs()) + U_EX2 + T * (U_EX2 + 2 * U32)
        PD = torch.where(live, P * dlt, torch.zeros_like(P))
        Dsum = PD.sum(-1, keepdim=True)
        out = P @ V
        A = P @ Va
        acc = u16 * A + PD @ Va + Dsum * out.abs() + nacc * U32 * (A + out.abs()) + t16 * Vsum
        res['out'].append((out, u16 * out.abs() + (1 + u16) * acc + TINY_OUT[dt]))
        if a['lse2']:
            lse = (m + torch.log2(l)).squeeze(-1)
            b = LOG2E * (Dsum.squeeze(-1) + nacc * U32) + 2 * U32 * (lse.abs() + torch.log2(l).squeeze(-1).abs())
            res['lse2'].append((lse, b + 2 ** -40))
        if a['probs'] or a['pcols']:
            Pb = P * (torch.where(live, dlt, torch.zeros_like(dlt)) + Dsum + (nk + 10) * U32) + FTZ
            if a['probs']:
                res['probs'].append((P, Pb))
            if a['pcols']:
                pos = _bh_rows(x['pos'].long().clamp(0, nk - 1), a['heads'])[:, None, :].expand(-1, q1 - q0, -1)
                res['pcols'].append((P.gather(2, pos), Pb.gather(2, pos)))
    out = {}
    for k, v in res.items():
        if v:
            out[k] = (torch.cat([r for r, _ in v], 1), torch.cat([b for _, b in v], 1))
    return out


def _bwd_reference(rec):
    a, x = rec['abi'], rec['in']
    d, nq, nk = a['head_dim'], a['nq'], a['nk']
    ub = U16[torch.bfloat16]
    scale = a['scale']
    c = scale * LOG2E
    Q, K, V, dO = (x[k][:, :, :d].double() for k in ('Q', 'K', 'V', 'dO'))
    Ka, Va = K.abs(), V.abs()
    lse, dl = x['lse2'].double(), x['delta'].double()
    dK, dV = torch.zeros_like(K), torch.zeros_like(K)
    dKb, dVb = torch.zeros_like(K), torch.zeros_like(K)
    dQ, dQb = [], []
    step = _q_chunk(rec, nk)
    for q0 in range(0, nq, step):
        q1 = min(nq, q0 + step)
        Qc, dOc = Q[:, q0:q1], dO[:, q0:q1]
        Xl = c * (Qc @ K.transpose(1, 2)) - lse[:, q0:q1, None]
        MS = abs(c) * (Qc.abs() @ Ka.transpose(1, 2))
        live = torch.ones_like(Xl, dtype=torch.bool)
        if a['causal']:
            live = ~_causal_mask(q0, q1, nk, Xl.device).expand_as(Xl)
        P = torch.where(live, torch.exp2(Xl), torch.zeros_like(Xl))
        Perr = torch.where(live, P * (LN2 * ((d + 4) * U32 * MS + U32 * Xl.abs()) + U_EX2) + FTZ, torch.zeros_like(P))
        dP = dOc @ V.transpose(1, 2) + _gcols_dense(rec, q0, q1, nk, Xl.device)
        Dv = dP - dl[:, q0:q1, None]
        eD = (d + 1) * U32 * (dOc.abs() @ Va.transpose(1, 2)) + U32 * dP.abs() + U32 * Dv.abs()
        dS = scale * P * Dv
        dSa = dS.abs()
        eS = scale * (Perr * Dv.abs() + P * eD + 2 * U32 * P * Dv.abs())
        ES = (1 + ub) * eS + ub * dSa + 2.0 ** -134
        EP = (1 + ub) * Perr + ub * P
        dQ.append(dS @ K)
        dQb.append((ES + (nk + 8) * U32 * (dSa + ES)) @ Ka)
        dK += dS.transpose(1, 2) @ Qc
        dKb += (ES + (nq + 8) * U32 * (dSa + ES)).transpose(1, 2) @ Qc.abs()
        dV += P.transpose(1, 2) @ dOc
        dVb += (EP + (nq + 8) * U32 * (P + EP)).transpose(1, 2) @ dOc.abs()
    dQ, dQb = torch.cat(dQ, 1), torch.cat(dQb, 1)
    to = TINY_OUT[torch.bfloat16]
    return {k: (r, ub * r.abs() + (1 + ub) * b + to) for k, r, b in (('dq', dQ, dQb), ('dk', dK, dKb), ('dv', dV, dVb))}


def _delta_reference(rec):
    a, x = rec['abi'], rec['in']
    B, H, d, N = a['batch'], a['heads'], a['head_dim'], a['N']
    dO = x['dO'][:, :, :d].double()                                          # [BH, N, d]
    O = x['O'].double().reshape(B * H, N, d)                                 # window [B, H, N, d]
    val, mag = (dO * O).sum(-1), (dO * O).abs().sum(-1)
    if x.get('pcols') is not None:
        pg = x['pcols'].double() * _bh_rows(x['gcols'].double(), H)
        val, mag = val + pg.sum(-1), mag + pg.abs().sum(-1)
    return {'delta': (val, U32 * val.abs() + (d + 4) * U32 * mag + TINY_OUT[torch.float32])}


def reference(rec):
    """float64 reference of every output target: {name: (ref, bound)}; heads_transpose: {name: (ref, None)} (exact)"""
    if rec['op'] == 'fwd':
        return _fwd_reference(rec)
    if rec['op'] == 'bwd':
        return _bwd_reference(rec)
    if rec['op'] == 'delta':
        return _delta_reference(rec)
    a = rec['abi']
    return {'dst': (rec['in']['src'][:, :a['R'], :a['DV']].transpose(1, 2), None)}


# --------------------------------------------------------------------------------------------------- checks
def window(rec, t, which):
    """target t of the 'before' / 'after' storage as its strided window"""
    return rec['mem'][t['mem']][which].as_strided(t['size'], t['stride'], t['off'])


def canonical(rec, t, w):
    """a target window in the reference's shape: [B, H, n, d] views -> [B*H, n, d]"""
    if len(t['size']) == 4:
        return w.reshape(t['size'][0] * t['size'][1], t['size'][2], t['size'][3])
    return w


def _tile_tol(rec, name):
    tol = TILE_TOL[name]
    return tol[rec['abi']['dt']] if isinstance(tol, dict) else tol


def check_launch(rec):
    """Checks (p) and (a)-(c) of one launch.  -> {'ratio': worst error / bound, 'tile_rel': worst tile rel-L2,
    'tile': worst fraction of the tile limit, 'errors': [messages]}"""
    errors = list(rec.get('pre', ()))
    ratio, worst_rel, worst_frac = 0.0, 0.0, 0.0
    refs = reference(rec)
    masks = {k: torch.zeros(st['after'].numel(), dtype=torch.bool, device=st['after'].device)
             for k, st in rec['mem'].items()}
    for t in rec['targets']:
        name = t['name']
        masks[t['mem']].as_strided(t['size'], t['stride'], t['off']).fill_(True)
        got = canonical(rec, t, window(rec, t, 'after'))
        ref, bound = refs[name]
        if bound is None:                                                   # exact copy
            if not torch.equal(got.reshape(-1).view(_BITS[got.element_size()]),
                               ref.reshape(-1).view(_BITS[ref.element_size()])):
                errors.append(f'(a) {name}: the transposed window differs from the source')
            continue
        gd = got.double()
        err = (gd - ref).abs()
        bad = ~(err <= bound)                                               # NaN counts as bad
        if bad.any():
            i = tuple(int(v) for v in bad.nonzero()[0])
            errors.append(f'(a) {name}: {int(bad.sum())} elements out of bound, first at {i}: got {gd[i].item():.6g} '
                          f'want {ref[i].item():.6g} bound {bound[i].item():.3g}')
        ratio = max(ratio, (err / bound).nan_to_num(nan=math.inf).max().item())
        # (b) per (bh, 128-row tile) of dimension 1 (queries; keys for dK / dV)
        n = got.shape[1]
        nt = -(-n // QT)
        pad = nt * QT - n
        e2 = torch.nn.functional.pad((err * err).reshape(got.shape[0], n, -1), (0, 0, 0, pad))
        r2 = torch.nn.functional.pad((ref * ref).reshape(got.shape[0], n, -1), (0, 0, 0, pad))
        e2 = e2.reshape(got.shape[0], nt, -1).sum(-1)       # reshape: the window may be a strided view (B = 1)
        if name == 'lse2':                                                  # absolute RMS per tile
            cnt = torch.full((nt,), float(QT), dtype=torch.float64, device=e2.device)
            cnt[-1] = QT - pad
            rel = (e2 / cnt).sqrt()
        else:
            r2 = r2.reshape(got.shape[0], nt, -1).sum(-1)
            rel = torch.where(e2 == 0, torch.zeros_like(e2), e2.sqrt() / r2.sqrt())
        rel = rel.nan_to_num(nan=math.inf)
        tol = _tile_tol(rec, name)
        worst_rel = max(worst_rel, rel.max().item())
        frac = rel.max().item() / tol
        worst_frac = max(worst_frac, frac)
        if not frac <= 1:
            bh, ti = divmod(int(rel.argmax()), nt)
            errors.append(f'(b) {name}: tile (bh {bh}, rows {ti * QT}..) rel-L2 {rel.max().item():.3e} > {tol:.1e}')
    for k, st in rec['mem'].items():
        es = st['after'].element_size()
        stray = (st['after'].view(_BITS[es]) != st['before'].view(_BITS[es])) & ~masks[k]
        if stray.any():
            errors.append(f'(c) storage {k[1]}: {int(stray.sum())} elements written outside the window, first at flat '
                          f'index {int(stray.nonzero()[0])}')
    return {'ratio': ratio, 'tile_rel': worst_rel, 'tile': worst_frac, 'errors': errors}


def simulate(rec):
    """Write the rounded reference into the 'after' storages: what a correct kernel leaves."""
    for st in rec['mem'].values():
        st['after'] = st['before'].clone()
    refs = reference(rec)
    for t in rec['targets']:
        w = window(rec, t, 'after')
        r = refs[t['name']][0]
        w.copy_(r.reshape(w.shape) if len(t['size']) == 4 else r)
    return rec


# --------------------------------------------------------------------------------------------------- records
_ARGS = {
    'mos_attention_fwd': ('Q', 'K', 'Vt', 'out', 'ldo', 'probs', 'batch', 'heads', 'head_dim', 'nq', 'nk', 'nk8',
                          'scale', 'act_dtype'),
    'mos_attention_fwd_train': ('Q', 'K', 'Vt', 'out', 'ldo', 'lse2', 'pcols', 'pos', 'batch', 'heads', 'head_dim',
                                'nq', 'nk', 'nk8', 'scale'),
    'mos_attention_fwd_causal': ('Q', 'K', 'Vt', 'out', 'ldo', 'batch', 'heads', 'head_dim', 'nq', 'nk8', 'scale',
                                 'lse2'),
    'mos_attention_bwd': ('Q', 'K', 'V', 'dO', 'Qt', 'Kt', 'dOt', 'lse2', 'delta', 'gcols', 'pos', 'dq', 'lddq', 'dk',
                          'lddk', 'dv', 'lddv', 'batch', 'heads', 'head_dim', 'nq', 'nk', 'nq8', 'nk8', 'scale',
                          'causal'),
    'mos_heads_transpose': ('src', 'BH', 'R', 'DP', 'DV', 'R8', 'dst'),
    'mos_attn_delta': ('dO', 'DP', 'O', 'ldo', 'batch', 'heads', 'head_dim', 'N', 'pcols', 'gcols', 'delta'),
}
ENTRY_POINTS = tuple(_ARGS)


def abi_of(entry, args):
    """the ctypes arguments of an entry point -> plain dict (pointers as ints, 0 for NULL; scale as the fp32 value)"""
    names = _ARGS[entry]
    a = {}
    for n, v in zip(names, args):
        v = getattr(v, 'value', v)
        a[n] = (0 if v is None else v) if n == 'scale' else (0 if v is None else int(v))
    if entry == 'mos_attention_fwd_causal':
        a['nk'] = a['nq']
        a['causal'] = 1
    if entry == 'mos_attention_fwd':
        a['dt'] = DT16[a.pop('act_dtype')]
    elif entry in ('mos_attention_fwd_train', 'mos_attention_fwd_causal', 'mos_attention_bwd'):
        a['dt'] = torch.bfloat16                                            # both are built for bf16 only
    for k in ('probs', 'lse2', 'pcols', 'pos', 'gcols', 'causal'):
        a.setdefault(k, 0)
    return a


def _bitnz(t):
    return (t.reshape(-1).view(_BITS[t.element_size()]) != 0).any().item() if t.numel() else False


def _pad_checks(pre, what, rows, d):
    """rows [BH, n, DP]: pad columns [d, DP) zero"""
    if _bitnz(rows[:, :, d:]):
        pre.append(f'(p) {what}: pad columns [{d}, {rows.shape[2]}) not zero')


def _transposed_checks(pre, what, tr, rows, d, n):
    """tr [BH, DV, n8] must be the bitwise transpose of rows[:, :n, :DV], pad rows [d, DV) and pad tokens [n, n8) zero"""
    DV = tr.shape[1]
    if _bitnz(tr[:, d:, :]):
        pre.append(f'(p) {what}: pad rows [{d}, {DV}) not zero')
    if _bitnz(tr[:, :, n:]):
        pre.append(f'(p) {what}: pad tokens [{n}, {tr.shape[2]}) not zero')
    if rows is not None:
        want = rows[:, :n, :d].transpose(1, 2)
        if not torch.equal(tr[:, :d, :n].reshape(-1).view(torch.int16), want.reshape(-1).view(torch.int16)):
            pre.append(f'(p) {what}: not the transpose of the rows passed')


def _pos_check(pre, pos, nk):
    if pos is not None and pos.numel() and not ((pos >= 0) & (pos < nk)).all():
        pre.append(f'(p) pos {pos.tolist()} not in [0, {nk})')


def record(entry, abi, S):
    """the launch record of one entry-point call (operand windows and written storages still live)"""
    a = abi
    x, targets, pre = {}, [], []

    def target(p, what, name, dtype, size, stride):
        base, off = S.find(p, what)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{what}: pointer not aligned to its element size'
        t = dict(name=name, mem=(base, dtype), off=off // es, size=tuple(size), stride=tuple(stride))
        S.flat(base, dtype).as_strided(t['size'], t['stride'], t['off'])     # raises if it runs past its storage
        targets.append(t)

    if entry == 'mos_heads_transpose':
        BH, R, DP, DV, R8 = a['BH'], a['R'], a['DP'], a['DV'], a['R8']
        x['src'] = S.window(a['src'], 'src', torch.bfloat16, (BH, R, DP), (R * DP, DP, 1))
        dst = S.window(a['dst'], 'dst', torch.bfloat16, (BH, DV, R8), (DV * R8, R8, 1))
        if _bitnz(dst[:, :, R:]):
            pre.append(f'(p) dst: pad tokens [{R}, {R8}) not zero before the launch')
        target(a['dst'], 'dst', 'dst', torch.bfloat16, (BH, DV, R), (DV * R8, R8, 1))
        return {'op': 'transpose', 'abi': a, 'in': x, 'targets': targets, 'pre': pre}
    B, H, d = a['batch'], a['heads'], a['head_dim']
    BH, DP, DV = B * H, _r(d, 64), _r(d, 16)
    bf = torch.bfloat16
    if entry == 'mos_attn_delta':
        N = a['N']
        x['dO'] = S.window(a['dO'], 'dO', bf, (BH, N, a['DP']), (N * a['DP'], a['DP'], 1))
        x['O'] = S.window(a['O'], 'O', bf, (B, H, N, d), (N * a['ldo'], d, a['ldo'], 1))
        if a['pcols']:
            x['pcols'] = S.window(a['pcols'], 'pcols', torch.float32, (BH, N, 2), (2 * N, 2, 1))
            x['gcols'] = S.window(a['gcols'], 'gcols', torch.float32, (B, N, 2), (2 * N, 2, 1))
        target(a['delta'], 'delta', 'delta', torch.float32, (BH, N), (N, 1))
        return {'op': 'delta', 'abi': a, 'in': x, 'targets': targets, 'pre': pre}
    dt = a['dt']
    nq, nk = a['nq'], a['nk']
    if entry == 'mos_attention_bwd':
        for k, n in (('Q', nq), ('K', nk), ('V', nk), ('dO', nq)):
            x[k] = S.window(a[k], k, bf, (BH, n, DP), (n * DP, DP, 1))
            _pad_checks(pre, k, x[k], d)
        for k, src, n, n8 in (('Qt', 'Q', nq, a['nq8']), ('Kt', 'K', nk, a['nk8']), ('dOt', 'dO', nq, a['nq8'])):
            x[k] = S.window(a[k], k, bf, (BH, DV, n8), (DV * n8, n8, 1))
            _transposed_checks(pre, k, x[k], x[src], d, n)
        x['lse2'] = S.window(a['lse2'], 'lse2', torch.float32, (BH, nq), (nq, 1))
        x['delta'] = S.window(a['delta'], 'delta', torch.float32, (BH, nq), (nq, 1))
        if a['gcols']:
            x['gcols'] = S.window(a['gcols'], 'gcols', torch.float32, (B, nq, 2), (2 * nq, 2, 1))
            x['pos'] = S.window(a['pos'], 'pos', torch.int32, (B, 2), (2, 1))
            _pos_check(pre, x['pos'], nk)
        for k, n in (('dq', nq), ('dk', nk), ('dv', nk)):
            ld = a['ld' + k]
            target(a[k], k, k, bf, (B, H, n, d), (n * ld, d, ld, 1))
        return {'op': 'bwd', 'abi': a, 'in': x, 'targets': targets, 'pre': pre}
    x['Q'] = S.window(a['Q'], 'Q', dt, (BH, nq, DP), (nq * DP, DP, 1))
    x['K'] = S.window(a['K'], 'K', dt, (BH, nk, DP), (nk * DP, DP, 1))
    x['Vt'] = S.window(a['Vt'], 'Vt', dt, (BH, DV, a['nk8']), (DV * a['nk8'], a['nk8'], 1))
    _pad_checks(pre, 'Q', x['Q'], d)
    _pad_checks(pre, 'K', x['K'], d)
    _transposed_checks(pre, 'Vt', x['Vt'], None, d, nk)
    if a['pcols']:
        x['pos'] = S.window(a['pos'], 'pos', torch.int32, (B, 2), (2, 1))
        _pos_check(pre, x['pos'], nk)
    target(a['out'], 'out', 'out', dt, (B, H, nq, d), (nq * a['ldo'], d, a['ldo'], 1))
    if a['lse2']:
        target(a['lse2'], 'lse2', 'lse2', torch.float32, (BH, nq), (nq, 1))
    if a['probs']:
        target(a['probs'], 'probs', 'probs', torch.float32, (BH, nq, nk), (nq * nk, nk, 1))
    if a['pcols']:
        target(a['pcols'], 'pcols', 'pcols', torch.float32, (BH, nq, 2), (2 * nq, 2, 1))
    return {'op': 'fwd', 'abi': a, 'in': x, 'targets': targets, 'pre': pre}


# --------------------------------------------------------------------------------------------------- recorder
_OPS = ('attention', 'attention_train', 'attention_causal', 'attention_bwd', 'attn_delta', 'heads_transpose')


class Recorder(ga.LaunchRecorder):
    """audits every attention-family launch made inside it"""
    OPS = _OPS
    ENTRY_POINTS = ENTRY_POINTS

    def record(self, entry, args, S):
        return record(entry, abi_of(entry, args[:len(_ARGS[entry])]), S)

    def key(self, rec):
        return attn_path(rec)

    def check(self, rec):
        return check_launch(rec)
