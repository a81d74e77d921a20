"""Launch audit of the wgmma GEMM: every `ops.gemm` / `ops.splitk_finalize` call of a real engine walk, checked on its own.

A launch record is a plain dict built from the `mos_gemm_args` struct that reaches `mos_gemm_bf16` (or from the arguments of
`mos_splitk_finalize`), not from the Python views the engine passed: every pointer is mapped into the storage of the
tensor argument that contains it, and the operand windows are read there at the ABI pitches.  A wrong pitch or offset in
`ops.gemm` is therefore checked as well.  Record layout:

    rec = {'op': 'gemm' | 'finalize', 'abi': {ABI fields}, 'in': {operand windows},
           'targets': [output windows], 'mem': {storage: {'before': flat, 'after': flat}}, 'zero': [storages]}

`reference` and `check_launch` are pure functions of a record (they run on CPU tensors too).  The reference is float64
and follows the contract of include/mos_sm100.h and csrc/gemm.cu:
- conv: 3x3 / pad 1 implicit GEMM over NHWC [B, H, W, C] at the pixel pitch, tap-major W [N, 9C];
- bias, bias_batch (row m uses batch m // rows_per_batch, rows at pitch bias_batch_ld);
- LoRA: segments of lora_seg columns, segment s uses rows 4s..4s+3 of down16, up fp32 [N, 4] with alpha folded in;
- residual (16-bit rows at ldr, added last; GEGLU and head-split take none);
- GEGLU: packed tile t = 80 `a` columns | 80 gate columns -> output columns 80t..80t+79 = a * gelu_erf(gate);
- head-split: Q/K [b*H+h, t, j] at pitch dpad with seg_rows_pad rows, V^T [b*H+h, j, t] at pitch seg_rows_pad;
- fp32 output, optionally accumulated onto what `out` held;
- split-K partials [splits, M, N]: split s covers k blocks [s * kb_per_split, (s + 1) * kb_per_split);
- `splitk_finalize` and the in-kernel finalize: the partials summed in split order, plus bias, bias_batch and residual.

Checks of every launch (`check_launch`):
  a. |got - ref| <= u_out |ref| + (1 + u_out) (K_eff + 8) 2^-24 mag for every output element, mag the float64 sum of the
     magnitudes of every term (GEGLU: carried through a * gelu(g), |gelu'| <= 1.13, a few ulp for erff);
  b. rel-L2 per 128 x 160 tile (128 x 80 for GEGLU; per segment and tile for head-split) within the GEMM tests' bounds;
  c. every byte of a written storage outside the launch's window is bitwise unchanged (the window excludes the Q/K pad
     columns, the V^T pad rows and the pad tokens); in-kernel split-K counters are back to zero.
The recorder adds (d) the operand windows are unchanged by the launch and (e) one more launch from the same bytes is
bit-identical.
"""
import math
import traceback

import torch
import torch.nn.functional as F

BM, BN = 128, 160
CHUNK_ROWS = 16384
U_OUT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
# half the smallest subnormal step of the output type: round-to-nearest there has an absolute, not a relative, error
TINY_OUT = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25, torch.float32: 2.0 ** -150}
# per-tile rel-L2 limits: the bounds of test_gemm_gpu.py / test_gemm_schedule_gpu.py.  The fp32 limit holds for reductions
# of up to 256; beyond, it grows as sqrt(K / 256), as the fp32 accumulation error of a K-term sum does (the wgmma
# accumulator adds about 1e-5 per tile at K = 1440 on an H100).  The element bound (a) is not relaxed.
TILE_TOL = {torch.bfloat16: 4e-3, torch.float16: 6e-4, torch.float32: 1e-5}
ACC_U = 2.0 ** -24
GELU_D = 1.13                  # max |gelu'(x)| (at x ~ 0.75 * sqrt(2))
GELU_ULP = 8 * ACC_U           # fp32 gelu_erf: erff and three roundings
DT16 = {0: torch.bfloat16, 1: torch.float16}
OUT_BF16, OUT_HEADS, OUT_F32 = 0, 1, 2
SEG_ROWS, SEG_TRANSPOSED = 0, 1
_BITS = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def _cdiv(a, b):
    return -(-a // b)


def conv_tiling(B, H, Wd):
    """(TW, TH, TB) of a conv launch: the pixel patch of one 128-row tile.  A copy of the host rule in csrc/gemm.cu,
    mos_gemm_bf16 (the TW / TH loop); keep the two in step."""
    TW = 1
    while TW * 2 <= 128 and Wd % (TW * 2) == 0:
        TW *= 2
    best_th, best_eff, TH = 1, -1.0, 1
    while TH * TW <= 128:
        TB = 128 // (TW * TH)
        if not (TB > 4 and TH * 2 * TW <= 128):
            eff = (H / (_cdiv(H, TH) * TH)) * (B / (_cdiv(B, TB) * TB))
            if eff > best_eff + 1e-9:
                best_eff, best_th = eff, TH
        TH *= 2
    return TW, best_th, 128 // (TW * best_th)


def gemm_path(rec, heads_copy=False):
    """Path key of a launch: the epilogue path `mos_gemm_bf16` picks, with the features that select code in the kernel.
    A copy of the host rule in csrc/gemm.cu, mos_gemm_bf16 (heads_tma, epi_tma, res_tma, epi_copy, epi_mode);
    keep the two in step.  heads_copy: MOS_GEMM_HEADS_COPY=1."""
    a = rec['abi']
    if rec['op'] == 'finalize':
        dt = 'fp16' if a['a_dtype'] == 1 else 'bf16'
        return '|'.join(['splitk_finalize', dt] + (['bb'] if a['bias_batch'] else []) + (['res'] if a['residual'] else []))
    N, M = a['N'], a['M']
    splits = max(a['splits'], 1)
    cols = N // 2 if a['geglu'] else N

    def tma_rows(base, ld):
        return bool(base) and ld >= cols and ld % 8 == 0 and base % 16 == 0

    T = a['tokens_per_batch'] if a['tokens_per_batch'] > 0 else 1
    heads = a['out_mode'] == OUT_HEADS
    nseg = N // (a['heads'] * a['head_dim']) if heads else 0
    heads_tma = heads and not heads_copy and (T == 64 or T % 128 == 0) and M % T == 0
    for s in range(nseg):
        if not heads_tma:
            break
        tr = a['seg_kind'][s] == SEG_TRANSPOSED
        heads_tma = (bool(a['seg_ptr'][s]) and a['seg_ptr'][s] % 16 == 0 and a['seg_rows_pad'][s] >= T and
                     (a['dv_pad'] >= a['head_dim'] and a['seg_rows_pad'][s] % 8 == 0 if tr
                      else a['dpad'] >= a['head_dim'] and a['dpad'] % 8 == 0))
    residual = None if a['geglu'] or heads else a['residual']
    epi_tma = (a['out_mode'] == OUT_BF16 and splits == 1 and tma_rows(a['out'], a['ldc'])) or heads_tma
    res_tma = epi_tma and bool(residual) and tma_rows(residual, a['ldr'])
    if splits > 1:
        mode, write = 'partial', 'global'
    elif a['out_mode'] == OUT_F32:
        mode, write = 'f32+acc' if a['accumulate'] else 'f32', 'global'
    else:
        write = 'tma' if epi_tma else 'copy'
        if heads:
            mode = 'heads_vt' if any(a['seg_kind'][s] == SEG_TRANSPOSED for s in range(nseg)) else 'heads'
        elif a['geglu']:
            mode = 'geglu'
        elif not residual:
            mode = 'rows'
        else:
            mode = 'rows+res_smem' if res_tma else 'rows+res_global'
    key = [mode, write, 'fp16' if a['a_dtype'] == 1 else 'bf16']
    if a['lora_down']:
        key.append('lora')
    if a['conv']:
        key.append('conv')
    if a['bias_batch'] and splits == 1:
        key.append('bb')
    if heads:
        key.append(f'T={T}')
    if splits > 1 and a['tile_counters']:
        key.append('fused')
    return '|'.join(key)


# --------------------------------------------------------------------------------------------------- reference
def _m_tile(rec, m):
    """output tile row index of rows m (conv: the TW x TH x TB pixel patch of the row)"""
    a = rec['abi']
    if rec['op'] == 'gemm' and a['conv']:
        TW, TH, TB = conv_tiling(a['B'], a['H'], a['Wd'])
        HW = a['H'] * a['Wd']
        b, hw = m // HW, m % HW
        h, w = hw // a['Wd'], hw % a['Wd']
        tiles_w, tiles_h = a['Wd'] // TW, _cdiv(a['H'], TH)
        return w // TW + tiles_w * (h // TH + tiles_h * (b // TB))
    return m // BM


def _m_tiles(rec):
    a = rec['abi']
    if rec['op'] == 'gemm' and a['conv']:
        TW, TH, TB = conv_tiling(a['B'], a['H'], a['Wd'])
        return a['Wd'] // TW * _cdiv(a['H'], TH) * _cdiv(a['B'], TB)
    return _cdiv(a['M'], BM)


def _a_rows(rec, m0, m1):
    """float64 rows [m0, m1) of the reduction operand: A, or for conv the im2col rows [rows, 9C] (tap-major)"""
    a, A = rec['abi'], rec['in']['A']
    if not a['conv']:
        return A[m0:m1].double()
    B, H, Wd, C = A.shape
    m = torch.arange(m0, m1, device=A.device)
    b, h, w = m // (H * Wd), (m // Wd) % H, m % Wd
    Ap = F.pad(A, (0, 0, 1, 1, 1, 1))                    # [B, H + 2, W + 2, C], zero padding 1
    return torch.cat([Ap[b, h + kh, w + kw] for kh in range(3) for kw in range(3)], 1).double()


def _batch_rows(rec, m0, m1, t):
    """rows [m0, m1) of a per-batch operand [nbatch, N]: row m uses batch m // rows_per_batch"""
    rpb = max(rec['abi']['rows_per_batch'], 1)
    return t[torch.arange(m0, m1, device=t.device) // rpb].double()


def _epilogue_terms(rec, m0, m1, val, mag):
    """+ bias, bias_batch and residual (in place)"""
    x = rec['in']
    if x.get('bias') is not None:
        val += x['bias'].double()
        mag += x['bias'].double().abs()
    if x.get('bias_batch') is not None:
        bb = _batch_rows(rec, m0, m1, x['bias_batch'])
        val += bb
        mag += bb.abs()
    if x.get('residual') is not None:
        r = x['residual'][m0:m1].double()
        val += r
        mag += r.abs()


def reference(rec, m0, m1):
    """float64 reference of rows [m0, m1) of every output target: a list of (ref [rows, cols], acc_bound [rows, cols]),
    one per entry of rec['targets'].  acc_bound is the error the fp32 arithmetic may add before the output rounding."""
    a, x = rec['abi'], rec['in']
    if rec['op'] == 'finalize':
        P = x['partial'][:, m0:m1].double()              # [splits, rows, N]
        val, mag = P.sum(0), P.abs().sum(0)
        _epilogue_terms(rec, m0, m1, val, mag)
        return [(val, (a['splits'] + 8) * ACC_U * mag)]
    Ar = _a_rows(rec, m0, m1)
    Aabs = Ar.abs()
    W = x['W'].double()
    N, Kw = W.shape
    splits = max(a['splits'], 1)
    if splits > 1:
        kb_total = Kw // 64
        kbps = _cdiv(kb_total, splits)
        out = []
        total, total_mag = 0, 0
        for s in range(splits):
            k0, k1 = s * kbps * 64, min(kb_total, (s + 1) * kbps) * 64
            v = Ar[:, k0:k1] @ W[:, k0:k1].t()
            mg = Aabs[:, k0:k1] @ W[:, k0:k1].abs().t()
            out.append((v, (k1 - k0 + 8) * ACC_U * mg))
            total, total_mag = total + v, total_mag + mg
        for t in rec['targets'][splits:]:                # in-kernel finalize: the 16-bit rows as well
            _epilogue_terms(rec, m0, m1, total, total_mag)
            out.append((total, (Kw + splits + 8) * ACC_U * total_mag))
        return out
    val = Ar @ W.t()
    mag = Aabs @ W.abs().t()
    if x.get('lora_down') is not None:
        D, U = x['lora_down'].double(), x['lora_up'].double()
        t, tm = Ar @ D.t(), Aabs @ D.abs().t()           # [rows, 16]
        seg = a['lora_seg']
        for s in range(_cdiv(N, seg)):
            c = slice(s * seg, min(N, (s + 1) * seg))
            val[:, c] += t[:, 4 * s:4 * s + 4] @ U[c].t()
            mag[:, c] += tm[:, 4 * s:4 * s + 4] @ U[c].abs().t()
    _epilogue_terms(rec, m0, m1, val, mag)
    acc = (Kw + 8) * ACC_U * mag
    if a['out_mode'] == OUT_F32 and a['accumulate']:
        before = gather(rec, 0, 'before', m0, m1).double()
        val += before
        acc += ACC_U * before.abs()
    if a['geglu']:
        rows = val.shape[0]
        v, e = val.view(rows, N // BN, 2, BN // 2), acc.view(rows, N // BN, 2, BN // 2)
        av, gv, ea, eg = v[:, :, 0], v[:, :, 1], e[:, :, 0], e[:, :, 1]
        gel = 0.5 * gv * (1 + torch.special.erf(gv / math.sqrt(2)))
        y = av * gel
        bound = ea * (gel.abs() + GELU_D * eg) + av.abs() * (GELU_D * eg + GELU_ULP * (gv.abs() + gel.abs()))
        return [(y.reshape(rows, N // 2), bound.reshape(rows, N // 2))]
    if a['out_mode'] == OUT_HEADS:
        seg_len = a['heads'] * a['head_dim']
        return [(val[:, t['col0']:t['col0'] + seg_len], acc[:, t['col0']:t['col0'] + seg_len]) for t in rec['targets']]
    return [(val, acc)]


def target_index(rec, t, m0, m1):
    """flat element indices [rows, cols] of rows [m0, m1) of output target t in its storage"""
    a = rec['abi']
    dev = rec['mem'][t['mem']]['after'].device
    m = torch.arange(m0, m1, device=dev)[:, None]
    c = torch.arange(t['cols'], device=dev)[None, :]
    if t['kind'] == 'rows':
        return t['off'] + m * t['ld'] + c
    if t['kind'] == 'partial':
        return t['off'] + (t['split'] * a['M'] + m) * a['N'] + c
    T, hd, H = a['tokens_per_batch'], a['head_dim'], a['heads']
    b, tok = m // T, m % T
    h, j = c // hd, c % hd
    if t['kind'] == 'qk':
        return t['off'] + ((b * H + h) * t['rows_pad'] + tok) * a['dpad'] + j
    return t['off'] + ((b * H + h) * a['dv_pad'] + j) * t['rows_pad'] + tok


def gather(rec, ti, which, m0, m1):
    t = rec['targets'][ti]
    return rec['mem'][t['mem']][which][target_index(rec, t, m0, m1)]


def _n_tile(rec, t, cols):
    c = torch.arange(cols)
    if rec['op'] == 'gemm' and rec['abi']['geglu']:
        return c // (BN // 2)
    return (t.get('col0', 0) + c) // BN


def tile_tol(rec, t, dtype):
    """per-tile rel-L2 limit of output target t"""
    if dtype != torch.float32:
        return TILE_TOL[dtype]
    a = rec['abi']
    if rec['op'] == 'finalize':
        k = a['splits']
    elif t['kind'] == 'partial':
        k = _cdiv(rec['in']['W'].shape[1] // 64, a['splits']) * 64
    else:
        k = rec['in']['W'].shape[1]
    return TILE_TOL[dtype] * max(1.0, math.sqrt(k / 256))


def chunk_rows(rec):
    a = rec['abi']
    width = a['N'] if rec['op'] == 'finalize' else rec['in']['W'].shape[1] + a['N']
    rows = min(CHUNK_ROWS, max(BM, (1 << 25) // max(width, 1)))
    return rows // BM * BM


def simulate(rec):
    """Write the rounded reference into the 'after' storages: what a correct kernel leaves (CPU tests)."""
    for st in rec['mem'].values():
        st['after'] = st['before'].clone()
    rec['zero_after'] = {k: torch.zeros(1, dtype=torch.int32) for k in rec['zero']}
    M = rec['abi']['M']
    step = chunk_rows(rec)
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        for t, (ref, _) in zip(rec['targets'], reference(rec, m0, m1)):
            st = rec['mem'][t['mem']]
            st['after'][target_index(rec, t, m0, m1)] = ref.to(st['after'].dtype)
    return rec


def check_launch(rec):
    """Checks (a)-(c) of one launch.  -> {'ratio': worst error / bound, 'tile': worst tile rel-L2 / its limit,
    'tile_rel': worst tile rel-L2, 'errors': [messages]}"""
    a = rec['abi']
    M = a['M']
    errors = []
    masks = {k: torch.zeros(st['after'].numel(), dtype=torch.bool, device=st['after'].device)
             for k, st in rec['mem'].items()}
    tiles = []
    for t in rec['targets']:
        dev = rec['mem'][t['mem']]['after'].device
        nt = _n_tile(rec, t, t['cols']).to(dev)
        shape = (_m_tiles(rec), int(nt.max()) + 1)
        tiles.append((torch.zeros(shape, dtype=torch.float64, device=dev),
                      torch.zeros(shape, dtype=torch.float64, device=dev), nt))
    ratio = 0.0
    step = chunk_rows(rec)
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        for ti, (t, (ref, accb)) in enumerate(zip(rec['targets'], reference(rec, m0, m1))):
            st = rec['mem'][t['mem']]
            dt = st['after'].dtype
            idx = target_index(rec, t, m0, m1)
            masks[t['mem']][idx.flatten()] = True
            got = st['after'][idx].double()
            err = (got - ref).abs()
            bound = U_OUT[dt] * ref.abs() + (1 + U_OUT[dt]) * accb + TINY_OUT[dt]
            bad = ~(err <= bound)                        # NaN counts as bad
            if bad.any():
                r, c = [int(v) for v in bad.nonzero()[0]]
                errors.append(f"(a) target {ti} ({t['kind']}): {int(bad.sum())} elements out of bound, first at row "
                              f"{m0 + r} col {c}: got {got[r, c].item():.6g} want {ref[r, c].item():.6g} bound "
                              f"{bound[r, c].item():.3g}")
            ratio = max(ratio, (err / bound).nan_to_num(nan=math.inf).max().item())
            e2, r2, nt = tiles[ti]
            mtile = _m_tile(rec, torch.arange(m0, m1, device=nt.device))
            key = (mtile[:, None] * e2.shape[1] + nt[None, :]).flatten()
            e2.view(-1).index_add_(0, key, (err * err).flatten())
            r2.view(-1).index_add_(0, key, (ref * ref).flatten())
    worst_rel, worst_frac = 0.0, 0.0
    for ti, (e2, r2, _) in enumerate(tiles):
        t = rec['targets'][ti]
        tol = tile_tol(rec, t, rec['mem'][t['mem']]['after'].dtype)
        rel = torch.where(e2 == 0, torch.zeros_like(e2), e2.sqrt() / r2.sqrt())
        worst_rel = max(worst_rel, rel.max().item())
        frac = rel.max().item() / tol
        worst_frac = max(worst_frac, frac)
        if not frac <= 1:
            mt, nt = divmod(int(rel.argmax()), rel.shape[1])
            errors.append(f'(b) target {ti}: tile ({mt}, {nt}) rel-L2 {rel.max().item():.3e} > {tol:.2e}')
    for k, st in rec['mem'].items():
        changed = st['after'].view(_BITS[st['after'].element_size()]) != st['before'].view(_BITS[st['before'].element_size()])
        stray = changed & ~masks[k]
        if stray.any():
            errors.append(f'(c) storage {k}: {int(stray.sum())} elements written outside the window, first at flat '
                          f'index {int(stray.nonzero()[0])}')
    for k in rec.get('zero', ()):
        if (rec['zero_after'][k] != 0).any():
            errors.append('(c) split-K tile counters not back to zero')
    return {'ratio': ratio, 'tile_rel': worst_rel, 'tile': worst_frac, 'errors': errors}


# --------------------------------------------------------------------------------------------------- recorder (GPU)
_PTRS = ('A', 'W', 'partial', 'bias', 'bias_batch', 'residual', 'lora_down', 'lora_up', 'out', 'tile_counters')
_INTS = ('M', 'N', 'K', 'lda', 'conv', 'B', 'H', 'Wd', 'C', 'splits', 'rows_per_batch', 'bias_batch_ld', 'ldr', 'geglu',
         'lora_seg', 'out_mode', 'ldc', 'heads', 'head_dim', 'dpad', 'dv_pad', 'tokens_per_batch', 'accumulate',
         'a_dtype', 'w_dtype', 'tile_counters_len')


def abi_of(args):
    """mos_gemm_args (ctypes) -> plain dict (pointers as ints, 0 for NULL)"""
    a = {f: int(getattr(args, f)) for f in _INTS}
    for f in _PTRS:
        a[f] = getattr(args, f) or 0
    a['seg_ptr'] = [args.seg_ptr[i] or 0 for i in range(3)]
    a['seg_kind'] = [int(args.seg_kind[i]) for i in range(3)]
    a['seg_rows_pad'] = [int(args.seg_rows_pad[i]) for i in range(3)]
    return a


class _Storages:
    """the storages of a call's tensor arguments; maps a device pointer to (storage, byte offset).  `extra`: storages
    that only pointers read from a device table may resolve into (find(..., table=True))"""

    def __init__(self, tensors, extra=()):
        self.st, self.extra = {}, {}
        for t in tensors:
            s = t.untyped_storage()
            self.st[s.data_ptr()] = (s, t.device)
        for t in extra:
            s = t.untyped_storage()
            self.extra.setdefault(s.data_ptr(), (s, t.device))

    def find(self, p, what, table=False):
        for pool in (self.st, self.extra) if table else (self.st,):
            for base, (s, dev) in pool.items():
                if base <= p < base + s.nbytes():
                    return base, p - base
        raise AssertionError(f'{what}: pointer {p:#x} lies in no ' +
                             ('tensor argument of the call or registered tensor' if table
                              else 'tensor argument of the call'))

    def flat(self, base, dtype):
        s, dev = self.st[base] if base in self.st else self.extra[base]
        es = torch.empty(0, dtype=dtype).element_size()
        return torch.empty(0, dtype=dtype, device=dev).set_(s, 0, (s.nbytes() // es,), (1,))

    def window(self, p, what, dtype, size, stride, table=False):
        base, off = self.find(p, what, table)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{what}: pointer not aligned to its element size'
        try:
            return self.flat(base, dtype).as_strided(size, stride, off // es)
        except RuntimeError as e:
            raise AssertionError(f'{what}: window {tuple(size)} at pitch {stride} runs past its storage: {e}')


def _site():
    for fr in reversed(traceback.extract_stack()[:-1]):
        f = fr.filename.replace('\\', '/')
        if f.endswith(('/ops.py', '/gemm_audit.py', '/attention_audit.py', '/norm_audit.py')) or \
                fr.name in ('gemm', '_audited', '_registering'):
            continue
        return f"{f.rsplit('/', 1)[-1]}:{fr.lineno}"
    return '?'


def _tensors(args, kwargs):
    """the tensors among a call's arguments: lists and tuples are flattened, a heads dict contributes its seg_ptr"""
    out = []
    for v in list(args) + list(kwargs.values()):
        if isinstance(v, torch.Tensor):
            out.append(v)
        elif isinstance(v, (list, tuple)):
            out += _tensors(v, {})
        elif isinstance(v, dict):
            out += _tensors(v.get('seg_ptr', ()), {})
    return out


def gemm_record(abi, S):
    """the launch record of a mos_gemm_bf16 call (operand windows and written storages still live)"""
    a = abi
    dt = DT16[a['a_dtype']]
    N, K, M = a['N'], a['K'], a['M']
    x = {}
    if a['conv']:
        ld = a['lda'] if a['lda'] > 0 else a['C']
        x['A'] = S.window(a['A'], 'A', dt, (a['B'], a['H'], a['Wd'], a['C']),
                          (a['H'] * a['Wd'] * ld, a['Wd'] * ld, ld, 1))
        Kw = 9 * K
    else:
        x['A'] = S.window(a['A'], 'A', dt, (M, K), (a['lda'], 1))
        Kw = K
    x['W'] = S.window(a['W'], 'W', DT16[a['w_dtype']], (N, Kw), (Kw, 1))
    if a['lora_down']:
        x['lora_down'] = S.window(a['lora_down'], 'lora_down', DT16[a['w_dtype']], (16, K), (K, 1))
        x['lora_up'] = S.window(a['lora_up'], 'lora_up', torch.float32, (N, 4), (4, 1))
    if a['bias']:
        x['bias'] = S.window(a['bias'], 'bias', torch.float32, (N,), (1,))
    if a['bias_batch'] and a['splits'] <= 1 or a['bias_batch'] and a['tile_counters']:
        rpb = max(a['rows_per_batch'], 1)
        nb = a['B'] if a['conv'] else _cdiv(M, rpb)
        x['bias_batch'] = S.window(a['bias_batch'], 'bias_batch', torch.float32, (nb, N),
                                   (a['bias_batch_ld'] or N, 1))
    heads = a['out_mode'] == OUT_HEADS
    if a['residual'] and not a['geglu'] and not heads and (a['splits'] <= 1 or a['tile_counters']):
        x['residual'] = S.window(a['residual'], 'residual', dt, (M, N), (a['ldr'], 1))
    targets, zero = [], []

    def target(p, what, dtype, **t):
        base, off = S.find(p, what)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{what}: pointer not aligned to its element size'
        targets.append(dict(mem=(base, dtype), off=off // es, **t))

    if a['splits'] > 1:
        for s in range(a['splits']):
            target(a['partial'], 'partial', torch.float32, kind='partial', split=s, cols=N)
        if a['tile_counters']:
            target(a['out'], 'out', dt, kind='rows', ld=a['ldc'], cols=N)
            zero.append(S.find(a['tile_counters'], 'tile_counters')[0])
    elif heads:
        seg_len = a['heads'] * a['head_dim']
        for s in range(N // seg_len):
            target(a['seg_ptr'][s], f'seg_ptr[{s}]', dt, kind='vt' if a['seg_kind'][s] == SEG_TRANSPOSED else 'qk',
                   rows_pad=a['seg_rows_pad'][s], col0=s * seg_len, cols=seg_len)
    elif a['out_mode'] == OUT_F32:
        target(a['out'], 'out', torch.float32, kind='rows', ld=a['ldc'], cols=N)
    else:
        target(a['out'], 'out', dt, kind='rows', ld=a['ldc'], cols=N // 2 if a['geglu'] else N)
    return {'op': 'gemm', 'abi': a, 'in': x, 'targets': targets, 'zero': zero}


def finalize_record(vals, S):
    partial, splits, M, N, bias, bias_batch, rpb, bbld, residual, ldr, out, ldc, adt = vals
    dt = DT16[adt]
    abi = dict(M=M, N=N, splits=splits, rows_per_batch=rpb, bias_batch_ld=bbld, ldr=ldr, ldc=ldc, a_dtype=adt,
               bias_batch=bias_batch or 0, residual=residual or 0)
    x = {'partial': S.window(partial, 'partial', torch.float32, (splits, M, N), (M * N, N, 1))}
    if bias:
        x['bias'] = S.window(bias, 'bias', torch.float32, (N,), (1,))
    if bias_batch:
        x['bias_batch'] = S.window(bias_batch, 'bias_batch', torch.float32, (_cdiv(M, max(rpb, 1)), N), (bbld or N, 1))
    if residual:
        x['residual'] = S.window(residual, 'residual', dt, (M, N), (ldr, 1))
    base, off = S.find(out, 'out')
    assert off % 2 == 0
    t = dict(mem=(base, dt), off=off // 2, kind='rows', ld=ldc, cols=N)
    return {'op': 'finalize', 'abi': abi, 'in': x, 'targets': [t], 'zero': []}


def attach_mem(rec, S):
    """snapshot the full bytes of every storage the launch may write into rec['mem'][...]['before']; -> the live flat
    views of those storages"""
    flats = {k: S.flat(*k) for k in {t['mem'] for t in rec['targets']}}
    rec['mem'] = {k: {'before': f.clone()} for k, f in flats.items()}
    return flats


class Stats:
    """per path key: launches, worst element ratio, worst tile rel-L2 (and its fraction of the limit), worst call site"""

    def __init__(self):
        self.rows, self.failures = {}, []

    def add(self, key, site, res):
        r = self.rows.setdefault(key, {'n': 0, 'ratio': 0.0, 'tile_rel': 0.0, 'tile': 0.0, 'site': site})
        r['n'] += 1
        r['tile_rel'] = max(r['tile_rel'], res['tile_rel'])
        if res['ratio'] >= r['ratio']:
            r['ratio'], r['site'] = res['ratio'], site
        r['tile'] = max(r['tile'], res['tile'])
        self.failures += [f'{key} @ {site}: {e}' for e in res['errors']]

    def merge(self, other):
        for k, o in other['rows'].items():
            r = self.rows.setdefault(k, {'n': 0, 'ratio': 0.0, 'tile_rel': 0.0, 'tile': 0.0, 'site': o['site']})
            r['n'] += o['n']
            r['tile_rel'] = max(r['tile_rel'], o['tile_rel'])
            r['tile'] = max(r['tile'], o['tile'])
            if o['ratio'] >= r['ratio']:
                r['ratio'], r['site'] = o['ratio'], o['site']
        self.failures += other['failures']

    def table(self):
        lines = [f"{'path key':<44} {'launches':>8} {'worst err/bound':>15} {'worst tile rel-L2':>17}  worst call site"]
        for k in sorted(self.rows):
            r = self.rows[k]
            lines.append(f"{k:<44} {r['n']:>8} {r['ratio']:>15.3e} {r['tile_rel']:>17.3e}  {r['site']}")
        return '\n'.join(lines)


class LaunchRecorder:
    """Context manager shared by the launch audits: wraps the `ops.*` functions named in OPS, proxies `_lib.lib()` so that
    every call of an entry point in ENTRY_POINTS made inside one of them is audited, and restores both on exit (eager
    walks only; it works on CPU tensors too, with a stand-in library in place of `_lib.lib()`).

    A subclass supplies `record(entry, args, S)` (the launch record, built from the ABI arguments and the storages S of
    the call's tensor arguments), `key(rec)` and `check(rec)`.  Each launch is checked by `check` ((p), (a)-(c)); the
    recorder adds (d) the operand windows rec['in'] are unchanged, except the names in rec['inplace'], and (e) one more
    launch from the same bytes is bit-identical.  The tensor arguments of the ops in REGISTER_OPS are kept as storages
    that device pointer tables may point into (S.find resolves them like tensor arguments).
    determinism: 'all' relaunches every launch once more, 'first' only the first launch of each path key."""
    OPS = ()
    ENTRY_POINTS = ()
    REGISTER_OPS = ()

    def __init__(self, stats=None, determinism='all'):
        self.stats = stats if stats is not None else Stats()
        self.determinism = determinism
        self._ctx = None
        self.registered = []
        self.last = None

    def register(self, *tensors):
        """storages a pointer table of a later launch may point into"""
        self.registered += _tensors(tensors, {})

    def record(self, entry, args, S):
        raise NotImplementedError

    def key(self, rec):
        raise NotImplementedError

    def check(self, rec):
        raise NotImplementedError

    def __enter__(self):
        from mos_b200 import _lib, ops
        self._ops, self._libmod = ops, _lib
        self._orig_ops = {n: getattr(ops, n) for n in self.OPS + self.REGISTER_OPS}
        self._orig_lib = _lib.lib
        real = _lib.lib()
        rec = self

        class Proxy:
            def __getattr__(self, name):
                fn = getattr(real, name)
                if name in rec.ENTRY_POINTS:
                    return lambda *args: rec._audit(name, lambda: fn(*args), args)
                return fn

        proxy = Proxy()

        def wrap(fn):
            def _audited(*args, **kwargs):
                assert self._ctx is None
                self._ctx = (_tensors(args, kwargs), _site(), (args, kwargs))
                try:
                    return fn(*args, **kwargs)
                finally:
                    self._ctx = None
            return _audited

        def registering(fn):
            def _registering(*args, **kwargs):
                self.register(*args, *kwargs.values())
                return fn(*args, **kwargs)
            return _registering

        for n, fn in self._orig_ops.items():
            setattr(ops, n, wrap(fn) if n in self.OPS else registering(fn))
        _lib.lib = lambda: proxy
        return self

    def __exit__(self, *exc):
        for n, fn in self._orig_ops.items():
            setattr(self._ops, n, fn)
        self._libmod.lib = self._orig_lib
        self.registered = []
        return False

    def _audit(self, entry, launch, args):
        assert self._ctx is not None, f'{entry} launched outside the audited ops.* wrappers'
        tensors, site = self._ctx[:2]
        cuda = any(t.is_cuda for t in tensors)
        if cuda:
            assert not torch.cuda.is_current_stream_capturing(), 'the launch audit needs an eager walk (use_graph=False)'
            torch.cuda.synchronize()
        S = _Storages(tensors, self.registered)
        rec = self.record(entry, args, S)
        key = self.key(rec)
        live, rec['in'] = rec['in'], {k: v.clone() for k, v in rec['in'].items()}   # the reference reads the snapshot
        flats = attach_mem(rec, S)
        zero = {k: S.flat(k, torch.int32) for k in rec.get('zero', ())}
        for k, z in zero.items():
            assert (z == 0).all(), 'split-K tile counters must be zero before the launch'

        def run():
            rc = launch()
            if cuda:
                torch.cuda.synchronize()
            return rc
        rc = run()
        if rc != 0:
            return rc
        for k, f in flats.items():
            rec['mem'][k]['after'] = f.clone()
        rec['zero_after'] = {k: z.clone() for k, z in zero.items()}
        res = self.check(rec)
        for k, v in rec['in'].items():
            if k in rec.get('inplace', ()):
                continue                                 # read and then overwritten by the launch
            if not torch.equal(v.reshape(-1).view(_BITS[v.element_size()]),
                               live[k].reshape(-1).view(_BITS[v.element_size()])):
                res['errors'].append(f'(d) operand {k} changed by the launch')
        if self.determinism == 'all' or key not in self.stats.rows:
            for k, f in flats.items():
                f.copy_(rec['mem'][k]['before'])
            assert run() == 0
            for k, f in flats.items():
                if not torch.equal(f.view(_BITS[f.element_size()]), rec['mem'][k]['after'].view(_BITS[f.element_size()])):
                    res['errors'].append('(e) a second launch from the same bytes is not bit-identical')
        self.stats.add(key, site, res)
        self.last = rec
        return rc


class Recorder(LaunchRecorder):
    """audits every ops.gemm / ops.splitk_finalize launch made inside it"""
    OPS = ('gemm', 'splitk_finalize')
    ENTRY_POINTS = ('mos_gemm_bf16', 'mos_splitk_finalize')

    def record(self, entry, args, S):
        if entry == 'mos_gemm_bf16':
            rec = gemm_record(abi_of(args[0]._obj), S)
            if rec['abi']['residual'] and rec['abi']['residual'] == rec['abi']['out']:
                rec['inplace'] = ('residual',)           # a residual that aliases `out` is read and then overwritten
            return rec
        vals = [getattr(v, 'value', v) for v in args[:13]]
        return finalize_record([0 if v is None else int(v) for v in vals], S)

    def key(self, rec):
        return gemm_path(rec)

    def check(self, rec):
        return check_launch(rec)
