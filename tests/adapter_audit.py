"""Launch audit of the T2I-Adapter's layout and elementwise kernels (csrc/adapter.cu): every call of an entry point in
ENTRY_POINTS made through its `adapter_ops.*` wrapper in a real engine walk, checked on its own.  The GEMM launches of the
adapter are audited by gemm_audit.Recorder.

As in norm_audit.py, the record is built from the arguments that reach the `mos_*` entry point: every pointer is mapped
into the storage of a tensor argument and each operand window is read there at the layout the kernel uses.  Record
layout: {'op', 'abi', 'in': {operand windows}, 'targets': [{'name', 'mem', 'off', 'size', 'stride'}], 'pre': [(p)
messages], 'inplace', 'mem': {storage: {'before', 'after'}}}.  `reference` and `check_launch` are pure functions of a record.

Element bound (a), with u = 2^-24 and the 16-bit output rounding of norm_audit (u16 |ref| + (1 + u16) e + t16):
- pixel_unshuffle: a copy rounded once to 16 bits: bit-exact.
- relu_rows: x < 0 ? 0 : x in 16 bits: bit-exact.
- avgpool2x: three fp32 adds of the four taps, times the exact 0.25: e = 5u sum |x / 4|.

Checks of every launch (`check_launch`):
  p. every tensor argument's row pitch equals the pitch the kernel reads it at; the image of pixel_unshuffle is dense;
  a. the element bound above; the bit-exact outputs bit for bit;
  c. every byte of a written storage outside the launch's window is bitwise unchanged (pitch pads included).
The recorder (gemm_audit.LaunchRecorder) adds (d) unchanged operands (ReLU's x is in place) and (e) a bit-identical
relaunch.
"""
import torch

import gemm_audit as ga
import norm_audit as na
from gemm_audit import Stats, _Storages  # noqa: F401  (the table and storage map of every audit)

F32 = torch.float32

_ARGS = {
    'mos_pixel_unshuffle': ('x', 'B', 'Cin', 'H', 'W', 'y', 'ldy', 'act_dtype'),
    'mos_relu_rows': ('x', 'ld', 'M', 'C', 'act_dtype'),
    'mos_avgpool2x': ('x', 'ldx', 'B', 'H', 'W', 'C', 'y', 'ldy', 'act_dtype'),
}
ENTRY_POINTS = tuple(_ARGS)
OPS = ('pixel_unshuffle', 'relu_rows', 'avgpool2x')


def abi_of(entry, args):
    """the ctypes arguments of an entry point -> plain dict (pointers as ints, 0 for NULL)"""
    return {n: (0 if getattr(v, 'value', v) is None else int(getattr(v, 'value', v))) for n, v in zip(_ARGS[entry], args)}


def _dt(a):
    return ga.DT16[a['act_dtype']]


def adapter_path(rec):
    """Path key of a launch: the entry point and its 16-bit type (the only feature that selects code)"""
    return f"{rec['op'][4:]}|{'fp16' if _dt(rec['abi']) == torch.float16 else 'bf16'}"


def record(entry, a, S, call=None):
    """the launch record of one entry-point call; call: the (args, kwargs) of the adapter_ops.* wrapper"""
    x, targets, pre, inplace, pitches = {}, [], [], [], {}
    dt = _dt(a)

    def win(name, dtype, size, stride, ld=None):
        x[name] = S.window(a[name], name, dtype, size, stride)
        if ld is not None:
            pitches[a[name]] = (name, ld)

    def target(name, dtype, size, stride, ld=None):
        p = a[name]
        if ld is not None:
            pitches[p] = (name, ld)
        base, off = S.find(p, name)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{name}: pointer not aligned to its element size'
        t = dict(name=name, mem=(base, dtype), off=off // es, size=tuple(size), stride=tuple(stride))
        S.flat(base, dtype).as_strided(t['size'], t['stride'], t['off'])     # raises if it runs past its storage
        targets.append(t)

    if entry == 'mos_pixel_unshuffle':
        B, Ci, H, W, ldy = a['B'], a['Cin'], a['H'], a['W'], a['ldy']
        win('x', F32, (B, Ci, H, W), (Ci * H * W, H * W, W, 1))
        img = call[0][0] if call and call[0] and isinstance(call[0][0], torch.Tensor) else None
        if img is not None and not img.is_contiguous():
            pre.append(f'(p) x: taken dense by the kernel, passed with strides {tuple(img.stride())}')
        Ho, Wo = H // 8, W // 8
        target('y', dt, (B, Ho, Wo, 64 * Ci), (Ho * Wo * ldy, Wo * ldy, ldy, 1), ld=ldy)
    elif entry == 'mos_relu_rows':
        win('x', dt, (a['M'], a['C']), (a['ld'], 1), ld=a['ld'])
        target('x', dt, (a['M'], a['C']), (a['ld'], 1))
        inplace.append('x')
    else:
        B, H, W, C, ldx, ldy = a['B'], a['H'], a['W'], a['C'], a['ldx'], a['ldy']
        win('x', dt, (B, H, W, C), (H * W * ldx, W * ldx, ldx, 1), ld=ldx)
        target('y', dt, (B, H // 2, W // 2, C), (H // 2 * W // 2 * ldy, W // 2 * ldy, ldy, 1), ld=ldy)
    for t in ga._tensors(*call) if call else ():
        hit = pitches.get(t.data_ptr())
        if hit is not None and t.dim() >= 2 and t.shape[-2] > 1 and t.stride(-2) != hit[1]:
            pre.append(f'(p) {hit[0]}: the kernel reads it at row pitch {hit[1]}, the tensor passed has strides '
                       f'{tuple(t.stride())}')
    return {'op': entry, 'abi': a, 'in': x, 'targets': targets, 'pre': pre, 'inplace': tuple(inplace)}


def reference(rec):
    """float64 reference of every output target: {name: (ref, fp32 error bound)}; bound None: bit-exact"""
    e, X = rec['op'], rec['in']['x'].double()
    if e == 'mos_pixel_unshuffle':
        B, Ci, H, W = X.shape
        return {'y': (X.view(B, Ci, H // 8, 8, W // 8, 8).permute(0, 2, 4, 1, 3, 5).reshape(B, H // 8, W // 8, 64 * Ci),
                      None)}
    if e == 'mos_relu_rows':
        return {'x': (torch.where(X < 0, torch.zeros_like(X), X), None)}
    B, H, W, C = X.shape
    terms = 0.25 * X.view(B, H // 2, 2, W // 2, 2, C)
    return {'y': (terms.sum((2, 4)), 5 * na.U32 * terms.abs().sum((2, 4)))}


def window(rec, t, which):
    return rec['mem'][t['mem']][which].as_strided(t['size'], t['stride'], t['off'])


def check_launch(rec):
    """Checks (p), (a) and (c) of one launch.  -> {'ratio': worst error / bound, 'tile_rel': 0, 'tile': 0, 'errors'}"""
    errors = list(rec.get('pre', ()))
    ratio = 0.0
    refs = reference(rec)
    masks = {k: torch.zeros(st['after'].numel(), dtype=torch.bool, device=st['after'].device)
             for k, st in rec['mem'].items()}
    for t in rec['targets']:
        name = t['name']
        masks[t['mem']].as_strided(t['size'], t['stride'], t['off']).fill_(True)
        got = window(rec, t, 'after')
        ref, bound = refs[name]
        bits = ga._BITS[got.element_size()]
        if bound is None:
            differ = got.reshape(-1).view(bits) != ref.to(got.dtype).reshape(-1).view(bits)
            if differ.any():
                errors.append(f'(a) {name}: {int(differ.sum())} elements differ from the exact result, first at flat '
                              f'{int(differ.nonzero()[0])}')
            continue
        gd = got.double()
        err = (gd - ref).abs()
        full = na.U16[got.dtype] * ref.abs() + (1 + na.U16[got.dtype]) * bound + na.TINY[got.dtype]
        bad = ~(err <= full)
        if bad.any():
            i = tuple(int(v) for v in bad.nonzero()[0])
            errors.append(f'(a) {name}: {int(bad.sum())} elements out of bound, first at {i}: got {gd[i].item():.6g} '
                          f'want {ref[i].item():.6g} bound {full[i].item():.3g}')
        ratio = max(ratio, (err / full).nan_to_num(nan=float('inf')).max().item())
    for k, st in rec['mem'].items():
        bits = ga._BITS[st['after'].element_size()]
        stray = (st['after'].view(bits) != st['before'].view(bits)) & ~masks[k]
        if stray.any():
            errors.append(f'(c) storage {k[1]}: {int(stray.sum())} elements written outside the window, first at flat '
                          f'index {int(stray.nonzero()[0])}')
    return {'ratio': ratio, 'tile_rel': 0.0, 'tile': 0.0, 'errors': errors}


def simulate(rec):
    """Write the rounded reference into the 'after' storages: what a correct kernel leaves (CPU tests)."""
    for st in rec['mem'].values():
        st['after'] = st['before'].clone()
    refs = reference(rec)
    for t in rec['targets']:
        window(rec, t, 'after').copy_(refs[t['name']][0])
    return rec


class Recorder(ga.LaunchRecorder):
    """audits every launch of ENTRY_POINTS made inside it through the mos_b200.adapter_ops wrappers (the shared loop of
    gemm_audit.LaunchRecorder with the wrappers taken from adapter_ops instead of ops)"""
    ENTRY_POINTS = ENTRY_POINTS

    def __enter__(self):
        from mos_b200 import adapter_ops
        super().__enter__()                       # OPS is empty: installs the library proxy only
        self._adapter_ops = adapter_ops
        self._orig_adapter_ops = {n: getattr(adapter_ops, n) for n in OPS}

        def wrap(fn):
            def _audited(*args, **kwargs):
                assert self._ctx is None
                self._ctx = (ga._tensors(args, kwargs), ga._site(), (args, kwargs))
                try:
                    return fn(*args, **kwargs)
                finally:
                    self._ctx = None
            return _audited

        for n, fn in self._orig_adapter_ops.items():
            setattr(adapter_ops, n, wrap(fn))
        return self

    def __exit__(self, *exc):
        for n, fn in self._orig_adapter_ops.items():
            setattr(self._adapter_ops, n, fn)
        return super().__exit__(*exc)

    def record(self, entry, args, S):
        return record(entry, abi_of(entry, args[:len(_ARGS[entry])]), S, self._ctx[2])

    def key(self, rec):
        return adapter_path(rec)

    def check(self, rec):
        return check_launch(rec)
