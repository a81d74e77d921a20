"""Launch audit of the normalisation, layout and elementwise kernels: every call of an entry point in ENTRY_POINTS made
through its `ops.*` wrapper in a real engine walk, checked on its own.

The record is built, as in gemm_audit.py and attention_audit.py, from the arguments that reach the `mos_*` entry point:
every pointer is mapped into the storage of a tensor argument and each operand window is read there at the layout the
kernel uses, which for some operands is not passed at all (implicit pitches: `conv_out` reads x at pitch C, `upsample2x`
writes y at pitch C, `im2col_s2` writes col at pitch 9C, `col2im_s2` reads dcol at pitch 9C, `add_noise` and
`cfg_dpmpp_step` take dense tensors).  Since a reference read at the ABI layout agrees with a kernel that reads the same
wrong rows, (p) also compares the Python layout of those tensor arguments with the layout the kernel assumes.  The region
pointers of `region_combine` and `lora_pack` live in device tables: only those are resolved against the tensors
registered with the recorder (the outputs of `ops.attention`, where the engines write the region outputs, and the
training state and GEMM operands a walk registers); every other pointer must lie in a tensor argument of the call.

Record layout (as attention_audit): {'op': entry, 'abi': {...}, 'in': {operand windows}, 'targets': [{'name', 'mem',
'off', 'size', 'stride', 'unit', 'scratch'}], 'pre': [(p) messages], 'inplace': (operands the launch overwrites),
'mem': {storage: {'before', 'after'}}}.  `reference` and `check_launch` are pure functions of a record.

Element bound (a).  u = 2^-24 (fp32), u16 = 2^-8 (bf16) / 2^-11 (fp16), t16 the half subnormal step of the output type
(gemm_audit.TINY_OUT); every 16-bit output adds u16 |ref| + t16 to the fp32 error e below: |got - ref| <= u16 |ref| +
(1 + u16) e + t16.  An fp32 sum of n terms in any order errs by at most (n - 1) u sum |terms| (plus second-order terms,
covered by using n + 8).
- upsample2x, im2col_s2 (taps and zero pads), clip_embed's pad columns [C, ld), t_out of cfg_dpmpp_step and
  region_combine where at most one region covers a pixel: bit-exact (e = 0, no output rounding).
- add_rows, clip_embed: one fp32 add, e = u |a + b|.
- upsample2x_bwd, col2im_s2 (with `add`): sums of at most 4 (5) terms, e = 5u sum |terms|.
- conv_out (9C products per output, lane sums, the butterfly and the bias) and conv_out_bwd (9 Cout products):
  e = (n + 8) u sum |terms| with n the number of products.
- region_combine with k >= 2 covering regions: the k-term sum and the product with the rounded 1 / k: e = (k + 2) u sum |r|/k.
- quick_gelu: y = x / (1 + __expf(-1.702 x)).  __expf has 2 + floor(1.173 |z|) ulp (2^-23 relative each) at argument z
  = -1.702 x, the argument's own rounding adds 2u |z| (the constant and the product), and 1 + E and the division one u
  each: with s = sigmoid(1.702 x), e = |y| ((1 - s) e_E + 3u), e_E = (2 + 1.173 |z| + 1) 2^-23 + 2u |z|.
  quick_gelu_bwd: g = s + 1.702 x s (1 - s); the error of s is s (1 - s) e_E + 3u s, carried through
  |dg/ds| = |1 + 1.702 x (1 - 2 s)|, plus 6u (s + |1.702 x| s (1 - s)) for its own five operations and u |dy g|.
- geglu_fwd: a * gelu_erf(g): 8u (|g| + |gelu|) |a| (gemm_audit.GELU_ULP) and the product u |y|.  geglu_bwd: erff has 2
  ulp, so cdf errs by 8u + 2u |g| pdf; pdf = 0.39894 __expf(-g^2 / 2) has e_E at z = g^2 / 2 plus 4u; da = dy g cdf
  errs by |dy g| e_cdf + 2u |da|, dg = dy a (cdf + g pdf) by |dy a| (e_cdf + |g| pdf (e_E + 4u) + u |cdf + g pdf|) +
  2u |dg|.
- add_noise: sqrtf is correctly rounded; 1 - ac rounds once (u ac absolute, so sqrt(1 - ac) errs by u ac / (2 sqrt(1 - ac))),
  then two products and the add: e = 4u (|sqrt(ac) x0| + |sqrt(1 - ac) n|) + u ac |n| / (2 sqrt(1 - ac)).
- cfg_dpmpp_step (fp32 coefficients as passed): eps = u + g (c - u) errs by e_eps = u (|c - u| |g| + |g (c - u)| + |eps|)
  (contracted FMAs only remove roundings), x0 = (x - sigma eps) / alpha by e_x0 = (|sigma| e_eps + u |sigma eps| +
  u |x - sigma eps|) / |alpha| + u |x0|, xn = c_x x + c_m0 x0 + c_m1 x0_prev by |c_m0| e_x0 + 5u (|c_x x| + |c_m0 x0| +
  |c_m1 x0_prev|); unet_in holds xn (both CFG halves).
- layernorm (one warp per row, C terms) and groupnorm (n = HW C / 32 terms per (sample, group), merged across lanes,
  chunks or the CTAs of a cluster): the mean errs by e_m = (n + 8) u mean|x|, the centred variance by
  e_v = (n + 8) u var + 2 e_m mean|x - mean| + e_m^2; rsqrtf has 2 ulp, so rstd errs relatively by
  r = e_v / (2 (var + eps)) + 2^-22 + 2u; xhat = (x - mean) rstd by e_h = |xhat| r + rstd e_m + u |xhat|; z = xhat gamma
  + beta by |gamma| e_h + 2u (|xhat gamma| + |beta|); SiLU (GroupNorm) carries it with |silu'| <= 1.1 and adds
  |silu(z)| ((1 - sigmoid(z)) e_E + 2u) at z.
- groupnorm_bwd / layernorm_bwd (frozen affine): the statistics errors above give e_h for xhat; g = dy gamma
  (GroupNorm: times silu'(z), which carries e_z with |silu''| <= 1/2 and __expf's e_E through s (1 - s)), the n-term
  sums sa = mean g, sb = mean g xhat ((n + 8) u plus the carried errors), dx = rstd (g - sa - xhat sb) with rstd's
  relative error r and three roundings, then + add.
- timestep_embedding: f = expf(-ln(1e4) i / half) has 2 ulp plus 3u |arg|; the angle t f errs by |t f| (e_f + u) and
  cosf / sinf add 2 ulp absolute.  gemv: (K + 40) u (|x| |W| + |bias|) (lane sums, butterfly, bias), SiLU on input
  or output as above.  conv_in: (9 Cin + 8) u sum |terms|; conv1x1_nchw: (Cin + 2) u; vae_moments: (2L + 2) u for the
  1x1 conv, then latents = scaling (mu + __expf(lv / 2) noise) with e_E and four roundings.
- softmax_rows: the logit v c - m c with the rounded c = scale log2(e) errs by 3u (|v c| + |m c|) + u |v c - m c|, exp2f
  has 2 ulp; with delta_k those relative errors, out errs by P_k (delta_k + sum_j P_j delta_j + (cols + 10) u).
- clip_embed_bwd: a sum over the k matching positions (+ the accumulated value): k u sum |terms|.  masked_mse: num and
  den per sample over Cc HW (HW) terms, the loss mean and dpred = 2 gs (p - t) m / (den B) with seven roundings.
- lora_grad: t = x D^T and s = dY U err by (K + 8) u |x| |D| and (N + 8) u |dY| |U|; dD = alpha s^T x and
  dU = alpha dY^T t by (M + 16) u over the magnitudes plus the carried errors of s and t, then + d_* when accumulating.
- attn_reg_group: cm is the mean of L heads x layers terms ((L H + 2) u); the statistics are checked against the launch's
  own cm: max and the tie / zero counts exactly, loss, S0, S1 over B N terms ((B N + 16) u).  attn_reg_grad: eight
  roundings of each term and four of the product with k; with reg_full_identity also the rounding of x1 / M1 before
  the target is subtracted (u |x1 / M1| twice: the difference cancels where the map is close to the target).  attn_reg_total: (ngroups + 2) u; NaN where the reference is.
- flat_adamw_step: per element from the fp32 hyper-parameters passed: p (1 - lr wd) 3u, m 4u and v 5u of their terms,
  sqrt(v) min(e_v / (2 sqrt v), sqrt e_v) + u, the denominator, the step (lr / bc1) m / denom with 4u plus the carried
  errors; the row-norm mean of the embedding rows (read from the launch's updated params): (dim + 8) u / 2 + 2u per norm.
- lora_pack: a copy (bf16 rounding only for the bf16 operands) and alpha times a copy (one rounding).
The bounds grow with magnitudes, not with the values; a ratio above 1 is a finding, not a reason to widen them.

Checks of every launch (`check_launch`):
  p. every tensor argument's row pitch equals the pitch the kernel reads it at (the ABI's, or the implicit one above),
     dense operands are contiguous, timesteps lie in [0, len(alphas_cumprod)), region boxes inside the map, and the
     pointers of the region and lora_pack tables resolve into registered storages (else the record cannot be built);
  a. the element bound above; the bit-exact outputs bit for bit;
  b. rel-L2 per natural unit within the existing kernel tests' limits: each (sample, group) for GroupNorm forward and
     backward (4e-3 bf16, 6e-4 fp16), each row for LayerNorm, GEGLU, QuickGELU and softmax_rows, each output channel of
     lora_grad (1e-4) and each AdamW parameter group (1e-5);
  c. every byte of a written storage outside the launch's window is bitwise unchanged: pitch pads (clip_embed's must
     become zero: they are in its window), and for the GroupNorm fallback's partial buffer, the GroupNorm backward
     workspace, the lora_grad workspace and mse_ws everything past the prefix the copied host rule uses.
The recorder (gemm_audit.LaunchRecorder) adds (d) unchanged operands (in-place targets exempt: their reference is built
from the snapshot taken before the launch) and (e) a bit-identical relaunch (none of these kernels uses atomics).
"""
import math
import os

import torch

import gemm_audit as ga
from gemm_audit import Stats, _Storages  # noqa: F401  (the table and storage map of every audit)

U32 = 2.0 ** -24
ULP = 2.0 ** -23
U16 = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}
TINY = {torch.bfloat16: ga.TINY_OUT[torch.bfloat16], torch.float16: ga.TINY_OUT[torch.float16], torch.float32: 0.0}
DT16 = ga.DT16
BF, F32 = torch.bfloat16, torch.float32
UNIT_TOL = {torch.bfloat16: 4e-3, torch.float16: 6e-4}
GN_GROUPS = 32
_BITS = ga._BITS
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
SMS = None                     # SM count for the GroupNorm rule; None: the current device's (132 without a GPU)


# --------------------------------------------------------------------------------------------------- ABI tables
_ARGS = {
    'mos_groupnorm_fwd': ('x', 'ldx', 'B', 'HW', 'C', 'gamma', 'beta', 'eps', 'silu', 'partial', 'partial_floats', 'y',
                          'ldy', 'act_dtype'),
    'mos_layernorm_fwd': ('x', 'ldx', 'M', 'C', 'gamma', 'beta', 'eps', 'y', 'ldy', 'act_dtype'),
    'mos_conv_out': ('x', 'B', 'H', 'W', 'C', 'w', 'bias', 'Cout', 'y', 'act_dtype'),
    'mos_upsample2x': ('x', 'ldx', 'B', 'H', 'W', 'C', 'y'),
    'mos_im2col_s2': ('x', 'ldx', 'B', 'H', 'W', 'C', 'pad', 'col'),
    'mos_add_rows': ('x', 'ldx', 'r', 'ldr', 'M', 'C', 'act_dtype'),
    'mos_clip_embed': ('ids', 'tok', 'pos', 'M', 'T', 'C', 'vocab', 'x', 'ld'),
    'mos_quick_gelu': ('x', 'ld', 'M', 'C'),
    'mos_quick_gelu_fwd': ('x', 'ldx', 'M', 'C', 'y', 'ldy'),
    'mos_quick_gelu_bwd': ('x', 'ldx', 'dy', 'lddy', 'M', 'C', 'dx', 'lddx'),
    'mos_cfg_dpmpp_step': ('noise_pred', 'latents', 'x0_prev', 'unet_in', 'n', 'cfg', 'guidance', 'c_x', 'c_m0', 'c_m1',
                           'alpha_s', 'sigma_s', 't_out', 't_count', 't_next'),
    'mos_region_combine': ('glob', 'table', 'n', 'boxes', 'B', 'FH', 'FW', 'C', 'ld', 'out', 'act_dtype'),
    'mos_geglu_fwd': ('z', 'ldz', 'M', 'H', 'y', 'ldy'),
    'mos_geglu_bwd': ('z', 'ldz', 'dy', 'lddy', 'M', 'H', 'dz', 'lddz'),
    'mos_upsample2x_bwd': ('dy', 'lddy', 'B', 'H', 'W', 'C', 'dx', 'lddx'),
    'mos_col2im_s2': ('dcol', 'B', 'H', 'W', 'C', 'add', 'ldadd', 'dx', 'lddx'),
    'mos_conv_out_bwd': ('dy', 'B', 'H', 'W', 'C', 'w', 'Cout', 'dx'),
    'mos_add_noise': ('x0', 'noise', 't', 'ac', 'B', 'per', 'out'),
    'mos_groupnorm_bwd': ('x', 'ldx', 'dy', 'lddy', 'B', 'HW', 'C', 'gamma', 'beta', 'eps', 'silu', 'ws', 'ws_floats',
                          'add', 'ldadd', 'dx', 'lddx'),
    'mos_layernorm_bwd': ('x', 'ldx', 'dy', 'lddy', 'M', 'C', 'gamma', 'eps', 'add', 'ldadd', 'dx', 'lddx'),
    'mos_timestep_embedding': ('t', 'B', 'dim', 'out'),
    'mos_gemv_bf16': ('x', 'nb', 'K', 'W', 'bias', 'N', 'act_in', 'act_out', 'out', 'ldo'),
    'mos_conv_in': ('x', 'B', 'Cin', 'H', 'W', 'w', 'bias', 'Cout', 'y', 'ldy', 'act_dtype'),
    'mos_softmax_rows': ('S', 'lds', 'rows', 'cols', 'scale', 'out', 'ldo', 'act_dtype'),
    'mos_conv1x1_nchw': ('x', 'B', 'Cin', 'HW', 'w', 'bias', 'Cout', 'y'),
    'mos_vae_moments': ('h', 'ldh', 'B', 'HW', 'L', 'w', 'bias', 'mean', 'logvar', 'noise', 'scaling', 'latents',
                        'act_dtype'),
    'mos_clip_embed_bwd': ('ids', 'dx', 'ld', 'M', 'C', 'rows', 'n_rows', 'accumulate', 'out'),
    'mos_masked_mse': ('pred', 'target', 'mask', 'B', 'Cc', 'HW', 'grad_scale', 'ws', 'loss', 'dpred'),
    'mos_lora_grad': ('x', 'ldx', 'dy', 'lddy', 'M', 'K', 'N', 'down', 'up', 'alpha', 'ws', 'ws_floats', 'accumulate',
                      'd_down', 'd_up'),
    'mos_attn_reg_group': ('pcols', 'L', 'B', 'heads', 'res', 'mask', 'MH', 'MW', 'full', 'weight', 'cm', 'stats'),
    'mos_attn_reg_grad': ('cm', 'mask', 'B', 'res', 'MH', 'MW', 'full', 'weight', 'stats_all', 'ngroups', 'group', 'L',
                          'heads', 'grad_scale', 'gcols'),
    'mos_attn_reg_total': ('mse', 'stats_all', 'ngroups', 'out'),
    'mos_flat_adamw_step': ('p', 'g', 'm', 'v', 'n', 'group_end', 'group_lr', 'beta1', 'beta2', 'eps', 'wd', 'step',
                            'grad_scale', 'emb_rows', 'emb_dim', 'norm_out'),
    'mos_lora_pack': ('table', 'n', 'alpha'),
}
ENTRY_POINTS = tuple(_ARGS)
_FLOATS = ('eps', 'guidance', 'c_x', 'c_m0', 'c_m1', 'alpha_s', 'sigma_s', 't_next', 'scale', 'scaling', 'grad_scale',
           'alpha', 'weight', 'beta1', 'beta2', 'wd')
# operands whose pitch the kernel assumes: entry -> [(position of the tensor in the ops.* call, name, pitch(abi))]
IMPLICIT = {
    'mos_add_noise': [(0, 'x0', None), (1, 'noise', None), (4, 'out', None)],
    'mos_cfg_dpmpp_step': [(0, 'noise_pred', None), (1, 'latents', None), (2, 'x0_prev', None), (3, 'unet_in', None)],
}


def abi_of(entry, args):
    """the ctypes arguments of an entry point -> plain dict (pointers as ints, 0 for NULL; floats as their fp32 value;
    region boxes as a list of 4-tuples)"""
    a = {}
    for n, v in zip(_ARGS[entry], args):
        if n == 'boxes':
            continue
        if hasattr(v, '_length_'):                                          # ctypes array: host table
            a[n] = [float(e) if n == 'group_lr' else int(e or 0) for e in v]
            continue
        v = getattr(v, 'value', v)
        a[n] = float(v) if n in _FLOATS else (0 if v is None else int(v))
    if entry == 'mos_region_combine':
        a['boxes'] = [tuple(int(args[3][4 * i + k]) for k in range(4)) for i in range(a['n'])]
    return a


def _dt(a):
    return DT16[a.get('act_dtype', 0)]


# --------------------------------------------------------------------------------------------------- host rules
def _sms():
    if SMS is not None:
        return SMS
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count \
        if torch.cuda.is_available() else 132


def gn_threads(C):
    oct_ = C // 8
    return oct_ * max(1, 320 // oct_)


def gn_rule(a):
    """(path, k, vec, nchunks) of a mos_groupnorm_fwd launch: a copy of the host rule in csrc/norm.cu, mos_groupnorm_fwd
    (MOS_GN_TWOPASS, MOS_GN_MIN_CTAS, the cluster widening loop, the shared-memory limit and the fallback's chunking);
    keep the two in step."""
    B, HW, C, ldx, ldy = a['B'], a['HW'], a['C'], a['ldx'], a['ldy']
    cpg = C // GN_GROUPS
    if os.environ.get('MOS_GN_TWOPASS', '')[:1] != '1':
        vec = 4 if cpg % 4 == 0 and ldx % 4 == 0 and ldy % 4 == 0 else 2
        slab = HW * cpg * 2
        try:
            min_ctas = int(os.environ['MOS_GN_MIN_CTAS'])
        except (KeyError, ValueError):
            min_ctas = 0
        if min_ctas < 1:
            min_ctas = 2 * _sms()
        k = 1
        while k < 8 and HW // (2 * k) >= 16 and (slab // k > 48 * 1024 or B * GN_GROUPS * k < min_ctas):
            k *= 2
        smem = -(-HW // k) * cpg * 2
        if smem <= 200 * 1024 and cpg % 2 == 0 and ldx % 2 == 0 and ldy % 2 == 0:
            return 'cluster', k, vec, 0
    threads = gn_threads(C)
    nchunks = -(-2368 // B)
    min_rows = 4 * (threads // (C // 8))
    nchunks = min(nchunks, -(-HW // min_rows), a['partial_floats'] // (B * GN_GROUPS * 2))
    nchunks = max(nchunks, 1)
    rows = -(-HW // nchunks)
    return 'fallback', 0, 0, -(-HW // rows)


def norm_path(rec):
    """Path key of a launch: the features that select code in csrc/norm.cu, elementwise.cu and backward.cu (a copy of
    their host rules; keep them in step)."""
    e, a = rec['op'], rec['abi']
    dt = 'fp16' if _dt(a) == torch.float16 else 'bf16'
    if e == 'mos_groupnorm_fwd':
        path, k, vec, _ = gn_rule(a)
        key = ['gn', dt, path] + ([f'k={k}', f'v{vec}'] if path == 'cluster' else [])
        return '|'.join(key + ['silu'] * bool(a['silu']))
    if e == 'mos_layernorm_fwd':
        return f"ln|{dt}|C={a['C']}" + ('|mtail' if a['M'] % 8 else '')
    if e == 'mos_im2col_s2':
        return f"im2col|pad={a['pad']}"
    if e == 'mos_region_combine':
        return f"region|{dt}|n={a['n']}" + ('|inplace' if a['glob'] == a['out'] else '')
    if e == 'mos_cfg_dpmpp_step':
        return 'cfg_step|' + ('cfg' if a['cfg'] else 'nocfg') + ('|t_out' if a['t_out'] else '') + \
            ('|unet_in' if a['unet_in'] else '')
    if e == 'mos_col2im_s2':
        return 'col2im' + ('|add' if a['add'] else '')
    if e in ('mos_conv_out', 'mos_add_rows', 'mos_conv_in', 'mos_softmax_rows', 'mos_vae_moments'):
        return f"{e[4:]}|{dt}" + ('|noise' if a.get('noise') else '')
    if e == 'mos_groupnorm_bwd':
        return 'gn_bwd' + ('|silu' if a['silu'] else '') + ('|add' if a['add'] else '')
    if e == 'mos_layernorm_bwd':
        return f"ln_bwd|C={a['C']}" + ('|mtail' if a['M'] % 8 else '') + ('|add' if a['add'] else '')
    if e == 'mos_gemv_bf16':
        return f"gemv|nb={a['nb']}" + ('|act_in' if a['act_in'] else '') + ('|act_out' if a['act_out'] else '')
    if e == 'mos_lora_grad':
        R, _, staged = lora_grad_rule(a)
        return f"lora_grad|R={R}|" + ('staged' if staged else 'global') + ('|acc' if a['accumulate'] else '')
    if e == 'mos_flat_adamw_step':
        return 'adamw' + ('|norm' if a['norm_out'] and a['emb_rows'] > 0 else '')
    if e == 'mos_clip_embed_bwd':
        return 'clip_embed_bwd' + ('|acc' if a['accumulate'] else '')
    if e == 'mos_attn_reg_group':
        return f"attn_reg_group|L={a['L']}" + ('|full' if a['full'] else '')
    return e[4:]


# --------------------------------------------------------------------------------------------------- records
def record(entry, a, S, call=None):
    """the launch record of one entry-point call (operand windows and written storages still live); call: the
    (args, kwargs) of the ops.* wrapper, for the implicit-pitch preconditions"""
    x, targets, pre, inplace, pitches = {}, [], [], [], {}

    def win(name, dtype, size, stride, p=None, ld=None, table=False):
        p = a[name] if p is None else p
        x[name] = S.window(p, name, dtype, size, stride, table=table)
        if ld is not None:
            pitches[p] = (name, ld)
        return x[name]

    def target(name, dtype, size, stride, unit=None, scratch=False, p=None, ld=None, table=False, **kw):
        p = a[name] if p is None else p
        if ld is not None:
            pitches[p] = (name, ld)
        base, off = S.find(p, name, table=table)
        es = torch.empty(0, dtype=dtype).element_size()
        assert off % es == 0, f'{name}: pointer not aligned to its element size'
        t = dict(name=name, mem=(base, dtype), off=off // es, size=tuple(size), stride=tuple(stride), unit=unit,
                 scratch=scratch, **kw)
        S.flat(base, dtype).as_strided(t['size'], t['stride'], t['off'])     # raises if it runs past its storage
        targets.append(t)

    args = call[0] if call else ()
    for pos, name, pitch in IMPLICIT.get(entry, ()):
        if pos >= len(args) or not isinstance(args[pos], torch.Tensor):
            continue
        t = args[pos]
        if pitch is None:
            if not t.is_contiguous():
                pre.append(f'(p) {name}: taken dense by the kernel, passed with strides {tuple(t.stride())}')
        elif t.stride(-1) != 1 or (t.dim() >= 2 and t.shape[-2] > 1 and t.stride(-2) != pitch(a)):
            pre.append(f'(p) {name}: the kernel assumes row pitch {pitch(a)}, the call passes strides {tuple(t.stride())}')

    if entry in ('mos_groupnorm_fwd', 'mos_layernorm_fwd'):
        dt = _dt(a)
        C = a['C']
        if entry == 'mos_groupnorm_fwd':
            B, HW, cpg = a['B'], a['HW'], C // GN_GROUPS
            win('x', dt, (B, HW, GN_GROUPS, cpg), (HW * a['ldx'], a['ldx'], cpg, 1), ld=a['ldx'])
            target('y', dt, (B, HW, GN_GROUPS, cpg), (HW * a['ldy'], a['ldy'], cpg, 1), unit=(1, 3), ld=a['ldy'])
            path, _, _, nchunks = gn_rule(a)
            if path == 'fallback':
                target('partial', F32, (B * nchunks * GN_GROUPS * 2,), (1,), scratch=True)
        else:
            win('x', dt, (a['M'], C), (a['ldx'], 1), ld=a['ldx'])
            target('y', dt, (a['M'], C), (a['ldy'], 1), unit=(1,), ld=a['ldy'])
        win('gamma', F32, (C,), (1,))
        win('beta', F32, (C,), (1,))
    elif entry == 'mos_conv_out':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        win('x', _dt(a), (B, H, W, C), (H * W * C, W * C, C, 1), ld=C)
        win('w', F32, (a['Cout'], 9, C), (9 * C, C, 1))
        win('bias', F32, (a['Cout'],), (1,))
        target('y', F32, (B, a['Cout'], H, W), (a['Cout'] * H * W, H * W, W, 1))
    elif entry == 'mos_upsample2x':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        win('x', BF, (B, H, W, C), (H * W * a['ldx'], W * a['ldx'], a['ldx'], 1), ld=a['ldx'])
        target('y', BF, (B, 2 * H, 2 * W, C), (4 * H * W * C, 2 * W * C, C, 1), ld=C)
    elif entry == 'mos_im2col_s2':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        win('x', BF, (B, H, W, C), (H * W * a['ldx'], W * a['ldx'], a['ldx'], 1), ld=a['ldx'])
        Ho, Wo = H // 2, W // 2
        target('col', BF, (B, Ho, Wo, 9, C), (Ho * Wo * 9 * C, Wo * 9 * C, 9 * C, C, 1), ld=9 * C)
    elif entry == 'mos_add_rows':
        dt = _dt(a)
        win('r', dt, (a['M'], a['C']), (a['ldr'], 1), ld=a['ldr'])
        win('x', dt, (a['M'], a['C']), (a['ldx'], 1), ld=a['ldx'])
        target('x', dt, (a['M'], a['C']), (a['ldx'], 1))
        inplace.append('x')
    elif entry == 'mos_clip_embed':
        M, C = a['M'], a['C']
        win('ids', torch.int32, (M,), (1,))
        win('tok', F32, (a['vocab'], C), (C, 1))
        win('pos', F32, (a['T'], C), (C, 1))
        target('x', BF, (M, a['ld']), (a['ld'], 1), ld=a['ld'])
    elif entry in ('mos_quick_gelu', 'mos_quick_gelu_fwd'):
        ldx = a['ld'] if entry == 'mos_quick_gelu' else a['ldx']
        win('x', BF, (a['M'], a['C']), (ldx, 1), ld=ldx)
        if entry == 'mos_quick_gelu':
            target('x', BF, (a['M'], a['C']), (ldx, 1), unit=(1,))
            inplace.append('x')
        else:
            target('y', BF, (a['M'], a['C']), (a['ldy'], 1), unit=(1,), ld=a['ldy'])
    elif entry == 'mos_quick_gelu_bwd':
        win('x', BF, (a['M'], a['C']), (a['ldx'], 1), ld=a['ldx'])
        win('dy', BF, (a['M'], a['C']), (a['lddy'], 1), ld=a['lddy'])
        target('dx', BF, (a['M'], a['C']), (a['lddx'], 1), unit=(1,), ld=a['lddx'])
    elif entry in ('mos_geglu_fwd', 'mos_geglu_bwd'):
        M, Hh = a['M'], a['H']
        win('z', BF, (M, Hh // 80, 2, 80), (a['ldz'], 160, 80, 1), ld=a['ldz'])
        if entry == 'mos_geglu_fwd':
            target('y', BF, (M, Hh // 80, 80), (a['ldy'], 80, 1), unit=(1, 2), ld=a['ldy'])
        else:
            win('dy', BF, (M, Hh // 80, 80), (a['lddy'], 80, 1), ld=a['lddy'])
            target('dz', BF, (M, Hh // 80, 2, 80), (a['lddz'], 160, 80, 1), unit=(1, 2, 3), ld=a['lddz'])
    elif entry == 'mos_upsample2x_bwd':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        win('dy', BF, (B, 2 * H, 2 * W, C), (4 * H * W * a['lddy'], 2 * W * a['lddy'], a['lddy'], 1), ld=a['lddy'])
        target('dx', BF, (B, H, W, C), (H * W * a['lddx'], W * a['lddx'], a['lddx'], 1), ld=a['lddx'])
    elif entry == 'mos_col2im_s2':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        Ho, Wo = H // 2, W // 2
        win('dcol', BF, (B, Ho, Wo, 9, C), (Ho * Wo * 9 * C, Wo * 9 * C, 9 * C, C, 1), ld=9 * C)
        if a['add']:
            win('add', BF, (B, H, W, C), (H * W * a['ldadd'], W * a['ldadd'], a['ldadd'], 1), ld=a['ldadd'])
        target('dx', BF, (B, H, W, C), (H * W * a['lddx'], W * a['lddx'], a['lddx'], 1), ld=a['lddx'])
        if a['add'] == a['dx']:
            inplace.append('add')
    elif entry == 'mos_conv_out_bwd':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        win('dy', F32, (B, a['Cout'], H, W), (a['Cout'] * H * W, H * W, W, 1))
        win('w', F32, (a['Cout'], 9, C), (9 * C, C, 1))
        target('dx', BF, (B, H, W, C), (H * W * C, W * C, C, 1), ld=C)
    elif entry == 'mos_add_noise':
        B, per = a['B'], a['per']
        win('x0', F32, (B, per), (per, 1))
        win('noise', F32, (B, per), (per, 1))
        ts = win('t', torch.int32, (B,), (1,))
        ac_arg = call[0][3] if call and len(call[0]) > 3 and isinstance(call[0][3], torch.Tensor) else None
        n_ac = ac_arg.numel() if ac_arg is not None else 1000
        win('ac', F32, (n_ac,), (1,))
        if not ((ts >= 0) & (ts < n_ac)).all():
            pre.append(f'(p) timesteps {ts.tolist()} not in [0, {n_ac})')
        target('out', F32, (B, per), (per, 1))
    elif entry == 'mos_cfg_dpmpp_step':
        n = a['n']
        win('noise_pred', F32, ((2 if a['cfg'] else 1) * n,), (1,))
        win('latents', F32, (n,), (1,))
        win('x0_prev', F32, (n,), (1,))
        target('latents', F32, (n,), (1,))
        target('x0_prev', F32, (n,), (1,))
        inplace += ['latents', 'x0_prev']
        if a['unet_in']:
            target('unet_in', F32, ((2 if a['cfg'] else 1) * n,), (1,))
        if a['t_out']:
            target('t_out', F32, (a['t_count'],), (1,))
    elif entry == 'mos_region_combine':
        dt = _dt(a)
        B, FH, FW, C, ld = a['B'], a['FH'], a['FW'], a['C'], a['ld']
        size, stride = (B, FH, FW, C), (FH * FW * ld, FW * ld, ld, 1)
        win('glob', dt, size, stride, ld=ld)
        table = win('table', torch.int64, (a['n'],), (1,))
        for i, p in enumerate(table.tolist()):
            try:
                win(f'region{i}', dt, size, stride, p=p, table=True)
            except AssertionError as e:
                pre.append(f'(p) region table entry {i}: {e}')
        for i, (sh, sw, eh, ew) in enumerate(a['boxes']):
            if not (0 <= sh <= eh <= FH and 0 <= sw <= ew <= FW):
                pre.append(f'(p) region box {i} {(sh, sw, eh, ew)} not inside the {FH} x {FW} map')
        target('out', dt, size, stride, ld=ld)
        if a['glob'] == a['out']:
            inplace.append('glob')
    else:
        _record_training(entry, a, S, x, win, target, pre, inplace)
    for t in ga._tensors(*call) if call else ():
        hit = pitches.get(t.data_ptr())
        if hit is not None and t.dim() >= 2 and t.shape[-2] > 1 and t.stride(-2) != hit[1]:
            pre.append(f'(p) {hit[0]}: the kernel reads it at row pitch {hit[1]}, the tensor passed has strides '
                       f'{tuple(t.stride())}')
    return {'op': entry, 'abi': a, 'in': x, 'targets': targets, 'pre': pre, 'inplace': tuple(inplace)}



def gn_bwd_chunks(a):
    """nchunks of a mos_groupnorm_bwd launch: a copy of the host rule in csrc/norm.cu, mos_groupnorm_bwd; keep the two
    in step.  The workspace prefix it uses is B * nchunks * 128 floats (the statistics, then the dy sums)."""
    B, HW, C = a['B'], a['HW'], a['C']
    nchunks = min(-(-1184 // B), -(-HW // (4 * (gn_threads(C) // (C // 8)))), a['ws_floats'] // (B * GN_GROUPS * 4))
    rows = -(-HW // nchunks)
    return -(-HW // rows)


def lora_grad_rule(a):
    """(R, nb, staged) of a mos_lora_grad launch: a copy of the host rule in csrc/backward.cu, mos_lora_grad (slab
    height, block count, D / U staged in shared memory); keep the two in step."""
    M, K, N = a['M'], a['K'], a['N']
    R = -(-(-(-M // 128)) // 16) * 16
    R = min(R, 1024)
    if R < 256:
        p2 = 16
        while p2 < R:
            p2 *= 2
        R = p2
    else:
        R = -(-R // 256) * 256
    staged = (R * 8 + 4 * 32 * 64) * 4 + (4 * K + 4 * N) * 4 <= 200 * 1024
    return R, -(-M // R), staged


def _record_training(entry, a, S, x, win, target, pre, inplace):
    """record builders of the backward, training-glue, VAE, time-embedding and optimizer entry points"""
    if entry in ('mos_groupnorm_bwd', 'mos_layernorm_bwd'):
        C = a['C']
        if entry == 'mos_groupnorm_bwd':
            B, HW, cpg = a['B'], a['HW'], C // GN_GROUPS
            shp = (B, HW, GN_GROUPS, cpg)
            st = lambda ld: (HW * ld, ld, cpg, 1)                                        # noqa: E731
            unit = (1, 3)
            win('beta', F32, (C,), (1,))
            target('ws', F32, (B * gn_bwd_chunks(a) * GN_GROUPS * 4,), (1,), scratch=True)
        else:
            shp, st, unit = (a['M'], C), (lambda ld: (ld, 1)), (1,)
        win('x', BF, shp, st(a['ldx']), ld=a['ldx'])
        win('dy', BF, shp, st(a['lddy']), ld=a['lddy'])
        win('gamma', F32, (C,), (1,))
        if a['add']:
            win('add', BF, shp, st(a['ldadd']), ld=a['ldadd'])
            if a['add'] == a['dx']:
                inplace.append('add')
        target('dx', BF, shp, st(a['lddx']), unit=unit, ld=a['lddx'])
    elif entry == 'mos_timestep_embedding':
        win('t', F32, (a['B'],), (1,))
        target('out', F32, (a['B'], a['dim']), (a['dim'], 1))
    elif entry == 'mos_gemv_bf16':
        win('x', F32, (a['nb'], a['K']), (a['K'], 1), ld=a['K'])
        win('W', BF, (a['N'], a['K']), (a['K'], 1), ld=a['K'])
        if a['bias']:
            win('bias', F32, (a['N'],), (1,))
        target('out', F32, (a['nb'], a['N']), (a['ldo'], 1), ld=a['ldo'])
    elif entry == 'mos_conv_in':
        B, Ci, H, W, Co = a['B'], a['Cin'], a['H'], a['W'], a['Cout']
        win('x', F32, (B, Ci, H, W), (Ci * H * W, H * W, W, 1))
        win('w', F32, (9 * Ci, Co), (Co, 1), ld=Co)
        win('bias', F32, (Co,), (1,))
        target('y', _dt(a), (B, H, W, Co), (H * W * a['ldy'], W * a['ldy'], a['ldy'], 1), ld=a['ldy'])
    elif entry == 'mos_softmax_rows':
        win('S', F32, (a['rows'], a['cols']), (a['lds'], 1), ld=a['lds'])
        target('out', _dt(a), (a['rows'], a['cols']), (a['ldo'], 1), unit=(1,), ld=a['ldo'])
    elif entry == 'mos_conv1x1_nchw':
        B, Ci, HW, Co = a['B'], a['Cin'], a['HW'], a['Cout']
        win('x', F32, (B, Ci, HW), (Ci * HW, HW, 1))
        win('w', F32, (Co, Ci), (Ci, 1))
        win('bias', F32, (Co,), (1,))
        target('y', F32, (B, Co, HW), (Co * HW, HW, 1))
    elif entry == 'mos_vae_moments':
        B, HW, L = a['B'], a['HW'], a['L']
        win('h', _dt(a), (B, HW, 2 * L), (HW * a['ldh'], a['ldh'], 1), ld=a['ldh'])
        win('w', F32, (2 * L, 2 * L), (2 * L, 1))
        win('bias', F32, (2 * L,), (1,))
        for n in ('mean', 'logvar'):
            target(n, F32, (B, L, HW), (L * HW, HW, 1))
        if a['noise']:
            win('noise', F32, (B, L, HW), (L * HW, HW, 1))
            target('latents', F32, (B, L, HW), (L * HW, HW, 1))
    elif entry == 'mos_clip_embed_bwd':
        win('ids', torch.int32, (a['M'],), (1,))
        win('dx', BF, (a['M'], a['C']), (a['ld'], 1), ld=a['ld'])
        win('rows', torch.int32, (a['n_rows'],), (1,))
        if a['accumulate']:
            win('out', F32, (a['n_rows'], a['C']), (a['C'], 1))
            inplace.append('out')
        target('out', F32, (a['n_rows'], a['C']), (a['C'], 1), ld=a['C'])
    elif entry == 'mos_masked_mse':
        B, Cc, HW = a['B'], a['Cc'], a['HW']
        for n in ('pred', 'target'):
            win(n, F32, (B, Cc, HW), (Cc * HW, HW, 1))
        win('mask', F32, (B, HW), (HW, 1))
        target('ws', F32, (B, 2), (2, 1))
        target('loss', F32, (1,), (1,))
        target('dpred', F32, (B, Cc, HW), (Cc * HW, HW, 1))
    elif entry == 'mos_lora_grad':
        M, K, N = a['M'], a['K'], a['N']
        win('x', BF, (M, K), (a['ldx'], 1), ld=a['ldx'])
        win('dy', BF, (M, N), (a['lddy'], 1), ld=a['lddy'])
        win('down', F32, (4, K), (K, 1))
        win('up', F32, (N, 4), (4, 1))
        R, nb, _ = lora_grad_rule(a)
        target('ws', F32, (nb * 4 * (K + N),), (1,), scratch=True)
        if a['accumulate']:
            win('d_down', F32, (4, K), (K, 1))
            win('d_up', F32, (N, 4), (4, 1))
            inplace += ['d_down', 'd_up']
        target('d_down', F32, (4, K), (K, 1), unit=(0,), tol=1e-4)
        target('d_up', F32, (N, 4), (4, 1), unit=(1,), tol=1e-4)
    elif entry == 'mos_attn_reg_group':
        B, Hh, N = a['B'], a['heads'], a['res'] * a['res']
        for l, p in enumerate(a['pcols'][:a['L']]):
            win(f'pcols{l}', F32, (B, Hh, N, 2), (Hh * N * 2, N * 2, 2, 1), p=p)
        win('mask', F32, (B, a['MH'], a['MW']), (a['MH'] * a['MW'], a['MW'], 1))
        target('cm', F32, (B, N, 2), (N * 2, 2, 1))
        target('stats', F32, (8,), (1,))
    elif entry == 'mos_attn_reg_grad':
        B, N = a['B'], a['res'] * a['res']
        win('cm', F32, (B, N, 2), (N * 2, 2, 1))
        win('mask', F32, (B, a['MH'], a['MW']), (a['MH'] * a['MW'], a['MW'], 1))
        win('stats_all', F32, (a['ngroups'], 8), (8, 1))
        if not 0 <= a['group'] < a['ngroups']:
            pre.append(f"(p) group {a['group']} not in [0, {a['ngroups']})")
        target('gcols', F32, (B, N, 2), (N * 2, 2, 1))
    elif entry == 'mos_attn_reg_total':
        win('mse', F32, (1,), (1,))
        win('stats_all', F32, (a['ngroups'], 8), (8, 1))
        target('out', F32, (2,), (1,))
    elif entry == 'mos_flat_adamw_step':
        n = a['n']
        for k in ('p', 'g', 'm', 'v'):
            win(k, F32, (n,), (1,))
        ge = a['group_end']
        if not (0 <= ge[0] <= ge[1] <= ge[2] == n):
            pre.append(f'(p) group ends {ge} not increasing to {n}')
        groups = [(0, ge[0]), (ge[0], ge[1]), (ge[1], ge[2])]
        for k in ('p', 'm', 'v'):
            target(k, F32, (n,), (1,), groups=groups if k == 'p' else None, tol=1e-5)
        inplace += ['p', 'm', 'v']
        if a['norm_out'] and a['emb_rows'] > 0:
            target('norm_out', F32, (1,), (1,))
    elif entry == 'mos_lora_pack':
        table = win('table', torch.int64, (a['n'], 8), (8, 1))
        for i, (D, U, K, N, fd, fu, bd, bu) in enumerate(table.tolist()):
            win(f'D{i}', F32, (4, K), (K, 1), p=D, table=True)
            win(f'U{i}', F32, (N, 4), (4, 1), p=U, table=True)
            target(f'fdown{i}', BF, (4, K), (K, 1), p=fd, table=True, src=('D', i))
            target(f'fup{i}', F32, (N, 4), (4, 1), p=fu, table=True, src=('U', i))
            if bd:
                target(f'bdown{i}', BF, (4, N), (N, 1), p=bd, table=True, src=('U', i))
            if bu:
                target(f'bup{i}', F32, (K, 4), (4, 1), p=bu, table=True, src=('D', i))
    else:
        raise AssertionError(f'no record builder for {entry}')


# --------------------------------------------------------------------------------------------------- references
def _e_exp(z):
    """relative error of __expf at argument z (its ulp bound plus the argument's rounding)"""
    return (3 + 1.173 * z.abs()) * ULP + 2 * U32 * z.abs()


def _norm_ref(rec, x, dims, silu):
    """float64 (x - mean) rstd gamma + beta (+ SiLU) over `dims`, with its fp32 error bound"""
    a, g, b = rec['abi'], rec['in']['gamma'].double(), rec['in']['beta'].double()
    n = 1
    for d in dims:
        n *= x.shape[d]
    mean = x.mean(dims, keepdim=True)
    dev = x - mean
    var = (dev * dev).mean(dims, keepdim=True)
    rstd = (var + a['eps']).rsqrt()
    xh = dev * rstd
    cn = (n + 8) * U32
    e_m = cn * x.abs().mean(dims, keepdim=True)
    e_v = cn * var + 2 * e_m * dev.abs().mean(dims, keepdim=True) + e_m * e_m
    r = e_v / (2 * (var + a['eps'])) + 2.0 ** -22 + 2 * U32
    e_h = xh.abs() * r + rstd * e_m + U32 * xh.abs()
    if x.dim() == 4:                                                     # GroupNorm: [B, HW, G, cpg]
        g, b = g.view(GN_GROUPS, -1), b.view(GN_GROUPS, -1)
    z = xh * g + b
    e_z = g.abs() * e_h + 2 * U32 * ((xh * g).abs() + b.abs())
    if not silu:
        return z, e_z
    s = torch.sigmoid(z)
    y = z * s
    return y, 1.1 * e_z + y.abs() * ((1 - s) * _e_exp(z) + 2 * U32)


def reference(rec):
    """float64 reference of every output target: {name: (ref, fp32 error bound)}; bound None: bit-exact"""
    e, a, x = rec['op'], rec['abi'], rec['in']
    if e == 'mos_groupnorm_fwd':
        return {'y': _norm_ref(rec, x['x'].double(), (1, 3), a['silu'])}
    if e == 'mos_layernorm_fwd':
        return {'y': _norm_ref(rec, x['x'].double(), (1,), False)}
    if e == 'mos_conv_out':
        X = x['x'].double().permute(0, 3, 1, 2)                            # [B, C, H, W]
        W = x['w'].double().view(a['Cout'], 3, 3, a['C']).permute(0, 3, 1, 2)
        y = torch.nn.functional.conv2d(X, W, x['bias'].double(), padding=1)
        mag = torch.nn.functional.conv2d(X.abs(), W.abs(), x['bias'].double().abs(), padding=1)
        return {'y': (y, (9 * a['C'] + 8) * U32 * mag)}
    if e == 'mos_upsample2x':
        return {'y': (x['x'].repeat_interleave(2, 1).repeat_interleave(2, 2), None)}
    if e == 'mos_im2col_s2':
        p = a['pad']
        X = torch.nn.functional.pad(x['x'], (0, 0, p, 2 - p, p, 2 - p))    # rows -p .. H + 1 - p
        B, H, W, C = x['x'].shape
        col = torch.stack([X[:, kh:kh + H:2, kw:kw + W:2] for kh in range(3) for kw in range(3)], 3)
        return {'col': (col, None)}
    if e == 'mos_add_rows':
        s = x['x'].double() + x['r'].double()
        return {'x': (s, U32 * s.abs())}
    if e == 'mos_clip_embed':
        ids = x['ids'].long().clamp(0, a['vocab'] - 1)
        v = x['tok'].double()[ids] + x['pos'].double()[torch.arange(a['M'], device=ids.device) % a['T']]
        out = torch.zeros(a['M'], a['ld'], dtype=torch.float64, device=v.device)
        bound = torch.zeros_like(out)
        out[:, :a['C']] = v
        bound[:, :a['C']] = U32 * v.abs()
        return {'x': (out, bound, 'pads_exact')}
    if e in ('mos_quick_gelu', 'mos_quick_gelu_fwd'):
        X = x['x'].double()
        s = torch.sigmoid(1.702 * X)
        y = X * s
        return {'x' if e == 'mos_quick_gelu' else 'y': (y, y.abs() * ((1 - s) * _e_exp(1.702 * X) + 3 * U32))}
    if e == 'mos_quick_gelu_bwd':
        X, dy = x['x'].double(), x['dy'].double()
        s = torch.sigmoid(1.702 * X)
        q = 1.702 * X * s * (1 - s)
        g = s + q
        e_s = s * (1 - s) * _e_exp(1.702 * X) + 3 * U32 * s
        e_g = (1 + 1.702 * X * (1 - 2 * s)).abs() * e_s + 6 * U32 * (s + q.abs())
        return {'dx': (dy * g, dy.abs() * e_g + U32 * (dy * g).abs())}
    if e in ('mos_geglu_fwd', 'mos_geglu_bwd'):
        z = x['z'].double()
        av, gv = z[:, :, 0], z[:, :, 1]
        cdf = 0.5 * (1 + torch.special.erf(gv / math.sqrt(2)))
        gel = gv * cdf
        if e == 'mos_geglu_fwd':
            y = av * gel
            return {'y': (y, av.abs() * ga.GELU_ULP * (gv.abs() + gel.abs()) + U32 * y.abs())}
        dy = x['dy'].double()
        pdf = torch.exp(-0.5 * gv * gv) / math.sqrt(2 * math.pi)
        e_cdf = 8 * U32 + 2 * U32 * gv.abs() * pdf
        da = dy * gv * cdf
        inner = cdf + gv * pdf
        dg = dy * av * inner
        e_da = (dy * gv).abs() * e_cdf + 2 * U32 * da.abs()
        e_dg = (dy * av).abs() * (e_cdf + (gv * pdf).abs() * (_e_exp(0.5 * gv * gv) + 4 * U32) + U32 * inner.abs()) + \
            2 * U32 * dg.abs()
        return {'dz': (torch.stack([da, dg], 2), torch.stack([e_da, e_dg], 2))}
    if e == 'mos_upsample2x_bwd':
        d = x['dy'].double()
        B, H2, W2, C = d.shape
        v = d.view(B, H2 // 2, 2, W2 // 2, 2, C)
        return {'dx': (v.sum((2, 4)), 5 * U32 * v.abs().sum((2, 4)))}
    if e == 'mos_col2im_s2':
        B, H, W, C = a['B'], a['H'], a['W'], a['C']
        dcol = x['dcol'].double()                                         # [B, Ho, Wo, 9, C]
        val = torch.zeros(B, H + 2, W + 2, C, dtype=torch.float64, device=dcol.device)
        mag = torch.zeros_like(val)
        for kh in range(3):
            for kw in range(3):
                val[:, kh:kh + H:2, kw:kw + W:2] += dcol[:, :, :, 3 * kh + kw]
                mag[:, kh:kh + H:2, kw:kw + W:2] += dcol[:, :, :, 3 * kh + kw].abs()
        val, mag = val[:, 1:H + 1, 1:W + 1], mag[:, 1:H + 1, 1:W + 1]
        if a['add']:
            val, mag = val + x['add'].double(), mag + x['add'].double().abs()
        return {'dx': (val, 5 * U32 * mag)}
    if e == 'mos_conv_out_bwd':
        dy, W = x['dy'].double(), x['w'].double().view(a['Cout'], 3, 3, a['C']).permute(0, 3, 1, 2)
        dx = torch.nn.functional.conv_transpose2d(dy, W, padding=1)
        mag = torch.nn.functional.conv_transpose2d(dy.abs(), W.abs(), padding=1)
        return {'dx': (dx.permute(0, 2, 3, 1), (9 * a['Cout'] + 8) * U32 * mag.permute(0, 2, 3, 1))}
    if e == 'mos_add_noise':
        ac = x['ac'].double()[x['t'].long().clamp(0, x['ac'].numel() - 1)][:, None]
        s0, s1 = ac.sqrt(), (1 - ac).sqrt()
        t0, t1 = s0 * x['x0'].double(), s1 * x['noise'].double()
        return {'out': (t0 + t1, 4 * U32 * (t0.abs() + t1.abs()) + U32 * ac / (2 * s1) * x['noise'].double().abs())}
    if e == 'mos_cfg_dpmpp_step':
        n = a['n']
        npred, X, x0p = x['noise_pred'].double(), x['latents'].double(), x['x0_prev'].double()
        if a['cfg']:
            uu, cc = npred[:n], npred[n:]
            d = cc - uu
            eps = uu + a['guidance'] * d
            e_eps = U32 * (d.abs() * abs(a['guidance']) + (a['guidance'] * d).abs() + eps.abs())
        else:
            eps, e_eps = npred, torch.zeros_like(npred)
        se = a['sigma_s'] * eps
        x0 = (X - se) / a['alpha_s']
        e_x0 = (abs(a['sigma_s']) * e_eps + U32 * se.abs() + U32 * (X - se).abs()) / abs(a['alpha_s']) + U32 * x0.abs()
        xn = a['c_x'] * X + a['c_m0'] * x0 + a['c_m1'] * x0p
        e_xn = abs(a['c_m0']) * e_x0 + 5 * U32 * ((a['c_x'] * X).abs() + (a['c_m0'] * x0).abs() + (a['c_m1'] * x0p).abs())
        out = {'latents': (xn, e_xn), 'x0_prev': (x0, e_x0)}
        if a['unet_in']:
            k = 2 if a['cfg'] else 1
            out['unet_in'] = (xn.repeat(k), e_xn.repeat(k))
        if a['t_out']:
            out['t_out'] = (torch.full((a['t_count'],), a['t_next'], dtype=torch.float32, device=X.device), None)
        return out
    if e == 'mos_region_combine':
        B, FH, FW, C = x['glob'].shape
        dev = x['glob'].device
        h = torch.arange(FH, device=dev)[:, None]
        w = torch.arange(FW, device=dev)[None, :]
        cnt = torch.zeros(FH, FW, dtype=torch.float64, device=dev)
        acc = torch.zeros(B, FH, FW, C, dtype=torch.float64, device=dev)
        mag = torch.zeros_like(acc)
        for i, (sh, sw, eh, ew) in enumerate(a['boxes']):
            cov = ((h >= sh) & (h < eh) & (w >= sw) & (w < ew)).double()
            cnt += cov
            r = x.get(f'region{i}')
            if r is not None:
                acc += cov[None, :, :, None] * r.double()
                mag += cov[None, :, :, None] * r.double().abs()
        k = cnt[None, :, :, None]
        ref = torch.where(k == 0, x['glob'].double(), acc / k.clamp(min=1))
        bound = torch.where(k <= 1, torch.zeros_like(ref), (k + 2) * U32 * mag / k.clamp(min=1))
        return {'out': (ref, bound, 'exact_le1')}
    return _reference_training(rec)



def _norm_bwd_ref(rec, dims):
    """float64 GroupNorm(+SiLU) / LayerNorm input gradient (frozen affine) with its fp32 error bound: the forward's
    statistics errors (see _norm_ref), g = dy gamma act'(z) with its own error, the n-term sums sa = mean g and
    sb = mean g xhat, dx = rstd (g - sa - xhat sb) (+ add)"""
    a, x = rec['abi'], rec['in']
    X, dy, gm = x['x'].double(), x['dy'].double(), x['gamma'].double()
    n = 1
    for d in dims:
        n *= X.shape[d]
    gn = X.dim() == 4
    if gn:
        gm = gm.view(GN_GROUPS, -1)
    mean = X.mean(dims, keepdim=True)
    dev = X - mean
    var = (dev * dev).mean(dims, keepdim=True)
    rstd = (var + a['eps']).rsqrt()
    xh = dev * rstd
    cn = (n + 8) * U32
    e_m = cn * X.abs().mean(dims, keepdim=True)
    e_v = cn * var + 2 * e_m * dev.abs().mean(dims, keepdim=True) + e_m * e_m
    r = e_v / (2 * (var + a['eps'])) + 2.0 ** -22 + 2 * U32
    e_h = xh.abs() * r + rstd * e_m + U32 * xh.abs()
    g = dy * gm
    e_g = 2 * U32 * g.abs()
    if gn and a['silu']:
        bt = x['beta'].double().view(GN_GROUPS, -1)
        z = xh * gm + bt
        e_z = gm.abs() * e_h + 2 * U32 * ((xh * gm).abs() + bt.abs())
        sg = torch.sigmoid(z)
        ds = sg * (1 + z * (1 - sg))
        e_ds = 0.5 * e_z + (1 + z * (1 - 2 * sg)).abs() * sg * (1 - sg) * _e_exp(z) + 5 * U32 * ds.abs()
        g, e_g = g * ds, (dy * gm).abs() * e_ds + 3 * U32 * (g * ds).abs()
    sa = g.mean(dims, keepdim=True)
    sb = (g * xh).mean(dims, keepdim=True)
    e_sa = cn * g.abs().mean(dims, keepdim=True) + e_g.mean(dims, keepdim=True)
    e_sb = cn * (g * xh).abs().mean(dims, keepdim=True) + (e_g * xh.abs() + g.abs() * e_h).mean(dims, keepdim=True)
    inner = g - sa - xh * sb
    e_in = e_g + e_sa + xh.abs() * e_sb + e_h * sb.abs() + 3 * U32 * (g.abs() + sa.abs() + (xh * sb).abs())
    dx = rstd * inner
    e = rstd * inner.abs() * r + rstd * e_in + U32 * dx.abs()
    if x.get('add') is not None:
        dx = dx + x['add'].double()
        e = e + U32 * dx.abs()
    return {'dx': (dx, e)}


def _silu_err(v, e_v):
    """silu(v) and its error given the error e_v of v (|silu'| <= 1.1, __expf at -v)"""
    sg = torch.sigmoid(v)
    y = v * sg
    return y, 1.1 * e_v + y.abs() * ((1 - sg) * _e_exp(v) + 2 * U32)


def _reg_gt(rec, B, res):
    """the nearest-resized mask [B, res * res] with the kernel's fp32 index arithmetic (reg_gt)"""
    a, mask = rec['abi'], rec['in']['mask']
    MH, MW = a['MH'], a['MW']
    n = torch.arange(res * res, device=mask.device)
    yy, xx = (n // res).float(), (n % res).float()
    sy = (yy * (torch.tensor(float(MH)) / torch.tensor(float(res))).to(mask.device)).floor().long().clamp(max=MH - 1)
    sx = (xx * (torch.tensor(float(MW)) / torch.tensor(float(res))).to(mask.device)).floor().long().clamp(max=MW - 1)
    return mask[:, sy, sx].double()


def _reference_training(rec):
    e, a, x = rec['op'], rec['abi'], rec['in']
    if e == 'mos_groupnorm_bwd':
        return _norm_bwd_ref(rec, (1, 3))
    if e == 'mos_layernorm_bwd':
        return _norm_bwd_ref(rec, (1,))
    if e == 'mos_timestep_embedding':
        half = a['dim'] // 2
        i = torch.arange(half, dtype=torch.float64, device=x['t'].device)
        arg = -math.log(10000.0) * i / half
        ang = x['t'].double()[:, None] * torch.exp(arg)[None, :]
        e_f = 2 * ULP + 3 * U32 * arg.abs()
        err = ang.abs() * (e_f + U32) + 2 * ULP
        return {'out': (torch.cat([ang.cos(), ang.sin()], 1), torch.cat([err, err], 1))}
    if e == 'mos_gemv_bf16':
        xv, W = x['x'].double(), x['W'].double()
        e_in = torch.zeros_like(xv)
        if a['act_in']:
            xv, e_in = _silu_err(xv, e_in)
        b = x['bias'].double() if x.get('bias') is not None else torch.zeros(a['N'], dtype=torch.float64,
                                                                            device=xv.device)
        v = xv @ W.t() + b
        e_v = (a['K'] + 40) * U32 * (xv.abs() @ W.abs().t() + b.abs()) + e_in @ W.abs().t()
        if a['act_out']:
            v, e_v = _silu_err(v, e_v)
        return {'out': (v, e_v)}
    if e == 'mos_conv_in':
        Ci, Co = a['Cin'], a['Cout']
        Wt = x['w'].double().view(3, 3, Ci, Co).permute(3, 2, 0, 1)
        X = x['x'].double()
        y = torch.nn.functional.conv2d(X, Wt, x['bias'].double(), padding=1)
        mag = torch.nn.functional.conv2d(X.abs(), Wt.abs(), x['bias'].double().abs(), padding=1)
        return {'y': (y.permute(0, 2, 3, 1), ((9 * Ci + 8) * U32 * mag).permute(0, 2, 3, 1))}
    if e == 'mos_softmax_rows':
        S = x['S'].double()
        c = a['scale'] * LOG2E
        X = S * c
        m = X.amax(1, keepdim=True)
        P = torch.softmax(X * LN2, 1)
        dlt = LN2 * (3 * U32 * (X.abs() + m.abs()) + U32 * (X - m).abs()) + 2 * ULP
        D = (P * dlt).sum(1, keepdim=True)
        return {'out': (P, P * (dlt + D + (a['cols'] + 10) * U32))}
    if e == 'mos_conv1x1_nchw':
        X, W, b = x['x'].double(), x['w'].double(), x['bias'].double()
        y = torch.einsum('oc,bcp->bop', W, X) + b[None, :, None]
        mag = torch.einsum('oc,bcp->bop', W.abs(), X.abs()) + b.abs()[None, :, None]
        return {'y': (y, (a['Cin'] + 2) * U32 * mag)}
    if e == 'mos_vae_moments':
        L = a['L']
        h, W, b = x['h'].double(), x['w'].double(), x['bias'].double()
        mo = (h @ W.t() + b).permute(0, 2, 1)                                  # [B, 2L, HW]
        e_mo = ((2 * L + 2) * U32 * (h.abs() @ W.abs().t() + b.abs())).permute(0, 2, 1)
        mu, lv = mo[:, :L], mo[:, L:].clamp(-30, 20)
        out = {'mean': (mu, e_mo[:, :L]), 'logvar': (lv, e_mo[:, L:])}
        if x.get('noise') is not None:
            sd = torch.exp(0.5 * lv)
            z = x['noise'].double()
            t = sd * z
            e_t = t.abs() * (0.5 * e_mo[:, L:] + _e_exp(0.5 * lv) + 2 * U32)
            lat = a['scaling'] * (mu + t)
            out['latents'] = (lat, abs(a['scaling']) * (e_mo[:, :L] + e_t + U32 * (mu + t).abs()) + U32 * lat.abs())
        return out
    if e == 'mos_clip_embed_bwd':
        ids, dx, rows = x['ids'].long(), x['dx'].double(), x['rows'].long()
        sel = (ids[None, :] == rows[:, None]).double()                           # [n_rows, M]
        val, mag = sel @ dx, sel @ dx.abs()
        cnt = sel.sum(1, keepdim=True)
        if a['accumulate']:
            val, mag, cnt = val + x['out'].double(), mag + x['out'].double().abs(), cnt + 1
        return {'out': (val, cnt * U32 * mag)}
    if e == 'mos_masked_mse':
        B, Cc, HW = a['B'], a['Cc'], a['HW']
        d = x['pred'].double() - x['target'].double()
        m = x['mask'].double()[:, None, :]
        num = (d * d * m).sum((1, 2))
        den = x['mask'].double().sum(1)
        e_num = (Cc * HW + 12) * U32 * num.abs() + 4 * U32 * (d * d * m.abs()).sum((1, 2))
        e_den = (HW + 8) * U32 * x['mask'].double().abs().sum(1)
        loss = (num / den).mean()
        r_b = e_num / num.abs().clamp(min=1e-300) + e_den / den.abs() + 2 * U32
        e_loss = ((num / den).abs() * r_b).mean() + (B + 3) * U32 * loss.abs()
        dp = a['grad_scale'] * 2 * d * m / (den[:, None, None] * B)
        e_dp = dp.abs() * (7 * U32 + (e_den / den.abs())[:, None, None])
        return {'ws': (torch.stack([num, den], 1), torch.stack([e_num, e_den], 1)),
                'loss': (loss.view(1), e_loss.view(1)), 'dpred': (dp, e_dp)}
    if e == 'mos_lora_grad':
        M, K, N = a['M'], a['K'], a['N']
        X, dy, D, U = x['x'].double(), x['dy'].double(), x['down'].double(), x['up'].double()
        t, st = X @ D.t(), dy @ U                                                  # [M, 4]
        e_t = (K + 8) * U32 * (X.abs() @ D.abs().t())
        e_s = (N + 8) * U32 * (dy.abs() @ U.abs())
        al = a['alpha']
        dD = al * (st.t() @ X)
        eD = abs(al) * ((M + 16) * U32 * (st.abs().t() @ X.abs()) + e_s.t() @ X.abs()) + U32 * dD.abs()
        dU = al * (dy.t() @ t)
        eU = abs(al) * ((M + 16) * U32 * (dy.abs().t() @ t.abs()) + dy.abs().t() @ e_t) + U32 * dU.abs()
        if a['accumulate']:
            dD, eD = dD + x['d_down'].double(), eD + U32 * (dD + x['d_down'].double()).abs()
            dU, eU = dU + x['d_up'].double(), eU + U32 * (dU + x['d_up'].double()).abs()
        return {'d_down': (dD, eD), 'd_up': (dU, eU)}
    if e == 'mos_attn_reg_group':
        B, Hh, res, L = a['B'], a['heads'], a['res'], a['L']
        P = torch.stack([x[f'pcols{l}'].double() for l in range(L)], 0)          # [L, B, H, N, 2]
        cm = P.mean((0, 2))
        e_cm = (L * Hh + 2) * U32 * P.abs().mean((0, 2))
        out = {'cm': (cm, e_cm)}
        got = rec.get('_got', {}).get('cm')
        cmk = got.double() if got is not None else cm                              # the stats read the launch's cm
        gt = _reg_gt(rec, B, res).reshape(-1)
        x0, x1 = cmk[..., 0].reshape(-1), cmk[..., 1].reshape(-1)
        M0, M1 = x0.max(), x1.max()
        zero = (gt == 0).double()
        Z = zero.sum()
        total = x0.numel()
        y0, y1 = x0 / M0, x1 / M1
        if a['full']:
            t1, g1 = (y1 - gt) ** 2 / total, 2 * (y1 - gt) / total
        else:
            t1, g1 = zero * y1 / Z, zero / Z
        ls = (t1 + zero * y0 / Z).sum()
        S0, S1 = ((zero / Z) * x0).sum(), (g1 * x1).sum()
        T0, T1 = (x0 == M0).double().sum(), (x1 == M1).double().sum()
        n = total + 16
        mag_l = (t1.abs() + zero * y0.abs() / Z).sum()
        st = torch.stack([M0, M1, T0, T1, Z, a['weight'] * ls, S0, S1])
        eb = torch.stack([M0 * 0, M1 * 0, T0 * 0, T1 * 0, Z * 0,
                          abs(a['weight']) * (n * U32 * mag_l + 6 * U32 * mag_l) + U32 * abs(a['weight'] * ls),
                          (n + 4) * U32 * ((zero / Z) * x0.abs()).sum(), (n + 6) * U32 * (g1.abs() * x1.abs()).sum()])
        out['stats'] = (st, eb, 'exact0')
        return out
    if e == 'mos_attn_reg_grad':
        B, res, g = a['B'], a['res'], a['group']
        sa = x['stats_all'].double()
        M0, M1, T0, T1, Z, S0, S1 = (sa[g, i] for i in (0, 1, 2, 3, 4, 6, 7))
        gt = _reg_gt(rec, B, res)
        zero = (gt == 0).double()
        x0, x1 = x['cm'][..., 0].double(), x['cm'][..., 1].double()
        total = x0.numel()
        g1 = 2 * (x1 / M1 - gt) / total if a['full'] else zero / Z
        g0 = zero / Z
        valid = bool((sa[:, 4] > 0).all())
        k = a['grad_scale'] * a['weight'] / (a['heads'] * a['L']) if valid else 0.0
        p0, q0 = g0 / M0, torch.where(x0 == M0, S0 / (M0 * M0 * T0), torch.zeros_like(x0))
        p1, q1 = g1 / M1, torch.where(x1 == M1, S1 / (M1 * M1 * T1), torch.zeros_like(x1))
        d = torch.stack([k * (p0 - q0), k * (p1 - q1)], -1)
        # full identity: x1 / M1 is rounded before the target is subtracted, and x1 / M1 - gt cancels where the map is
        # close to the target, so that rounding is bounded by |x1 / M1|, not by |g1|
        e_g1 = 2 * U32 * 2 * (x1 / M1).abs() / total if a['full'] else torch.zeros_like(x1)
        eb = torch.stack([abs(k) * 8 * U32 * (p0.abs() + q0.abs()),
                          abs(k) * (8 * U32 * (p1.abs() + q1.abs()) + e_g1 / M1)], -1)
        return {'gcols': (d, eb + 4 * U32 * d.abs())}
    if e == 'mos_attn_reg_total':
        ls = x['stats_all'][:, 5].double()
        s1 = ls.sum()
        s0 = x['mse'].double()[0] + (0.0 if torch.isnan(s1) else s1)
        e1 = (ls.numel() + 2) * U32 * ls.abs().sum()
        return {'out': (torch.stack([s0, s1]), torch.stack([e1 + U32 * (x['mse'].double()[0].abs() + s0.abs()), e1]))}
    if e == 'mos_flat_adamw_step':
        n = a['n']
        dev = x['p'].device
        i = torch.arange(n, device=dev)
        ge, gl = a['group_end'], [float(torch.tensor(v, dtype=torch.float32)) for v in a['group_lr']]
        lr = torch.where(i < ge[0], gl[0], torch.where(i < ge[1], gl[1], gl[2])).double()
        b1, b2, eps, wd, step = a['beta1'], a['beta2'], a['eps'], a['wd'], a['step']
        bc1, bc2s = 1 - b1 ** step, math.sqrt(1 - b2 ** step)
        gi = x['g'].double() * a['grad_scale']
        p0, m0, v0 = x['p'].double(), x['m'].double(), x['v'].double()
        pw = p0 * (1 - lr * wd)
        mi = b1 * m0 + (1 - b1) * gi
        vi = b2 * v0 + (1 - b2) * gi * gi
        e_pw = 3 * U32 * p0.abs()
        e_m = 4 * U32 * ((b1 * m0).abs() + ((1 - b1) * gi).abs())
        e_v = 5 * U32 * ((b2 * v0).abs() + (1 - b2) * gi * gi)
        sq = vi.sqrt()
        e_sq = torch.minimum(e_v / (2 * sq).clamp(min=1e-300), e_v.sqrt()) + U32 * sq
        den = sq / bc2s + eps
        e_den = e_sq / bc2s + 3 * U32 * sq / bc2s + U32 * den
        upd = (lr / bc1) * (mi / den)
        e_upd = upd.abs() * (4 * U32 + e_den / den) + (lr / bc1) * e_m / den
        pn = pw - upd
        out = {'p': (pn, e_pw + e_upd + U32 * pn.abs()), 'm': (mi, e_m), 'v': (vi, e_v)}
        if a['norm_out'] and a['emb_rows'] > 0:
            R, Dm = a['emb_rows'], a['emb_dim']
            got = rec.get('_got', {}).get('p')
            pr = (got.double() if got is not None else pn)[:R * Dm].view(R, Dm)   # the norms read the updated params
            nr = pr.norm(dim=1)
            val = nr.mean()
            err = ((Dm + 8) * U32 * 0.5 + 2 * U32) * nr.sum() / R + (R + 2) * U32 * val
            out['norm_out'] = (val.view(1), err.view(1))
        return out
    if e == 'mos_lora_pack':
        out = {}
        for t in rec['targets']:
            src, i = t['src']
            v = x[f'{src}{i}'].double()
            if t['name'].startswith('fdown'):
                out[t['name']] = (v, torch.zeros_like(v))
            elif t['name'].startswith('fup'):
                out[t['name']] = (a['alpha'] * v, U32 * (a['alpha'] * v).abs())
            elif t['name'].startswith('bdown'):
                out[t['name']] = (v.t(), torch.zeros_like(v.t()))
            else:
                out[t['name']] = (a['alpha'] * v.t(), U32 * (a['alpha'] * v.t()).abs())
        return out
    raise AssertionError(f'no reference for {e}')


# --------------------------------------------------------------------------------------------------- checks
def window(rec, t, which):
    return rec['mem'][t['mem']][which].as_strided(t['size'], t['stride'], t['off'])


def check_launch(rec):
    """Checks (p) and (a)-(c) of one launch.  -> {'ratio': worst error / bound, 'tile_rel': worst unit rel-L2,
    'tile': worst fraction of the unit limit, 'errors': [messages]}"""
    errors = list(rec.get('pre', ()))
    ratio, worst_rel, worst_frac = 0.0, 0.0, 0.0
    rec['_got'] = {t['name']: window(rec, t, 'after') for t in rec['targets']}   # second stages read the first's output
    refs = reference(rec)
    masks = {k: torch.zeros(st['after'].numel(), dtype=torch.bool, device=st['after'].device)
             for k, st in rec['mem'].items()}
    for t in rec['targets']:
        name = t['name']
        masks[t['mem']].as_strided(t['size'], t['stride'], t['off']).fill_(True)
        if t['scratch']:
            continue
        got = window(rec, t, 'after')
        ref, bound = refs[name][:2]
        dt = got.dtype
        if bound is None:                                                   # bit-exact
            want = ref.to(dt)
            if not torch.equal(got.reshape(-1).view(_BITS[got.element_size()]),
                               want.reshape(-1).view(_BITS[got.element_size()])):
                bad = (got.reshape(-1).view(_BITS[got.element_size()]) !=
                       want.reshape(-1).view(_BITS[got.element_size()])).nonzero()
                errors.append(f'(a) {name}: {bad.numel()} elements differ from the exact result, first at flat '
                              f'{int(bad[0])}')
            continue
        gd = got.double()
        err = (gd - ref).abs()
        full = U16[dt] * ref.abs() + (1 + U16[dt]) * bound + TINY[dt]
        mode = refs[name][2] if len(refs[name]) > 2 else None
        if mode == 'pads_exact':                                            # clip_embed: pad columns exactly zero
            full[:, rec['abi']['C']:] = 0
        elif mode in ('exact_le1', 'exact0'):          # region_combine: one region or none; attn_reg stats: max, counts
            full = torch.where(bound == 0, torch.zeros_like(full), full)
        exact = full == 0
        bad = ~(err <= full) & ~(ref.isnan() & gd.isnan())                 # NaN counts as bad unless the reference is NaN
        if exact.any():
            bits = _BITS[got.element_size()]
            differ = got.view(bits) != ref.to(dt).view(bits)
            bad = bad | (exact & differ)
        if bad.any():
            i = tuple(int(v) for v in bad.nonzero()[0])
            errors.append(f'(a) {name}: {int(bad.sum())} elements out of bound, first at {i}: got {gd[i].item():.6g} '
                          f'want {ref[i].item():.6g} bound {full[i].item():.3g}')
        r = torch.where(exact, torch.zeros_like(err), err / full)
        ratio = max(ratio, r.nan_to_num(nan=math.inf).max().item())
        tol = t.get('tol') or UNIT_TOL.get(dt)
        if tol and (t['unit'] is not None or t.get('groups')):
            if t.get('groups'):                                             # AdamW: one unit per parameter group
                e2 = torch.stack([(err[g0:g1] ** 2).sum() for g0, g1 in t['groups'] if g1 > g0])
                r2 = torch.stack([(ref[g0:g1] ** 2).sum() for g0, g1 in t['groups'] if g1 > g0])
            else:
                e2 = (err * err).sum(t['unit'])
                r2 = (ref * ref).sum(t['unit'])
            rel = torch.where(e2 == 0, torch.zeros_like(e2), e2.sqrt() / r2.sqrt()).nan_to_num(nan=math.inf)
            worst_rel = max(worst_rel, rel.max().item())
            worst_frac = max(worst_frac, rel.max().item() / tol)
            if not rel.max().item() <= tol:
                u = tuple(int(v) for v in (rel == rel.max()).nonzero()[0])
                errors.append(f'(b) {name}: unit {u} rel-L2 {rel.max().item():.3e} > {tol:.1e}')
    for k, st in rec['mem'].items():
        es = st['after'].element_size()
        stray = (st['after'].view(_BITS[es]) != st['before'].view(_BITS[es])) & ~masks[k]
        if stray.any():
            errors.append(f'(c) storage {k[1]}: {int(stray.sum())} elements written outside the window, first at flat '
                          f'index {int(stray.nonzero()[0])}')
    return {'ratio': ratio, 'tile_rel': worst_rel, 'tile': worst_frac, 'errors': errors}


def simulate(rec):
    """Write the rounded reference into the 'after' storages: what a correct kernel leaves (CPU tests).  Scratch
    windows are filled with ones (a correct kernel may leave anything there)."""
    for st in rec['mem'].values():
        st['after'] = st['before'].clone()
    refs = reference(rec)
    for t in rec['targets']:
        w = window(rec, t, 'after')
        w.copy_(torch.ones_like(w) if t['scratch'] else refs[t['name']][0].to(w.dtype))
    return rec


# --------------------------------------------------------------------------------------------------- recorder
_OPS = ('groupnorm', 'layernorm', 'conv_out', 'upsample2x', 'im2col_s2', 'add_rows', 'clip_embed', 'quick_gelu',
        'quick_gelu_fwd', 'quick_gelu_bwd', 'cfg_dpmpp_step', 'region_combine', 'geglu_fwd', 'geglu_bwd',
        'upsample2x_bwd', 'col2im_s2', 'conv_out_bwd', 'add_noise', 'groupnorm_bwd', 'layernorm_bwd', 'timestep_embedding',
        'gemv', 'conv_in', 'softmax_rows', 'conv1x1_nchw', 'vae_moments', 'clip_embed_bwd', 'masked_mse', 'lora_grad',
        'attn_reg_group', 'attn_reg_grad', 'attn_reg_total', 'flat_adamw_step', 'lora_pack')


class Recorder(ga.LaunchRecorder):
    """audits every launch of ENTRY_POINTS made inside it; the outputs of ops.attention are registered as storages the
    region table of region_combine may point into"""
    OPS = _OPS
    ENTRY_POINTS = ENTRY_POINTS
    REGISTER_OPS = ('attention',)

    def record(self, entry, args, S):
        return record(entry, abi_of(entry, args[:len(_ARGS[entry])]), S, self._ctx[2])

    def key(self, rec):
        return norm_path(rec)

    def check(self, rec):
        return check_launch(rec)
