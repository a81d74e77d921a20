"""The norm / elementwise launch audit (tests/norm_audit.py) on the CPU: its float64 references against independent
torch statements of the same operations, and its checks against a stand-in library.

Launches are made by the real `ops.*` wrappers with CPU tensors through the audit's own Recorder, so the records come
from the ABI arguments exactly as on the GPU.  The stand-in writes the rounded reference of each entry point into the
windows it reads from those arguments; every mutation case breaks it (or its inputs) the way a faulty kernel or engine
would, and the check it targets must flag it while the unbroken stand-in passes every check.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import norm_audit as na

BF, F16 = torch.bfloat16, torch.float16


def rnd(shape, seed, scale=1.0, dtype=torch.float32, shift=0.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale + shift).to(dtype)


class StandIn:
    """writes the rounded float64 reference of every audited entry point; `mut` names one defect to inject"""

    def __init__(self, mut=None):
        self.mut, self.calls, self.recorder = mut, 0, None

    def __getattr__(self, name):
        if name not in na.ENTRY_POINTS:
            raise AttributeError(name)
        return lambda *args: self._launch(name, args)

    def _launch(self, entry, args):
        S = na._Storages(self.recorder._ctx[0], self.recorder.registered)
        rec = na.record(entry, na.abi_of(entry, args[:len(na._ARGS[entry])]), S, self.recorder._ctx[2])
        a, m = rec['abi'], self.mut
        if m == 'im2col_pad' and entry == 'mos_im2col_s2':
            a = dict(a, pad=1 - a['pad'])
        if m == 'region_edge' and entry == 'mos_region_combine':
            a = dict(a, boxes=[(sh, sw, eh + 1, ew) for sh, sw, eh, ew in a['boxes']])
        if m == 'noise_t+1' and entry == 'mos_add_noise':
            rec['in']['t'] = rec['in']['t'] + 1
        if m == 'adamw_bc_late' and entry == 'mos_flat_adamw_step':
            a = dict(a, step=a['step'] - 1)
        snap = dict(rec)
        snap['abi'], snap['in'] = a, {k: v.clone() for k, v in rec['in'].items()}
        refs = na.reference(snap)
        for t in rec['targets']:
            w = S.flat(*t['mem']).as_strided(t['size'], t['stride'], t['off'])
            if t['scratch']:
                w.fill_(1)
                continue
            r = refs[t['name']][0]
            if m == 'gn_neighbour' and entry == 'mos_groupnorm_fwd':
                x = rec['in']['x'].double()
                g = x[:, :, 5:6]                                            # group 4 normalised with group 5's statistics
                mean, var = g.mean((1, 3), keepdim=True), g.var((1, 3), unbiased=False, keepdim=True)
                r = r.clone()
                gm, bt = rec['in']['gamma'].double().view(32, -1), rec['in']['beta'].double().view(32, -1)
                r[:, :, 4] = (x[:, :, 4] - mean[:, :, 0]) * (var[:, :, 0] + a['eps']).rsqrt() * gm[4] + bt[4]
            if m == 'ln_skip_tail' and entry == 'mos_layernorm_fwd':
                r = r.clone()
                r[-1] = w[-1].double()
            if m == 'clip_pad' and entry == 'mos_clip_embed':
                r = r.clone()
                r[3, a['C'] + 2] = 1.0
            if m == 'geglu_tanh' and entry == 'mos_geglu_bwd':
                z = rec['in']['z'].double()
                av, gv = z[:, :, 0], z[:, :, 1].clone().requires_grad_()
                gel = F.gelu(gv, approximate='tanh')
                (dg,) = torch.autograd.grad((gel * av * rec['in']['dy'].double()).sum(), gv)
                r = torch.stack([rec['in']['dy'].double() * gel.detach(), dg], 2)
            if m == 'gn_bwd_drop_add' and entry == 'mos_groupnorm_bwd':
                nch = na.gn_bwd_chunks(a)
                r0 = (nch - 1) * -(-a['HW'] // nch)                         # the last chunk's rows lose `add`
                r = r.clone()
                r[:, r0:] -= rec['in']['add'].double()[:, r0:]
            if m == 'mse_count' and t['name'] == 'dpred':
                den = rec['in']['mask'].double().sum(1)
                r = r * (den / (den + 1))[:, None, None]
            w.copy_(r.to(w.dtype))
            if m == 'nondet' and self.calls % 2:                     # the relaunch differs in one last bit
                S.flat(t['mem'][0], torch.int16)[t['off']] ^= 1
        if m == 'write_past' and entry == 'mos_upsample2x':
            t = rec['targets'][0]
            S.flat(*t['mem'])[t['off'] + math.prod(t['size'])] = 1.0
        if m == 'lora_ws_past' and entry == 'mos_lora_grad':
            t = next(t for t in rec['targets'] if t['name'] == 'ws')
            S.flat(*t['mem'])[t['off'] + t['size'][0]] = 1.0
        if m == 'qg_bwd_into_x' and entry == 'mos_quick_gelu_bwd':
            rec['in']['x'][0, 0] = 7.0
        self.calls += 1
        return 0


@pytest.fixture
def audit(monkeypatch):
    """audit(mut=None) -> a Recorder over the stand-in library (CPU tensors)"""
    from mos_b200 import _lib, ops
    monkeypatch.setattr(ops, 'current_stream', lambda: None)
    monkeypatch.setattr(na, 'SMS', 132)

    def make(mut=None):
        lib = StandIn(mut)
        monkeypatch.setattr(_lib, 'lib', lambda: lib)
        r = na.Recorder()
        lib.recorder = r
        return r
    return make


def ok(r):
    assert not r.stats.failures, '\n'.join(r.stats.failures)
    return r


def flagged(r, letter):
    assert any(f'({letter})' in e for e in r.stats.failures), r.stats.failures


def keys(r):
    return set(r.stats.rows)


# ---------------------------------------------------------------------------------------------------- launches
def run_gn(audit, mut=None, B=2, HW=4096, C=320, ld=None, dtype=F16, silu=True, partial_floats=None):
    from mos_b200 import ops
    ld = ld or C
    x = rnd((B, HW, ld), 1, 2.0, dtype, shift=0.5)
    y = torch.full((B, HW, ld), 3.0, dtype=dtype)
    gamma, beta = rnd((C,), 2, 0.3) + 1, rnd((C,), 3, 0.2)
    partial = torch.zeros(partial_floats or B * 64 * 64)
    with audit(mut) as r:
        ops.groupnorm(x, gamma, beta, y, partial, B=B, HW=HW, C=C, eps=1e-5, silu=silu, ldx=ld, ldy=ld)
    return r, dict(x=x, y=y, gamma=gamma, beta=beta, partial=partial)


def run_ln(audit, mut=None, M=157, C=768, ld=800):
    from mos_b200 import ops
    x = rnd((M, ld), 4, 1.5, BF, shift=0.3)
    y = torch.full((M, ld), 2.0, dtype=BF)
    gamma, beta = rnd((C,), 5, 0.3) + 1, rnd((C,), 6, 0.2)
    with audit(mut) as r:
        ops.layernorm(x, gamma, beta, y, M=M, C=C, ldx=ld, ldy=ld)
    return r, dict(x=x, y=y, gamma=gamma, beta=beta)


def run_resample(audit, mut=None, B=2, H=6, W=10, C=16, pad=1):
    from mos_b200 import ops
    x = rnd((B * H * W, C + 8), 7, dtype=BF)                               # pitched rows: ldx = C + 8
    y = torch.zeros(B * 4 * H * W + 1, C, dtype=BF)                        # one spare row past the window
    col = torch.zeros(B * (H // 2) * (W // 2), 9 * C, dtype=BF)
    with audit(mut) as r:
        ops.upsample2x(x, y, B=B, H=H, W=W, C=C, ldx=C + 8)
        ops.im2col_s2(x, col, B=B, H=H, W=W, C=C, ldx=C + 8, pad=pad)
    return r, dict(x=x[:, :C].reshape(B, H, W, C), y=y[:-1].view(B, 2 * H, 2 * W, C), col=col)


def run_region(audit, mut=None, n=3, B=2, FH=12, FW=24, C=40, dtype=F16):
    from mos_b200 import ops
    o = rnd((B, FH * FW, C), 8, dtype=dtype)
    regs = [rnd((B, FH * FW, C), 9 + i, dtype=dtype) for i in range(n)]
    boxes = [(i, 2 * i, FH - (i % 2), 2 * i + 9) for i in range(n)]       # overlapping boxes, one touching the edge
    o0 = o.clone()
    with audit(mut) as r:
        r.register(*regs)
        ptrs = torch.tensor([t.data_ptr() for t in regs], dtype=torch.int64)
        ops.region_combine(o, ptrs, boxes, o, B=B, FH=FH, FW=FW, C=C, ld=C)
    return r, dict(o0=o0, o=o, regs=regs, boxes=boxes)


def run_pointwise(audit, mut=None, M=157, C=768):
    """QuickGELU (in place, forward, backward), GEGLU forward / backward, add_rows at pitched rows"""
    from mos_b200 import ops
    x = rnd((M, C + 32), 11, 3.0, BF)
    y, dx = torch.zeros(M, C + 32, dtype=BF), torch.zeros(M, C, dtype=BF)
    dy = rnd((M, C), 12, dtype=BF)
    xi = x.clone()
    z = rnd((M, 2 * 320), 13, 2.0, BF)
    gy, dz = torch.zeros(M, 320, dtype=BF), torch.zeros(M, 2 * 320, dtype=BF)
    gdy = rnd((M, 320), 14, dtype=BF)
    a, rr = rnd((M, 336), 15, dtype=BF), rnd((M, 320), 16, dtype=BF)
    with audit(mut) as r:
        ops.quick_gelu(xi, M=M, C=C)
        ops.quick_gelu_fwd(x, y, M=M, C=C)
        ops.quick_gelu_bwd(x, dy, dx, M=M, C=C)
        ops.geglu_fwd(z, gy, M=M, H=320)
        ops.geglu_bwd(z, gdy, dz, M=M, H=320)
        ops.add_rows(a, rr, M=M, C=320, ldx=336, ldr=320)
    return r, dict(x=x, xi=xi, y=y, dx=dx, dy=dy, z=z, gy=gy, dz=dz, gdy=gdy)


def run_training_glue(audit, mut=None, t=(77, 640)):
    from mos_b200 import ops
    B, C, H, W = 2, 320, 8, 8
    x0, noise = rnd((B, 4, H, W), 17), rnd((B, 4, H, W), 18)
    ac = torch.cumprod(1 - torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2, 0).float()
    out = torch.zeros(B, 4, H, W)
    dy = rnd((B, 4, H, W), 19)
    w = rnd((4, 9 * C), 20, 0.05)
    dxo = torch.zeros(B * H * W, C, dtype=BF)
    dcol = rnd((B * (H // 2) * (W // 2), 9 * C), 21, dtype=BF)
    dxc = torch.zeros(B * H * W, C, dtype=BF)
    up = rnd((B * 2 * H * 2 * W, C), 22, dtype=BF)
    dxu = torch.zeros(B * H * W, C, dtype=BF)
    with audit(mut) as r:
        ops.add_noise(x0, noise, torch.tensor(t, dtype=torch.int32), ac, out)
        ops.conv_out_bwd(dy, w, dxo, B=B, H=H, W=W, C=C)
        ops.col2im_s2(dcol, dxc, B=B, H=H, W=W, C=C, add=dxo)
        ops.upsample2x_bwd(up, dxu, B=B, H=H, W=W, C=C)
    return r, dict(x0=x0, noise=noise, ac=ac, out=out, dy=dy, w=w, dxo=dxo, dcol=dcol, dxc=dxc, up=up, dxu=dxu)


def run_conv_out(audit, mut=None, x=None):
    from mos_b200 import ops
    B, H, W, C = 2, 8, 8, 320
    x = rnd((B * H * W, C), 23, dtype=F16) if x is None else x
    w, b = rnd((4, 9 * C), 24, 0.05), rnd((4,), 25)
    y = torch.zeros(B, 4, H, W)
    with audit(mut) as r:
        ops.conv_out(x, w, b, y, B=B, H=H, W=W, C=C)
    return r, dict(x=x, w=w, b=b, y=y)


def run_clip_embed(audit, mut=None):
    from mos_b200 import ops
    T, C, ld = 77, 768, 800
    ids = torch.randint(0, 100, (2 * T,), generator=torch.Generator().manual_seed(26), dtype=torch.int32)
    tok, pos = rnd((100, C), 27, 0.02), rnd((T, C), 28, 0.01)
    x = torch.full((2 * T, ld), 5.0, dtype=BF)
    with audit(mut) as r:
        ops.clip_embed(ids, tok, pos, x, T=T, C=C)
    return r, dict(ids=ids, tok=tok, pos=pos, x=x)


def run_cfg_step(audit, mut=None, cfg=True):
    from mos_b200 import ops
    n = 4 * 8 * 8
    npred = rnd(((2 if cfg else 1) * n,), 29)
    lat, x0p = rnd((n,), 30), rnd((n,), 31)
    unet_in, t_out = torch.zeros((2 if cfg else 1) * n), torch.zeros(2)
    lat0, x0p0 = lat.clone(), x0p.clone()
    coef = (0.93, 0.41, -0.12, 0.87, 0.49)
    with audit(mut) as r:
        ops.cfg_dpmpp_step(npred, lat, x0p, unet_in, cfg=cfg, guidance=7.5, coef=coef, t_out=t_out, t_next=501.0)
    return r, dict(npred=npred, lat0=lat0, x0p0=x0p0, lat=lat, x0p=x0p, unet_in=unet_in, t_out=t_out, coef=coef)


# ------------------------------------------------------------------------------------- reference vs restatements
@pytest.mark.parametrize('B,HW,C,dtype', [(2, 4096, 320, F16), (1, 4096, 128, BF), (2, 1152, 1280, F16)])
def test_groupnorm_reference_vs_torch(audit, B, HW, C, dtype):
    r, o = run_gn(audit, B=B, HW=HW, C=C, dtype=dtype)
    ok(r)
    x = o['x'][..., :C].double().transpose(1, 2)
    want = F.silu(F.group_norm(x, 32, o['gamma'].double(), o['beta'].double(), 1e-5)).transpose(1, 2)
    assert torch.allclose(o['y'][..., :C].double(), want, rtol=2e-2, atol=2e-2)
    ref = na.reference(r.last)['y'][0].reshape(B, HW, C)
    assert torch.allclose(ref, want, rtol=1e-10, atol=1e-10)


def test_groupnorm_fallback_workspace_prefix(audit):
    """VAE-sized map: the fallback writes only the B * nchunks * 64 prefix of the partial workspace"""
    r, o = run_gn(audit, B=1, HW=262144, C=128, dtype=F16, partial_floats=1 << 16)
    ok(r)
    (key,) = keys(r)
    assert key == 'gn|fp16|fallback|silu'
    _, _, _, nchunks = na.gn_rule(r.last['abi'])
    assert (o['partial'][:nchunks * 64] == 1).all() and (o['partial'][nchunks * 64:] == 0).all()


@pytest.mark.parametrize('M', [157, 8, 1])
def test_layernorm_reference_vs_autograd_free_torch(audit, M):
    r, o = run_ln(audit, M=M)
    ok(r)
    want = F.layer_norm(o['x'][:, :768].double(), (768,), o['gamma'].double(), o['beta'].double(), 1e-5)
    assert torch.allclose(na.reference(r.last)['y'][0], want, rtol=1e-10, atol=1e-10)
    assert keys(r) == ({'ln|bf16|C=768|mtail'} if M % 8 else {'ln|bf16|C=768'})
    assert torch.equal(o['y'][:, 768:], torch.full((M, 32), 2.0, dtype=BF))


@pytest.mark.parametrize('pad', [0, 1])
def test_resampling_references_vs_torch(audit, pad):
    r, o = run_resample(audit, pad=pad)
    ok(r)
    x = o['x'].permute(0, 3, 1, 2).double()
    assert torch.equal(o['y'].permute(0, 3, 1, 2).double(), F.interpolate(x, scale_factor=2, mode='nearest'))
    xp = F.pad(x, (pad, 2 - pad, pad, 2 - pad))
    B, C = x.shape[0], x.shape[1]
    cols = F.unfold(xp, 3, stride=2)                                       # [B, C * 9, L] channel-major
    want = cols.view(B, C, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * C)
    assert torch.equal(o['col'].double(), want)
    assert keys(r) == {'upsample2x', f'im2col|pad={pad}'}


def test_training_glue_references_vs_torch(audit):
    r, o = run_training_glue(audit)
    ok(r)
    B, C, H, W = 2, 320, 8, 8
    ac = o['ac'].double()[torch.tensor([77, 640])].view(2, 1, 1, 1)
    assert torch.allclose(o['out'].double(), ac.sqrt() * o['x0'].double() + (1 - ac).sqrt() * o['noise'].double(),
                          rtol=1e-6, atol=1e-6)
    Wt = o['w'].double().view(4, 3, 3, C).permute(0, 3, 1, 2)
    xin = torch.zeros(B, C, H, W, dtype=torch.float64, requires_grad=True)
    (gx,) = torch.autograd.grad((F.conv2d(xin, Wt, padding=1) * o['dy'].double()).sum(), xin)
    assert torch.allclose(o['dxo'].double().view(B, H, W, C).permute(0, 3, 1, 2), gx, rtol=1e-2, atol=1e-2)
    dcol = o['dcol'].double().view(B, (H // 2) * (W // 2), 9, C).permute(0, 3, 2, 1).reshape(B, 9 * C, -1)
    fold = F.fold(dcol, (H + 2, W + 2), 3, stride=2)[:, :, 1:H + 1, 1:W + 1]
    want = fold + o['dxo'].double().view(B, H, W, C).permute(0, 3, 1, 2)
    assert torch.allclose(o['dxc'].double().view(B, H, W, C).permute(0, 3, 1, 2), want, rtol=1e-2, atol=1e-2)
    up = o['up'].double().view(B, 2 * H, 2 * W, C).permute(0, 3, 1, 2)
    assert torch.allclose(o['dxu'].double().view(B, H, W, C).permute(0, 3, 1, 2), F.avg_pool2d(up, 2) * 4,
                          rtol=1e-2, atol=1e-2)


def test_conv_out_reference_vs_conv2d(audit):
    r, o = run_conv_out(audit)
    ok(r)
    x = o['x'].double().view(2, 8, 8, 320).permute(0, 3, 1, 2)
    want = F.conv2d(x, o['w'].double().view(4, 3, 3, 320).permute(0, 3, 1, 2), o['b'].double(), padding=1)
    assert torch.allclose(na.reference(r.last)['y'][0], want, rtol=1e-10, atol=1e-10)


def test_pointwise_references_vs_torch(audit):
    r, o = run_pointwise(audit)
    ok(r)
    x = o['x'][:, :768].double()
    qg = x * torch.sigmoid(1.702 * x)
    assert torch.allclose(o['xi'][:, :768].double(), qg, rtol=1e-2, atol=1e-2)
    assert torch.equal(o['xi'][:, 768:], o['x'][:, 768:])
    xg = x.clone().requires_grad_()
    (g,) = torch.autograd.grad((xg * torch.sigmoid(1.702 * xg) * o['dy'].double()).sum(), xg)
    assert torch.allclose(o['dx'].double(), g, rtol=1e-2, atol=1e-2)
    z = o['z'].double().view(-1, 4, 2, 80)
    a, gt = z[:, :, 0].reshape(-1, 320), z[:, :, 1].reshape(-1, 320).requires_grad_()
    ar = a.clone().requires_grad_()
    y = ar * F.gelu(gt)
    assert torch.allclose(o['gy'].double(), y.detach(), rtol=1e-2, atol=1e-2)
    da, dg = torch.autograd.grad((y * o['gdy'].double()).sum(), (ar, gt))
    dz = o['dz'].double().view(-1, 4, 2, 80)
    assert torch.allclose(dz[:, :, 0].reshape(-1, 320), da, rtol=1e-2, atol=1e-2)
    assert torch.allclose(dz[:, :, 1].reshape(-1, 320), dg, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize('n', [1, 3, 8])
def test_region_combine_reference(audit, n):
    r, o = run_region(audit, n=n)
    ok(r)
    assert keys(r) == {f'region|fp16|n={n}|inplace'}
    B, FH, FW, C = 2, 12, 24, 40
    want = o['o0'].double().view(B, FH, FW, C).clone()
    acc, cnt = torch.zeros_like(want), torch.zeros(FH, FW, dtype=torch.float64)
    for reg, (sh, sw, eh, ew) in zip(o['regs'], o['boxes']):
        acc[:, sh:eh, sw:ew] += reg.double().view(B, FH, FW, C)[:, sh:eh, sw:ew]
        cnt[sh:eh, sw:ew] += 1
    want = torch.where(cnt[None, :, :, None] > 0, acc / cnt.clamp(min=1)[None, :, :, None], want)
    assert torch.allclose(o['o'].double().view(B, FH, FW, C), want, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize('cfg', [True, False])
def test_cfg_step_reference_vs_scheduler_update(audit, cfg):
    """the DPM-Solver++(2M) update and the CFG combine of mos_b200/scheduler.py, restated in float64"""
    r, o = run_cfg_step(audit, cfg=cfg)
    ok(r)
    n = o['lat0'].numel()
    c_x, c_m0, c_m1, a_s, s_s = o['coef']
    e = o['npred'].double()
    eps = e[:n] + 7.5 * (e[n:] - e[:n]) if cfg else e
    x0 = (o['lat0'].double() - s_s * eps) / a_s
    xn = c_x * o['lat0'].double() + c_m0 * x0 + c_m1 * o['x0p0'].double()
    assert torch.allclose(o['lat'].double(), xn, rtol=1e-5, atol=1e-5)
    assert torch.allclose(o['x0p'].double(), x0, rtol=1e-5, atol=1e-5)
    assert torch.equal(o['t_out'], torch.full((2,), 501.0))
    assert keys(r) == {'cfg_step|' + ('cfg' if cfg else 'nocfg') + '|t_out|unet_in'}


def test_clip_embed_reference(audit):
    r, o = run_clip_embed(audit)
    ok(r)
    want = o['tok'].double()[o['ids'].long()] + o['pos'].double().repeat(2, 1)
    assert torch.allclose(o['x'][:, :768].double(), want, rtol=1e-2, atol=1e-3)
    assert not o['x'][:, 768:].any()


def test_groupnorm_path_keys(audit):
    """132 SMs: clusters are widened until 2 * 132 CTAs; a 48 KiB slab per CTA at most; vec 4 needs 4 | C / 32"""
    assert keys(ok(run_gn(audit)[0])) == {'gn|fp16|cluster|k=8|v2|silu'}
    assert keys(ok(run_gn(audit, B=2, HW=64, C=640, dtype=BF, silu=False)[0])) == {'gn|bf16|cluster|k=4|v4'}
    assert keys(ok(run_gn(audit, B=16, HW=4096, C=1280, dtype=BF)[0])) == {'gn|bf16|cluster|k=8|v4|silu'}


# -------------------------------------------------------------------------------------------------- mutation cases
def test_mutation_gn_neighbour_group_statistics(audit):
    r, _ = run_gn(audit, 'gn_neighbour')
    flagged(r, 'a')
    flagged(r, 'b')


def test_mutation_ln_skips_last_row_of_tail(audit):
    flagged(run_ln(audit, 'ln_skip_tail')[0], 'a')


def test_mutation_conv_out_pitched_x(audit):
    x = rnd((2 * 8 * 8, 336), 23, dtype=F16)[:, :320]
    flagged(run_conv_out(audit, x=x)[0], 'p')


def test_mutation_upsample_writes_past_window(audit):
    flagged(run_resample(audit, 'write_past')[0], 'c')


@pytest.mark.parametrize('pad', [0, 1])
def test_mutation_im2col_wrong_pad(audit, pad):
    flagged(run_resample(audit, 'im2col_pad', pad=pad)[0], 'a')


def test_mutation_region_box_edge_off_by_one(audit):
    flagged(run_region(audit, 'region_edge')[0], 'a')


def test_mutation_clip_embed_pad_not_zero(audit):
    flagged(run_clip_embed(audit, 'clip_pad')[0], 'a')


def test_mutation_geglu_bwd_tanh_gelu(audit):
    flagged(run_pointwise(audit, 'geglu_tanh')[0], 'a')


def test_mutation_add_noise_reads_next_timestep(audit):
    flagged(run_training_glue(audit, 'noise_t+1')[0], 'a')


def test_mutation_quick_gelu_bwd_writes_into_x(audit):
    flagged(run_pointwise(audit, 'qg_bwd_into_x')[0], 'd')


def test_mutation_nondeterministic_relaunch(audit):
    flagged(run_ln(audit, 'nondet')[0], 'e')


def test_timestep_out_of_range(audit):
    flagged(run_training_glue(audit, t=(77, 1000))[0], 'p')


def test_region_box_outside_map(audit):
    from mos_b200 import ops
    o = rnd((1, 64, 8), 40, dtype=F16)
    reg = rnd((1, 64, 8), 41, dtype=F16)
    with audit() as r:
        r.register(reg)
        ops.region_combine(o, torch.tensor([reg.data_ptr()]), [(0, 0, 9, 8)], o, B=1, FH=8, FW=8, C=8, ld=8)
    flagged(r, 'p')


# ------------------------------------------------------------------------------ backward, training state, VAE, time
def run_gn_bwd(audit, mut=None, B=2, HW=1024, C=320, silu=True, add=True, ws=1 << 16):
    from mos_b200 import ops
    x = rnd((B, HW, C), 50, 2.0, BF, shift=0.5)
    dy = rnd((B, HW, C), 51, 1.0, BF)
    gamma, beta = rnd((C,), 52, 0.3) + 1, rnd((C,), 53, 0.2)
    ad = rnd((B, HW, C), 54, 1.0, BF) if add else None
    dx = torch.zeros(B, HW, C, dtype=BF)
    wsb = torch.zeros(ws)
    with audit(mut) as r:
        ops.groupnorm_bwd(x, dy, gamma, beta, dx, wsb, B=B, HW=HW, C=C, eps=1e-5, silu=silu, add=ad)
    return r, dict(x=x, dy=dy, gamma=gamma, beta=beta, add=ad, dx=dx, ws=wsb)


def test_groupnorm_bwd_reference_vs_autograd(audit):
    r, o = run_gn_bwd(audit)
    ok(r)
    assert keys(r) == {'gn_bwd|silu|add'}
    x = o['x'].double().transpose(1, 2).requires_grad_()
    y = F.silu(F.group_norm(x, 32, o['gamma'].double(), o['beta'].double(), 1e-5))
    (g,) = torch.autograd.grad((y * o['dy'].double().transpose(1, 2)).sum(), x)
    want = g.transpose(1, 2) + o['add'].double()
    assert torch.allclose(na.reference(r.last)['dx'][0].reshape(want.shape), want, rtol=1e-9, atol=1e-9)
    nch = na.gn_bwd_chunks(r.last['abi'])
    assert (o['ws'][:2 * nch * 128] == 1).all() and (o['ws'][2 * nch * 128:] == 0).all()


@pytest.mark.parametrize('M', [157, 8])
def test_layernorm_bwd_reference_vs_autograd(audit, M):
    from mos_b200 import ops
    C = 768
    x, dy, ad = rnd((M, C), 55, 1.5, BF), rnd((M, C), 56, 1.0, BF), rnd((M, C), 57, 1.0, BF)
    gamma = rnd((C,), 58, 0.3) + 1
    dx = torch.zeros(M, C, dtype=BF)
    with audit() as r:
        ops.layernorm_bwd(x, dy, gamma, dx, M=M, C=C, add=ad)
    ok(r)
    assert keys(r) == {f"ln_bwd|C=768{'|mtail' if M % 8 else ''}|add"}
    xd = x.double().requires_grad_()
    (g,) = torch.autograd.grad((F.layer_norm(xd, (C,), gamma.double(), None, 1e-5) * dy.double()).sum(), xd)
    assert torch.allclose(na.reference(r.last)['dx'][0], g + ad.double(), rtol=1e-9, atol=1e-9)


def run_adamw(audit, mut=None, step=3, norm=True):
    from mos_b200 import ops
    n = 3 * 768 + 1000 + 2000
    p, g = rnd((n,), 60, 0.1), rnd((n,), 61, 0.01)
    m, v = rnd((n,), 62, 0.001), rnd((n,), 63, 1e-4).abs()
    ends, lrs = (3 * 768, 3 * 768 + 1000, n), (1e-3, 1e-5, 1e-4)
    out = torch.zeros(1)
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    with audit(mut) as r:
        ops.flat_adamw_step(p, g, m, v, ends, lrs, step=step, grad_scale=0.5, emb_rows=3, emb_dim=768,
                            norm_mean_out=out if norm else None)
    return r, dict(p=p, g=g, m=m, v=v, p0=p0, m0=m0, v0=v0, ends=ends, lrs=lrs, out=out, step=step)


def test_adamw_reference_vs_torch_optim(audit):
    r, o = run_adamw(audit)
    ok(r)
    assert keys(r) == {'adamw|norm'}
    want = []
    for (g0, g1), lr in zip([(0, o['ends'][0]), (o['ends'][0], o['ends'][1]), (o['ends'][1], o['ends'][2])], o['lrs']):
        prm = torch.nn.Parameter(o['p0'][g0:g1].double().clone())
        opt = torch.optim.AdamW([prm], lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
        opt.state[prm] = {'step': torch.tensor(float(o['step'] - 1)), 'exp_avg': o['m0'][g0:g1].double().clone(),
                          'exp_avg_sq': o['v0'][g0:g1].double().clone()}
        prm.grad = o['g'][g0:g1].double() * 0.5
        opt.step()
        want.append(prm.detach())
    want = torch.cat(want)
    ref = na.reference(r.last)['p'][0]
    assert torch.allclose(ref, want, rtol=1e-6, atol=1e-8)          # the fp32 betas and rates the kernel is given
    assert torch.allclose(o['p'].double(), want, rtol=1e-5, atol=1e-9)
    assert abs(o['out'].item() - want[:3 * 768].view(3, 768).norm(dim=1).mean().item()) < 1e-6


def test_lora_grad_reference_vs_autograd(audit):
    from mos_b200 import ops
    M, K, N = 300, 320, 640
    x, dy = rnd((M, K), 64, 1.0, BF), rnd((M, N), 65, 1.0, BF)
    D, U = rnd((4, K), 66, 0.1), rnd((N, 4), 67, 0.1)
    ws = torch.zeros(1 << 17)
    dd, du = torch.zeros(4, K), torch.zeros(N, 4)
    with audit() as r:
        ops.lora_grad(x, dy, D, U, 0.7, ws, dd, du, M=M, K=K, N=N)
    ok(r)
    Dd, Ud = D.double().requires_grad_(), U.double().requires_grad_()
    y = r.last['abi']['alpha'] * (x.double() @ Dd.t()) @ Ud.t()          # the fp32 alpha the kernel is given
    gD, gU = torch.autograd.grad((y * dy.double()).sum(), (Dd, Ud))
    ref = na.reference(r.last)
    assert torch.allclose(ref['d_down'][0], gD, rtol=1e-9, atol=1e-9) and torch.allclose(ref['d_up'][0], gU, rtol=1e-9, atol=1e-9)
    (key,) = keys(r)
    assert key == 'lora_grad|R=16|staged'


def test_masked_mse_reference_vs_oracle(audit):
    from mos_b200 import ops
    from oracle.train_ref import masked_mse
    B, HW = 2, 64
    pred, target = rnd((B, 4, 8, 8), 68), rnd((B, 4, 8, 8), 69)
    mask = (rnd((B, 1, 8, 8), 70) > 0).float()
    ws, loss, dp = torch.zeros(2 * B + 5), torch.zeros(1), torch.zeros(B, 4, 8, 8)
    with audit() as r:
        ops.masked_mse(pred, target, mask, ws, loss, dp)
    ok(r)
    pd = pred.double().requires_grad_()
    want = masked_mse(pd, target.double(), mask.double())
    (g,) = torch.autograd.grad(want, pd)
    assert abs(loss.item() - want.item()) < 1e-5 * abs(want.item())
    assert torch.allclose(dp.double(), g, rtol=1e-5, atol=1e-9)
    assert (ws[2 * B:] == 0).all()
    del HW


def test_mutation_gn_bwd_drops_add_on_last_chunk(audit):
    flagged(run_gn_bwd(audit, 'gn_bwd_drop_add')[0], 'a')


def test_mutation_lora_grad_writes_past_workspace_prefix(audit):
    from mos_b200 import ops
    M, K, N = 300, 320, 640
    with audit('lora_ws_past') as r:
        ops.lora_grad(rnd((M, K), 64, 1.0, BF), rnd((M, N), 65, 1.0, BF), rnd((4, K), 66, 0.1), rnd((N, 4), 67, 0.1),
                      0.7, torch.zeros(1 << 17), torch.zeros(4, K), torch.zeros(N, 4), M=M, K=K, N=N)
    flagged(r, 'c')


def test_mutation_masked_mse_wrong_count(audit):
    from mos_b200 import ops
    pred, target = rnd((2, 4, 8, 8), 68), rnd((2, 4, 8, 8), 69)
    mask = (rnd((2, 1, 8, 8), 70) > 0).float()
    with audit('mse_count') as r:
        ops.masked_mse(pred, target, mask, torch.zeros(4), torch.zeros(1), torch.zeros(2, 4, 8, 8))
    flagged(r, 'a')


def test_mutation_adamw_bias_correction_one_step_late(audit):
    flagged(run_adamw(audit, 'adamw_bc_late')[0], 'a')


def test_small_kernels_pass_clean(audit):
    """time embedding, GEMV nb = 1..8, conv_in, softmax rows, 1x1 conv, VAE moments with noise, clip_embed_bwd"""
    from mos_b200 import ops
    with audit() as r:
        ops.timestep_embedding(torch.tensor([981.0, 1.0]), torch.zeros(2, 320))
        for nb in range(1, 9):
            ops.gemv(rnd((nb, 320), 71 + nb), rnd((1280, 320), 80, 0.05, BF), rnd((1280,), 81), torch.zeros(nb, 1280),
                     act_in=nb % 2 == 0, act_out=nb % 3 == 0)
        ops.conv_in(rnd((2, 4, 8, 8), 82), rnd((36, 320), 83, 0.1), rnd((320,), 84), torch.zeros(128, 336, dtype=F16),
                    ldy=336)
        ops.softmax_rows(rnd((64, 68), 85, 3.0)[:, :64], torch.zeros(64, 64, dtype=F16), rows=64, cols=64, scale=0.125)
        ops.conv1x1_nchw(rnd((2, 4, 8, 8), 86), rnd((4, 4), 87), rnd((4,), 88), torch.zeros(2, 4, 8, 8))
        ops.vae_moments(rnd((128, 8), 89, dtype=BF), rnd((8, 8), 90, 0.3), rnd((8,), 91), torch.zeros(2, 4, 64),
                        torch.zeros(2, 4, 64), B=2, HW=64, L=4, noise=rnd((2, 4, 64), 92), scaling=0.18215,
                        latents=torch.zeros(2, 4, 64))
        ids = torch.tensor([1, 5, 7, 5, 2, 5], dtype=torch.int32)
        ops.clip_embed_bwd(ids, rnd((6, 768), 93, dtype=BF), torch.tensor([5, 9], dtype=torch.int32),
                           torch.zeros(2, 768), C=768)
    ok(r)
    assert {f'gemv|nb={nb}' + ('|act_in' if nb % 2 == 0 else '') + ('|act_out' if nb % 3 == 0 else '')
            for nb in range(1, 9)} <= keys(r)


def test_pitched_operand_without_its_pitch(audit):
    """upsample2x_bwd called without lddy on a pitched dy: the kernel reads it at pitch C"""
    from mos_b200 import ops
    dy = rnd((2 * 8 * 8, 336), 94, dtype=BF)[:, :320]
    with audit() as r:
        ops.upsample2x_bwd(dy, torch.zeros(2 * 4 * 4, 320, dtype=BF), B=2, H=4, W=4, C=320)
    flagged(r, 'p')
