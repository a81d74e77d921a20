"""Backward kernels of the training step vs torch.autograd (fp32) on the same bf16-rounded inputs.

Tolerances: outputs are bf16 (one rounding: rel-L2 ~2e-3); attention backward additionally rounds P and dS to bf16
before the tensor-core products (as every flash backward does): rel-L2 <= 2e-2.  fp32 outputs (loss, LoRA grads with
fixed-order fp32 reductions): 1e-4 .. 2e-3 as stated.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def mk(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(BF)


def _row_offsets(M, dev, ratio, seed):
    """a per-row offset of `ratio` x the rows' std (1.5), with a random sign per row"""
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0) * 1.5 * ratio).to(dev)


def _check_layernorm_bwd(cuda, M, C, ld=None, off=0):
    """x rows with pitch ld (default C) and a per-row offset of `off` x the rows' std, vs float64 autograd"""
    from mos_b200 import ops
    ld = C if ld is None else ld
    buf = (mk((M, ld), cuda, 1.5, 1).float() + _row_offsets(M, cuda, off, 4)).to(BF)
    x = buf[:, :C]
    dy, add = mk((M, C), cuda, 1.0, 2), mk((M, C), cuda, 1.0, 3)
    gamma, beta = torch.randn(C, device=cuda), torch.randn(C, device=cuda)
    xr = x.double().requires_grad_(True)
    F.layer_norm(xr, (C,), gamma.double(), beta.double(), 1e-5).backward(dy.double())
    dx = torch.empty(M, C, device=cuda, dtype=BF)
    ops.layernorm_bwd(buf, dy, gamma, dx, M=M, C=C, ldx=ld)
    assert rel_l2(dx, xr.grad) < 4e-3
    ops.layernorm_bwd(buf, dy, gamma, dx, M=M, C=C, add=add, ldx=ld)
    assert rel_l2(dx, xr.grad + add.double()) < 4e-3


@pytest.mark.parametrize('M,C', [(8192, 320), (2048, 640), (300, 1280)])
def test_layernorm_bwd(cuda, M, C):
    _check_layernorm_bwd(cuda, M, C)


# C = 768 with ldx = 800 is the CLIP engines' hidden-state pitch; off: row mean / std
@pytest.mark.parametrize('off', [0, 100])
def test_layernorm_bwd_pitched_offset(cuda, off):
    _check_layernorm_bwd(cuda, 154, 768, ld=800, off=off)


# off: group mean / std (a per-(sample, group) offset); pad: extra columns of dy, dx and add (lddy = lddx = ldadd = C + pad);
# ws: workspace floats (B * 128 holds one chunk of both partial tables)
# outlier: (layout, K) of gpu_helpers.plant_outlier: the group's first element of row 0, or all of row 0, K std from its
# mean
def _check_groupnorm_bwd(cuda, B, HW, C, ld, silu, off=0, pad=0, ws=1 << 18, outlier=None):
    from gpu_helpers import canary, plant_outlier, untouched, window_mask, worst_group_rel_l2
    from mos_b200 import ops
    g = torch.Generator(device='cpu').manual_seed(5)
    sign = torch.where(torch.rand(B, 1, 32, 1, generator=g) < 0.5, -1.0, 1.0)
    shift = (sign * 1.5 * off).expand(B, 1, 32, C // 32).reshape(B, 1, C).to(cuda)
    buf = mk((B, HW, ld), cuda, 1.5, 1).float() + 0.3
    buf[..., :C] += shift
    buf = buf.to(BF)
    if outlier is not None:
        buf, _ = plant_outlier(buf, C, *outlier, seed=6)
    x = buf[..., :C]
    ldp = C + pad
    dyb = torch.full((B, HW, ldp), float('nan'), device=cuda, dtype=BF)
    addb = torch.full((B, HW, ldp), float('nan'), device=cuda, dtype=BF)
    dyb[..., :C], addb[..., :C] = mk((B, HW, C), cuda, 1.0, 2), mk((B, HW, C), cuda, 1.0, 3)
    dy, add = dyb[..., :C], addb[..., :C]
    gamma, beta = torch.randn(C, device=cuda), torch.randn(C, device=cuda)
    xr = x.double().permute(0, 2, 1).contiguous().requires_grad_(True)       # [B, C, HW]
    y = F.group_norm(xr, 32, gamma.double(), beta.double(), 1e-5)
    if silu:
        y = F.silu(y)
    y.backward(dy.double().permute(0, 2, 1))
    ref = xr.grad.permute(0, 2, 1)
    wsb = torch.empty(ws, device=cuda)
    dxb = canary((B * HW + 2, ldp), cuda, BF)
    dx = dxb[:B * HW, :C].view(B, HW, C)
    ops.groupnorm_bwd(x, dy, gamma, beta, dx, wsb, B=B, HW=HW, C=C, eps=1e-5, silu=silu, ldx=ld, lddy=ldp, lddx=ldp)
    assert untouched(dxb, window_mask(dxb, slice(0, B * HW), slice(0, C)))
    e = rel_l2(dx, ref)
    # the planted element must not hide a bad group behind the global norm; without add, so that add does not dilute it
    e_group = worst_group_rel_l2(dx, ref, C) if outlier is not None else None
    ops.groupnorm_bwd(x, dy, gamma, beta, dx, wsb, B=B, HW=HW, C=C, eps=1e-5, silu=silu, ldx=ld, lddy=ldp, lddx=ldp,
                      add=add, ldadd=ldp)
    e_add = rel_l2(dx, ref + add.double())
    print(f'GN bwd B={B} HW={HW} C={C} offset {off} pad {pad} ws {ws} outlier {outlier}: rel-L2 {e:.2e}, '
          f'with add {e_add:.2e}')
    assert e < 5e-3 and e_add < 5e-3
    if outlier is not None:
        e_group_add = worst_group_rel_l2(dx, ref + add.double(), C)
        print(f'  worst group rel-L2 {e_group:.2e}, with add {e_group_add:.2e}')
        assert e_group < 5e-3 and e_group_add < 5e-3


GN_BWD_SHAPES = [(2, 4096, 320, 320, True), (2, 1024, 1920, 1920, True), (2, 256, 640, 1280, False),
                 (3, 64, 1280, 1280, True), (1, 1024, 960, 960, True)]


@pytest.mark.parametrize('B,HW,C,ld,silu', GN_BWD_SHAPES)
def test_groupnorm_bwd(cuda, B, HW, C, ld, silu):
    _check_groupnorm_bwd(cuda, B, HW, C, ld, silu)


@pytest.mark.parametrize('B,HW,C,ld,silu,off,pad,ws', [
    (2, 4096, 320, 320, True, 10, 32, 1 << 18), (2, 1024, 640, 1280, True, 30, 16, 1 << 18),
    (1, 1024, 960, 960, True, 100, 40, 1 << 18), (2, 256, 1280, 1280, False, 100, 8, 1 << 18),
    (2, 4096, 320, 320, True, 100, 0, 2 * 128), (3, 64, 1280, 1280, True, 30, 24, 3 * 128)])
def test_groupnorm_bwd_offset_pitched(cuda, B, HW, C, ld, silu, off, pad, ws):
    """group means up to 100 x their std, dy / dx / add pitches above C, and a one-chunk workspace"""
    _check_groupnorm_bwd(cuda, B, HW, C, ld, silu, off, pad, ws)


@pytest.mark.parametrize('K', [30, 100, 300, 'max'])
@pytest.mark.parametrize('layout', ['pivot', 'corner'])
@pytest.mark.parametrize('B,HW,C,ld,silu', GN_BWD_SHAPES)
def test_groupnorm_bwd_outlier(cuda, B, HW, C, ld, silu, layout, K):
    """the group's first element of row 0, or the whole first pixel, K x the group's std from its mean: the recomputed
    statistics must not lose the variance to cancellation against it"""
    _check_groupnorm_bwd(cuda, B, HW, C, ld, silu, outlier=(layout, K))


@pytest.mark.parametrize('K', [30, 300, 'max'])
@pytest.mark.parametrize('layout', ['pivot', 'corner'])
def test_groupnorm_bwd_outlier_one_chunk(cuda, layout, K):
    """a workspace of one chunk per sample: each statistics thread runs over HW / lanes = 512 rows, the outlier first"""
    _check_groupnorm_bwd(cuda, 2, 4096, 320, 320, True, ws=2 * 128, outlier=(layout, K))


def test_geglu_fwd_bwd(cuda):
    from mos_b200 import ops
    M, H = 1024, 1280
    z, dy = mk((M, 2 * H), cuda, 1.0, 1), mk((M, H), cuda, 1.0, 2)
    zt = z.float().view(M, H // 80, 2, 80).requires_grad_(True)
    y_ref = (zt[:, :, 0] * F.gelu(zt[:, :, 1])).reshape(M, H)
    y_ref.backward(dy.float())
    y, dz = torch.empty(M, H, device=cuda, dtype=BF), torch.empty(M, 2 * H, device=cuda, dtype=BF)
    ops.geglu_fwd(z, y, M=M, H=H)
    ops.geglu_bwd(z, dy, dz, M=M, H=H)
    assert rel_l2(y, y_ref) < 4e-3
    assert rel_l2(dz, zt.grad.reshape(M, 2 * H)) < 4e-3


def test_resample_bwd(cuda):
    from mos_b200 import ops
    B, H, W, C = 2, 16, 12, 320
    dy = mk((B, 2 * H, 2 * W, C), cuda, 1.0, 1)
    dx = torch.empty(B, H, W, C, device=cuda, dtype=BF)
    ops.upsample2x_bwd(dy, dx, B=B, H=H, W=W, C=C)
    ref = dy.float().view(B, H, 2, W, 2, C).sum((2, 4))
    assert rel_l2(dx, ref) < 4e-3
    # col2im: backward of mos_im2col_s2 (3x3, stride 2, pad 1, tap-major columns)
    x = mk((B, H, W, C), cuda, 1.0, 2)
    col = torch.empty(B * (H // 2) * (W // 2), 9 * C, device=cuda, dtype=BF)
    ops.im2col_s2(x, col, B=B, H=H, W=W, C=C)
    dcol = mk(tuple(col.shape), cuda, 1.0, 3)
    xr = x.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    un = F.unfold(xr, 3, padding=1, stride=2)                                  # [B, C*9, L], rows ordered (c, kh, kw)
    un = un.view(B, C, 9, -1).permute(0, 3, 2, 1).reshape(B * (H // 2) * (W // 2), 9 * C)
    assert torch.equal(un.detach().to(BF), col)
    (un * dcol.float()).sum().backward()
    add = mk((B, H, W, C), cuda, 1.0, 4)
    dxc = torch.empty(B, H, W, C, device=cuda, dtype=BF)
    ops.col2im_s2(dcol, dxc, B=B, H=H, W=W, C=C, add=add)
    assert rel_l2(dxc, xr.grad.permute(0, 2, 3, 1) + add.float()) < 4e-3


def test_conv_out_bwd_mse_noise(cuda):
    from mos_b200 import ops
    B, H, W, C = 2, 16, 16, 320
    w = torch.randn(4, 9, C, device=cuda) * 0.05
    dy = torch.randn(B, 4, H, W, device=cuda)
    xr = torch.randn(B, C, H, W, device=cuda, requires_grad=True)
    w4 = w.view(4, 3, 3, C).permute(0, 3, 1, 2).contiguous()
    F.conv2d(xr, w4, padding=1).backward(dy)
    dx = torch.empty(B * H * W, C, device=cuda, dtype=BF)
    ops.conv_out_bwd(dy, w, dx, B=B, H=H, W=W, C=C)
    assert rel_l2(dx.view(B, H, W, C), xr.grad.permute(0, 2, 3, 1)) < 4e-3
    # masked MSE (trainer_edlora.py:251-252) and its gradient
    pred = torch.randn(B, 4, H, W, device=cuda, requires_grad=True)
    target = torch.randn(B, 4, H, W, device=cuda)
    mask = (torch.rand(B, 1, H, W, device=cuda) > 0.4).float()
    l = F.mse_loss(pred.float(), target.float(), reduction='none')
    l = ((l * mask).sum([1, 2, 3]) / mask.sum([1, 2, 3])).mean()
    l.backward()
    ws, loss, dp = torch.empty(2 * B, device=cuda), torch.empty(1, device=cuda), torch.empty_like(target)
    ops.masked_mse(pred.detach(), target, mask, ws, loss, dp)
    assert abs(loss.item() - l.item()) < 1e-5 * abs(l.item()) + 1e-7
    assert rel_l2(dp, pred.grad) < 1e-5
    # add_noise
    from oracle.schedulers import DDPMScheduler
    sch = DDPMScheduler()
    t = torch.tensor([7, 933], device=cuda)
    noise = torch.randn_like(target)
    out = torch.empty_like(target)
    ops.add_noise(target, noise, t.int(), sch.alphas_cumprod.to(cuda), out)
    assert rel_l2(out, sch.add_noise(target, noise, t)) < 1e-6


@pytest.mark.parametrize('M,K,N', [(8192, 320, 320), (154, 768, 640), (1000, 1280, 1280), (20001, 640, 320),
                                   (70000, 320, 320)])
def test_lora_grad(cuda, M, K, N):
    from mos_b200 import ops
    x, dy = mk((M, K), cuda, 1.0, 1), mk((M, N), cuda, 1.0, 2)
    down = (torch.randn(4, K, device=cuda) * 0.1).requires_grad_(True)
    up = (torch.randn(N, 4, device=cuda) * 0.1).requires_grad_(True)
    alpha = 0.7
    (alpha * (x.float() @ down.T) @ up.T * dy.float()).sum().backward()
    ws = torch.empty(128 * 4 * (K + N), device=cuda)      # <= 128 row slabs, one partial [4K + 4N] each
    dd, du = torch.empty(4, K, device=cuda), torch.empty(N, 4, device=cuda)
    ops.lora_grad(x, dy, down.detach(), up.detach(), alpha, ws, dd, du, M=M, K=K, N=N)
    assert rel_l2(dd, down.grad) < 1e-4
    assert rel_l2(du, up.grad) < 1e-4
    ops.lora_grad(x, dy, down.detach(), up.detach(), alpha, ws, dd, du, M=M, K=K, N=N, accumulate=True)
    assert rel_l2(dd, 2 * down.grad) < 1e-4


def _pack_rows(t, dp):
    """[B, H, n, d] -> [B*H, n, dp] zero padded"""
    B, H, n, d = t.shape
    out = torch.zeros(B * H, n, dp, device=t.device, dtype=BF)
    out[..., :d] = t.reshape(B * H, n, d)
    return out


@pytest.mark.parametrize('d,nq,nk,reg', [(40, 512, 512, False), (40, 1000, 300, False), (80, 256, 256, False),
                                         (160, 200, 200, False), (160, 64, 64, False), (40, 1024, 77, True),
                                         (80, 256, 77, True), (160, 64, 77, True), (40, 4096, 4096, False)])
def test_attention_fwd_train_and_bwd(cuda, d, nq, nk, reg):
    from mos_b200 import ops
    B, H = 2, 8
    dp, dvp = (d + 63) // 64 * 64, (d + 15) // 16 * 16
    nq8, nk8 = (nq + 7) // 8 * 8, (nk + 7) // 8 * 8
    q, k, v = mk((B, H, nq, d), cuda, 1.0, 1), mk((B, H, nk, d), cuda, 1.0, 2), mk((B, H, nk, d), cuda, 1.0, 3)
    do = mk((B, H, nq, d), cuda, 1.0, 4)
    Q, K, V, dO = _pack_rows(q, dp), _pack_rows(k, dp), _pack_rows(v, dp), _pack_rows(do, dp)
    Qt = torch.zeros(B * H, dvp, nq8, device=cuda, dtype=BF)
    Kt, Vt, dOt = torch.zeros(B * H, dvp, nk8, device=cuda, dtype=BF), torch.zeros(B * H, dvp, nk8, device=cuda, dtype=BF), \
        torch.zeros_like(Qt)
    for s, t in ((Q, Qt), (K, Kt), (V, Vt), (dO, dOt)):
        ops.heads_transpose(s, t)
    assert torch.equal(Vt[:, :d, :nk], v.reshape(B * H, nk, d).transpose(1, 2))
    assert dvp == d or Vt[:, d:].abs().max().item() == 0
    pos = torch.tensor([[3, 9], [5, 6]], device=cuda, dtype=torch.int32) if reg else None
    gcols = (torch.randn(B, nq, 2, device=cuda) * 0.5) if reg else None
    pcols = torch.empty(B * H, nq, 2, device=cuda) if reg else None
    out = torch.empty(B, nq, H * d, device=cuda, dtype=BF)
    lse2 = torch.empty(B * H, nq, device=cuda)
    ops.attention_train(Q, K, Vt, out, lse2, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, pcols=pcols, pos=pos)
    # ---- reference (fp32 autograd)
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    S = (qr @ kr.transpose(-1, -2)) * d ** -0.5
    P = S.softmax(-1)
    O = P @ vr
    loss = (O * do.float()).sum()
    if reg:
        for b in range(B):
            for c in range(2):
                loss = loss + (P[b, :, :, int(pos[b, c])] * gcols[b, :, c][None]).sum()
    loss.backward()
    ref_lse2 = torch.logsumexp(S.detach(), -1) * 1.4426950408889634
    assert rel_l2(out, O.detach().permute(0, 2, 1, 3).reshape(B, nq, H * d)) < 8e-3
    assert (lse2 - ref_lse2.reshape(B * H, nq)).abs().max().item() < 2e-3
    if reg:
        pr = torch.stack([torch.stack([P[b, :, :, int(pos[b, c])] for c in range(2)], -1) for b in range(B)])
        assert rel_l2(pcols, pr.detach().reshape(B * H, nq, 2)) < 2e-3
    # ---- backward kernels
    delta = torch.empty(B * H, nq, device=cuda)
    ops.attn_delta(dO, out, delta, batch=B, heads=H, head_dim=d, N=nq, pcols=pcols, gcols=gcols)
    dref = (O.detach() * do.float()).sum(-1)
    if reg:
        dref = dref + (pr.detach() * gcols[:, None]).sum(-1)
    assert rel_l2(delta, dref.reshape(B * H, nq)) < 1e-2
    dq = torch.full((B * nq, H * d), float('nan'), device=cuda, dtype=BF)
    dk = torch.full((B * nk, H * d), float('nan'), device=cuda, dtype=BF)
    dv = torch.full((B * nk, H * d), float('nan'), device=cuda, dtype=BF)
    ops.attention_bwd(Q, K, V, dO, Qt, Kt, dOt, lse2, delta, dq, dk, dv, batch=B, heads=H, head_dim=d, nq=nq, nk=nk,
                      gcols=gcols, pos=pos)
    torch.cuda.synchronize()

    def tok(g, n):
        return g.permute(0, 2, 1, 3).reshape(B * n, H * d)
    eq, ek, ev = rel_l2(dq, tok(qr.grad, nq)), rel_l2(dk, tok(kr.grad, nk)), rel_l2(dv, tok(vr.grad, nk))
    print(f'attention bwd d={d} nq={nq} nk={nk} reg={reg}: dq {eq:.2e} dk {ek:.2e} dv {ev:.2e}')
    assert eq < 2e-2 and ek < 2e-2 and ev < 2e-2
