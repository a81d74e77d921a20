"""Parity of the attention / norm / elementwise kernels vs plain PyTorch fp32 references of the same op.

Tolerances (stated per test): outputs are bf16, so one final rounding gives rel-L2 ~2e-3; attention additionally
rounds P to bf16 before the PV product (as every flash kernel does): rel-L2 <= 8e-3.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def mk(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(torch.bfloat16)


def pack_heads(q, k, v, d):
    """q [B,H,nq,d], k/v [B,H,nk,d] bf16 -> padded device layouts"""
    B, H, nq, _ = q.shape
    nk = k.shape[2]
    dp = ((d + 63) // 64) * 64
    dv = ((d + 15) // 16) * 16
    nk8 = ((nk + 7) // 8) * 8
    Q = torch.zeros(B * H, nq, dp, device=q.device, dtype=torch.bfloat16)
    K = torch.zeros(B * H, nk, dp, device=q.device, dtype=torch.bfloat16)
    Vt = torch.zeros(B * H, dv, nk8, device=q.device, dtype=torch.bfloat16)
    Q[..., :d] = q.reshape(B * H, nq, d)
    K[..., :d] = k.reshape(B * H, nk, d)
    Vt[:, :d, :nk] = v.reshape(B * H, nk, d).transpose(1, 2)
    return Q, K, Vt


@pytest.mark.parametrize('d,nq,nk', [(40, 4096, 4096), (40, 1000, 300), (80, 1024, 1024), (160, 256, 256),
                                     (160, 64, 64), (40, 4096, 77), (80, 1024, 77), (160, 256, 77), (40, 130, 1)])
def test_attention(cuda, d, nq, nk):
    from mos_b200 import ops
    B, H = 2, 8
    q, k, v = mk((B, H, nq, d), cuda, seed=1), mk((B, H, nk, d), cuda, seed=2), mk((B, H, nk, d), cuda, seed=3)
    Q, K, Vt = pack_heads(q, k, v, d)
    out = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float())  # [B,H,nq,d]
    ref = ref.permute(0, 2, 1, 3).reshape(B, nq, H * d)
    assert rel_l2(out, ref) < 8e-3


@pytest.mark.parametrize('d,nq,nk,amp', [(40, 256, 1024, 4.0), (40, 256, 1024, 16.0), (40, 384, 1000, 60.0),
                                         (80, 256, 1024, 16.0), (80, 128, 600, 60.0), (160, 128, 512, 16.0),
                                         (160, 128, 500, 60.0)])
def test_attention_growing_logits(cuda, d, nq, nk, amp):
    """Later key tiles carry ever larger logits, so the running maximum of the online softmax has to move and O be
    rescaled, by large factors for the large amplitudes.  Same tolerance as test_attention."""
    from mos_b200 import ops
    B, H = 1, 8
    q, k, v = mk((B, H, nq, d), cuda, seed=4), mk((B, H, nk, d), cuda, seed=5), mk((B, H, nk, d), cuda, seed=6)
    ramp = (0.1 + torch.arange(nk, device=cuda).float() / nk).view(1, 1, nk, 1)
    k = (k.float() * ramp * amp).to(torch.bfloat16)
    Q, K, Vt = pack_heads(q, k, v, d)
    out = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float())
    ref = ref.permute(0, 2, 1, 3).reshape(B, nq, H * d)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < 8e-3


@pytest.mark.parametrize('d,nq', [(40, 4096), (80, 1024), (160, 256), (160, 64)])
def test_attention_probs(cuda, d, nq):
    """probability maps for the attention controller (edlora.py:81-82): [B*heads, N, 77], rows sum to 1."""
    from mos_b200 import ops
    B, H, nk = 2, 8, 77
    q, k, v = mk((B, H, nq, d), cuda, seed=1), mk((B, H, nk, d), cuda, seed=2), mk((B, H, nk, d), cuda, seed=3)
    Q, K, Vt = pack_heads(q, k, v, d)
    out = torch.empty((B, nq, H * d), device=cuda, dtype=torch.bfloat16)
    probs = torch.full((B * H, nq, nk), float('nan'), device=cuda)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, probs=probs)
    ref = ((q.float() @ k.float().transpose(-1, -2)) * d ** -0.5).softmax(-1).reshape(B * H, nq, nk)
    assert rel_l2(probs, ref) < 1e-4          # fp32 in, fp32 out: only exp2 / summation-order differences
    assert (probs.sum(-1) - 1).abs().max().item() < 1e-5


@pytest.mark.parametrize('B,HW,C,ld,silu', [(2, 4096, 320, 320, True), (2, 1024, 640, 1280, True),
                                             (2, 256, 2560, 2560, True), (2, 64, 1280, 1280, False),
                                             (1, 4096, 960, 960, True), (2, 1024, 1920, 1920, True),
                                             (3, 288, 320, 320, False)])
def test_groupnorm(cuda, B, HW, C, ld, silu):
    from mos_b200 import ops
    buf = mk((B, HW, ld), cuda, seed=1) * 1.5 + 0.3
    x = buf[..., :C]
    gamma, beta = torch.randn(C, device=cuda), torch.randn(C, device=cuda)
    y = torch.empty((B, HW, C), device=cuda, dtype=torch.bfloat16)
    partial = torch.zeros(B * 592 * 64, device=cuda)   # the engines' workspace: enough for any B, HW
    ops.groupnorm(buf, gamma, beta, y, partial, B=B, HW=HW, C=C, eps=1e-5, silu=silu, ldx=ld)
    ref = F.group_norm(x.float().transpose(1, 2), 32, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    assert rel_l2(y, ref.transpose(1, 2)) < 4e-3


def _check_layernorm(cuda, M, C, ld=None, off=0):
    """x rows with pitch ld (default C) and a per-row offset of `off` x the rows' std, vs float64"""
    from mos_b200 import ops
    ld = C if ld is None else ld
    g = torch.Generator(device='cpu').manual_seed(2)
    shift = (torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0) * 2 * off).to(cuda)
    buf = (mk((M, ld), cuda, seed=1).float() * 2 + 0.5 + shift).to(torch.bfloat16)
    x = buf[:, :C]
    gamma, beta = torch.randn(C, device=cuda), torch.randn(C, device=cuda)
    y = torch.empty(M, C, device=cuda, dtype=torch.bfloat16)
    ops.layernorm(buf, gamma, beta, y, M=M, C=C, ldx=ld)
    ref = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5)
    assert rel_l2(y, ref) < 4e-3


@pytest.mark.parametrize('M,C', [(8192, 320), (2048, 640), (512, 1280), (154, 320)])
def test_layernorm(cuda, M, C):
    _check_layernorm(cuda, M, C)


# C = 768 with ldx = 800 is the CLIP engines' hidden-state pitch; off: row mean / std
@pytest.mark.parametrize('off', [0, 100])
def test_layernorm_pitched_offset(cuda, off):
    _check_layernorm(cuda, 154, 768, ld=800, off=off)


def test_time_embedding_and_gemv(cuda):
    from mos_b200 import ops
    t = torch.tensor([999.0, 981.0, 3.0], device=cuda)
    emb = torch.empty(3, 320, device=cuda)
    ops.timestep_embedding(t, emb)
    half = 160
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, device=cuda) / half)
    ref = torch.cat([torch.cos(t[:, None] * freqs), torch.sin(t[:, None] * freqs)], -1)
    assert (emb - ref).abs().max().item() < 2e-3   # sin/cos of arguments up to 1e3 in fp32
    W = mk((1280, 320), cuda, 320 ** -0.5, seed=2)
    b = torch.randn(1280, device=cuda)
    out = torch.empty(3, 1280, device=cuda)
    ops.gemv(ref.contiguous(), W, b, out, act_in=False, act_out=True)
    assert rel_l2(out, F.silu(ref @ W.float().t() + b)) < 1e-5
    out2 = torch.empty(3, 1280, device=cuda)
    ops.gemv(ref.contiguous(), W, b, out2, act_in=True, act_out=False)
    assert rel_l2(out2, F.silu(ref) @ W.float().t() + b) < 1e-5


def test_conv_in_out(cuda):
    from mos_b200 import ops
    B, H, W = 2, 64, 64
    x = torch.randn(B, 4, H, W, device=cuda)
    w = torch.randn(320, 4, 3, 3, device=cuda) * 0.2
    b = torch.randn(320, device=cuda)
    y = torch.empty(B, H, W, 320, device=cuda, dtype=torch.bfloat16)
    ops.conv_in(x, w.permute(2, 3, 1, 0).reshape(36, 320).contiguous(), b, y)
    ref = F.conv2d(x, w, b, padding=1).permute(0, 2, 3, 1)
    assert rel_l2(y, ref) < 4e-3
    xo = mk((B, H, W, 320), cuda, seed=4)
    wo = torch.randn(4, 320, 3, 3, device=cuda) * 0.05
    bo = torch.randn(4, device=cuda)
    yo = torch.empty(B, 4, H, W, device=cuda)
    ops.conv_out(xo, wo.permute(0, 2, 3, 1).reshape(4, 9, 320).contiguous(), bo, yo, B=B, H=H, W=W, C=320)
    assert rel_l2(yo, F.conv2d(xo.float().permute(0, 3, 1, 2), wo, bo, padding=1)) < 1e-5


def test_upsample_im2col_add(cuda):
    from mos_b200 import ops
    B, H, W, C = 2, 16, 16, 640
    x = mk((B, H, W, C), cuda, seed=1)
    y = torch.empty(B, 2 * H, 2 * W, C, device=cuda, dtype=torch.bfloat16)
    ops.upsample2x(x, y, B=B, H=H, W=W, C=C)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode='nearest').permute(0, 2, 3, 1)
    assert torch.equal(y.float(), ref)
    # stride-2 conv via im2col + GEMM == Downsample2D
    w = mk((C, C, 3, 3), cuda, (9 * C) ** -0.5, seed=2)
    bias = torch.randn(C, device=cuda)
    col = torch.empty(B * (H // 2) * (W // 2), 9 * C, device=cuda, dtype=torch.bfloat16)
    ops.im2col_s2(x, col, B=B, H=H, W=W, C=C)
    out = torch.empty(B * (H // 2) * (W // 2), C, device=cuda, dtype=torch.bfloat16)
    ops.gemm(col, w.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous(), out, bias=bias)
    refc = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, stride=2, padding=1).permute(0, 2, 3, 1)
    assert rel_l2(out, refc.reshape(-1, C)) < 4e-3
    a, r = mk((100, 640), cuda, seed=5), mk((100, 320), cuda, seed=6)
    a0 = a.clone()
    ops.add_rows(a, r, M=100, C=320, ldx=640, ldr=320)
    assert rel_l2(a[:, :320], a0[:, :320].float() + r.float()) < 4e-3 and torch.equal(a[:, 320:], a0[:, 320:])


def test_cfg_dpm_step_and_region_combine(cuda):
    from mos_b200 import ops
    n = 4 * 64 * 64
    npred = torch.randn(2 * n, device=cuda)
    lat, x0p = torch.randn(n, device=cuda), torch.randn(n, device=cuda)
    lat0, x0p0 = lat.clone(), x0p.clone()
    uin = torch.empty(2 * n, device=cuda)
    coef = (0.9, 0.12, -0.03, 0.2, 0.98)
    ops.cfg_dpmpp_step(npred, lat, x0p, uin, cfg=True, guidance=7.5, coef=coef)
    eps = npred[:n] + 7.5 * (npred[n:] - npred[:n])
    x0 = (lat0 - coef[4] * eps) / coef[3]
    ref = coef[0] * lat0 + coef[1] * x0 + coef[2] * x0p0
    assert torch.allclose(lat, ref, rtol=1e-5, atol=1e-5) and torch.allclose(x0p, x0, rtol=1e-5, atol=1e-5)
    assert torch.equal(uin[:n], lat) and torch.equal(uin[n:], lat)
    # region combine
    B, FH, FW, C = 2, 12, 24, 320
    glob = mk((B, FH * FW, C), cuda, seed=1)
    regs = [mk((B, FH * FW, C), cuda, seed=2 + i) for i in range(3)]
    boxes = [(0, 1, 12, 9), (1, 7, 12, 16), (0, 18, 11, 24)]
    ptrs = torch.tensor([r.data_ptr() for r in regs], dtype=torch.int64, device=cuda)
    out = torch.empty_like(glob)
    ops.region_combine(glob, ptrs, boxes, out, B=B, FH=FH, FW=FW, C=C, ld=C)
    count = torch.zeros(FH, FW, device=cuda)
    acc = torch.zeros(B, FH, FW, C, device=cuda)
    for r, (sh, sw, eh, ew) in zip(regs, boxes):
        count[sh:eh, sw:ew] += 1
        acc[:, sh:eh, sw:ew] += r.float().view(B, FH, FW, C)[:, sh:eh, sw:ew]
    ref = torch.where(count[None, :, :, None] == 0, glob.float().view(B, FH, FW, C),
                      acc / count.clamp_min(1)[None, :, :, None])
    assert rel_l2(out.view(B, FH, FW, C), ref) < 4e-3
    assert torch.equal(out.view(B, FH, FW, C)[:, count == 0], glob.view(B, FH, FW, C)[:, count == 0])
