"""Kernels of the ED-LoRA training state against plain references: the LoRA re-pack after each optimiser step
(mos_lora_pack), the flat AdamW step over three learning-rate groups (mos_flat_adamw_step, against AdamW written out in
float64), the gradient of the concept-token embedding rows (mos_clip_embed_bwd), the CLIP MLP activation
(mos_quick_gelu_fwd / _bwd) and the masked MSE of the UNet loss (mos_masked_mse).  Output buffers are canaries wherever
the kernel writes into a window of a larger allocation."""
import pytest
import torch

from gpu_helpers import bits, canary, mk, rel_l2_64, same_bits, untouched, window_mask

pytestmark = pytest.mark.gpu
F64 = torch.float64


# ================================================================================================= lora_pack
def test_lora_pack_layouts_and_canaries(cuda):
    """Hand-built pack table at SD1.5 projection sizes, ~100 modules, alpha 0.9, with and without backward packs.
    Forward down rows live at segment `seg` of a [16, K] bf16 block and forward up rows at segment `seg` of a [3N, 4]
    fp32 buffer (the fused q/k/v packs); the backward "down" is a [16, N] bf16 block (rows 0..3 = U^T) and the backward
    "up" a [Kp, 4] fp32 block (= alpha D^T), padded to 800 rows for the 768-wide text K / V inputs.  Bitwise."""
    from mos_b200 import ops
    alpha = 0.9
    sizes = [(320, 320), (320, 768), (768, 320), (640, 640), (1280, 1280)]
    g = torch.Generator().manual_seed(0)
    mods, rows = [], []
    for i in range(100):
        K, N = sizes[i % len(sizes)]
        seg = i % 3
        D = (torch.randn(4, K, generator=g) * 0.3).cuda()
        U = (torch.randn(N, 4, generator=g) * 0.3).cuda()
        fd = canary((16, K), cuda, torch.bfloat16)
        fu = canary((3 * N, 4), cuda, torch.float32)
        has_bwd = i % 7 != 3
        kp = 800 if K == 768 else K
        bd = canary((16, N), cuda, torch.bfloat16) if has_bwd else None
        bu = canary((kp, 4), cuda, torch.float32) if has_bwd else None
        mods.append(dict(D=D, U=U, K=K, N=N, seg=seg, fd=fd, fu=fu, bd=bd, bu=bu))
        rows.append([D.data_ptr(), U.data_ptr(), K, N, fd[4 * seg].data_ptr(), fu[seg * N].data_ptr(),
                     bd.data_ptr() if has_bwd else 0, bu.data_ptr() if has_bwd else 0])
    table = torch.tensor(rows, dtype=torch.int64, device=cuda)
    ops.lora_pack(table, len(rows), alpha)
    torch.cuda.synchronize()
    a = torch.tensor(alpha, dtype=torch.float32, device=cuda)
    for i, m in enumerate(mods):
        K, N, s = m['K'], m['N'], m['seg']
        assert same_bits(m['fd'][4 * s:4 * s + 4], m['D'].bfloat16()), i
        assert untouched(m['fd'], window_mask(m['fd'], slice(4 * s, 4 * s + 4))), i
        assert same_bits(m['fu'][s * N:(s + 1) * N], a * m['U']), i
        assert untouched(m['fu'], window_mask(m['fu'], slice(s * N, (s + 1) * N))), i
        if m['bd'] is None:
            continue
        assert same_bits(m['bd'][:4], m['U'].t().bfloat16()), i
        assert untouched(m['bd'], window_mask(m['bd'], slice(0, 4))), i
        assert same_bits(m['bu'][:K], a * m['D'].t()), i
        assert untouched(m['bu'], window_mask(m['bu'], slice(0, K))), i


# ================================================================================================= flat AdamW
def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _adamw64(p, g, m, v, ends, lrs, step, grad_scale, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.01):
    """torch.optim.AdamW's update (decoupled weight decay, bias corrections) written out in float64, with the
    hyper-parameters rounded to fp32 as the kernel receives them (1 - fp32(0.999) is 1.3e-5 off 0.001)"""
    p, g, m, v = (t.to(F64) for t in (p, g, m, v))
    lrs, beta1, beta2, eps, wd = [_f32(r) for r in lrs], _f32(beta1), _f32(beta2), _f32(eps), _f32(wd)
    lr = torch.empty_like(p)
    lo = 0
    for e, r in zip(ends, lrs):
        lr[lo:e] = r
        lo = e
    g = g * grad_scale
    m = beta1 * m + (1 - beta1) * g
    v = beta2 * v + (1 - beta2) * g * g
    bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
    p = p * (1 - lr * wd) - (lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + eps)
    return p, m, v, lr


@pytest.mark.parametrize('ends,step', [
    ((24909, 30012, 110101), 1),            # group ends off every multiple of 256 / 1024
    ((24909, 24909, 101113), 1000),         # no text-encoder LoRA (empty middle group), preloaded moments
    ((24576, 24576 + 33 * 1024, 24576 + 33 * 1024 + 1_300_001), 7),   # more elements than one grid-stride pass
])
def test_flat_adamw_vs_float64(cuda, ends, step):
    """Per element, the fp32 step may differ from float64 by rounding only: |p - p64| <= 1e-3 * lr_i (a parameter in the
    wrong learning-rate group would be off by ~lr).  Measured worst on an H100 80GB HBM3 (700 W): 2.8e-5 * lr_i;
    exp_avg / exp_avg_sq rel-L2 3.8e-8; Norm_mean 1.2e-7."""
    from mos_b200 import ops
    n = ends[2]
    lrs = (1e-3, 1e-5, 1e-4)
    g = torch.Generator().manual_seed(step)
    p0 = (torch.randn(n, generator=g) * 1e-3).cuda()
    grad = torch.randn(n, generator=g).cuda()
    if step == 1:
        m0, v0 = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    else:
        m0 = (torch.randn(n, generator=g) * 0.1).cuda()
        v0 = (torch.rand(n, generator=g) * 0.02).cuda()
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    norm = torch.full((1,), float('nan'), device=cuda)
    ops.flat_adamw_step(p, grad, m, v, ends, lrs, step=step, grad_scale=0.5, emb_rows=32, emb_dim=768,
                        norm_mean_out=norm)
    torch.cuda.synchronize()
    pr, mr, vr, lr = _adamw64(p0, grad, m0, v0, ends, lrs, step, 0.5)
    e_p = ((p.double() - pr).abs() / lr).max().item()
    e_m, e_v = rel_l2_64(m.double(), mr), rel_l2_64(v.double(), vr)
    norm_ref = p[:32 * 768].double().view(32, 768).norm(dim=1).mean().item()
    e_n = abs(norm.item() - norm_ref) / norm_ref
    print(f'adamw ends={ends} step={step}: |dp|/lr {e_p:.2e}, exp_avg {e_m:.2e}, exp_avg_sq {e_v:.2e}, norm {e_n:.2e}')
    assert e_p < 1e-3
    assert e_m < 1e-6 and e_v < 1e-6
    assert e_n < 1e-6


# ================================================================================================= clip_embed_bwd
def test_clip_embed_bwd(cuda):
    """d(token embedding row) = sum of the output gradient over the positions holding that token, over 2 x 16 layer
    prompts of 77 tokens with rows of pitch 800 (NaN in the pad columns, which must not be read).  Concept tokens repeat
    within and across sequences; a requested token that never occurs gets exactly 0.  fp32 sums in a fixed order against
    float64: measured worst rel-L2 3.3e-8 on an H100 80GB HBM3 (700 W)."""
    from mos_b200 import ops
    n_seq, T, C, ld = 2 * 16, 77, 768, 800
    M = n_seq * T
    ids = torch.full((n_seq, T), 49407, dtype=torch.int32)
    ids[:, 0] = 49406
    for s in range(n_seq):
        ids[s, 3] = 49408 + s % 16                   # one concept token per layer prompt, in both samples
        ids[s, 4 + s % 5] = 49424 + s % 16
        ids[s, 40] = 49408                            # a token that repeats in every sequence
        if s % 3 == 0:
            ids[s, 41] = 49408
    ids = ids.flatten().cuda()
    rows = torch.tensor([49408 + i for i in range(32)] + [49500], dtype=torch.int32, device=cuda)
    dx = torch.full((M, ld), float('nan'), device=cuda, dtype=torch.bfloat16)
    dx[:, :C] = mk((M, C), cuda, seed=5)
    nr = rows.numel()
    buf = canary(((nr + 2) * C,), cuda, torch.float32)
    out = buf[:nr * C].view(nr, C)
    ops.clip_embed_bwd(ids, dx, rows, out, C=C)
    first = out.clone()
    ops.clip_embed_bwd(ids, dx, rows, out, C=C)
    torch.cuda.synchronize()
    assert same_bits(out, first)
    assert untouched(buf, window_mask(buf, slice(0, nr * C)))
    want = torch.zeros(nr, C, dtype=F64, device=cuda)
    for r in range(nr):
        sel = ids == rows[r]
        want[r] = dx[sel, :C].double().sum(0)
    assert not bits(out[-1]).any()
    e = rel_l2_64(out.double(), want)
    base = torch.randn(nr, C, generator=torch.Generator().manual_seed(6)).cuda()
    out.copy_(base)
    ops.clip_embed_bwd(ids, dx, rows, out, C=C, accumulate=True)
    torch.cuda.synchronize()
    e_acc = rel_l2_64(out.double(), want + base.double())
    print(f'clip_embed_bwd: rel-L2 {e:.2e}, accumulate {e_acc:.2e}')
    assert e < 1e-6 and e_acc < 1e-6
    assert untouched(buf, window_mask(buf, slice(0, nr * C)))


# ================================================================================================= quick GELU
def _ulp_bf16(x):
    """one bf16 ulp at |x| (the normal-range spacing; x == 0 -> the smallest normal's)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def test_quick_gelu_fwd_bwd(cuda):
    """x sigmoid(1.702 x) and its derivative at C = 3072 on pitched rows, for x in +-30 with exact zeros and values
    where the sigmoid saturates, against float64 of the same bf16 inputs.  The bf16 result may be off by its rounding
    (half an ulp) plus the error of __expf: bound 1 ulp of the reference, and for the derivative, whose two terms cancel
    near x = -1.28, 1e-5 |dy| on top.  Measured worst on an H100 80GB HBM3 (700 W): fwd 0.50 ulp, bwd 0.50 ulp."""
    from mos_b200 import ops
    M, C = 154, 3072
    g = torch.Generator().manual_seed(0)
    x = torch.randn(M, C, generator=g) * 6
    x[:, :64] = torch.linspace(-30, 30, 64)
    x[::7, 64:128] = 0.0
    x[1::7, 64:96], x[1::7, 96:128] = 30.0, -30.0
    x[2::7, 64:128] = torch.linspace(-12, -8, 64)
    x = x.clamp(-30, 30).bfloat16().cuda()
    xs = torch.full((M, C + 64), float('nan'), device=cuda, dtype=torch.bfloat16)
    xs[:, :C] = x
    dy = mk((M, C), cuda, seed=1)
    dys = torch.full((M, C + 32), float('nan'), device=cuda, dtype=torch.bfloat16)
    dys[:, :C] = dy
    y = canary((M + 1, C + 128), cuda, torch.bfloat16)
    dx = canary((M + 1, C + 96), cuda, torch.bfloat16)
    ops.quick_gelu_fwd(xs, y, M=M, C=C)
    ops.quick_gelu_bwd(xs, dys, dx, M=M, C=C)
    torch.cuda.synchronize()
    assert untouched(y, window_mask(y, slice(0, M), slice(0, C)))
    assert untouched(dx, window_mask(dx, slice(0, M), slice(0, C)))
    xd = x.double()
    s = torch.sigmoid(1.702 * xd)
    y_ref = xd * s
    dx_ref = dy.double() * (s + 1.702 * xd * s * (1 - s))
    e_f = ((y[:M, :C].double() - y_ref).abs() / _ulp_bf16(y_ref)).max().item()
    e_b = (((dx[:M, :C].double() - dx_ref).abs() - 1e-5 * dy.double().abs()).clamp_min(0) / _ulp_bf16(dx_ref)).max().item()
    print(f'quick_gelu: fwd {e_f:.2f} ulp, bwd {e_b:.2f} ulp')
    assert (y[:M, :C][x == 0] == 0).all()
    assert e_f <= 1.0 and e_b <= 1.0


# ================================================================================================= masked MSE
def test_masked_mse_fractional_mask(cuda):
    """trainer_edlora.py:251-252 at the engine shape [2, 4, 64, 64] with a fractional mask (zeros included) and
    grad_scale 0.5, against float64.  Measured worst on an H100 80GB HBM3 (700 W): loss 6.2e-9 rel, gradient 4.7e-8
    rel-L2."""
    from mos_b200 import ops
    B, Cc, H = 2, 4, 64
    g = torch.Generator().manual_seed(0)
    pred, target = torch.randn(B, Cc, H, H, generator=g).cuda(), torch.randn(B, Cc, H, H, generator=g).cuda()
    mask = torch.rand(B, 1, H, H, generator=g)
    mask[mask < 0.2] = 0.0
    mask[1, :, :32] *= 0.25                       # the two samples' mask sums differ
    mask = mask.cuda()
    ws, loss, dp = torch.empty(2 * B, device=cuda), torch.empty(1, device=cuda), torch.empty_like(pred)
    ops.masked_mse(pred, target, mask, ws, loss, dp, grad_scale=0.5)
    torch.cuda.synchronize()
    p = pred.double().requires_grad_(True)
    m = mask.double()
    ref = (((p - target.double()) ** 2 * m).sum([1, 2, 3]) / m.sum([1, 2, 3])).mean()
    (ref * 0.5).backward()
    e_l = abs(loss.item() - ref.item()) / ref.item()
    e_g = rel_l2_64(dp.double(), p.grad)
    print(f'masked_mse: loss {e_l:.2e}, grad {e_g:.2e}')
    assert e_l < 1e-6 and e_g < 1e-6
