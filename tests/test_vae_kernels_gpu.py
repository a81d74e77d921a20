"""The VAE glue kernels (csrc/elementwise.cu) against fp32 / fp64 PyTorch statements of the same operation, at the shapes and
pitches `mos_b200/vae_engine.py` passes for 512 x 512 images.

- softmax_rows: the mid-block attention's row softmax, 4096 keys at 512^2 with a logit pitch rounded up to 160 (4160).
- vae_moments: quant_conv + mean / logvar (clamped to [-30, 20]) + the scaled latent sample.
- conv1x1_nchw: the decoder's post_quant_conv.
- im2col_s2(pad=0): the encoder's Downsample2D (pad right / bottom by one, 3x3 stride 2).
- upsample2x: the decoder's Upsample2D input, read with the engine's pixel pitch.

Bounds: 16-bit outputs carry one rounding (rel-L2 < 6e-4 for fp16, 4e-3 for bf16); fp32 outputs only see summation-order
and fast-exp differences (1e-5 relative or tighter, as stated); copies are exact.
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_helpers import canary, rel_l2, rup, untouched, window_mask

pytestmark = pytest.mark.gpu
BF, H16 = torch.bfloat16, torch.float16
TOL = {BF: 4e-3, H16: 6e-4}


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


@pytest.mark.parametrize('dtype', [H16, BF], ids=['fp16', 'bf16'])
@pytest.mark.parametrize('amp', [1.0, 16.0, 60.0])
@pytest.mark.parametrize('n,lds', [(4096, 4160), (1024, 1120)])
def test_softmax_rows(cuda, n, lds, amp, dtype):
    """rows = cols = n over fp32 logits with pitch lds (NaN in the pitch columns); scaled logits reach +-amp.  The output
    goes into a canary buffer with a wider pitch and spare rows."""
    from mos_b200 import ops
    scale = 512 ** -0.5
    g = _gen(cuda, 1)
    S = torch.full((n, lds), float('nan'), device=cuda)
    ramp = torch.linspace(0.1, 1.0, n, device=cuda)                       # rows of growing spread
    S[:, :n] = torch.randn(n, n, generator=g, device=cuda) * ramp[:, None] * (amp / 3 / scale)
    ldo = n + 64
    out = canary((n + 2, ldo), cuda, dtype)
    ops.softmax_rows(S, out, rows=n, cols=n, scale=scale)
    torch.cuda.synchronize()
    P = out[:n, :n]
    ref = torch.softmax(S[:, :n].double() * scale, -1)
    assert untouched(out, window_mask(out, slice(0, n), slice(0, n)))
    assert torch.isfinite(P).all()
    e = rel_l2(P, ref)
    rows = (P.double().sum(-1) - 1).abs().max().item()
    print(f'softmax_rows {n}x{n} lds={lds} amp={amp} {dtype}: rel-L2 {e:.2e}, max |row sum - 1| {rows:.2e}')
    assert e < TOL[dtype]
    assert rows < (1e-3 if dtype == H16 else 8e-3)


@pytest.mark.parametrize('with_noise', [False, True], ids=['moments', 'sample'])
def test_vae_moments(cuda, with_noise):
    """h: fp16 [B*HW, 160] with the 2L = 8 moment channels first (NaN beyond); quant_conv is a 1x1 8 -> 8 conv.  The logvar
    channels are built to cross both clamp bounds: clamped entries must be exactly -30 / 20."""
    from mos_b200 import ops
    B, HW, L, ldh, scaling = 2, 4096, 4, 160, 0.18215
    g = _gen(cuda, 2)
    h = torch.full((B * HW, ldh), float('nan'), device=cuda, dtype=H16)
    amp = torch.tensor([1.0] * L + [25.0] * L, device=cuda)
    h[:, :2 * L] = (torch.randn(B * HW, 2 * L, generator=g, device=cuda) * amp).to(H16)
    w = torch.eye(2 * L, device=cuda) + torch.randn(2 * L, 2 * L, generator=g, device=cuda) * 0.05
    bias = torch.cat([torch.randn(L, generator=g, device=cuda), torch.full((L,), -5.0, device=cuda)])
    mean, logvar = torch.empty(B, L, HW, device=cuda), torch.empty(B, L, HW, device=cuda)
    noise = torch.randn(B, L, HW, generator=g, device=cuda) if with_noise else None
    lat = torch.empty(B, L, HW, device=cuda) if with_noise else None
    ops.vae_moments(h, w, bias, mean, logvar, B=B, HW=HW, L=L, noise=noise, scaling=scaling, latents=lat)
    torch.cuda.synchronize()
    mo = (h[:, :2 * L].double() @ w.double().t() + bias.double()).view(B, HW, 2 * L).permute(0, 2, 1)   # [B, 2L, HW]
    mean_ref, lv_raw = mo[:, :L], mo[:, L:]
    hi, lo = lv_raw > 20 + 1e-3, lv_raw < -30 - 1e-3
    assert hi.sum().item() > 100 and lo.sum().item() > 100                 # both bounds are exercised
    assert (logvar[hi] == 20.0).all() and (logvar[lo] == -30.0).all()
    lv_ref = lv_raw.clamp(-30, 20)
    mid = ~(hi | lo)
    assert torch.allclose(logvar.double()[mid], lv_ref[mid], rtol=1e-5, atol=5e-5)       # 8 fp32 products of up to ~30
    assert torch.allclose(mean.double(), mean_ref, rtol=1e-5, atol=5e-5)
    if with_noise:
        # from the kernel's own mean / logvar: what is left is the fast __expf and the fp32 rounding
        term = torch.exp(0.5 * logvar.double()) * noise.double()
        ref = scaling * (mean.double() + term)
        err = (lat.double() - ref).abs()
        assert (err <= 1e-5 * scaling * (mean.double().abs() + term.abs()) + 1e-12).all(), err.max().item()


@pytest.mark.parametrize('cin,cout', [(4, 4), (8, 8)])
def test_conv1x1_nchw(cuda, cin, cout):
    from mos_b200 import ops
    B, H, W = 2, 64, 48
    g = _gen(cuda, 3)
    x = torch.randn(B, cin, H, W, generator=g, device=cuda)
    w = torch.randn(cout, cin, generator=g, device=cuda)
    bias = torch.randn(cout, generator=g, device=cuda)
    buf = canary((B * cout * H * W + 64,), cuda, torch.float32)
    y = buf[:B * cout * H * W].view(B, cout, H, W)
    ops.conv1x1_nchw(x, w, bias, y)
    torch.cuda.synchronize()
    ref = F.conv2d(x.double(), w.double().view(cout, cin, 1, 1), bias.double())
    assert untouched(buf, window_mask(buf, slice(0, B * cout * H * W)))
    assert rel_l2(y, ref) < 1e-6


@pytest.mark.parametrize('B,H,W,C,ldx', [(2, 16, 24, 128, 160), (1, 32, 8, 256, 320), (2, 8, 8, 512, 512)])
def test_im2col_s2_pad0(cuda, B, H, W, C, ldx):
    """The VAE's asymmetric Downsample2D: F.pad(x, (0, 1, 0, 1)) then a 3x3 / stride-2 conv.  The columns are an exact copy
    of F.unfold in tap-major order, and the GEMM over them matches F.conv2d."""
    from mos_b200 import ops
    g = _gen(cuda, 4)
    xb = torch.full((B, H, W, ldx), float('nan'), device=cuda, dtype=H16)
    xb[..., :C] = torch.randn(B, H, W, C, generator=g, device=cuda).to(H16)
    x = xb[..., :C]
    Ho, Wo = H // 2, W // 2
    col = canary((B * Ho * Wo + 2, 9 * C), cuda, H16)
    ops.im2col_s2(xb, col, B=B, H=H, W=W, C=C, ldx=ldx, pad=0)
    torch.cuda.synchronize()
    xp = F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    un = F.unfold(xp, 3, stride=2)                                        # [B, C*9, L], rows ordered (c, kh, kw)
    un = un.view(B, C, 9, -1).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C)
    assert untouched(col, window_mask(col, slice(0, B * Ho * Wo)))
    assert torch.equal(col[:B * Ho * Wo].float(), un)
    # the engine's packing: output channels padded to the GEMM's 160-column tile with zero weight rows and bias
    wt = torch.randn(C, C, 3, 3, generator=g, device=cuda) * (9 * C) ** -0.5
    bias = torch.randn(C, generator=g, device=cuda)
    Np = rup(C, 160)
    Wp = torch.zeros(Np, 9 * C, device=cuda, dtype=H16)
    Wp[:C] = wt.permute(0, 2, 3, 1).reshape(C, 9 * C).to(H16)
    bp = torch.zeros(Np, device=cuda)
    bp[:C] = bias
    out = torch.empty(B * Ho * Wo, Np, device=cuda, dtype=H16)
    ops.gemm(col[:B * Ho * Wo], Wp, out, bias=bp)
    torch.cuda.synchronize()
    ref = F.conv2d(xp.double(), wt.to(H16).double(), bias.double(), stride=2).permute(0, 2, 3, 1).reshape(-1, C)
    assert rel_l2(out[:, :C], ref) < TOL[H16]
    assert not out[:, C:].any()


@pytest.mark.parametrize('B,H,W,C,ldx', [(2, 16, 12, 128, 160), (1, 8, 8, 512, 640)])
def test_upsample2x_pitched(cuda, B, H, W, C, ldx):
    """Nearest 2x upsampling reading x with the engine's pixel pitch ldx > C (NaN pad columns) into [B, 2H, 2W, C]."""
    from mos_b200 import ops
    g = _gen(cuda, 5)
    xb = torch.full((B, H, W, ldx), float('nan'), device=cuda, dtype=H16)
    xb[..., :C] = torch.randn(B, H, W, C, generator=g, device=cuda).to(H16)
    n = B * 4 * H * W
    buf = canary((n + 3, C), cuda, H16)
    ops.upsample2x(xb, buf, B=B, H=H, W=W, C=C, ldx=ldx)
    torch.cuda.synchronize()
    ref = F.interpolate(xb[..., :C].float().permute(0, 3, 1, 2), scale_factor=2.0, mode='nearest').permute(0, 2, 3, 1)
    assert untouched(buf, window_mask(buf, slice(0, n)))
    assert torch.equal(buf[:n].view(B, 2 * H, 2 * W, C).float(), ref)
