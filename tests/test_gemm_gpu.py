"""K1/K4 parity: wgmma GEMM / implicit-GEMM conv vs a plain PyTorch fp32 reference of the same op.

Tolerance: inputs are bf16-exact in both paths, accumulation is fp32 in both, so the only differences are
summation order and the final bf16 rounding of the output: rel-L2 <= 4e-3 (bf16 eps = 3.9e-3), typically ~2e-3.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def mk(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(torch.bfloat16)


@pytest.mark.parametrize('M,N,K', [(128, 160, 64), (256, 320, 320), (8192, 320, 320), (154, 640, 768),
                                   (1000, 1280, 1280), (128, 160, 2880)])
def test_gemm_plain(cuda, M, N, K):
    from mos_b200 import ops
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    out = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, out)
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t()
    assert rel_l2(out, ref) < 4e-3


def test_gemm_bias_residual_batchbias(cuda):
    from mos_b200 import ops
    M, N, K = 2 * 1024, 640, 640
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    bias = torch.randn(N, device=cuda)
    bb = torch.randn(2, N, device=cuda)
    res = mk((M, N), cuda, seed=3)
    out = torch.empty((M, N), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, out, bias=bias, bias_batch=bb, rows_per_batch=1024, residual=res)
    ref = A.float() @ W.float().t() + bias + bb.repeat_interleave(1024, 0) + res.float()
    assert rel_l2(out, ref) < 4e-3


def test_gemm_strided_out(cuda):
    """ldc > N: producer writes straight into a channel-concat buffer."""
    from mos_b200 import ops
    M, N, K = 512, 320, 320
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    buf = torch.zeros((M, 960), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, buf[:, 320:640])
    ref = A.float() @ W.float().t()
    assert rel_l2(buf[:, 320:640], ref) < 4e-3
    assert buf[:, :320].abs().max().item() == 0 and buf[:, 640:].abs().max().item() == 0


@pytest.mark.parametrize('M,N,K,nseg', [(4096, 320, 320, 1), (154, 640, 768, 1), (300, 960, 320, 3)])
def test_gemm_lora(cuda, M, N, K, nseg):
    """y = x W^T + alpha * up(down(x))   (mixofshow/models/edlora.py:244-246), rank 4, up to 3 fused segments."""
    from mos_b200 import ops
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    alpha = 0.7
    seg = N // nseg
    downs = [mk((4, K), cuda, K ** -0.5, seed=10 + s) for s in range(nseg)]
    ups = [torch.randn(seg, 4, device=cuda) * 0.5 for s in range(nseg)]
    down16 = torch.zeros(16, K, device=cuda, dtype=torch.bfloat16)
    for s in range(nseg):
        down16[4 * s:4 * s + 4] = downs[s]
    up_all = (torch.cat(ups, 0) * alpha).contiguous()
    out = torch.empty((M, N), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, out, lora_down=down16, lora_up=up_all, lora_seg=seg)
    ref = A.float() @ W.float().t()
    for s in range(nseg):
        ref[:, s * seg:(s + 1) * seg] += alpha * (A.float() @ downs[s].float().t()) @ ups[s].t()
    assert rel_l2(out, ref) < 4e-3


def test_gemm_geglu(cuda):
    from mos_b200 import ops
    M, C = 1024, 320
    N = 8 * C
    A, W = mk((M, C), cuda, seed=1), mk((N, C), cuda, C ** -0.5, seed=2)
    bias = torch.randn(N, device=cuda) * 0.1
    # pack: tile t holds [a cols 80t..80t+79 | gate cols 80t..80t+79]
    half = N // 2
    idx = torch.cat([torch.cat([torch.arange(80 * t, 80 * t + 80), half + torch.arange(80 * t, 80 * t + 80)])
                     for t in range(half // 80)]).to(cuda)
    Wp, bp = W[idx].contiguous(), bias[idx].contiguous()
    out = torch.empty((M, half), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, Wp, out, bias=bp, geglu=True)
    h = A.float() @ W.float().t() + bias
    ref = h[:, :half] * torch.nn.functional.gelu(h[:, half:])
    assert rel_l2(out, ref) < 4e-3


@pytest.mark.parametrize('d,heads', [(40, 8), (80, 8), (160, 8)])
def test_gemm_heads(cuda, d, heads):
    from mos_b200 import ops
    from mos_b200._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED
    Bn, T = 2, 200
    C = d * heads
    M = Bn * T
    A, W = mk((M, C), cuda, seed=1), mk((3 * C, C), cuda, C ** -0.5, seed=2)
    Tp = 256
    dpad = ((d + 63) // 64) * 64
    dv = ((d + 15) // 16) * 16
    Q = torch.zeros(Bn, heads, Tp, dpad, device=cuda, dtype=torch.bfloat16)
    Kt = torch.zeros_like(Q)
    Vt = torch.zeros(Bn, heads, dv, Tp, device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, heads=dict(seg_ptr=[Q, Kt, Vt], seg_kind=[MOS_SEG_ROWS, MOS_SEG_ROWS, MOS_SEG_TRANSPOSED],
                              seg_rows_pad=[Tp, Tp, Tp], heads=heads, head_dim=d, dpad=dpad, dv_pad=dv,
                              tokens_per_batch=T))
    ref = (A.float() @ W.float().t()).view(Bn, T, 3, heads, d)
    q_ref = ref[:, :, 0].permute(0, 2, 1, 3)
    k_ref = ref[:, :, 1].permute(0, 2, 1, 3)
    v_ref = ref[:, :, 2].permute(0, 2, 3, 1)
    assert rel_l2(Q[:, :, :T, :d], q_ref) < 4e-3
    assert rel_l2(Kt[:, :, :T, :d], k_ref) < 4e-3
    assert rel_l2(Vt[:, :, :d, :T], v_ref) < 4e-3
    assert Q[:, :, T:].abs().max().item() == 0 and Q[..., d:].abs().max().item() == 0
    assert Vt[..., T:].abs().max().item() == 0
    if dv > d:
        assert Vt[:, :, d:].abs().max().item() == 0


@pytest.mark.parametrize('B,H,Wd,Cin,Cout', [(2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 8, 8, 1280, 1280),
                                              (1, 16, 16, 1920, 640), (2, 12, 24, 320, 320), (3, 4, 8, 64, 160)])
def test_conv3x3(cuda, B, H, Wd, Cin, Cout):
    from mos_b200 import ops
    x = mk((B, H, Wd, Cin), cuda, seed=1)
    w = mk((Cout, Cin, 3, 3), cuda, (9 * Cin) ** -0.5, seed=2)
    bias = torch.randn(Cout, device=cuda) * 0.1
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    out = torch.empty((B * H * Wd, Cout), device=cuda, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, bias=bias, conv=(B, H, Wd, Cin))
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * Wd, Cout)
    assert rel_l2(out, ref) < 4e-3


@pytest.mark.parametrize('splits', [2, 5, 9])
def test_conv3x3_splitk(cuda, splits):
    from mos_b200 import ops
    B, H, Wd, Cin, Cout = 2, 8, 8, 1280, 1280
    x = mk((B, H, Wd, Cin), cuda, seed=1)
    w = mk((Cout, Cin, 3, 3), cuda, (9 * Cin) ** -0.5, seed=2)
    bias = torch.randn(Cout, device=cuda) * 0.1
    res = mk((B * H * Wd, Cout), cuda, seed=3)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous()
    M = B * H * Wd
    partial = torch.empty((splits, M, Cout), device=cuda, dtype=torch.float32)
    out = torch.empty((M, Cout), device=cuda, dtype=torch.bfloat16)
    ops.gemm(x, wp, None, conv=(B, H, Wd, Cin), splits=splits, partial=partial)
    ops.splitk_finalize(partial, splits, M, Cout, out, bias=bias, residual=res)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(M, Cout) + res.float()
    assert rel_l2(out, ref) < 4e-3


@pytest.mark.parametrize('case', [dict(conv=(2, 8, 8, 1280), N=1280, splits=15), dict(conv=(2, 16, 16, 1280), N=1280, splits=4),
                                  dict(conv=(2, 12, 24, 320), N=320, splits=3), dict(M=512, K=2560, N=1280, splits=4),
                                  dict(M=200, K=1280, N=640, splits=5), dict(conv=(2, 32, 32, 640), N=640, splits=2),
                                  dict(conv=(2, 32, 32, 640), N=640, splits=4)])    # last: 256 work items > 132 CTAs
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_splitk_in_kernel_finalize(cuda, case, dtype):
    """mos_gemm_args.tile_counters: the `splits` CTAs of every output tile reduce the partials themselves.  Same summation
    order as mos_splitk_finalize, so the result must be BIT-identical to the two-launch path; three back-to-back launches
    check that the counters return to zero (CUDA-graph replay relies on it)."""
    from mos_b200 import ops
    conv, N, S = case.get('conv'), case['N'], case['splits']
    if conv is not None:
        B, H, Wd, C = conv
        M, K = B * H * Wd, 9 * C
        x = mk((B, H, Wd, C), cuda, seed=1).to(dtype)
        rows_per_batch = H * Wd
    else:
        M, K = case['M'], case['K']
        x = mk((M, K), cuda, seed=1).to(dtype)
        B, rows_per_batch = 2, M // 2
    w = mk((N, K), cuda, K ** -0.5, seed=2).to(dtype)
    bias = torch.randn(N, device=cuda) * 0.1
    bias_batch = torch.randn(B, N + 40, device=cuda) * 0.1           # pitched like the engine's time-embedding table
    res = mk((M, N + 8), cuda, seed=3).to(dtype)[:, :N]              # pitched residual
    partial = torch.empty((S, M, N), device=cuda, dtype=torch.float32)
    ref = torch.empty((M, N), device=cuda, dtype=dtype)
    kw = dict(conv=conv, M=M)
    ops.gemm(x, w, None, splits=S, partial=partial, **kw)
    ops.splitk_finalize(partial, S, M, N, ref, bias=bias, bias_batch=bias_batch, rows_per_batch=rows_per_batch, residual=res,
                        bias_batch_ld=N + 40)
    counters = torch.zeros(256, device=cuda, dtype=torch.int32)
    for rep in range(3):
        out = torch.full((M, N), float('nan'), device=cuda, dtype=dtype)
        partial.fill_(float('nan'))
        ops.gemm(x, w, out, splits=S, partial=partial, bias=bias, bias_batch=bias_batch, rows_per_batch=rows_per_batch,
                 bias_batch_ld=N + 40, residual=res, counters=counters, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), f'launch {rep}'
        assert int(counters.abs().sum()) == 0, f'counters not reset after launch {rep}'


def test_gemm_bad_args(cuda):
    """Error behaviour mirrors the reference's fail-fast asserts: ValueError, not a crash."""
    from mos_b200 import ops
    A, W = mk((128, 64), cuda), mk((100, 64), cuda)
    out = torch.empty((128, 100), device=cuda, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.gemm(A, W, out)


# ---------------------------------------------------------------------------------------------- fp16 operands
# Sampling runs the GEMMs on fp16 operands (weights AND activations, mos_b200/engine.py).  wgmma takes ONE operand
# type for A and B, so the C ABI rejects mixed operand types up front.  Tolerance: operands are exact in both paths, fp32 accumulation, final fp16
# rounding (eps 4.9e-4): rel-L2 <= 6e-4.
def test_gemm_f16(cuda):
    from mos_b200 import ops
    M, N, K = 2 * 1024, 640, 640
    g = torch.Generator().manual_seed(5)
    A = torch.randn(M, K, generator=g).to(cuda).half()
    W = (torch.randn(N, K, generator=g) * K ** -0.5).to(cuda).half()
    bias = torch.randn(N, device=cuda)
    res = torch.randn(M, N, generator=g).to(cuda).half()
    down16 = torch.zeros(16, K, device=cuda, dtype=torch.float16)
    down16[:4] = (torch.randn(4, K, generator=g) * K ** -0.5).to(cuda).half()
    up = (torch.randn(N, 4, device=cuda) * 0.5).contiguous()
    out = torch.empty((M, N), device=cuda, dtype=torch.float16)
    ops.gemm(A, W, out, bias=bias, residual=res, lora_down=down16, lora_up=up, lora_seg=N)
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t() + bias + res.float() + (A.float() @ down16[:4].float().t()) @ up.t()
    e = rel_l2(out, ref)
    print(f'fp16 gemm rel-L2 {e:.2e}')
    assert e < 6e-4
    # mixed 16-bit types in one call are a caller bug: refused before any launch
    with pytest.raises(TypeError):
        ops.gemm(A, W, out.to(torch.bfloat16))
    with pytest.raises(ValueError):
        ops.gemm(A, W.to(torch.bfloat16), out)


def test_conv3x3_and_splitk_f16(cuda):
    from mos_b200 import ops
    B, H, Wd, C, N = 2, 16, 16, 1280, 1280
    g = torch.Generator().manual_seed(6)
    x = torch.randn(B, H, Wd, C, generator=g).to(cuda).half()
    w = (torch.randn(N, C, 3, 3, generator=g) * (9 * C) ** -0.5).to(cuda).half()
    Wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    bias = torch.randn(N, device=cuda)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    out = torch.empty(B * H * Wd, N, device=cuda, dtype=torch.float16)
    ops.gemm(x, Wp, out, bias=bias, conv=(B, H, Wd, C))
    assert rel_l2(out, ref.reshape(-1, N)) < 6e-4
    partial = torch.empty(4 * B * H * Wd * N, device=cuda)
    ops.gemm(x, Wp, None, conv=(B, H, Wd, C), splits=4, partial=partial)
    out2 = torch.empty_like(out)
    ops.splitk_finalize(partial, 4, B * H * Wd, N, out2, bias=bias)
    assert rel_l2(out2, ref.reshape(-1, N)) < 6e-4
