"""The GEMM epilogue paths that the engines rarely take, against a float64 reference.

Each output path of `gemm_kernel` is compiled separately, so each one needs a test of its own:
- 16-bit rows that TMA cannot address (row pitch not a multiple of 8 elements): the consumers copy them out;
- a residual that TMA cannot address, read from global memory, with TMA-store or copied-out output;
- fp32 output, with and without accumulation, with LoRA, and with more column tiles than SMs and a row count that is not
  a multiple of 8, so that a CTA runs a second tile after a tail tile whose last rows are outside the output.
Every case runs with fp16 and bf16 operands, and with and without the fused LoRA branch (two segments).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def operands(M, N, K, dtype, dev, lora, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    A = (torch.randn(M, K, generator=g)).to(dtype).to(dev)
    W = (torch.randn(N, K, generator=g) * K ** -0.5).to(dtype).to(dev)
    bias = (torch.randn(N, generator=g) * 0.5).to(dev)
    ref = A.double() @ W.double().t() + bias.double()
    kw = dict(bias=bias)
    if lora:
        nseg = 2
        seg = N // nseg
        down16 = torch.zeros(16, K, dtype=dtype)
        up = torch.randn(N, 4, generator=g) * 0.5
        for s in range(nseg):
            down16[4 * s:4 * s + 4] = (torch.randn(4, K, generator=g) * K ** -0.5).to(dtype)
        down16, up = down16.to(dev), up.to(dev)
        t = A.double() @ down16.double().t()                      # [M, 16]
        for s in range(nseg):
            ref[:, s * seg:(s + 1) * seg] += t[:, 4 * s:4 * s + 4] @ up[s * seg:(s + 1) * seg].double().t()
        kw.update(lora_down=down16, lora_up=up.contiguous(), lora_seg=seg)
    return A, W, ref, kw


def tol16(dtype):
    return 4e-3 if dtype == torch.bfloat16 else 1e-3


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('lora', [False, True])
def test_rows_copy_out(cuda, dtype, lora):
    from mos_b200 import ops
    M, N, K = 300, 320, 320
    A, W, ref, kw = operands(M, N, K, dtype, cuda, lora, seed=1)
    buf = torch.full((M, N + 4), float('nan'), device=cuda, dtype=dtype)     # pitch N + 4: TMA cannot address it
    ops.gemm(A, W, buf[:, :N], **kw)
    torch.cuda.synchronize()
    assert rel_l2(buf[:, :N], ref) < tol16(dtype)
    assert torch.isnan(buf[:, N:]).all()


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('lora', [False, True])
@pytest.mark.parametrize('out_tma', [True, False])
def test_residual_from_global(cuda, dtype, lora, out_tma):
    from mos_b200 import ops
    M, N, K = 300, 320, 320
    A, W, ref, kw = operands(M, N, K, dtype, cuda, lora, seed=2)
    rbuf = torch.randn(M, N + 4, generator=torch.Generator().manual_seed(3)).to(dtype).to(cuda)
    res = rbuf[:, :N]                                                       # pitch N + 4: read from global memory
    ref = ref + res.double()
    if out_tma:
        out = torch.full((M, N), float('nan'), device=cuda, dtype=dtype)
    else:
        out = torch.full((M, N + 4), float('nan'), device=cuda, dtype=dtype)[:, :N]
    ops.gemm(A, W, out, residual=res, **kw)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < tol16(dtype)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('lora', [False, True])
@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('M,N', [(91, 320), (91, 160 * 133)])
def test_f32_output(cuda, dtype, lora, accumulate, M, N):
    from mos_b200 import ops
    K = 128
    A, W, ref, kw = operands(M, N, K, dtype, cuda, lora, seed=4)
    if accumulate:
        out = torch.randn(M, N, generator=torch.Generator().manual_seed(5)).to(cuda)
        ref = ref + out.double()
    else:
        out = torch.full((M, N), float('nan'), device=cuda)
    ops.gemm(A, W, out, out_f32=True, accumulate=accumulate, **kw)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < 1e-5
