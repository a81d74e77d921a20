"""Schedule, operand-form and write-bound tests of the persistent wgmma GEMM / implicit-GEMM conv (csrc/gemm.cu).

The kernel runs min(work items, SM count) CTAs and each CTA loops over its items, so the parts that only run on a CTA's
second and later item (the smem ring carried across items, the producer fetching the next tile during the epilogue, the
per-item accumulator reset) are only exercised by launches with several items per CTA.  The tests here use at least
3 x SM-count items where the schedule is the subject.

Bitwise properties: the k order inside a 128 x 160 tile does not depend on the schedule, the pipeline depth or the operand
pitch, so those variations must give bit-identical outputs.  Tolerances against the fp32 PyTorch reference (TF32 off) are
those of test_gemm_gpu.py: rel-L2 <= 4e-3 for bf16 outputs (one bf16 rounding), 6e-4 for fp16, and 1e-5 for fp32 outputs
(no output rounding; only the summation order differs).
"""
import math

import pytest
import torch

from gpu_helpers import canary, mk, num_sms, rel_l2, rup, same_bits, untouched, window_mask

pytestmark = pytest.mark.gpu
BM, BN = 128, 160
TOL = {torch.bfloat16: 4e-3, torch.float16: 6e-4, torch.float32: 1e-5}


def _ref(A, W):
    return A.float() @ W.float().t()


def _lora(N, K, nseg, dev, dtype, seed=10):
    """rank-4 LoRA over `nseg` equal output segments, packed as the engines pack it: down [16, K] (segment s in rows
    4s..4s+3), up [N, 4] fp32 with alpha folded in.  Returns (down16, up, term(A) -> fp32 [M, N])."""
    seg = N // nseg
    downs = [mk((4, K), dev, K ** -0.5, seed + s, dtype) for s in range(nseg)]
    g = torch.Generator().manual_seed(seed + 100)
    up = (torch.randn(N, 4, generator=g) * 0.5).to(dev)
    down16 = torch.zeros(16, K, device=dev, dtype=dtype)
    for s in range(nseg):
        down16[4 * s:4 * s + 4] = downs[s]

    def term(A):
        return torch.cat([(A.float() @ downs[s].float().t()) @ up[s * seg:(s + 1) * seg].t() for s in range(nseg)], 1)
    return down16, up, term


def _geglu_perm(N, dev):
    """tile t of the packed weight holds [a columns 80t..80t+79 | gate columns 80t..80t+79] (engine.py)"""
    half = N // 2
    return torch.cat([torch.cat([torch.arange(80 * t, 80 * t + 80), half + torch.arange(80 * t, 80 * t + 80)])
                      for t in range(half // 80)]).to(dev)


def _conv_tiling(B, H, Wd):
    """(m tiles, batches per tile) of the conv schedule: the host's choice of the TW x TH x TB pixel patch"""
    TW = 1
    while TW * 2 <= 128 and Wd % (TW * 2) == 0:
        TW *= 2
    best, best_eff, TH = 1, -1.0, 1
    while TH * TW <= 128:
        TB = 128 // (TW * TH)
        if not (TB > 4 and TH * 2 * TW <= 128):
            eff = (H / (math.ceil(H / TH) * TH)) * (B / (math.ceil(B / TB) * TB))
            if eff > best_eff + 1e-9:
                best, best_eff = TH, eff
        TH *= 2
    TB = 128 // (TW * best)
    return (Wd // TW) * math.ceil(H / best) * math.ceil(B / TB), TB


# ------------------------------------------------------------------------------------------------ tile locality
PLAIN_MODES = ['plain', 'bias_batchbias_residual', 'geglu', 'geglu_lora', 'lora1', 'lora3', 'lora4', 'f32', 'f32_accumulate']


def _plain_case(mode, dev):
    """A row-major launch of >= 3 x SM-count items with an M tail.  Returns the operands, the fp32 reference and a
    launch(r0, r1, out) that runs rows [r0, r1) into out[r0:r1]."""
    K = 320
    geglu = mode.startswith('geglu')
    M, N = (32 * BM - 21, 2560) if geglu else (72 * BM - 37, {'lora3': 960}.get(mode, 1280))
    A, W = mk((M, K), dev, seed=1), mk((N, K), dev, K ** -0.5, seed=2)
    ref = _ref(A, W)
    kw, rows = {}, {}
    rpb = 64                        # batch boundaries at tile rows 0 and 64: every tile straddles one
    bb = None
    if mode in ('bias_batchbias_residual', 'geglu', 'geglu_lora'):
        bias = torch.randn(N, device=dev) * 0.1
        kw['bias'] = bias
        ref += bias
    if mode == 'bias_batchbias_residual':
        bb = torch.randn(math.ceil(M / rpb), N, device=dev) * 0.5
        res = mk((M, N), dev, seed=3)
        rows['residual'] = res
        ref += bb.repeat_interleave(rpb, 0)[:M] + res.float()
    if mode.startswith('lora') or mode == 'geglu_lora':
        nseg = int(mode[-1]) if mode.startswith('lora') else 1
        down16, up, term = _lora(N, K, nseg, dev, torch.bfloat16)
        ref += term(A)
        kw.update(lora_down=down16, lora_up=up, lora_seg=N // nseg)
    if geglu:
        perm = _geglu_perm(N, dev)
        kw['geglu'] = True
        W = W[perm].contiguous()
        if 'bias' in kw:
            kw['bias'] = kw['bias'][perm].contiguous()
        if 'lora_up' in kw:
            kw['lora_up'] = kw['lora_up'][perm].contiguous()
        ref = ref[:, :N // 2] * torch.nn.functional.gelu(ref[:, N // 2:])
    out_dtype = torch.float32 if mode.startswith('f32') else torch.bfloat16
    if out_dtype == torch.float32:
        kw['out_f32'] = True
    init = None
    if mode == 'f32_accumulate':
        kw['accumulate'] = True
        init = torch.randn(M, ref.shape[1], device=dev)
        ref += init

    def launch(r0, r1, out):
        extra = {k: v[r0:r1] for k, v in rows.items()}
        if bb is not None:
            extra.update(bias_batch=bb[r0 // rpb:], rows_per_batch=rpb)
        from mos_b200 import ops
        ops.gemm(A[r0:r1], W, out[r0:r1], **kw, **extra)
    n_items = math.ceil(M / BM) * (N // BN)
    return M, ref, out_dtype, init, launch, n_items


@pytest.mark.parametrize('mode', PLAIN_MODES)
def test_tile_locality_plain(cuda, mode):
    """Every tile of a launch with several items per CTA is bit-identical to the same tile computed by a launch of its
    row block alone; the large launch matches the fp32 reference, and nothing outside out[:M, :N] is written (rows >= M,
    the gap between N and ldc)."""
    M, ref, out_dtype, init, launch, n_items = _plain_case(mode, cuda)
    assert n_items >= 3 * num_sms()
    Nout = ref.shape[1]
    bufs = []
    for whole in (True, False):
        buf = canary((M + 3, Nout + 32), cuda, out_dtype)
        if init is not None:
            buf[:M, :Nout] = init
        out = buf[:M, :Nout]
        if whole:
            launch(0, M, out)
        else:
            for r0 in range(0, M, BM):
                launch(r0, min(M, r0 + BM), out)
        bufs.append(buf)
    torch.cuda.synchronize()
    big, small = bufs
    assert untouched(big, window_mask(big, slice(0, M), slice(0, Nout)))
    assert same_bits(big, small)
    e = rel_l2(big[:M, :Nout], ref)
    print(f'{mode}: rel-L2 {e:.2e}')
    assert e < TOL[out_dtype]


def _heads_case(dtype, T, nseg, dev):
    """QKV (3 segments) or KV (2 segments: K rows, V transposed) head-split projection with a 3-segment / 2-segment LoRA,
    8 heads of 40.  The segment buffers carry pads beyond T rows, beyond d columns and (V^T) beyond d rows."""
    from mos_b200._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED
    H, d = 8, 40
    C, dp, dvp = H * d, 64, 48
    B, K = (256, 768) if nseg == 2 else (48, 320)
    N, M = nseg * C, B * T
    A, W = mk((M, K), dev, seed=1, dtype=dtype), mk((N, K), dev, K ** -0.5, seed=2, dtype=dtype)
    down16, up, term = _lora(N, K, nseg, dev, dtype)
    ref = (_ref(A, W) + term(A)).view(B, T, nseg, H, d)
    kinds = [MOS_SEG_ROWS] * (nseg - 1) + [MOS_SEG_TRANSPOSED]
    pads = [T + 5] * (nseg - 1) + [rup(T, 8) + 8]

    def alloc():
        return [canary((B * H, r, dp), dev, dtype) if k == MOS_SEG_ROWS else canary((B * H, dvp, r), dev, dtype)
                for k, r in zip(kinds, pads)]

    def launch(b0, b1, segs):
        from mos_b200 import ops
        ops.gemm(A[b0 * T:b1 * T], W, None, lora_down=down16, lora_up=up, lora_seg=C,
                 heads=dict(seg_ptr=[s[b0 * H:b1 * H] for s in segs], seg_kind=kinds, seg_rows_pad=pads, heads=H,
                            head_dim=d, dpad=dp, dv_pad=dvp, tokens_per_batch=T))

    def check(segs):
        for s, (buf, kind) in enumerate(zip(segs, kinds)):
            r = ref[:, :, s]
            if kind == MOS_SEG_ROWS:
                got, want = buf[:, :T, :d], r.permute(0, 2, 1, 3).reshape(B * H, T, d)
                win = window_mask(buf, slice(None), slice(0, T), slice(0, d))
            else:
                got, want = buf[:, :d, :T], r.permute(0, 2, 3, 1).reshape(B * H, d, T)
                win = window_mask(buf, slice(None), slice(0, d), slice(0, T))
            e = rel_l2(got, want)
            print(f'heads {dtype} T={T} segment {s}: rel-L2 {e:.2e}')
            assert e < TOL[dtype]
            assert untouched(buf, win), f'segment {s}: write outside the head-split window'
    return B, M, N, alloc, launch, check


@pytest.mark.parametrize('dtype,T,nseg', [(torch.bfloat16, 77, 2), (torch.float16, 77, 2), (torch.bfloat16, 200, 3),
                                          (torch.float16, 200, 3)])
def test_tile_locality_heads(cuda, dtype, T, nseg):
    """Head-split epilogue with LoRA: the large launch is bit-identical to launches over subsets of whole batches whose
    first row starts a tile (77 tokens: 128 batches; 200 tokens: 16 batches), matches the reference and leaves every
    pad (beyond T, beyond d, V^T beyond d) untouched."""
    B, M, N, alloc, launch, check = _heads_case(dtype, T, nseg, cuda)
    assert math.ceil(M / BM) * (N // BN) >= 3 * num_sms()
    unit = math.lcm(T, BM) // T
    big, small = alloc(), alloc()
    launch(0, B, big)
    for b0 in range(0, B, unit):
        launch(b0, min(B, b0 + unit), small)
    torch.cuda.synchronize()
    for x, y in zip(big, small):
        assert same_bits(x, y)
    check(big)


def test_tile_locality_conv(cuda):
    """Implicit-GEMM conv with a batch tail and a height tail (9 rows in 2-row patches, 7 batches in 4-batch patches):
    bit-identical to launches over whole-batch subsets aligned to the batch patch, and matches F.conv2d."""
    from mos_b200 import ops
    B, H, Wd, C, N = 7, 9, 16, 128, 6400
    m_tiles, TB = _conv_tiling(B, H, Wd)
    assert TB > 1 and B % TB != 0 and H % 2 != 0
    assert m_tiles * (N // BN) >= 3 * num_sms()
    x = mk((B, H, Wd, C), cuda, seed=1)
    w = mk((N, C, 3, 3), cuda, (9 * C) ** -0.5, seed=2)
    bias = torch.randn(N, device=cuda) * 0.1
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    M, HW = B * H * Wd, H * Wd
    big, small = canary((M + 3, N + 32), cuda, torch.bfloat16), canary((M + 3, N + 32), cuda, torch.bfloat16)
    ops.gemm(x, wp, big[:M, :N], bias=bias, conv=(B, H, Wd, C))
    for b0 in range(0, B, TB):
        b1 = min(B, b0 + TB)
        ops.gemm(x[b0:b1], wp, small[b0 * HW:b1 * HW, :N], bias=bias, conv=(b1 - b0, H, Wd, C))
    torch.cuda.synchronize()
    assert untouched(big, window_mask(big, slice(0, M), slice(0, N)))
    assert same_bits(big, small)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    assert rel_l2(big[:M, :N], ref.permute(0, 2, 3, 1).reshape(M, N)) < 4e-3


# ------------------------------------------------------------------------------------------------ pipeline depth
@pytest.mark.parametrize('kb', [1, 2, 5, 7, 20, 45])
@pytest.mark.parametrize('lora', [False, True])
def test_stages_sweep(cuda, kb, lora):
    """Pipeline depths 2..5, an over-large request (clamped to what fits in shared memory) and the default, on a launch
    of ~2 items per CTA: the smem ring wraps inside a tile and across items.  All depths are bit-identical."""
    from mos_b200 import ops
    M, N, K = 32 * BM - 40, 1280, 64 * kb
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    ref = _ref(A, W)
    kw = {}
    if lora:
        down16, up, term = _lora(N, K, 4, cuda, torch.bfloat16)
        ref += term(A)
        kw = dict(lora_down=down16, lora_up=up, lora_seg=N // 4)
    outs = {}
    for st in (2, 3, 4, 5, 8, 0):
        out = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
        ops.gemm(A, W, out, stages=st, **kw)
        outs[st] = out
    torch.cuda.synchronize()
    for st, out in outs.items():
        assert same_bits(out, outs[0]), f'stages={st} differs from the default depth'
    assert rel_l2(outs[0], ref) < 4e-3


# ------------------------------------------------------------------------------------------------ operand forms
@pytest.mark.parametrize('mult,col', [(2, 0), (2, 1), (3, 1), (3, 2)])
def test_lda_column_slice(cuda, mult, col):
    """A read as a column slice of a [M, mult*C] buffer (dK / dV out of dkv, dQ / dK / dV out of dqkv), written into the
    middle column slice of a wider output: bit-identical to the contiguous operand, neighbours untouched."""
    from mos_b200 import ops
    M, C, N = 1000, 320, 640
    A_all = mk((M, mult * C), cuda, seed=1)
    A = A_all[:, col * C:(col + 1) * C]
    W = mk((N, C), cuda, C ** -0.5, seed=2)
    buf = canary((M + 2, 3 * N), cuda, torch.bfloat16)
    ops.gemm(A, W, buf[:M, N:2 * N], lda=mult * C)
    want = torch.empty(M, N, device=cuda, dtype=torch.bfloat16)
    ops.gemm(A.contiguous(), W, want)
    torch.cuda.synchronize()
    assert untouched(buf, window_mask(buf, slice(0, M), slice(N, 2 * N)))
    assert same_bits(buf[:M, N:2 * N], want)
    assert rel_l2(want, _ref(A, W)) < 4e-3


@pytest.mark.parametrize('splits', [1, 3])
def test_conv_pixel_pitch(cuda, splits):
    """Conv input with a pixel pitch of 2C (the second half of a channel-concat buffer), single pass and two-launch
    split-K: bit-identical to the contiguous input."""
    from mos_b200 import ops
    B, H, Wd, C, N = 2, 16, 16, 320, 640
    x_all = mk((B, H, Wd, 2 * C), cuda, seed=1)
    x = x_all[..., C:]
    w = mk((N, C, 3, 3), cuda, (9 * C) ** -0.5, seed=2)
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    bias = torch.randn(N, device=cuda) * 0.1
    M = B * H * Wd

    def run(inp, lda):
        out = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
        if splits == 1:
            ops.gemm(inp, wp, out, bias=bias, conv=(B, H, Wd, C), lda=lda)
        else:
            partial = torch.full((splits, M, N), float('nan'), device=cuda)
            ops.gemm(inp, wp, None, conv=(B, H, Wd, C), lda=lda, splits=splits, partial=partial)
            ops.splitk_finalize(partial, splits, M, N, out, bias=bias)
        return out
    got, want = run(x, 2 * C), run(x.contiguous(), None)
    torch.cuda.synchronize()
    assert same_bits(got, want)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1)
    assert rel_l2(got, ref.permute(0, 2, 3, 1).reshape(M, N)) < 4e-3


@pytest.mark.parametrize('path', ['single', 'splitk_two_launch', 'splitk_in_kernel'])
def test_residual_is_out(cuda, path):
    """out += A W^T + bias with `residual` being the output buffer itself (the engines accumulate dX over the q / k / v
    projections this way): bit-identical to a separate residual buffer, and correct."""
    from mos_b200 import ops
    M, N, K, S = 1000, 640, 1280, 4
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    R = mk((M, N), cuda, seed=3)
    bias = torch.randn(N, device=cuda) * 0.1

    def run(out, res):
        if path == 'single':
            ops.gemm(A, W, out, bias=bias, residual=res)
            return
        partial = torch.full((S, M, N), float('nan'), device=cuda)
        if path == 'splitk_two_launch':
            ops.gemm(A, W, None, splits=S, partial=partial, M=M)
            ops.splitk_finalize(partial, S, M, N, out, bias=bias, residual=res)
        else:
            counters = torch.zeros(math.ceil(M / BM) * (N // BN), device=cuda, dtype=torch.int32)
            ops.gemm(A, W, out, splits=S, partial=partial, bias=bias, residual=res, counters=counters)
    buf = canary((M + 2, N + 32), cuda, torch.bfloat16)
    out = buf[:M, :N]
    out.copy_(R)
    run(out, out)
    sep = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
    run(sep, R)
    torch.cuda.synchronize()
    assert untouched(buf, window_mask(buf, slice(0, M), slice(0, N)))
    assert same_bits(out, sep)
    assert rel_l2(out, _ref(A, W) + bias + R.float()) < 4e-3


@pytest.mark.parametrize('rpb', [77, 100, 200, 1000])
def test_rows_per_batch_pitched_bias(cuda, rpb):
    """Per-batch bias with batch boundaries inside tiles, read from a pitched table (bias_batch_ld > N), on the
    single-pass epilogue and the in-kernel split-K reduction."""
    from mos_b200 import ops
    M, N, K, S = 1997, 640, 640, 2
    nb = math.ceil(M / rpb)
    A, W = mk((M, K), cuda, seed=1), mk((N, K), cuda, K ** -0.5, seed=2)
    bias = torch.randn(N, device=cuda) * 0.1
    table = torch.randn(nb, N + 24, device=cuda)
    ref = _ref(A, W) + bias + table[:, :N].repeat_interleave(rpb, 0)[:M]
    kw = dict(bias=bias, bias_batch=table, rows_per_batch=rpb, bias_batch_ld=N + 24)
    out = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.gemm(A, W, out, **kw)
    out_sk = torch.full((M, N), float('nan'), device=cuda, dtype=torch.bfloat16)
    partial = torch.empty((S, M, N), device=cuda)
    counters = torch.zeros(math.ceil(M / BM) * (N // BN), device=cuda, dtype=torch.int32)
    ops.gemm(A, W, out_sk, splits=S, partial=partial, counters=counters, **kw)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < 4e-3
    assert rel_l2(out_sk, ref) < 4e-3


@pytest.mark.parametrize('rpb', [1, 16, 31])
def test_rows_per_batch_below_32_rejected(cuda, rpb):
    from mos_b200 import ops
    A, W = mk((256, 64), cuda, seed=1), mk((160, 64), cuda, seed=2)
    out = torch.empty((256, 160), device=cuda, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.gemm(A, W, out, bias_batch=torch.zeros(256, 160, device=cuda), rows_per_batch=rpb)
