"""The GEMM launch audit (tests/gemm_audit.py) on the CPU: its float64 reference against independent statements of the same
operation at the edges where the kernel's tiling goes wrong, and its checker against corrupted outputs.

Launches are built by the real `ops.gemm` / `ops.splitk_finalize` with CPU tensors and a stand-in library that keeps the
`mos_gemm_args` struct, so the records come from the ABI exactly as on the GPU.  The stand-in "kernel" is the rounded
reference (`gemm_audit.simulate`); every mutation case corrupts it the way a broken epilogue would, and the checker must
flag it while passing the uncorrupted output.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_audit as ga

F16, BF16 = torch.float16, torch.bfloat16


@pytest.fixture
def launch(monkeypatch):
    """launch(fn, *args, **kw): run ops.gemm / ops.splitk_finalize against a stand-in library; -> the simulated record"""
    from mos_b200 import _lib, ops
    calls = []

    class Lib:
        def mos_gemm_bf16(self, argref, stream):
            calls.append(('gemm', ga.abi_of(argref._obj)))
            return 0

        def mos_splitk_finalize(self, *args):
            calls.append(('finalize', [0 if getattr(v, 'value', v) is None else int(getattr(v, 'value', v))
                                       for v in args[:13]]))
            return 0

    monkeypatch.setattr(_lib, 'lib', lambda: Lib())
    monkeypatch.setattr(ops, 'current_stream', lambda: None)

    def run(name, *args, **kw):
        getattr(ops, name)(*args, **kw)
        op, vals = calls[-1]
        S = ga._Storages(ga._tensors(args, kw))
        rec = ga.gemm_record(vals, S) if op == 'gemm' else ga.finalize_record(vals, S)
        flats = ga.attach_mem(rec, S)
        ga.simulate(rec)
        for k, f in flats.items():                       # the stand-in kernel's output lands in the arguments too
            f.copy_(rec['mem'][k]['after'])
        return rec
    return run


def rnd(shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dtype)


def out_rows(rec, ti=0):
    """the whole output of target ti as written ('after'), [M, cols]"""
    return ga.gather(rec, ti, 'after', 0, rec['abi']['M'])


def ok(rec):
    res = ga.check_launch(rec)
    assert not res['errors'], res['errors']
    return res


def flagged(rec, letter):
    errs = ga.check_launch(rec)['errors']
    assert any(e.startswith(f'({letter})') for e in errs), errs


# ------------------------------------------------------------------------------------------- reference vs restatements
@pytest.mark.parametrize('dtype', [F16, BF16])
def test_rows_unaligned_m_pitched(launch, dtype):
    """M = 300 (a tail tile), A and out read / written at pitches wider than the row, bias + residual"""
    M, N, K = 300, 320, 128
    Abuf, W = rnd((M, K + 64), 1, dtype=dtype), rnd((N, K), 2, K ** -0.5, dtype)
    bias, res = rnd(N, 3), rnd((M, N), 4, dtype=dtype)
    out = torch.zeros(M, N + 8, dtype=dtype)
    rec = launch('gemm', Abuf[:, :K], W, out[:, :N], bias=bias, residual=res)
    want = Abuf[:, :K].double() @ W.double().t() + bias.double() + res.double()
    assert (out_rows(rec).double() - want).abs().max() <= ga.U_OUT[dtype] * want.abs().max()
    assert ga.gemm_path(rec) == f"rows+res_smem|tma|{'fp16' if dtype == F16 else 'bf16'}"
    ok(rec)


@pytest.mark.parametrize('B,H,Wd', [(2, 12, 24), (3, 12, 24), (1, 8, 8)], ids=['TH8-TB2', 'batch-tail', 'one-tile'])
def test_conv_tails_vs_conv2d(launch, B, H, Wd):
    """3x3 implicit GEMM with bias_batch at non-square latents: F.conv2d + repeat_interleave of the batch bias"""
    C, N = 64, 160
    if (B, H, Wd) == (2, 12, 24):
        assert ga.conv_tiling(B, H, Wd) == (8, 8, 2)     # the 12 x 24 level of a 96 x 192 latent: the last patch runs past H
    A = rnd((B, H, Wd, C), 5, dtype=F16)
    Wt = rnd((N, 3, 3, C), 6, (9 * C) ** -0.5)           # [N, kh, kw, C]: tap-major rows
    W = Wt.reshape(N, 9 * C).to(F16)
    temb = rnd((B, 3 * N), 7)
    bias = rnd(N, 8)
    out = torch.zeros(B * H * Wd, N, dtype=F16)
    rec = launch('gemm', A, W, out, conv=(B, H, Wd, C), bias=bias, bias_batch=temb[:, N:2 * N], rows_per_batch=H * Wd,
                 bias_batch_ld=3 * N)
    y = F.conv2d(A.permute(0, 3, 1, 2).double(), W.double().view(N, 3, 3, C).permute(0, 3, 1, 2), padding=1)
    want = y.permute(0, 2, 3, 1).reshape(-1, N) + bias.double() + temb[:, N:2 * N].double().repeat_interleave(H * Wd, 0)
    ref = ga.reference(rec, 0, B * H * Wd)[0][0]
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)
    assert ga.gemm_path(rec) == 'rows|tma|fp16|conv|bb'
    ok(rec)


def test_bias_batch_spanning_tiles(launch):
    """rows_per_batch = 96: a 128-row tile spans two or three batches"""
    M, N, K = 300, 160, 64
    A, W = rnd((M, K), 9, dtype=BF16), rnd((N, K), 10, K ** -0.5, BF16)
    bb = rnd((4, N), 11)
    out = torch.zeros(M, N, dtype=BF16)
    rec = launch('gemm', A, W, out, bias_batch=bb, rows_per_batch=96)
    want = A.double() @ W.double().t() + bb.double().repeat_interleave(96, 0)[:M]
    assert torch.allclose(ga.reference(rec, 0, M)[0][0], want, rtol=1e-12, atol=1e-12)
    ok(rec)


def _heads_launch(launch, T, B, nseg, lora, dtype=F16, d=40, H=8, K=128):
    from mos_b200._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED
    C = H * d
    M, N = B * T, nseg * C
    A, W = rnd((M, K), 12, dtype=dtype), rnd((N, K), 13, K ** -0.5, dtype)
    kinds = [MOS_SEG_ROWS] * min(nseg, 2) + [MOS_SEG_TRANSPOSED] * (nseg - 2)
    dp, dvp = 64, 48
    pads = [T + 3 if k == MOS_SEG_ROWS else (T + 7) // 8 * 8 + 8 for k in kinds]
    segs = [torch.zeros(B * H, r, dp, dtype=dtype) if k == MOS_SEG_ROWS else torch.zeros(B * H, dvp, r, dtype=dtype)
            for k, r in zip(kinds, pads)]
    kw = {}
    want = A.double() @ W.double().t()
    if lora:
        down = torch.zeros(16, K, dtype=dtype)
        down[:4 * nseg] = rnd((4 * nseg, K), 14, K ** -0.5, dtype)
        up = rnd((N, 4), 15, 0.5)
        for s in range(nseg):
            want[:, s * C:(s + 1) * C] += (A.double() @ down[4 * s:4 * s + 4].double().t()) @ up[s * C:(s + 1) * C].double().t()
        kw = dict(lora_down=down, lora_up=up, lora_seg=C)
    rec = launch('gemm', A, W, None, heads=dict(seg_ptr=segs, seg_kind=kinds, seg_rows_pad=pads, heads=H, head_dim=d,
                                                dpad=dp, dv_pad=dvp, tokens_per_batch=T), **kw)
    return rec, segs, kinds, want


@pytest.mark.parametrize('T,B', [(77, 3), (64, 3), (128, 2)])
def test_heads_vs_per_head_loops(launch, T, B):
    """head-split Q | K | V^T against explicit per-batch, per-head slices (T = 77: tiles cross batches mid-tile; T = 64:
    two batches per tile, the last tile half outside)"""
    H, d, nseg = 8, 40, 3
    rec, segs, kinds, want = _heads_launch(launch, T, B, nseg, lora=True)
    for s, kind in enumerate(kinds):
        for b in range(B):
            for h in range(H):
                w = want[b * T:(b + 1) * T, s * H * d + h * d:s * H * d + (h + 1) * d]
                got = segs[s][b * H + h, :T, :d] if kind == ga.SEG_ROWS else segs[s][b * H + h, :d, :T].t()
                assert (got.double() - w).abs().max() <= 2 ** -10 * w.abs().max() + 1e-6
        pad = segs[s][:, :, d:] if kind == ga.SEG_ROWS else segs[s][:, d:, :]
        assert not pad.any() and not (segs[s][:, T:, :] if kind == ga.SEG_ROWS else segs[s][:, :, T:]).any()
    assert ga.gemm_path(rec).startswith('heads_vt|' + ('copy' if T == 77 else 'tma'))
    ok(rec)


@pytest.mark.parametrize('nseg', [1, 2, 3, 4])
def test_lora_segments(launch, nseg):
    """1-4 LoRA segments of 160 columns: column n uses the 4 down rows of its segment n // 160"""
    M, K, N = 200, 64, 160 * nseg
    A, W = rnd((M, K), 16, dtype=BF16), rnd((N, K), 17, K ** -0.5, BF16)
    down = rnd((16, K), 18, K ** -0.5, BF16)
    up = rnd((N, 4), 19, 0.5)
    rec = launch('gemm', A, W, torch.zeros(M, N, dtype=BF16), lora_down=down, lora_up=up, lora_seg=160)
    want = A.double() @ W.double().t()
    for n in range(N):
        s = n // 160
        want[:, n] += (A.double() @ down[4 * s:4 * s + 4].double().t()) @ up[n].double()
    assert torch.allclose(ga.reference(rec, 0, M)[0][0], want, rtol=1e-10, atol=1e-10)
    ok(rec)


def _geglu(launch, M=200, Hh=160, K=64, lora=False):
    from mos_b200.engine import geglu_perm
    Wn, bn = rnd((2 * Hh, K), 20, K ** -0.5), rnd(2 * Hh, 21)
    perm = geglu_perm(2 * Hh)
    A = rnd((M, K), 22, dtype=F16)
    kw = {}
    if lora:
        down = torch.zeros(16, K, dtype=F16)
        down[:4] = rnd((4, K), 23, K ** -0.5, F16)
        upn = rnd((2 * Hh, 4), 24, 0.5)
        kw = dict(lora_down=down, lora_up=upn[perm].contiguous(), lora_seg=2 * Hh)
    rec = launch('gemm', A, Wn[perm].to(F16), torch.zeros(M, Hh, dtype=F16), bias=bn[perm].contiguous(), geglu=True, **kw)
    h = A.double() @ Wn.to(F16).double().t() + bn.double()
    if lora:
        h += (A.double() @ down[:4].double().t()) @ upn.double().t()
    return rec, h[:, :Hh], h[:, Hh:]


@pytest.mark.parametrize('lora', [False, True])
def test_geglu_vs_natural_layout(launch, lora):
    """GEGLU over the packed rows (engine.geglu_perm) against a * gelu(gate) of the natural projection"""
    rec, a, g = _geglu(launch, lora=lora)
    want = a * F.gelu(g)
    assert torch.allclose(ga.reference(rec, 0, a.shape[0])[0][0], want, rtol=1e-10, atol=1e-10)
    ok(rec)


@pytest.mark.parametrize('accumulate', [False, True])
def test_f32_output(launch, accumulate):
    M, N, K = 150, 320, 128
    A, W = rnd((M, K), 25, dtype=F16), rnd((N, K), 26, K ** -0.5, F16)
    out = rnd((M, N), 27)
    before = out.double().clone()
    rec = launch('gemm', A, W, out, out_f32=True, accumulate=accumulate)
    want = A.double() @ W.double().t() + (before if accumulate else 0)
    assert torch.allclose(ga.reference(rec, 0, M)[0][0], want, rtol=1e-12, atol=1e-12)
    ok(rec)


@pytest.mark.parametrize('fused', [False, True])
def test_splitk_partials_and_finalize(launch, fused):
    """split-K over 9 k blocks in 4 splits (3, 3, 3, 0 -> normalised by the engine to 3 splits; here 2 x 5 + 4): each
    partial covers its k range, and the finalize sums them in split order plus bias, bias_batch and residual"""
    M, N, K, splits = 260, 320, 64 * 9, 2
    A, W = rnd((M, K), 28, dtype=BF16), rnd((N, K), 29, K ** -0.5, BF16)
    bias, bb, res = rnd(N, 30), rnd((3, N), 31), rnd((M, N), 32, dtype=BF16)
    partial = torch.zeros(splits * M * N + 64)
    out = torch.zeros(M, N, dtype=BF16)
    kw = dict(bias=bias, bias_batch=bb, rows_per_batch=100, residual=res)
    if fused:
        rec = launch('gemm', A, W, out, splits=splits, partial=partial, counters=torch.zeros(64, dtype=torch.int32), **kw)
    else:
        rec = launch('gemm', A, W, None, splits=splits, partial=partial)
    P = partial[:splits * M * N].view(splits, M, N).double()
    Ad, Wd = A.double(), W.double()
    assert torch.allclose(P[0], (Ad[:, :320] @ Wd[:, :320].t()), rtol=1e-6, atol=1e-5)
    assert torch.allclose(P[1], (Ad[:, 320:] @ Wd[:, 320:].t()), rtol=1e-6, atol=1e-5)
    ok(rec)
    if not fused:
        rec = launch('splitk_finalize', partial, splits, M, N, out, **kw)
        ok(rec)
    want = P.sum(0) + bias.double() + bb.double().repeat_interleave(100, 0)[:M] + res.double()
    assert ga.gemm_path(rec) == ('partial|global|bf16|fused' if fused else 'splitk_finalize|bf16|bb|res')
    assert (out.double() - want).abs().max() <= 2 ** -8 * want.abs().max()


def test_pointer_outside_arguments():
    S = ga._Storages([torch.zeros(16)])
    with pytest.raises(AssertionError, match='lies in no tensor argument'):
        S.find(torch.zeros(4).data_ptr(), 'A')
    with pytest.raises(AssertionError, match='runs past its storage'):
        S.window(S.st and next(iter(S.st)), 'A', torch.float32, (4, 8), (8, 1))


# -------------------------------------------------------------------------------------------------- mutation cases
def _conv_bb(launch):
    B, H, Wd, C, N = 2, 12, 24, 64, 160
    A, W = rnd((B, H, Wd, C), 40, dtype=F16), rnd((N, 9 * C), 41, (9 * C) ** -0.5, F16)
    bb = rnd((B, N), 42)
    return launch('gemm', A, W, torch.zeros(B * H * Wd, N, dtype=F16), conv=(B, H, Wd, C), bias_batch=bb,
                  rows_per_batch=H * Wd), bb


def _set(rec, ti, m, c, value):
    t = rec['targets'][ti]
    st = rec['mem'][t['mem']]
    st['after'][ga.target_index(rec, t, m, m + 1)[0, c]] = value


def test_mutation_tail_row_gets_neighbour_batch_bias(launch):
    rec, bb = _conv_bb(launch)
    ok(rec)
    m = rec['abi']['M'] - 1                              # last row: batch 1, in the last (tail) patch
    row = out_rows(rec)[m].double() - bb[1].double() + bb[0].double()
    t = rec['targets'][0]
    rec['mem'][t['mem']]['after'][ga.target_index(rec, t, m, m + 1)[0]] = row.to(F16)
    flagged(rec, 'a')


def test_mutation_one_element_loses_residual(launch):
    M, N, K = 200, 160, 64
    A, W, res = rnd((M, K), 43, dtype=BF16), rnd((N, K), 44, K ** -0.5, BF16), rnd((M, N), 45, dtype=BF16)
    rec = launch('gemm', A, W, torch.zeros(M, N, dtype=BF16), residual=res)
    ok(rec)
    _set(rec, 0, 150, 77, (out_rows(rec)[150, 77].double() - res[150, 77].double()).to(BF16))
    flagged(rec, 'a')


def test_mutation_byte_in_qk_pad_column(launch):
    rec, segs, kinds, _ = _heads_launch(launch, 77, 2, 2, lora=False)
    ok(rec)
    t = rec['targets'][0]
    st = rec['mem'][t['mem']]
    i = int(ga.target_index(rec, t, 5, 6)[0, 39]) + 3   # token 5, head 0: column 42 (head_dim 40, dpad 64)
    st['after'].view(torch.uint8)[2 * i + 1] ^= 0x10
    flagged(rec, 'c')


def test_mutation_vt_pad_row_written(launch):
    rec, segs, kinds, _ = _heads_launch(launch, 64, 3, 3, lora=False)
    ok(rec)
    t = rec['targets'][2]
    assert t['kind'] == 'vt'
    st = rec['mem'][t['mem']]
    i = int(ga.target_index(rec, t, 0, 1)[0, 39]) + t['rows_pad']   # head 0, row j = 40 (a pad row), token 0
    st['after'][i] = 1.0
    flagged(rec, 'c')


def test_mutation_geglu_pair_swapped(launch):
    rec, a, g = _geglu(launch, lora=True)
    ok(rec)
    _set(rec, 0, 17, 90, (g[17, 90] * F.gelu(a[17, 90])).to(F16))
    flagged(rec, 'a')


def test_mutation_lora_segment_boundary_moved(launch):
    M, K, N = 200, 64, 320
    A, W = rnd((M, K), 46, dtype=BF16), rnd((N, K), 47, K ** -0.5, BF16)
    down, up = rnd((16, K), 48, K ** -0.5, BF16), rnd((N, 4), 49, 0.5)
    rec = launch('gemm', A, W, torch.zeros(M, N, dtype=BF16), lora_down=down, lora_up=up, lora_seg=160)
    ok(rec)
    t = A.double() @ down.double().t()
    c = slice(160, 168)                                  # segment 1's first 8 columns take segment 0's ranks
    wrong = out_rows(rec)[:, c].double() + (t[:, 0:4] - t[:, 4:8]) @ up[c].double().t()
    tg = rec['targets'][0]
    rec['mem'][tg['mem']]['after'][ga.target_index(rec, tg, 0, M)[:, c]] = wrong.to(BF16)
    flagged(rec, 'a')


def test_mutation_f32_accumulate_drops_out_before_in_one_tile(launch):
    M, N, K = 256, 320, 64
    A, W = rnd((M, K), 50, dtype=F16), rnd((N, K), 51, K ** -0.5, F16)
    out = rnd((M, N), 52)
    before = out.clone()
    rec = launch('gemm', A, W, out, out_f32=True, accumulate=True)
    ok(rec)
    tg = rec['targets'][0]
    idx = ga.target_index(rec, tg, 128, 256)[:, 160:320]
    rec['mem'][tg['mem']]['after'][idx] -= before[128:256, 160:320]
    flagged(rec, 'a')
    flagged(rec, 'b')


def test_mutation_tile_staged_from_another_tile(launch):
    M, N, K = 256, 320, 64
    A, W = rnd((M, K), 53, dtype=F16), rnd((N, K), 54, K ** -0.5, F16)
    rec = launch('gemm', A, W, torch.zeros(M, N, dtype=F16), bias=rnd(N, 55))
    ok(rec)
    tg = rec['targets'][0]
    after = rec['mem'][tg['mem']]['after']
    after[ga.target_index(rec, tg, 128, 256)[:, 160:]] = after[ga.target_index(rec, tg, 0, 128)[:, :160]]
    flagged(rec, 'a')
    flagged(rec, 'b')


def test_path_keys_follow_host_rule(launch):
    """unaligned pitches leave TMA: copy-out rows, global residual"""
    M, N, K = 130, 160, 64
    A, W = rnd((M, K), 56, dtype=F16), rnd((N, K), 57, K ** -0.5, F16)
    rbuf = rnd((M, N + 4), 58, dtype=F16)
    rec = launch('gemm', A, W, torch.zeros(M, N, dtype=F16), residual=rbuf[:, :N])
    assert ga.gemm_path(rec) == 'rows+res_global|tma|fp16'
    ok(rec)
    rec = launch('gemm', A, W, torch.zeros(M, N + 4, dtype=F16)[:, :N])
    assert ga.gemm_path(rec) == 'rows|copy|fp16'
    ok(rec)
    assert math.isfinite(ga.check_launch(rec)['ratio'])
