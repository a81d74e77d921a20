"""CPU emulation of the GroupNorm statistics of the fallback and the backward (csrc/norm.cu: gn_stats_kernel and
gn_merge_chunks) in fp32, operation by operation and in the kernels' order, against float64.

The kernels' arithmetic:
  - each thread of a chunk's block owns row lane l (rows r0 + l + j * lanes) and 8 channels, and keeps a Welford
    (mean, M2) per channel: inv = rn(1 / count), m = fma(d, inv, m), M2 = fma(d, x - m_new, M2);
  - thread g < 32 of the block merges its group's cpg x lanes partials in (channel, lane) order about the first
    partial's mean: lane l holds q0 + (l < rem) rows;
  - gn_merge_chunks merges the chunks: 4 threads over strided chunks, the last chunk ragged, about the first chunk's
    mean, then an xor-shuffle tree (2, then 1).
The emulation pins these formulas (lane weights, the ragged last chunk, centring about the first partial) without a GPU:
with an outlier in lane 0 of chunk 0 (the group's first element, or the whole first pixel) the variance stays within
1e-4 of float64, while the sums about that element that the kernels used before lose it.
"""
import math

import numpy as np
import pytest

F32 = np.float32


def fma(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 values is exact in float64"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def block_threads(C):
    """gn_block_threads in csrc/norm.cu (keep in step)"""
    oct = C // 8
    return oct * max(1, 320 // oct)


def fwd_chunks(B, HW, C, capacity):
    """the fallback's chunking in mos_groupnorm_fwd (keep in step): returns (nchunks, rows_per_chunk)"""
    nchunks = -(-2368 // B)
    min_rows = 4 * (block_threads(C) // (C // 8))
    nchunks = min(nchunks, -(-HW // min_rows), capacity // (B * 64))
    nchunks = max(nchunks, 1)
    rpc = -(-HW // nchunks)
    return -(-HW // rpc), rpc


def bwd_chunks(B, HW, C, workspace):
    """the backward's chunking in mos_groupnorm_bwd (keep in step)"""
    nchunks = -(-1184 // B)
    min_rows = 4 * (block_threads(C) // (C // 8))
    nchunks = min(nchunks, -(-HW // min_rows), workspace // (B * 128))
    rpc = -(-HW // nchunks)
    return -(-HW // rpc), rpc


def stats_kernel(x, C, nchunks, rpc):
    """gn_stats_kernel for one sample: x [HW, C] fp32 -> (mean, M2) [nchunks, 32]"""
    HW = x.shape[0]
    oct, cpg = C // 8, C // 32
    lanes = block_threads(C) // oct
    per_lane = -(-rpc // lanes)
    m = np.zeros((nchunks, lanes, C), F32)
    m2 = np.zeros((nchunks, lanes, C), F32)
    cnt = np.zeros((nchunks, lanes, 1), np.int64)
    r0 = (np.arange(nchunks) * rpc)[:, None]
    r1 = np.minimum(HW, r0 + rpc)
    for j in range(per_lane):                       # the thread's rows in increasing order
        r = r0 + np.arange(lanes)[None, :] + j * lanes
        live = (r < r1)[..., None]
        v = x[np.minimum(r, HW - 1)]
        cnt = cnt + live
        inv = (1.0 / np.maximum(cnt, 1)).astype(F32)
        d = (v - m).astype(F32)
        mn = fma(d, inv, m)
        m2n = fma(d, (v - mn).astype(F32), m2)
        m, m2 = np.where(live, mn, m), np.where(live, m2n, m2)
    rows = (r1 - r0)[:, 0]
    q0, rem = rows // lanes, rows % lanes
    out_m = np.zeros((nchunks, 32), F32)
    out_q = np.zeros((nchunks, 32), F32)
    for g in range(32):
        m0 = m[:, 0, g * cpg]
        s = np.zeros(nchunks, F32)
        for c in range(g * cpg, (g + 1) * cpg):
            for lane in range(lanes):
                s = fma((q0 + (lane < rem)).astype(F32), (m[:, lane, c] - m0).astype(F32), s)
        mu = (m0 + (s / (rows.astype(F32) * F32(cpg))).astype(F32)).astype(F32)
        q = np.zeros(nchunks, F32)
        for c in range(g * cpg, (g + 1) * cpg):
            for lane in range(lanes):
                d = (m[:, lane, c] - mu).astype(F32)
                q = (q + fma(((q0 + (lane < rem)).astype(F32) * d).astype(F32), d, m2[:, lane, c])).astype(F32)
        out_m[:, g], out_q[:, g] = mu, q
    return out_m, out_q


def merge_chunks(pm, pq, HW, cpg, rpc):
    """gn_merge_chunks for one sample: per-chunk (mean, M2) [nchunks, 32] -> (mean, var) [32]"""
    nchunks = pm.shape[0]
    rows = (np.minimum(HW, (np.arange(nchunks) + 1) * rpc) - np.arange(nchunks) * rpc).astype(F32)
    m0 = pm[0]

    def tree(v):      # xor 2, then xor 1: thread 0 ends with (v0 + v2) + (v1 + v3)
        a = [(v[i] + v[i ^ 2]).astype(F32) for i in range(4)]
        return (a[0] + a[1]).astype(F32)

    s = [np.zeros(32, F32) for _ in range(4)]
    for c in range(nchunks):
        s[c % 4] = fma(rows[c], (pm[c] - m0).astype(F32), s[c % 4])
    mu = (m0 + (tree(s) / F32(HW)).astype(F32)).astype(F32)
    q = [np.zeros(32, F32) for _ in range(4)]
    for c in range(nchunks):
        d = (pm[c] - mu).astype(F32)
        q[c % 4] = (q[c % 4] + fma((F32(rows[c] * F32(cpg)) * d).astype(F32), d, pq[c])).astype(F32)
    return mu, (tree(q) / (F32(HW) * F32(cpg))).astype(F32)


def pivoted_stats(x, C, nchunks, rpc):
    """the earlier arithmetic: sums of x - p and (x - p)^2 about the group's first element, var = Q/n - (S/n)^2"""
    HW, cpg = x.shape[0], C // 32
    p = np.repeat(x[0, ::cpg], cpg)
    d = (x - p).astype(F32)
    s = np.zeros(C, F32)
    q = np.zeros(C, F32)
    for c in range(nchunks):        # per-chunk fp32 partials, summed in chunk order
        blk = d[c * rpc:(c + 1) * rpc]
        s = (s + blk.sum(0, dtype=F32)).astype(F32)
        q = (q + (blk * blk).sum(0, dtype=F32)).astype(F32)
    n = F32(HW * cpg)
    sg, qg = s.reshape(32, cpg).sum(1, dtype=F32), q.reshape(32, cpg).sum(1, dtype=F32)
    dm = (sg / n).astype(F32)
    return (x[0, ::cpg] + dm).astype(F32), (qg / n - dm * dm).astype(F32)


def sample(HW, C, layout, K, ratio, dtype, seed):
    """one sample [HW, C] in the 16-bit type: group mean ~ ratio x std, then the outlier K std from the mean in lane 0
    of chunk 0 (row 0): the group's first element ('pivot') or every channel of row 0 ('corner')"""
    rng = np.random.default_rng(seed)
    cpg = C // 32
    body = (rng.standard_normal((HW, 32, cpg)) + ratio * rng.choice([-1.0, 1.0], (1, 32, 1))).astype(np.float64)
    if K == 'max':
        K = math.sqrt(HW * cpg) / 2
    mean, std = body.mean(axis=(0, 2)), body.std(axis=(0, 2))
    if layout == 'pivot':
        body[0, :, 0] = mean + K * std
    else:
        body[0] = (mean + K * std)[:, None]
    import torch
    t = torch.from_numpy(body.reshape(HW, C)).to(dtype).float()
    return t.numpy().astype(F32)


def reference(x, C):
    g = x.astype(np.float64).reshape(x.shape[0], 32, C // 32)
    return g.mean(axis=(0, 2)), g.var(axis=(0, 2))


# (name, HW, C, chunking): the VAE's full-resolution layer with the engines' workspace (592 chunks of 443 rows over 20
# lanes, a last chunk of 331 rows), a UNet map on the backward's chunking, and the backward with a one-chunk workspace
# (512 rows per thread)
CASES = [('vae-fwd', 262144, 128, lambda HW, C: fwd_chunks(1, HW, C, 592 * 64)),
         ('unet-bwd', 4096, 320, lambda HW, C: bwd_chunks(2, HW, C, 2 * 1184 * 128)),
         ('unet-bwd-one-chunk', 4096, 320, lambda HW, C: bwd_chunks(2, HW, C, 2 * 128))]


def test_chunking_reaches_ragged_lanes_and_chunks():
    nchunks, rpc = fwd_chunks(1, 262144, 128, 592 * 64)
    assert (nchunks, rpc, 262144 - (nchunks - 1) * rpc) == (592, 443, 331)
    assert rpc % (block_threads(128) // 16) != 0
    assert bwd_chunks(2, 4096, 320, 2 * 128) == (1, 4096)


@pytest.mark.parametrize('K', [300, 'max'])
@pytest.mark.parametrize('layout', ['pivot', 'corner'])
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_stats_centred_against_float64(case, layout, K):
    import torch
    name, HW, C, chunking = case
    nchunks, rpc = chunking(HW, C)
    x = sample(HW, C, layout, K, ratio=3.0, dtype=torch.bfloat16, seed=len(name))
    want_m, want_v = reference(x, C)
    pm, pq = stats_kernel(x, C, nchunks, rpc)
    got_m, got_v = merge_chunks(pm, pq, HW, C // 32, rpc)
    err_v = np.abs(got_v / want_v - 1).max()
    err_m = (np.abs(got_m - want_m) / np.sqrt(want_v)).max()
    old_m, old_v = pivoted_stats(x, C, nchunks, rpc)
    err_old = np.abs(np.maximum(old_v, 0) / want_v - 1).max()
    print(f'{name} {layout} K={K}: var rel err {err_v:.1e} (pivoted sums {err_old:.1e}), mean err / std {err_m:.1e}')
    assert err_v < 1e-4 and err_m < 1e-5
    assert err_old > 1e-4         # the sums about the outlier fail the same bound on this input


def test_constant_groups_exact():
    """every group one value: the mean is that value and M2 is 0, bit for bit"""
    HW, C = 4096, 320
    vals = np.linspace(-110.0, 110.0, 32).astype(F32)
    x = np.repeat(vals, C // 32)[None, :].repeat(HW, 0).astype(F32)
    nchunks, rpc = bwd_chunks(2, HW, C, 2 * 1184 * 128)
    m, v = merge_chunks(*stats_kernel(x, C, nchunks, rpc), HW, C // 32, rpc)
    assert np.array_equal(m, vals) and not v.any()
