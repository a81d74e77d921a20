"""The pipelined multi-tile forward attention kernel (csrc/attention.cu, nk > 128) against a float64 reference.

The multi-tile kernel overlaps each KV tile's softmax with the tensor-core work of its neighbours and masks only the
last, partial tile, so these tests sit on the pipeline's edges: T = 2 and 3 full tiles, and a partial last tile of 1, 15,
16, 17 and BKV - 1 keys (BKV = 128 for d = 40 and 80, 64 for d = 160), T >= 4 tiles (more tiles than K/V stages, so the
producer waits for released stages and the ring wraps), query tails, pitched output, the training
forward's lse2, and run-to-run bit identity.  d = 80 with nk = 77 (probs, pcols) now runs the single-tile kernel.

Tolerances against float64: out rel-L2 1e-3 (fp16) / 8e-3 (bf16), lse2 2e-3 absolute, probabilities 1e-4.
"""
import pytest
import torch

from gpu_helpers import canary, mk, pack_rows, pack_vt, rel_l2_64, rup, same_bits, untouched, window_mask

pytestmark = pytest.mark.gpu
B, H, NQ = 2, 2, 200
OUT_TOL = {torch.float16: 1e-3, torch.bfloat16: 8e-3}
DTYPES = [pytest.param(torch.float16, id='fp16'), pytest.param(torch.bfloat16, id='bf16')]


def _bkv(d):
    return 128 if d <= 80 else 64


def _nks(d):
    """T = 2 and 3 full tiles, 2 full tiles and a partial one of r keys, and T >= 4 with and without a partial tile;
    only nk > 128 (the multi-tile kernel)"""
    b = _bkv(d)
    nks = [2 * b, 3 * b] + [2 * b + r for r in (1, 15, 16, 17, b - 1)] + [4 * b + 1, 5 * b + 17, 7 * b]
    return [n for n in nks if n > 128]


CASES = [(d, nk) for d in (40, 80, 160) for nk in _nks(d)]


def _setup(d, nq, nk, dt, dev, seed=3):
    q, k, v = (mk((B, H, n, d), dev, seed=seed + i, dtype=dt) for i, n in enumerate((nq, nk, nk)))
    dp, dv = rup(d, 64), rup(d, 16)
    return (q, k, v), (pack_rows(q, dp), pack_rows(k, dp), pack_vt(v, dv))


def _reference(q, k, v):
    """float64: out [B, nq, H*d], lse2 [B*H, nq] (log2 of sum 2^(scale log2e S)), P [B*H, nq, nk]"""
    d = q.shape[-1]
    s = (q.double() @ k.double().transpose(-1, -2)) * d ** -0.5
    p = torch.softmax(s, -1)
    out = (p @ v.double()).permute(0, 2, 1, 3).reshape(B, q.shape[2], H * d)
    lse2 = torch.logsumexp(s, -1) / torch.log(torch.tensor(2.0, dtype=torch.float64))
    return out, lse2.reshape(B * H, -1), p.reshape(B * H, q.shape[2], -1)


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('d,nk', CASES)
def test_multi_tile_forward_matches_float64(cuda, dt, d, nk):
    from mos_b200 import ops
    (q, k, v), (Q, K, Vt) = _setup(d, NQ, nk, dt, cuda)
    out = torch.full((B, NQ, H * d), float('nan'), device=cuda, dtype=dt)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=NQ, nk=nk)
    torch.cuda.synchronize()
    ref, _, _ = _reference(q, k, v)
    e = rel_l2_64(out, ref)
    print(f'd={d} nk={nk} {dt}: rel-L2 {e:.2e}')
    assert e < OUT_TOL[dt]


@pytest.mark.parametrize('d,nk', CASES)
def test_multi_tile_train_forward_lse2(cuda, d, nk):
    """mos_attention_fwd_train (bf16, the training operand type) at the same shapes: out as above, lse2 within 2e-3 of
    the float64 log2-sum-exp"""
    from mos_b200 import ops
    dt = torch.bfloat16
    (q, k, v), (Q, K, Vt) = _setup(d, NQ, nk, dt, cuda, seed=11)
    out = torch.full((B, NQ, H * d), float('nan'), device=cuda, dtype=dt)
    lse2 = torch.full((B * H, NQ), float('nan'), device=cuda)
    ops.attention_train(Q, K, Vt, out, lse2, batch=B, heads=H, head_dim=d, nq=NQ, nk=nk)
    torch.cuda.synchronize()
    ref, ref_lse2, _ = _reference(q, k, v)
    assert rel_l2_64(out, ref) < OUT_TOL[dt]
    assert (lse2.double() - ref_lse2).abs().max().item() < 2e-3


@pytest.mark.parametrize('d,nk,nq', [(40, 257, 129), (80, 143, 1), (160, 129, 383)])
def test_multi_tile_query_tails_and_pitched_output(cuda, d, nk, nq):
    """ldo > H*d: only the window is written, bit-identical to a dense output; nq not a multiple of 128"""
    from mos_b200 import ops
    dt = torch.float16
    (q, k, v), (Q, K, Vt) = _setup(d, nq, nk, dt, cuda, seed=21)
    ldo = H * d + 24
    buf = canary((B * nq + 3, ldo), cuda, dt)
    ops.attention(Q, K, Vt, buf, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, ldo=ldo)
    dense = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=dt)
    ops.attention(Q, K, Vt, dense, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    assert untouched(buf, window_mask(buf, slice(0, B * nq), slice(0, H * d)))
    assert same_bits(buf[:B * nq, :H * d], dense.view(B * nq, H * d))
    ref, _, _ = _reference(q, k, v)
    assert rel_l2_64(dense, ref) < OUT_TOL[dt]


@pytest.mark.parametrize('d,nk', [(40, 4096), (80, 1024), (160, 333)])
def test_multi_tile_run_to_run_bitwise(cuda, d, nk):
    from mos_b200 import ops
    (_, _, _), (Q, K, Vt) = _setup(d, 640, nk, torch.float16, cuda, seed=31)
    outs = []
    for _ in range(3):
        out = torch.empty((B, 640, H * d), device=cuda, dtype=torch.float16)
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=640, nk=nk)
        outs.append(out)
    torch.cuda.synchronize()
    assert same_bits(outs[0], outs[1]) and same_bits(outs[0], outs[2])


@pytest.mark.parametrize('dt', DTYPES)
def test_d80_cross_attention_probs_single_tile(cuda, dt):
    """d = 80, nk = 77 with the controller's probability maps: out and probs against float64"""
    from mos_b200 import ops
    d, nk = 80, 77
    (q, k, v), (Q, K, Vt) = _setup(d, NQ, nk, dt, cuda, seed=41)
    out = torch.full((B, NQ, H * d), float('nan'), device=cuda, dtype=dt)
    probs = torch.full((B * H, NQ, nk), float('nan'), device=cuda)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=NQ, nk=nk, probs=probs)
    torch.cuda.synchronize()
    ref, _, P = _reference(q, k, v)
    assert rel_l2_64(out, ref) < OUT_TOL[dt]
    assert rel_l2_64(probs, P) < 1e-4


def test_d80_cross_attention_pcols_single_tile(cuda):
    """d = 80, nk = 77 training forward with the regulariser columns: pcols and lse2 against float64"""
    from mos_b200 import ops
    d, nk, dt = 80, 77, torch.bfloat16
    (q, k, v), (Q, K, Vt) = _setup(d, NQ, nk, dt, cuda, seed=51)
    pos = torch.tensor([[3, 40], [0, 76]], device=cuda, dtype=torch.int32)
    out = torch.full((B, NQ, H * d), float('nan'), device=cuda, dtype=dt)
    lse2 = torch.full((B * H, NQ), float('nan'), device=cuda)
    pcols = torch.full((B * H, NQ, 2), float('nan'), device=cuda)
    ops.attention_train(Q, K, Vt, out, lse2, batch=B, heads=H, head_dim=d, nq=NQ, nk=nk, pcols=pcols, pos=pos)
    torch.cuda.synchronize()
    ref, ref_lse2, P = _reference(q, k, v)
    idx = pos.long().repeat_interleave(H, 0)[:, None, :].expand(-1, NQ, -1)
    assert rel_l2_64(out, ref) < OUT_TOL[dt]
    assert (lse2.double() - ref_lse2).abs().max().item() < 2e-3
    assert rel_l2_64(pcols, P.gather(2, idx)) < 1e-4
