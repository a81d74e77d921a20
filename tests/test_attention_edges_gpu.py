"""Edge cases of the wgmma flash-attention forward (csrc/attention.cu) and backward (csrc/attention_bwd.cu) kernels.

Query tails against the 128-query tile together with several key tiles, key tails against the backward's 64-key inner
tile, concept-token columns in either 64-key tile, large logits, pitched and sliced outputs with canaries, and causal
self-attention at the lengths around the tile edges.  Inputs follow the layout the engines allocate: zero pads in Q / K /
V / dO beyond d and in the transposed copies beyond n.

Tolerances are those of test_kernels_gpu.py / test_backward_gpu.py against fp32 PyTorch references of the same op
(TF32 off): forward rel-L2 <= 8e-3 (bf16 output, P rounded to bf16 before PV), backward <= 2e-2 (P and dS rounded to bf16
before the tensor-core products), fp32 probabilities <= 1e-4 (only exp2 / summation-order differences).
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_helpers import bits, canary, mk, pack_rows, pack_vt, rel_l2, rup, same_bits, untouched, window_mask

pytestmark = pytest.mark.gpu
LOG2E = 1.4426950408889634


def _dims(d):
    return rup(d, 64), rup(d, 16)


def _inputs(B, H, d, nq, nk, dev, seed=1, amp=None):
    q, k, v = mk((B, H, nq, d), dev, seed=seed), mk((B, H, nk, d), dev, seed=seed + 1), mk((B, H, nk, d), dev, seed=seed + 2)
    if amp is not None:    # key ramp: later keys carry ever larger logits
        ramp = (0.1 + torch.arange(nk, device=dev).float() / nk).view(1, 1, nk, 1)
        k = (k.float() * ramp * amp).to(torch.bfloat16)
    return q, k, v


def _tok(x):
    """[B, H, n, d] -> token-major [B, n, H*d]"""
    B, H, n, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(B, n, H * d)


# ================================================================================================= forward
@pytest.mark.parametrize('d,nq,nk', [(40, 129, 515), (40, 1000, 300), (80, 200, 333), (80, 383, 1000), (160, 333, 200),
                                     (160, 130, 129)])
def test_forward_query_tails_several_key_tiles(cuda, d, nq, nk):
    from mos_b200 import ops
    B, H = 2, 8
    q, k, v = _inputs(B, H, d, nq, nk, cuda)
    dp, dv = _dims(d)
    out = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(pack_rows(q, dp), pack_rows(k, dp), pack_vt(v, dv), out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    e = rel_l2(out, _tok(F.scaled_dot_product_attention(q.float(), k.float(), v.float())))
    print(f'forward d={d} nq={nq} nk={nk}: rel-L2 {e:.2e}')
    assert e < 8e-3


@pytest.mark.parametrize('d,nk', [(40, 77), (40, 300), (80, 77), (80, 300), (160, 77), (160, 300)])
def test_forward_pitched_output(cuda, d, nk):
    """ldo > H*d: the output rows live in a wider buffer; columns beyond H*d and rows beyond B*nq stay untouched, and
    the values are bit-identical to a dense output."""
    from mos_b200 import ops
    B, H, nq = 2, 8, 200
    q, k, v = _inputs(B, H, d, nq, nk, cuda)
    dp, dv = _dims(d)
    Q, K, Vt = pack_rows(q, dp), pack_rows(k, dp), pack_vt(v, dv)
    ldo = H * d + 24
    buf = canary((B * nq + 3, ldo), cuda, torch.bfloat16)
    ops.attention(Q, K, Vt, buf, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, ldo=ldo)
    dense = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q, K, Vt, dense, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    assert untouched(buf, window_mask(buf, slice(0, B * nq), slice(0, H * d)))
    assert same_bits(buf[:B * nq, :H * d], dense.view(B * nq, H * d))
    assert rel_l2(dense, _tok(F.scaled_dot_product_attention(q.float(), k.float(), v.float()))) < 8e-3


@pytest.mark.parametrize('d,nq,nk', [(40, 300, 77), (80, 200, 333), (160, 130, 200)])
def test_forward_head_placement_bitwise(cuda, d, nq, nk):
    """The output of one (batch, head) does not depend on the batch count or on where the head sits in the grid: a
    3-batch launch, a 1-batch launch of each batch and a 1-head launch of all heads in a shuffled order agree bitwise."""
    from mos_b200 import ops
    B, H = 3, 8
    q, k, v = _inputs(B, H, d, nq, nk, cuda)
    dp, dv = _dims(d)
    Q, K, Vt = pack_rows(q, dp), pack_rows(k, dp), pack_vt(v, dv)
    full = torch.full((B, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q, K, Vt, full, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    for b in range(B):
        one = torch.full((1, nq, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
        hs = slice(b * H, (b + 1) * H)
        ops.attention(Q[hs].contiguous(), K[hs].contiguous(), Vt[hs].contiguous(), one, batch=1, heads=H, head_dim=d,
                      nq=nq, nk=nk)
        assert same_bits(one[0], full[b]), f'batch {b}'
    perm = torch.randperm(B * H, generator=torch.Generator().manual_seed(0)).to(cuda)
    solo = torch.full((B * H, nq, d), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q[perm].contiguous(), K[perm].contiguous(), Vt[perm].contiguous(), solo, batch=B * H, heads=1,
                  head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    want = full.view(B, nq, H, d).permute(0, 2, 1, 3).reshape(B * H, nq, d)[perm]
    assert same_bits(solo, want)


@pytest.mark.parametrize('d', [40, 80, 160])
def test_forward_probs_and_pcols_edge_positions(cuda, d):
    """Probability maps and the concept-token columns at key positions 0, 63, 64 and 76 of a 77-token prompt."""
    from mos_b200 import ops
    B, H, nq, nk = 2, 8, 200, 77
    q, k, v = _inputs(B, H, d, nq, nk, cuda)
    dp, dv = _dims(d)
    Q, K, Vt = pack_rows(q, dp), pack_rows(k, dp), pack_vt(v, dv)
    pos = torch.tensor([[0, 63], [64, 76]], device=cuda, dtype=torch.int32)
    probs = torch.full((B * H, nq, nk), float('nan'), device=cuda)
    out = torch.empty((B, nq, H * d), device=cuda, dtype=torch.bfloat16)
    ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, probs=probs)
    out2 = torch.empty_like(out)
    lse2 = torch.full((B * H, nq), float('nan'), device=cuda)
    pcols = torch.full((B * H, nq, 2), float('nan'), device=cuda)
    ops.attention_train(Q, K, Vt, out2, lse2, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, pcols=pcols, pos=pos)
    torch.cuda.synchronize()
    S = (q.float() @ k.float().transpose(-1, -2)) * d ** -0.5
    P = S.softmax(-1)
    assert rel_l2(probs, P.reshape(B * H, nq, nk)) < 1e-4
    pc = torch.stack([P[b][..., pos[b].long()] for b in range(B)]).reshape(B * H, nq, 2)
    assert rel_l2(pcols, pc) < 1e-4
    assert same_bits(out, out2)
    assert (lse2 - (torch.logsumexp(S, -1) * LOG2E).reshape(B * H, nq)).abs().max().item() < 2e-3


# ================================================================================================= backward
def _fwd_bwd(B, H, d, nq, nk, dev, pos=None, amp=None, seed=1, outputs=None, do_scale=1.0):
    """attention_train + attn_delta + attention_bwd as the training engine chains them, against fp32 autograd.
    outputs(M_q, M_k, C) -> (dq, dk, dv) views to write into (default: dense [B*n, H*d] buffers)."""
    from mos_b200 import ops
    dp, dvp = _dims(d)
    C = H * d
    q, k, v = _inputs(B, H, d, nq, nk, dev, seed=seed, amp=amp)
    do = mk((B, H, nq, d), dev, do_scale, seed=seed + 3)
    Q, K, V, dO = pack_rows(q, dp), pack_rows(k, dp), pack_rows(v, dp), pack_rows(do, dp)
    Qt, dOt = (torch.zeros(B * H, dvp, rup(nq, 8), device=dev, dtype=torch.bfloat16) for _ in range(2))
    Kt, Vt = (torch.zeros(B * H, dvp, rup(nk, 8), device=dev, dtype=torch.bfloat16) for _ in range(2))
    for s, t in ((Q, Qt), (K, Kt), (V, Vt), (dO, dOt)):
        ops.heads_transpose(s, t)
    reg = pos is not None
    posd = torch.tensor(pos, device=dev, dtype=torch.int32) if reg else None
    gcols = torch.randn(B, nq, 2, generator=torch.Generator().manual_seed(seed + 7)).to(dev) * 0.5 if reg else None
    pcols = torch.empty(B * H, nq, 2, device=dev) if reg else None
    out = torch.empty(B, nq, C, device=dev, dtype=torch.bfloat16)
    lse2 = torch.empty(B * H, nq, device=dev)
    ops.attention_train(Q, K, Vt, out, lse2, batch=B, heads=H, head_dim=d, nq=nq, nk=nk, pcols=pcols, pos=posd)
    delta = torch.empty(B * H, nq, device=dev)
    ops.attn_delta(dO, out, delta, batch=B, heads=H, head_dim=d, N=nq, pcols=pcols, gcols=gcols)
    if outputs is None:
        dq, dk, dv = (torch.full((B * n, C), float('nan'), device=dev, dtype=torch.bfloat16) for n in (nq, nk, nk))
    else:
        dq, dk, dv = outputs(B * nq, B * nk, C)

    def run():
        ops.attention_bwd(Q, K, V, dO, Qt, Kt, dOt, lse2, delta, dq, dk, dv, batch=B, heads=H, head_dim=d, nq=nq, nk=nk,
                          gcols=gcols, pos=posd)
    run()
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    P = ((qr @ kr.transpose(-1, -2)) * d ** -0.5).softmax(-1)
    loss = ((P @ vr) * do.float()).sum()
    if reg:
        for b in range(B):
            for c in range(2):
                loss = loss + (P[b, :, :, pos[b][c]] * gcols[b, :, c][None]).sum()
    loss.backward()
    refs = [_tok(g).reshape(-1, C) for g in (qr.grad, kr.grad, vr.grad)]
    return (dq, dk, dv), refs, run


def _check(got, refs, tag, tol=2e-2):
    errs = [rel_l2(g, r) for g, r in zip(got, refs)]
    print(f'{tag}: dq {errs[0]:.2e} dk {errs[1]:.2e} dv {errs[2]:.2e}')
    assert max(errs) < tol, errs


@pytest.mark.parametrize('B', [1, 4])
@pytest.mark.parametrize('d,nq,nk', [(40, 333, 201), (80, 200, 139), (160, 130, 77), (160, 257, 333)])
def test_backward_tails(cuda, B, d, nq, nk):
    """nq % 128 != 0 and nk % 64 != 0 for all three head dims, at B x H = 1 x 8 and 4 x 8."""
    got, refs, _ = _fwd_bwd(B, 8, d, nq, nk, cuda)
    torch.cuda.synchronize()
    _check(got, refs, f'B={B} d={d} nq={nq} nk={nk}')


@pytest.mark.parametrize('only_reg', [False, True])
@pytest.mark.parametrize('d', [40, 80, 160])
def test_backward_regulariser_positions(cuda, d, only_reg):
    """Concept-token columns on both sides of the 64-key tile edge and at the last key of a 77-token prompt.  With
    only_reg the output gradient is zero, so dQ and dK come from the probability gradient alone (dV is exactly zero):
    a gradient applied at the wrong key cannot hide under the dO term."""
    pos = [[0, 1], [62, 63], [63, 64], [75, 76]]
    (dq, dk, dv), refs, _ = _fwd_bwd(4, 8, d, 200, 77, cuda, pos=pos, do_scale=0.0 if only_reg else 1.0)
    torch.cuda.synchronize()
    if not only_reg:
        _check((dq, dk, dv), refs, f'regulariser d={d}')
        return
    assert dv.abs().max().item() == 0
    eq, ek = rel_l2(dq, refs[0]), rel_l2(dk, refs[1])
    print(f'regulariser only d={d}: dq {eq:.2e} dk {ek:.2e}')
    assert eq < 2e-2 and ek < 2e-2


@pytest.mark.parametrize('amp', [16.0, 60.0])
@pytest.mark.parametrize('d', [40, 80, 160])
def test_backward_large_logits(cuda, d, amp):
    """Key ramp as in test_attention_growing_logits: P is recomputed from the saved log2-sum-exp with ex2.approx, where
    large logits leave the least headroom."""
    got, refs, _ = _fwd_bwd(1, 8, d, 256, 333, cuda, amp=amp)
    torch.cuda.synchronize()
    assert all(torch.isfinite(g.float()).all() for g in got)
    _check(got, refs, f'large logits d={d} amp={amp}')


@pytest.mark.parametrize('d', [40, 80, 160])
def test_backward_into_engine_slices(cuda, d):
    """dQ dense with dK / dV in the two halves of dkv (pitch 2C, cross-attention over 77 tokens), and dQ / dK / dV in the
    three thirds of dqkv (pitch 3C, self-attention), exactly as the training engine passes them.  Bit-identical to
    dense outputs; the rows past the end of each buffer stay untouched."""
    B, H, nq = 2, 8, 200
    C = H * d
    for nk, split in ((77, 'dkv'), (nq, 'dqkv')):
        bufs = {}

        def outputs(Mq, Mk, C_):
            dq = torch.full((Mq, C_), float('nan'), device=cuda, dtype=torch.bfloat16)
            if split == 'dkv':
                bufs['dkv'] = canary((Mk + 2, 2 * C_), cuda, torch.bfloat16)
                return dq, bufs['dkv'][:Mk, :C_], bufs['dkv'][:Mk, C_:]
            bufs['dqkv'] = canary((Mq + 2, 3 * C_), cuda, torch.bfloat16)
            b = bufs['dqkv']
            return b[:Mq, :C_], b[:Mq, C_:2 * C_], b[:Mq, 2 * C_:]
        got, refs, _ = _fwd_bwd(B, H, d, nq, nk, cuda, outputs=outputs)
        dense, _, _ = _fwd_bwd(B, H, d, nq, nk, cuda)
        torch.cuda.synchronize()
        buf = bufs[split]
        rows = B * nk
        assert untouched(buf, window_mask(buf, slice(0, rows), slice(None))), split
        for g, w in zip(got, dense):
            assert same_bits(g, w), split
        _check(got, refs, f'{split} d={d}')


@pytest.mark.parametrize('n', [1, 8, 64, 65, 128])
def test_backward_causal(cuda, n):
    """Causal self-attention backward at d = 80 (all 80 dimensions in use) around the 64-key and 128-query tile edges,
    against autograd of F.scaled_dot_product_attention(is_causal=True).  n = 1: dS = P (dP - delta) is zero up to
    rounding, so dQ and dK are checked for being negligible against dV instead of by relative error."""
    from mos_b200 import ops
    B, H, d = 2, 8, 80
    dp, dvp, n8 = 128, 80, rup(n, 8)
    q, k, v = _inputs(B, H, d, n, n, cuda)
    do = mk((B, H, n, d), cuda, seed=9)
    Q, K, V, dO = pack_rows(q, dp), pack_rows(k, dp), pack_rows(v, dp), pack_rows(do, dp)
    Qt, Kt, Vt, dOt = (torch.zeros(B * H, dvp, n8, device=cuda, dtype=torch.bfloat16) for _ in range(4))
    for s, t in ((Q, Qt), (K, Kt), (V, Vt), (dO, dOt)):
        ops.heads_transpose(s, t)
    o = torch.full((B, n, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
    lse2 = torch.full((B * H, n), float('nan'), device=cuda)
    ops.attention_causal(Q, K, Vt, o, batch=B, heads=H, head_dim=d, n=n, scale=d ** -0.5, lse2=lse2)
    delta = torch.empty(B * H, n, device=cuda)
    ops.attn_delta(dO, o, delta, batch=B, heads=H, head_dim=d, N=n)
    dq, dk, dv = (torch.full((B * n, H * d), float('nan'), device=cuda, dtype=torch.bfloat16) for _ in range(3))
    ops.attention_bwd(Q, K, V, dO, Qt, Kt, dOt, lse2, delta, dq, dk, dv, batch=B, heads=H, head_dim=d, nq=n, nk=n,
                      causal=True)
    torch.cuda.synchronize()
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    out = F.scaled_dot_product_attention(qr, kr, vr, is_causal=True)
    out.backward(do.float())
    assert rel_l2(o, _tok(out.detach())) < 8e-3
    refs = [_tok(g).reshape(B * n, H * d) for g in (qr.grad, kr.grad, vr.grad)]
    if n == 1:
        assert rel_l2(dv, refs[2]) < 2e-2
        scale = refs[2].norm().item()
        assert dq.float().norm().item() < 1e-3 * scale and dk.float().norm().item() < 1e-3 * scale
    else:
        _check((dq, dk, dv), refs, f'causal n={n}')


@pytest.mark.parametrize('d,nk,pos', [(40, 201, None), (80, 201, None), (160, 201, None), (80, 77, [[3, 70], [64, 0]])])
def test_backward_deterministic(cuda, d, nk, pos):
    """No atomics in either backward kernel: two identical calls give bit-identical gradients."""
    (dq, dk, dv), _, run = _fwd_bwd(2, 8, d, 333, nk, cuda, pos=pos)
    first = [t.clone() for t in (dq, dk, dv)]
    for t in (dq, dk, dv):
        bits(t).fill_(0x7FA5)
    run()
    torch.cuda.synchronize()
    for a, b in zip(first, (dq, dk, dv)):
        assert same_bits(a, b)
