"""The attention regulariser of ED-LoRA (cal_attn_reg, trainer_edlora.py:263-313) on the GPU: the kernels
mos_attn_reg_group / total / grad against float64 autograd of oracle.train_ref.cal_attn_reg (itself pinned to the
reference's output by tests/golden/reference_golden.pt['attn_reg']); the backward chain attention_train -> regulariser ->
attn_delta -> attention_bwd with a zero output gradient, so that only the regulariser drives dQ and dK; and, in the
training engine, the share of the LoRA and text-embedding gradients that the regulariser contributes.

The oracle evaluates the full-identity subject MSE through `.float()`, as the reference does, so that one term of the
float64 reference carries fp32 rounding (~1e-7 relative), far below the bounds used here.
"""
import math

import pytest
import torch

from gpu_helpers import mk, pack_rows, pack_vt, rel_l2, rel_l2_64, rup

pytestmark = pytest.mark.gpu
HEADS = 8
F64 = torch.float64


def _groups(maps):
    """{N: [maps_l of the group, in layer order]}, ordered as the engine runs them (largest N first)."""
    g = {}
    for lst in maps.values():
        for m in lst:
            g.setdefault(m.shape[1], []).append(m)
    return {N: g[N] for N in sorted(g, reverse=True)}


def _pcols(m, pos):
    """pcols[(b, h), n, c] = m[(b, h), n, pos[b][c]] as the forward emits them (fp32 [B*heads, N, 2])"""
    B = m.shape[0] // HEADS
    idx = torch.tensor(pos, device=m.device).repeat_interleave(HEADS, 0)          # [B*heads, 2]
    return torch.gather(m, 2, idx[:, None, :].expand(-1, m.shape[1], -1)).float().contiguous()


def _run_kernels(maps, masks, pos, full, weight, grad_scale, mse=0.3125):
    from mos_b200 import ops
    B = masks.shape[0]
    mask = masks.float().cuda().contiguous()
    groups = _groups(maps)
    stats = torch.full((len(groups), 8), float('nan'), device='cuda')
    cms = {}
    for g, (N, lst) in enumerate(groups.items()):
        cm = torch.full((B, N, 2), float('nan'), device='cuda')
        ops.attn_reg_group([_pcols(m, pos) for m in lst], mask, cm, stats[g], B=B, heads=HEADS, res=math.isqrt(N),
                           full_identity=full, weight=weight)
        cms[N] = cm
    mse_t = torch.tensor([mse], device='cuda')
    out = torch.full((2,), float('nan'), device='cuda')
    ops.attn_reg_total(mse_t, stats, out)
    gcols = {}
    for g, (N, lst) in enumerate(groups.items()):
        gc = torch.full((B, N, 2), float('nan'), device='cuda')
        ops.attn_reg_grad(cms[N], mask, stats, gc, B=B, res=math.isqrt(N), full_identity=full, weight=weight, group=g,
                          L=len(lst), heads=HEADS, grad_scale=grad_scale)
        gcols[N] = gc
    torch.cuda.synchronize()
    return dict(stats=stats, cm=cms, out=out, gcols=gcols, mse=mse_t)


def _reference(maps, masks, pos, full, weight, grad_scale):
    """float64 cal_attn_reg on the same maps; per group the mean map [B, N, 2] and d(grad_scale * loss)/d maps_l."""
    from oracle import train_ref
    leaves = {k: [m.to(F64).requires_grad_(True) for m in v] for k, v in maps.items()}
    loss = train_ref.cal_attn_reg(leaves, masks.to(F64).cuda(), pos, reg_full_identity=full, attn_reg_weight=weight)
    if not torch.isnan(loss):
        (loss * grad_scale).backward()
    grads, cms = {}, {}
    for k, lst in leaves.items():
        for m in lst:
            N = m.shape[1]
            B = m.shape[0] // HEADS
            grads.setdefault(N, []).append(m.grad)
            sel = torch.stack([m.detach()[b * HEADS:(b + 1) * HEADS, :, pos[b]] for b in range(B)])   # [B, H, N, 2]
            cms.setdefault(N, []).append(sel)
    cms = {N: torch.cat(v, 1).mean(1) for N, v in cms.items()}
    return loss.detach(), grads, cms


def _softmax_maps(ress, B, seed, nk=77):
    """fresh softmax maps {place: [[B*heads, r*r, nk] ...]} for the given resolutions, on the GPU"""
    g = torch.Generator().manual_seed(seed)
    return {'cross': [(torch.randn(B * HEADS, r, r, nk, generator=g) * 2.0).softmax(-1).reshape(B * HEADS, r * r, nk)
                      .cuda() for r in ress]}


def _sd15_maps(B):
    from oracle import train_ref
    maps, masks, ids, pos = train_ref.attn_reg_inputs(B)
    return {k: [m.cuda() for m in v] for k, v in maps.items()}, masks, pos[:B]


def _make_ties(maps, pos, masks):
    """For the groups of res 64 and 8: copy the probability rows of each column's arg-max position (every layer and head
    of the group) to two further positions of the same sample, so that the mean map has an exact three-way tie of its
    maximum, in fp32 as in float64."""
    B = masks.shape[0]
    groups = _groups(maps)
    for N in (4096, 64):
        lst = groups[N]
        cm = torch.stack([torch.stack([m[b * HEADS:(b + 1) * HEADS, :, pos[b]] for b in range(B)]) for m in lst]).mean((0, 2))
        used = set()
        for c in range(2):
            flat = int(cm[..., c].flatten().argmax())
            b, n = divmod(flat, N)
            dst = [x for x in range(N) if x != n and (b, x) not in used][:2]
            used.update({(b, n), *[(b, x) for x in dst]})
            for m in lst:
                for x in dst:
                    m[b * HEADS:(b + 1) * HEADS, x] = m[b * HEADS:(b + 1) * HEADS, n]
    return maps


def _masks_split(B, size):
    m = torch.ones(B, 1, size, size)
    m[0, :, : size // 2] = 0.0
    m[-1, :, :, size // 3:] = 0.0
    return m


def _case(name, B):
    if name in ('sd15', 'tie'):
        maps, masks, pos = _sd15_maps(B)
        if name == 'tie':
            maps = _make_ties(maps, pos, masks)
        return maps, masks, pos
    pos = [[4, 5], [2, 9]][:B]
    if name == 'lat96':                           # 96x96 latents: groups 96 / 48 / 24 / 12 with 5 / 5 / 5 / 1 layers
        maps = _softmax_maps([96, 96, 48, 48, 24, 24, 12, 24, 24, 24, 48, 48, 48, 96, 96, 96], B, 3)
        masks = (torch.rand(B, 1, 96, 96, generator=torch.Generator().manual_seed(4)) > 0.5).float()
        return maps, masks, pos
    if name == 'split_masks':                     # the two samples' masks differ in shape and zero count
        maps, _, pos = _sd15_maps(B)
        return maps, _masks_split(B, 64), pos
    raise ValueError(name)


# fp32 kernels against float64.  Measured worst over the cases below on an H100 80GB HBM3 (700 W): mean map 3.0e-7
# max-rel, loss 6.1e-8 rel, gcols 3.5e-7 rel-L2 (per layer and head), arg-max / tie elements 3.6e-7 of max|ref|
TOL_CM, TOL_LOSS, TOL_G, TOL_G_ELEM = 2e-6, 1e-6, 2e-6, 2e-6


@pytest.mark.parametrize('name,B,full,weight,grad_scale', [
    ('sd15', 2, True, 0.01, 1.0),
    ('sd15', 2, False, 1.0, 0.5),
    ('sd15', 1, True, 1.0, 0.5),
    ('sd15', 1, False, 0.01, 1.0),
    ('lat96', 2, True, 0.01, 1.0),
    ('lat96', 1, False, 1.0, 0.5),
    ('split_masks', 2, True, 1.0, 1.0),
    ('split_masks', 2, False, 0.01, 0.5),
    ('tie', 2, True, 1.0, 1.0),
    ('tie', 2, False, 0.01, 0.5),
])
def test_attn_reg_kernels_vs_float64(cuda, name, B, full, weight, grad_scale):
    maps, masks, pos = _case(name, B)
    got = _run_kernels(maps, masks, pos, full, weight, grad_scale)
    ref_loss, ref_grads, ref_cm = _reference(maps, masks, pos, full, weight, grad_scale)
    assert not torch.isnan(ref_loss)
    worst = dict(cm=0.0, g=0.0, elem=0.0)
    for g, N in enumerate(_groups(maps)):
        res = math.isqrt(N)
        cm, st, gc = got['cm'][N], got['stats'][g], got['gcols'][N]
        worst['cm'] = max(worst['cm'], ((cm.double() - ref_cm[N]).abs().max() / ref_cm[N].abs().max()).item())
        gt = torch.nn.functional.interpolate(masks.float(), size=(res, res), mode='nearest').squeeze(1)
        assert st[4].item() == (gt == 0).sum().item(), 'zero count'
        for c in range(2):
            mx = cm[..., c].max()
            assert st[c].item() == mx.item(), 'max of the fp32 mean map'
            ties = cm[..., c] == mx
            assert st[2 + c].item() == ties.sum().item(), 'tie count'
            ref_arg = int(ref_cm[N][..., c].flatten().argmax())
            assert ties.flatten()[ref_arg], 'the float64 arg-max is not a maximum of the fp32 map'
            if name == 'tie' and N in (4096, 64):
                assert ties.sum().item() == 3
        # every layer and head of the group carries the same gradient on its concept columns
        for l, rg in enumerate(ref_grads[N]):
            want = torch.stack([rg[b * HEADS:(b + 1) * HEADS, :, pos[b]] for b in range(B)])    # [B, H, N, 2]
            per_head = torch.linalg.vector_norm(gc.double()[:, None] - want, dim=(0, 2, 3))
            e = (per_head / torch.linalg.vector_norm(want, dim=(0, 2, 3))).max().item()
            worst['g'] = max(worst['g'], e)
            assert e < TOL_G, (N, l, e)
            # the arg-max correction lands on the maxima only: check those elements on their own
            scale = want.abs().max().item()
            for c in range(2):
                idx = (cm[..., c] == cm[..., c].max()).nonzero()
                for b, n in idx.tolist():
                    e = (gc[b, n, c].double() - want[b, :, n, c]).abs().max().item() / scale
                    worst['elem'] = max(worst['elem'], e)
                    assert e < TOL_G_ELEM, (N, b, n, c, e)
    e_loss = abs(got['out'][1].item() - ref_loss.item()) / abs(ref_loss.item())
    print(f'[{name} B={B} full={full} w={weight} gs={grad_scale}] cm {worst["cm"]:.2e} loss {e_loss:.2e} '
          f'gcols {worst["g"]:.2e} arg-max elements {worst["elem"]:.2e}')
    assert worst['cm'] < TOL_CM
    assert e_loss < TOL_LOSS
    assert torch.equal(got['out'][0:1], got['mse'] + got['out'][1:2])


@pytest.mark.parametrize('kind', ['pixel33', 'ones'])
def test_attn_reg_skip_path(cuda, kind):
    """A resized mask without a zero pixel makes the reference loss NaN, and the trainer then skips the regulariser
    (trainer_edlora.py:257).  With one zero pixel at (3, 3), off the stride-2 grid that nearest resizing samples for
    res 32 / 16 / 8, only res 64 sees it."""
    maps, masks, pos = _sd15_maps(2)
    masks = torch.ones_like(masks)
    if kind == 'pixel33':
        masks[:, :, 3, 3] = 0.0
    got = _run_kernels(maps, masks, pos, True, 0.01, 1.0)
    ref_loss, _, _ = _reference(maps, masks, pos, True, 0.01, 1.0)
    assert torch.isnan(ref_loss)
    assert torch.isnan(got['out'][1]).item()
    assert torch.equal(got['out'][0:1], got['mse'])
    zeros = got['stats'][:, 4].tolist()
    assert zeros == ([2.0, 0.0, 0.0, 0.0] if kind == 'pixel33' else [0.0] * 4)
    for gc in got['gcols'].values():
        assert not torch.isnan(gc).any()
        assert (gc == 0).all()


# ================================================================================================= backward chain
def _tok(t):
    """[B, H, n, d] -> token-major rows [B*n, H*d]"""
    B, H, n, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * n, H * d)


@pytest.mark.parametrize('full', [True, False])
@pytest.mark.parametrize('d,res', [(160, 16), (40, 64)])
def test_regulariser_backward_chain(cuda, d, res, full):
    """One resolution group of two cross-attention layers, composed as train_engine composes them: attention_train
    (pcols) -> attn_reg_group / total / grad -> attn_delta(pcols, gcols) -> attention_bwd(gcols), with dO = 0.  Against
    float64 autograd of softmax attention -> cal_attn_reg.  Bound: the attention backward's rel-L2 2e-2 (P and dS are
    rounded to bf16 before the tensor-core products); measured worst 3.6e-3 on an H100 80GB HBM3 (700 W)."""
    from mos_b200 import ops
    from oracle import train_ref
    B, H, nk, L, weight = 1, HEADS, 77, 2, 1.0
    N = res * res
    dp, dvp = rup(d, 64), rup(d, 16)
    pos = [[5, 70]]
    posd = torch.tensor(pos, device=cuda, dtype=torch.int32)
    masks = torch.ones(B, 1, 64, 64)
    masks[:, :, 10:30, 5:50] = 0.0
    mask = masks.cuda()
    layers = []
    for l in range(L):
        q, k, v = (mk((B, H, n, d), cuda, 1.5 if i < 2 else 1.0, seed=10 * l + i)
                   for i, n in enumerate((N, nk, nk)))
        Q, K, V = pack_rows(q, dp), pack_rows(k, dp), pack_rows(v, dp)
        out = torch.empty(B, N, H * d, device=cuda, dtype=torch.bfloat16)
        lse2 = torch.empty(B * H, N, device=cuda)
        pcols = torch.full((B * H, N, 2), float('nan'), device=cuda)
        ops.attention_train(Q, K, pack_vt(v, dvp), out, lse2, batch=B, heads=H, head_dim=d, nq=N, nk=nk, pcols=pcols,
                            pos=posd)
        layers.append(dict(q=q, k=k, v=v, Q=Q, K=K, V=V, out=out, lse2=lse2, pcols=pcols))
    stats = torch.empty(1, 8, device=cuda)
    cm = torch.empty(B, N, 2, device=cuda)
    ops.attn_reg_group([x['pcols'] for x in layers], mask, cm, stats[0], B=B, heads=H, res=res, full_identity=full,
                       weight=weight)
    loss_out = torch.empty(2, device=cuda)
    ops.attn_reg_total(torch.zeros(1, device=cuda), stats, loss_out)
    gcols = torch.empty(B, N, 2, device=cuda)
    ops.attn_reg_grad(cm, mask, stats, gcols, B=B, res=res, full_identity=full, weight=weight, group=0, L=L, heads=H)
    errs = []
    maps = []
    ref_leaves = []
    for x in layers:
        dO = torch.zeros(B * H, N, dp, device=cuda, dtype=torch.bfloat16)
        Qt, dOt = (torch.zeros(B * H, dvp, rup(N, 8), device=cuda, dtype=torch.bfloat16) for _ in range(2))
        Kt = torch.zeros(B * H, dvp, rup(nk, 8), device=cuda, dtype=torch.bfloat16)
        for s, t in ((x['Q'], Qt), (dO, dOt), (x['K'], Kt)):
            ops.heads_transpose(s, t)
        delta = torch.empty(B * H, N, device=cuda)
        ops.attn_delta(dO, x['out'], delta, batch=B, heads=H, head_dim=d, N=N, pcols=x['pcols'], gcols=gcols)
        x['dq'], x['dk'], x['dv'] = (torch.full((B * n, H * d), float('nan'), device=cuda, dtype=torch.bfloat16)
                                     for n in (N, nk, nk))
        ops.attention_bwd(x['Q'], x['K'], x['V'], dO, Qt, Kt, dOt, x['lse2'], delta, x['dq'], x['dk'], x['dv'], batch=B,
                          heads=H, head_dim=d, nq=N, nk=nk, gcols=gcols, pos=posd)
        qr, kr = x['q'].to(F64).requires_grad_(True), x['k'].to(F64).requires_grad_(True)
        ref_leaves.append((qr, kr))
        maps.append(((qr @ kr.transpose(-1, -2)) * d ** -0.5).softmax(-1).reshape(B * H, N, nk))
    torch.cuda.synchronize()
    loss = train_ref.cal_attn_reg({'cross': maps}, masks.to(F64).cuda(), pos, reg_full_identity=full,
                                  attn_reg_weight=weight)
    loss.backward()
    assert abs(loss_out[1].item() - loss.item()) < 1e-5 * abs(loss.item())   # measured < 3e-6
    for x, (qr, kr) in zip(layers, ref_leaves):
        eq, ek = rel_l2(x['dq'], _tok(qr.grad)), rel_l2(x['dk'], _tok(kr.grad))
        errs += [eq, ek]
        assert x['dv'].abs().max().item() == 0
    print(f'chain d={d} res={res} full={full}: loss {loss_out[1].item():.6e} vs {loss.item():.6e}; '
          f'dq/dk rel-L2 {" ".join(f"{e:.2e}" for e in errs)}')
    assert max(errs) < 2e-2


@pytest.mark.parametrize('case', ['pcols', 'plain', 'pcols_zero_do'])
@pytest.mark.parametrize('d', [40, 80, 160])
def test_attn_delta_vs_float64(cuda, d, case):
    """delta[bh, q] = dO . O (+ sum_c pcols * gcols) with dO in the padded head-split layout [B*H, N, DP] (NaN in the pad
    columns, which must not be read) and O in a pitched token-major buffer (NaN beyond H*d).  fp32 accumulation of at most
    160 products against float64 of the same bf16 values: measured worst 8.5e-8 rel-L2 on an H100 80GB HBM3 (700 W)."""
    from mos_b200 import ops
    B, H, N = 2, HEADS, 333
    C, dp = H * d, rup(d, 64)
    ldo = C + 24
    do = mk((B * H, N, d), cuda, 0.0 if case == 'pcols_zero_do' else 1.0, seed=1)
    dO = torch.full((B * H, N, dp), float('nan'), device=cuda, dtype=torch.bfloat16)
    dO[..., :d] = do
    o = mk((B * N, C), cuda, seed=2)
    O = torch.full((B * N, ldo), float('nan'), device=cuda, dtype=torch.bfloat16)
    O[:, :C] = o
    reg = case != 'plain'
    pcols = torch.rand(B * H, N, 2, generator=torch.Generator().manual_seed(3)).cuda() if reg else None
    gcols = torch.randn(B, N, 2, generator=torch.Generator().manual_seed(4)).cuda() if reg else None
    delta = torch.full((B * H, N), float('nan'), device=cuda)
    ops.attn_delta(dO, O, delta, batch=B, heads=H, head_dim=d, N=N, ldo=ldo, pcols=pcols, gcols=gcols)
    torch.cuda.synchronize()
    o4 = o.to(F64).view(B, N, H, d).permute(0, 2, 1, 3).reshape(B * H, N, d)
    want = (do.to(F64) * o4).sum(-1)
    if reg:
        want = want + (pcols.to(F64) * gcols.to(F64).repeat_interleave(H, 0)).sum(-1)
    e = rel_l2_64(delta, want)
    print(f'attn_delta d={d} {case}: rel-L2 {e:.2e}')
    assert e < 1e-6


# ================================================================================================= engine
def _setup(reg_weight, full_identity, seed=0):
    """The tiny-topology training step of test_train_gpu.py; the oracle's gradient is that of the attention term only."""
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle import unet as ou
    from oracle.schedulers import DDPMScheduler
    ref = ou.build_unet(seed, ou.TINY)
    lora = inject.random_lora_state(ref, seed=10)
    leaves = {k: v.clone().requires_grad_(True) for k, v in lora.items()}
    alpha = 0.9
    inject.inject_lora(ref, leaves, alpha)
    ctl = AttentionStore(training=True)
    n_layers = inject.install_control_processors(ref, ctl)
    g = torch.Generator().manual_seed(21)
    B, H = 2, 16
    x0 = torch.randn(B, 4, H, H, generator=g)
    noise = torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([130, 811])
    ehs = torch.randn(B, n_layers, 77, 768, generator=g).to(torch.bfloat16).float().requires_grad_(True)
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    pos = [[3, 4], [2, 7]]
    noisy = DDPMScheduler().add_noise(x0, noise, t)
    _, _, attn = train_ref.train_loss(ref, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                      reg_full_identity=full_identity, attn_reg_weight=reg_weight)
    names = sorted(leaves)
    gr = torch.autograd.grad(attn, [leaves[k] for k in names] + [ehs], allow_unused=True)
    grads = {k: torch.zeros_like(leaves[k]) if v is None else v for k, v in zip(names, gr)}
    return dict(ref=ref, lora=lora, alpha=alpha, n_layers=n_layers, x0=x0, noise=noise, t=t, ehs=ehs.detach(),
                ehs_grad=gr[-1], masks=masks, pos=pos, attn=attn.detach(), grads=grads)


@pytest.mark.parametrize('full', [True, False])
def test_engine_regulariser_gradient(cuda, full):
    """TrainEngine.forward_backward with attn_reg_weight = 1.0 and with None: the forward is bit-identical, and the
    difference of the LoRA gradients (and of d(text embeddings)) is the oracle's autograd of the attention term alone.
    The difference keeps the bf16 rounding of the activation gradients it passed through, so the bounds are those of
    test_train_gpu.py's flat gradient.  Measured worst on an H100 80GB HBM3 (700 W): attention loss 4.1e-4 rel, flat
    LoRA rel-L2 1.1e-2 (cosine 0.99994), d(ehs) rel-L2 1.0e-2."""
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import unet as ou
    w = 1.0
    S = _setup(w, full)
    sd = {k: v.detach() for k, v in S['ref'].state_dict().items()}
    runs = {}
    for reg in (w, None):
        eng = TrainEngine(sd, 2, 16, 16, lora=S['lora'], lora_alpha=S['alpha'], attn_reg_weight=reg,
                          reg_full_identity=full, text_grad=True, block_out=ou.TINY['block_out_channels'],
                          layers=ou.TINY['layers_per_block'])
        out = eng.forward_backward(S['x0'].cuda(), S['noise'].cuda(), S['t'].cuda(),
                                   ehs_to_layer_major(S['ehs'].cuda(), S['n_layers'], torch.bfloat16), S['masks'].cuda(),
                                   token_pos=S['pos'])
        torch.cuda.synchronize()
        runs[reg] = dict(eps=eng.out_eps.clone(), out=out.clone(), grads=eng.lora_grad_dict(),
                         d_ehs=eng.d_ehs[:, :768].float().clone())
        del eng
    a, b = runs[w], runs[None]
    assert torch.equal(a['eps'], b['eps'])
    e_attn = abs(a['out'][1].item() - S['attn'].item()) / abs(S['attn'].item())
    fg, fr = [], []
    for m, (gD, gU) in a['grads'].items():
        nD, nU = b['grads'][m]
        fg += [(gD - nD).flatten().cpu(), (gU - nU).flatten().cpu()]
        fr += [S['grads'][m + '.lora_down.weight'].flatten(), S['grads'][m + '.lora_up.weight'].flatten()]
    fg, fr = torch.cat(fg), torch.cat(fr)
    e_lora = rel_l2(fg, fr)
    cos = torch.nn.functional.cosine_similarity(fg.double(), fr.double(), dim=0).item()
    nl = S['n_layers']
    d_ehs = (a['d_ehs'] - b['d_ehs']).view(nl, 2, 77, 768).cpu()
    e_ehs = rel_l2(d_ehs, S['ehs_grad'].permute(1, 0, 2, 3))
    print(f'[full={full}] attn loss rel {e_attn:.2e}; regulariser share of the LoRA gradient: rel-L2 {e_lora:.3e} '
          f'cosine {cos:.6f} (|ref| {fr.norm():.3e}); of d(ehs): rel-L2 {e_ehs:.3e}')
    assert e_attn < 2e-3
    assert e_lora < 3e-2 and cos > 0.9995
    assert e_ehs < 3e-2
