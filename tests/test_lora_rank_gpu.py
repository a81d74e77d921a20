"""ED-LoRA at LoRA ranks 1-3 on the GPU, from training to sampling and fusion.

A rank below 4 reaches the kernels as zero padding, not as a code path of its own: the flat training state keeps four
rank slots per module, loading zeroes them and writes the first r, the fused epilogue packs rank r into its 4-wide
`down16` / `up` operands, and saving cuts back to r.  So a rank-r model is right only if the pad slots stay exactly zero
through the LoRA-gradient kernels, the flat AdamW step and lora_pack, and loading and saving put the r live rows where
they belong.  These tests hold that:

- the captured step at ranks 1-3 (both placement pairs, and text / UNet ranks that differ) against fp32 autograd, live
  rows and columns only, at the bound of test_finetune_groups_gpu.py::test_step_vs_autograd;
- three optimiser steps at rank r: every pad of the flat parameters, gradients and AdamW moments, of the forward and
  backward GEMM packs and of the CLIP head pads stays +0.0 as raw bits;
- the padded twin: the rank-r checkpoint zero-padded to rank 4 and trained under `rank: 4` gives bit-identical losses,
  parameters, gradients and moments, and saves the rank-r checkpoint in its first r rows / columns;
- checkpoints at rank r: reference shapes and keys, a bit-exact save -> load -> save, and the refusal of a mismatched one;
- sampling at ranks 1-3 (UNetEngine, CLIPTextEngine, merged weights, test_edlora.py) against the fp32 oracle;
- gradient fusion with concepts of ranks 1, 3 and 4: merges against float64, and every stage bit-identical whether a
  concept is given at rank r or zero-padded to rank 4;
- launch audits of a rank-2 training step, a rank-1 sampling call and a mixed-rank fusion."""
import os
import time

import pytest
import torch
import yaml

from test_finetune_groups import finetune_cfg
from test_trainer_full_gpu import _base_dir, _cos, rel_l2

pytestmark = pytest.mark.gpu

PROMPTS = ['photo of a <c1> <c2>', 'the <c1> <c2> on a beach']
ATT, WB = ('CLIPAttention', 'Attention'), ('CLIPEncoderLayer', 'Transformer2DModel')
# (text rank, UNet rank, placements): ranks 1-3 on both placement pairs, and text / UNet ranks that differ
CASES = [(r, r, w) for r in (1, 2, 3) for w in (ATT, WB)] + [(1, 3, ATT), (3, 1, WB)]


def case_id(c):
    return f'text{c[0]}-unet{c[1]}-{"attention" if c[2] == ATT else "whole_block"}'


def _int(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _assert_zero_bits(t, what):
    n = int(_int(t).ne(0).sum())
    assert n == 0, f'{what}: {n} of {t.numel()} pad values are not +0.0'


def _trainer(base, text_rank, unet_rank, wheres, tok=None):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    cfg = finetune_cfg(True, True, True, *wheres)
    cfg['text_encoder']['lora_cfg']['rank'] = text_rank
    cfg['unet']['lora_cfg']['rank'] = unet_rank
    return EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=cfg, attn_reg_weight=0.05,
                         reg_full_identity=False, use_mask_loss=True, tokenizer=tok or WordTokenizer(),
                         latent_size=(16, 16))


def _data(ref_unet, clip, text_rank, unet_rank, wheres):
    """a rank-r checkpoint (random LoRA with non-zero up) and one batch -> (delta, latents, noise, timesteps, masks)"""
    from oracle import inject
    g = torch.Generator().manual_seed(5)
    d = {'new_concept_embedding': {c: torch.randn(16, 768, generator=g) * 0.02 for c in ('<c1>', '<c2>')},
         'text_encoder': inject.random_lora_state(clip, seed=3, rank=text_rank, where=wheres[0], up_std=0.05),
         'unet': inject.random_lora_state(ref_unet, seed=10, rank=unet_rank, where=wheres[1])}
    B, H = 2, 16
    lat, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    return d, lat, noise, torch.tensor([130, 811]), masks


def pad_to_rank4(lora):
    """rank-r checkpoint tensors -> rank 4 with zero rows (down) / columns (up), 4-D 1x1-conv tensors included"""
    out = {}
    for k, v in lora.items():
        if k.endswith('lora_down.weight'):
            p = v.new_zeros((4,) + tuple(v.shape[1:]))
            p[:v.shape[0]] = v
        else:
            p = v.new_zeros((v.shape[0], 4) + tuple(v.shape[2:]))
            p[:, :v.shape[1]] = v
        out[k] = p
    return out


# ================================================================================================ (a) step vs autograd
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_step_vs_autograd(cuda, tmp_path, case):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle.schedulers import DDPMScheduler
    rt, ru, wheres = case
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    tr = _trainer(base, rt, ru, wheres, tok)
    delta, lat, noise, t, masks = _data(ref_unet, clip, rt, ru, wheres)
    tr.load_delta_state_dict(delta)
    loss = tr(lat, PROMPTS, masks, torch.ones_like(masks), noise=noise, timesteps=t)
    torch.cuda.synchronize()
    ids_concept = tr.get_all_concept_token_ids()
    clip.resize_token_embeddings(49408 + 32)
    emb = clip.get_input_embeddings().weight
    with torch.no_grad():
        emb[49408:49408 + 16] = delta['new_concept_embedding']['<c1>']
        emb[49408 + 16:49408 + 32] = delta['new_concept_embedding']['<c2>']
    for p in list(clip.parameters()) + list(ref_unet.parameters()):
        p.requires_grad_(False)
    emb.requires_grad_(True)
    t_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['text_encoder'].items()}
    u_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['unet'].items()}
    inject.inject_lora(clip, t_leaves, 1.0)
    inject.inject_lora(ref_unet, u_leaves, 1.0)
    ids = tok(bind_concept_prompt(PROMPTS, tr.new_concept_cfg), padding='max_length', max_length=77,
              return_tensors='pt').input_ids
    pos = train_ref.concept_token_positions(ids, 2, ids_concept)
    noisy = DDPMScheduler().add_noise(lat, noise, t)
    # the engines' gradients of the r live rows / columns, in the engines' module order
    ours, order = {'rows': tr.text_engine.emb_grad.flatten().cpu()}, {}
    for name, eng, leaves, r in (('text', tr.text_engine, t_leaves, rt), ('unet', tr.engine, u_leaves, ru)):
        grads = eng.lora_grad_dict()
        assert sorted(f'{m}.lora_{s}.weight' for m in grads for s in ('down', 'up')) == sorted(leaves)
        order[name] = [(m, (r, gd.shape[1]), (gu.shape[0], r)) for m, (gd, gu) in grads.items()]
        ours[name] = torch.cat([x.flatten().cpu() for gd, gu in grads.values() for x in (gd[:r], gu[:, :r])])

    def autograd(bf16):
        for p in [emb, *t_leaves.values(), *u_leaves.values()]:
            p.grad = None
        ctl = AttentionStore(training=True)
        inject.install_control_processors(ref_unet, ctl)
        with torch.autocast('cpu', dtype=torch.bfloat16, enabled=bf16):
            ehs = clip(ids)[0].view(2, 16, 77, 768)
            loss_r, _, _ = train_ref.train_loss(ref_unet, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                                reg_full_identity=False, attn_reg_weight=0.05)
        loss_r.float().backward()
        out = {'rows': emb.grad[49408:49408 + 32].float().flatten().clone()}
        for name, leaves in (('text', t_leaves), ('unet', u_leaves)):
            out[name] = torch.cat([leaves[m + f'.lora_{s}.weight'].grad.float().reshape(shp).flatten()
                                   for m, sd, su in order[name] for s, shp in (('down', sd), ('up', su))])
        return loss_r.item(), out

    loss_bf, g_bf = autograd(True)
    loss_ref, g_ref = autograd(False)
    msg = [f'{case_id(case)}: loss {loss.item():.6f} vs {loss_ref:.6f}']
    assert abs(loss.item() - loss_ref) < 2e-2 * abs(loss_ref)
    for name, g in ours.items():
        r, c = rel_l2(g, g_ref[name]), _cos(g, g_ref[name])
        r_bf, c_bf = rel_l2(g_bf[name], g_ref[name]), _cos(g_bf[name], g_ref[name])
        msg.append(f'{name}: rel-L2 {r:.3e} cos {c:.5f} (bf16 autocast autograd: {r_bf:.3e} / {c_bf:.5f})')
        assert r < max(4e-2, 2 * r_bf) and c > min(0.998, 1 - 2 * (1 - c_bf)), msg[-1]
    print('  ' + ';  '.join(msg))


# ================================================================================================ (b, c, d) training
def _flat_pad_mask(tr, rt, ru):
    """bool mask over the flat state: the rank pads of every LoRA (down rows r..3, up columns r..3) and the CLIP GEMM pads
    (q / k / v up rows and out_proj down columns at the head pads dims d..dh-1 of every head, fc1 up rows and fc2 down
    columns beyond the MLP width) - derived from the layout, not from the engines' own loading code"""
    st = tr.state
    mask = torch.zeros(st.params.numel(), dtype=torch.bool)
    p0 = st.params.data_ptr()
    for eng, r, is_clip in ((tr.engine, ru, False), (tr.text_engine, rt, True)):
        for m, (D, U, _, _, K, N) in eng.lora_views.items():
            md = torch.ones(4, K, dtype=torch.bool)
            md[:r] = False
            mu = torch.ones(N, 4, dtype=torch.bool)
            mu[:, :r] = False
            if is_clip:
                if m.endswith('out_proj'):
                    md[:, torch.arange(K) % eng.dh >= eng.d] = True
                elif m.endswith('fc2'):
                    md[:, eng.I:] = True
                if m.endswith(('q_proj', 'k_proj', 'v_proj')):
                    mu[torch.arange(N) % eng.dh >= eng.d] = True
                elif m.endswith('fc1'):
                    mu[eng.I:] = True
            od, ou = (D.data_ptr() - p0) // 4, (U.data_ptr() - p0) // 4
            mask[od:od + 4 * K] = md.flatten()
            mask[ou:ou + 4 * N] = mu.flatten()
    return mask.to(st.params.device)


def _lora_packs(tr):
    """(label, GEMM pack entry, rank, network) of every forward and backward pack that carries a LoRA term"""
    out = []
    for net, eng, r in (('unet', tr.engine, tr.unet_rank), ('text', tr.text_engine, tr.text_rank)):
        fwd = eng.w.items() if net == 'unet' else [(f'{i}.{k}', e) for i, ent in eng.w.items() for k, e in ent.items()]
        for kind, items in (('fwd', fwd), ('bwd', eng.wb.items())):
            for key, e in items:
                if isinstance(e, dict) and isinstance(e.get('lora_down'), torch.Tensor):
                    out.append((f'{net} {kind} {key}', e, r, net, kind, key))
    return out


def _assert_pads_zero(tr, mask, step):
    st = tr.state
    n = st.params.numel()
    for name, t in (('params', st.params), ('grads', st.grads[:n]), ('exp_avg', st.exp_avg),
                    ('exp_avg_sq', st.exp_avg_sq)):
        _assert_zero_bits(t[mask], f'step {step}: flat {name}')
    assert _int(st.params[~mask]).ne(0).any()
    te = tr.text_engine
    for label, e, r, net, kind, key in _lora_packs(tr):
        down, up = e['lora_down'], e['lora_up']                  # [16, *] 16-bit rows / [*, 4] fp32 columns
        _assert_zero_bits(down[torch.arange(16, device=down.device) % 4 >= r], f'step {step}: {label} lora_down rows')
        _assert_zero_bits(up[:, r:], f'step {step}: {label} lora_up columns')
        if net == 'text' and kind == 'fwd':                       # head / MLP pads of the CLIP packs
            if key.endswith('.qkv'):
                _assert_zero_bits(up[torch.arange(up.shape[0], device=up.device) % te.dh >= te.d], f'{label} head rows')
            elif key.endswith('.out'):
                _assert_zero_bits(down[:, torch.arange(te.Ca, device=up.device) % te.dh >= te.d], f'{label} head cols')
                _assert_zero_bits(up[te.C:], f'{label} rows beyond 768')
            elif key.endswith('.fc1'):
                _assert_zero_bits(up[te.I:], f'{label} rows beyond the MLP width')
            elif key.endswith('.fc2'):
                _assert_zero_bits(down[:, te.I:], f'{label} columns beyond the MLP width')
        if net == 'text' and kind == 'bwd' and key.endswith(('q_proj', 'k_proj', 'v_proj')):
            _assert_zero_bits(down[:, torch.arange(down.shape[1], device=up.device) % te.dh >= te.d], f'{label} head cols')
            _assert_zero_bits(up[te.C:], f'{label} rows beyond 768')


def _state(tr):
    st = tr.state
    return {k: getattr(st, k).clone() for k in ('params', 'grads', 'exp_avg', 'exp_avg_sq')}


def _train3(tr, batch, delta, check_pads=None):
    """load, then 3 x (captured step, flat AdamW, refresh); -> (losses, flat state after every step)"""
    from mos_b200.dp import optimizer_step
    lat, noise, t, masks = batch
    tr.load_delta_state_dict(delta)
    losses, states = [], []
    for step in range(3):
        loss = tr(lat, PROMPTS, masks, torch.ones_like(masks), noise=noise, timesteps=t)
        optimizer_step(tr.state, 1.0)
        tr.refresh()
        torch.cuda.synchronize()
        losses.append(loss.detach().clone())
        states.append(_state(tr))
        if check_pads is not None:
            check_pads(step)
    return losses, states


_RUNS = {}


def _run_pair(case, tmp_path_factory):
    """the rank-r run and its padded rank-4 twin of one case, trained once per module"""
    if case not in _RUNS:
        rt, ru, wheres = case
        base, ref_unet, clip = _base_dir(tmp_path_factory.mktemp('rank'), clip_layers=1)
        delta, lat, noise, t, masks = _data(ref_unet, clip, rt, ru, wheres)
        batch = (lat, noise, t, masks)
        tr = _trainer(base, rt, ru, wheres)
        tr._build(2)
        mask = _flat_pad_mask(tr, rt, ru)
        _assert_pads_zero(tr, mask, 'init')
        pad_checks = []

        def check(step):
            _assert_pads_zero(tr, mask, step)
            pad_checks.append(step)
        losses, states = _train3(tr, batch, delta, check)
        twin = _trainer(base, 4, 4, wheres)
        padded = dict(delta, text_encoder=pad_to_rank4(delta['text_encoder']), unet=pad_to_rank4(delta['unet']))
        t_losses, t_states = _train3(twin, batch, padded)
        _RUNS[case] = dict(tr=tr, twin=twin, losses=losses, states=states, t_losses=t_losses, t_states=t_states,
                           delta=delta, padded=padded, ref_unet=ref_unet, clip=clip, pad_checks=pad_checks, mask=mask)
    return _RUNS[case]


@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_train_loop_keeps_rank_pads_zero(cuda, tmp_path_factory, case):
    run = _run_pair(case, tmp_path_factory)
    assert run['pad_checks'] == [0, 1, 2]
    tr = run['tr']
    packs = _lora_packs(tr)
    assert {(net, kind) for _, _, _, net, kind, _ in packs} == {('unet', 'fwd'), ('unet', 'bwd'), ('text', 'fwd'),
                                                               ('text', 'bwd')}
    # the live slots did train: every LoRA's live rows moved away from the loaded checkpoint
    d = tr.delta_state_dict()
    for part in ('text_encoder', 'unet'):
        moved = sum(not torch.equal(d[part][k], run['delta'][part][k].float()) for k in d[part])
        assert moved == len(d[part]), (part, moved, len(d[part]))
    print(f'  {case_id(case)}: {int(run["mask"].sum())} flat pad values and {len(packs)} LoRA packs +0.0 after 3 steps')


@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_padded_rank4_twin_bit_identical(cuda, tmp_path_factory, case):
    run = _run_pair(case, tmp_path_factory)
    rt, ru, _ = case
    for step, (a, b) in enumerate(zip(run['losses'], run['t_losses'])):
        assert torch.equal(_int(a), _int(b)), f'step {step}: loss {a.item()} vs rank-4 twin {b.item()}'
    for step, (s, ts) in enumerate(zip(run['states'], run['t_states'])):
        for k in s:
            diff = int(_int(s[k]).ne(_int(ts[k])).sum())
            assert diff == 0, f'step {step}: flat {k} differs from the rank-4 twin at {diff} of {s[k].numel()} values'
    d, td = run['tr'].delta_state_dict(), run['twin'].delta_state_dict()
    for part, r in (('text_encoder', rt), ('unet', ru)):
        assert set(td[part]) == set(d[part])
        for k, v in td[part].items():
            live, pad = (v[:r], v[r:]) if k.endswith('lora_down.weight') else (v[:, :r], v[:, r:])
            assert torch.equal(_int(live), _int(d[part][k])), k
            _assert_zero_bits(pad, f'twin checkpoint {k}')
    for c in ('<c1>', '<c2>'):
        assert torch.equal(_int(td['new_concept_embedding'][c]), _int(d['new_concept_embedding'][c]))


@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_checkpoints_at_rank(cuda, tmp_path_factory, tmp_path, case):
    from oracle import inject
    run = _run_pair(case, tmp_path_factory)
    rt, ru, wheres = case
    tr = run['tr']
    d = tr.delta_state_dict()
    for part, model, where, r in (('text_encoder', run['clip'], wheres[0], rt), ('unet', run['ref_unet'], wheres[1], ru)):
        want = inject.random_lora_state(model, rank=r, where=where)      # the reference's module walk and shapes
        assert set(d[part]) == set(want)
        for k, v in want.items():
            assert tuple(d[part][k].shape) == tuple(v.shape), (k, tuple(d[part][k].shape), tuple(v.shape))
    if wheres == WB:
        assert d['unet']['down_blocks.0.attentions.0.proj_in.lora_down.weight'].shape == (ru, 320, 1, 1)
        assert d['unet']['down_blocks.0.attentions.0.proj_in.lora_up.weight'].shape == (320, ru, 1, 1)
    # save -> load -> save, bit for bit
    path = tmp_path / 'edlora.pth'
    torch.save({'params': d}, path)
    tr.load_delta_state_dict(torch.load(path)['params'])
    d2 = tr.delta_state_dict()
    for part in d:
        assert set(d2[part]) == set(d[part])
        for k in d[part]:
            assert torch.equal(_int(d2[part][k]), _int(d[part][k])), k
    # a checkpoint of another rank is refused, and leaves the trained state untouched
    before = _state(tr)
    for part, r in (('text_encoder', rt), ('unet', ru)):
        wrong = dict(d, **{part: pad_to_rank4(d[part])})
        with pytest.raises(ValueError, match=f'{part} LoRA of .*: rank 4, the config trains rank {r}'):
            tr.load_delta_state_dict(wrong)
    after = _state(tr)
    assert all(torch.equal(_int(before[k]), _int(after[k])) for k in before)


# ================================================================================================ (e) sampling
@pytest.mark.parametrize('rank', [1, 2, 3])
@pytest.mark.parametrize('where', ['Attention', 'Transformer2DModel'])
def test_unet_engine_at_rank(cuda, rank, where):
    """fp16 UNetEngine with the fused epilogue vs the fp32 oracle (bound of test_unet_gpu.py), vs merged weights, and
    the LoRA must matter"""
    from mixofshow.utils.convert_edlora_to_diffusers import merge_lora_into_weight
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, ou.TINY)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10 + rank, rank=rank, where=where, up_std=0.05)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    inject.inject_lora(unet, lora, 0.8)
    g = torch.Generator().manual_seed(1)
    B, H = 2, 32
    lat = torch.randn(B, 4, H, H, generator=g)
    ehs = torch.randn(B, 16, 77, 768, generator=g)
    tt = torch.tensor([501.0, 501.0])
    with torch.no_grad():
        ref = unet(lat, tt, ehs).sample
    kw = dict(block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])

    def run(sd_, **k):
        eng = UNetEngine(sd_, B, H, H, **kw, **k)
        nx = len(eng.xattn_names)
        return eng.forward(lat.cuda(), tt.cuda(), ehs_to_layer_major(ehs[:, :nx].cuda(), nx)).clone()
    eps = run(sd, lora=lora, lora_alpha=0.8)
    eps_m = run(sd, lora=lora, lora_alpha=0.8, merge_lora=True)
    eps_w = run(merge_lora_into_weight(sd, lora, 'unet', 0.8))
    base = run(sd)
    torch.cuda.synchronize()
    e, e_m, e_w, e_base = rel_l2(eps, ref), rel_l2(eps, eps_m), rel_l2(eps_w, eps_m), rel_l2(base, ref)
    print(f'  UNet rank {rank} {where}: eps rel-L2 {e:.3e} (without the LoRA {e_base:.3e}); fused vs merge_lora {e_m:.3e}; '
          f'merged state dict vs merge_lora {e_w:.3e}')
    assert e < 5e-3 and e_base > 2 * e
    assert e_m < 5e-3 and e_w < 5e-3


@pytest.mark.parametrize('rank', [1, 2, 3])
@pytest.mark.parametrize('where', ['CLIPAttention', 'CLIPEncoderLayer'])
def test_clip_engine_at_rank(cuda, rank, where):
    """CLIPTextEngine with the fused LoRA vs transformers fp32 (bound of test_clip_gpu.py), and vs merge_lora=True"""
    from transformers import CLIPTextConfig, CLIPTextModel
    from mos_b200.clip_engine import CLIPTextEngine
    from oracle import inject
    torch.manual_seed(0)
    model = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                                         num_attention_heads=12, max_position_embeddings=77)).eval()
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    lora = inject.random_lora_state(model, seed=7 + rank, rank=rank, where=where, up_std=0.05)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 49407, (16, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 9:] = 49407
    inject.inject_lora(model, lora, 0.8)
    with torch.no_grad():
        ref = model(ids)[0]
    out = CLIPTextEngine(sd, 16, lora=lora, lora_alpha=0.8)(ids)
    out_m = CLIPTextEngine(sd, 16, lora=lora, lora_alpha=0.8, merge_lora=True)(ids)
    base = CLIPTextEngine(sd, 16)(ids)
    torch.cuda.synchronize()
    e, e_m, e_fm, e_base = rel_l2(out, ref), rel_l2(out_m, ref), rel_l2(out, out_m), rel_l2(base, ref)
    print(f'  CLIP rank {rank} {where}: rel-L2 {e:.3e} (merged {e_m:.3e}, fused vs merged {e_fm:.3e}, '
          f'without the LoRA {e_base:.3e})')
    assert e < 2e-2 and e_m < 2e-2 and e_fm < 2e-2 and e_base > 2 * e


def test_test_edlora_rank2_checkpoint(cuda, tmp_path):
    """`test_edlora.py -opt` samples a rank-2 checkpoint on the synthetic model directory; the pipeline it loads
    (load_pipeline: the LoRA merged at alpha) matches the fp32 oracle with the rank-2 LoRA injected after the first step
    of a 50-step schedule, per sample of a 4-prompt CFG call (test_validation_sampling_gpu.py's bound)"""
    import test_edlora
    from synth import make_pretrained_dir
    from test_validation_sampling_gpu import _val_vis, random_edlora_checkpoint
    from mixofshow.utils import model_io
    from oracle import edlora_ref as er
    from oracle import inject
    from oracle import unet as ou
    from oracle.schedulers import DPMSolverMultistepScheduler
    base = make_pretrained_dir(str(tmp_path / 'base'))
    ckpt = random_edlora_checkpoint(base, str(tmp_path / 'edlora_rank2.pth'), seed=1, rank=2)
    lora = torch.load(ckpt)['params']
    assert {v.shape[1] for k, v in lora['unet'].items() if 'lora_up' in k} == {2}
    vis = tmp_path / 'vis'
    opt = {'name': 'rank2', 'manual_seed': 0, 'datasets': {'val_vis': _val_vis(n_samples=1)},
           'models': {'pretrained_path': base, 'enable_edlora': True},
           'path': {'lora_path': ckpt, 'visualization': str(vis)},
           'val': {'compose_visualize': False, 'alpha_list': [0.7], 'sample': {'num_inference_steps': 2,
                                                                              'guidance_scale': 7.5}}}
    yml = tmp_path / 'test.yml'
    yml.write_text(yaml.safe_dump(opt))
    test_edlora.main(['-opt', str(yml)])
    pngs = sorted(os.listdir(vis / 'PromptDataset' / 'validation_edlora_0.7'))
    assert len(pngs) == 3 and all(p.endswith('---validation_edlora_0.7.png') for p in pngs)
    # the pipeline test_edlora.main sampled with, against the oracle loop
    pipe = test_edlora.load_pipeline(base, ckpt, 0.7)
    ref = ou.build_unet(0, ou.TINY)            # the synthetic directory's topology
    ref.load_state_dict(model_io.load_unet(base).state_dict())
    inject.install_edlora_processors(ref)
    inject.inject_lora(ref, lora['unet'], 0.7)
    n = 4
    lat = torch.randn(n, 4, 32, 32, generator=torch.Generator().manual_seed(3))
    pe = torch.randn(n, 16, 77, 768, generator=torch.Generator().manual_seed(4))
    ne = torch.randn(n, 77, 768, generator=torch.Generator().manual_seed(5))
    first = []
    pipe(prompt_embeds=pe.cuda(), negative_prompt_embeds=ne.cuda(), latents=lat.clone(), height=64, width=64,
         num_inference_steps=50, guidance_scale=7.5, output_type='latent',
         callback=lambda i, t, x: first.append(x.clone()) if i == 0 else None)     # the tiny VAE is one 2x level
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(50)
    t0 = int(sched.timesteps[0])
    emb = torch.cat([ne.view(n, 1, 77, 768).repeat(1, 16, 1, 1), pe])
    with torch.no_grad():
        eps = ref(torch.cat([lat, lat]), torch.tensor([t0] * 2 * n), emb).sample
    want = sched.step(er.cfg_combine(eps, 7.5), t0, lat).prev_sample
    errs = [rel_l2(first[0][i], want[i]) for i in range(n)]
    print(f'  test_edlora.py rank-2 checkpoint: per-sample latents rel-L2 after step 1: {errs}')
    assert max(errs) < 1e-3


# ================================================================================================ (f) gradient fusion
FUSION_RANKS = [1, 3, 4]


def _merge_bound(W0, down, up, alpha):
    """float64 W0 + alpha up @ down and the fp32 rounding bound of its evaluation (r + 2 roundings per element)"""
    d, u = down.double().reshape(down.shape[0], -1), up.double().reshape(up.shape[0], -1)
    ref = W0.double().reshape(W0.shape[0], -1) + alpha * (u @ d)
    mag = W0.double().abs().reshape(W0.shape[0], -1) + abs(alpha) * (u.abs() @ d.abs())
    return ref, (d.shape[0] + 2) * 2.0 ** -24 * mag


@pytest.mark.parametrize('rank', FUSION_RANKS)
def test_merges_vs_float64(cuda, rank):
    import gradient_fusion as gf
    from oracle import inject
    from oracle import unet as ou
    u0 = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in u0.state_dict().items()}
    lora = inject.random_lora_state(u0, seed=30 + rank, rank=rank, where='Transformer2DModel', up_std=0.05)
    names = sorted(k.replace('.lora_down', '') for k in lora if 'lora_down' in k)
    assert any(sd[n].ndim == 4 for n in names)
    out = gf.merge_lora_into_weight(sd, lora, names, 'unet', 0.7, 'cuda')
    worst = 0.0
    for n in names:
        dn, up = lora[n.replace('.weight', '.lora_down.weight')], lora[n.replace('.weight', '.lora_up.weight')]
        ref, bound = _merge_bound(sd[n], dn, up, 0.7)
        got = out[n].cpu()
        assert got.shape == sd[n].shape
        err = (got.double().reshape(ref.shape) - ref).abs()
        assert bool((err <= bound).all()), n
        worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
        Wc = gf._merged(sd[n], dn, up, 0.7, 'cuda').cpu()
        assert torch.equal(Wc.reshape(ref.shape), got.reshape(ref.shape)), n          # one kernel, one result
    print(f'  rank {rank}: {len(names)} merged weights, worst error / bound {worst:.3f}')


def _cross_kv_case(ranks, seed=21):
    g = torch.Generator().manual_seed(seed)
    C, D = 320, 768
    names = [(0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight'),
             (0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_v.weight'),
             (1, 'down_blocks.0.attentions.1.transformer_blocks.0.attn2.to_k.weight')]
    sd = {n: torch.randn(C, D, generator=g) * D ** -0.5 for _, n in names}
    feats = [{l: torch.randn(6, D, generator=g) for l in (0, 1)} for _ in ranks]
    tuned = []
    for r in ranks:
        t = {}
        for _, n in names:
            dn = n.replace('.weight', '.lora_down.weight')
            t[dn] = torch.randn(r, D, generator=g) * D ** -0.5
            t[dn.replace('lora_down', 'lora_up')] = torch.randn(C, r, generator=g) * 0.1
        tuned.append(t)
    return sd, names, feats, tuned


def _same_weights(a, b, what):
    assert set(a) == set(b), what
    for k in a:
        assert torch.equal(_int(a[k].float().contiguous()), _int(b[k].float().contiguous())), f'{what}: {k}'


def test_cross_kv_fusion_mixed_ranks(cuda):
    """concepts of ranks 1, 3 and 4: bit-identical to the same concepts zero-padded to rank 4, and against the
    reference's construction (test_fusion_gpu.py's bounds)"""
    from gradient_fusion import merge_kv_in_cross_attention
    from oracle import edlora_ref as er
    sd, names, feats, tuned = _cross_kv_case(FUSION_RANKS)
    alphas, iters = [1.0, 0.7, 1.3], 200
    new_w = merge_kv_in_cross_attention(sd, names, feats, tuned, alphas, iters, device='cuda')
    padded = merge_kv_in_cross_attention(sd, names, feats, [pad_to_rank4(t) for t in tuned], alphas, iters, device='cuda')
    _same_weights(new_w, padded, 'cross-K/V stage, rank r vs zero-padded rank 4')
    for layer_idx, n in names:
        dn = n.replace('.weight', '.lora_down.weight')
        X = torch.cat([feats[c][layer_idx] for c in range(3)], 0)
        V = torch.cat([(((sd[n] + alphas[c] * tuned[c][dn.replace('lora_down', 'lora_up')] @ tuned[c][dn])
                         @ feats[c][layer_idx].T).T) for c in range(3)], 0)
        Wref = er.update_quasi_newton(X, V, sd[n].clone(), iters)
        Wn = new_w[n]
        r0 = (X @ sd[n].t() - V).norm().item()
        rr, rn = (X @ Wref.t() - V).norm().item(), (X @ Wn.t() - V).norm().item()
        e_w, e_d = rel_l2(Wn, Wref), rel_l2(Wn - sd[n], Wref - sd[n])
        print(f'  mixed-rank cross-KV {n.split(".")[-2]}[{layer_idx}]: W rel-Frob {e_w:.2e}, update {e_d:.2e}; '
              f'residual ours {rn:.3e} reference {rr:.3e} start {r0:.3e}')
        assert e_w < 5e-4 and e_d < 5e-2
        assert rn <= max(rr * 1.02, 1e-5 * r0)


def _text_case(ranks):
    from transformers import CLIPTextConfig, CLIPTextModel
    from oracle import inject
    cfg = CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                         num_attention_heads=12, max_position_embeddings=77, eos_token_id=999, bos_token_id=998,
                         pad_token_id=999)
    torch.manual_seed(0)
    base = CLIPTextModel(cfg).eval()
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    loras = [inject.random_lora_state(base, seed=40 + c, rank=r, where='CLIPEncoderLayer', up_std=0.05)
             for c, r in enumerate(ranks)]
    g = torch.Generator().manual_seed(9)
    prompts = [[torch.cat([torch.tensor([998]), torch.randint(0, 990, (n,), generator=g), torch.tensor([999])])
                for n in (5, 2, 5, 2)] for _ in ranks]
    return sd, loras, prompts


def test_text_encoder_fusion_rank_r_equals_padded(cuda):
    from gradient_fusion import merge_text_encoder
    sd, loras, prompts = _text_case(FUSION_RANKS)
    alphas = [1.0, 0.7, 0.9]
    a = merge_text_encoder(sd, loras, alphas, prompts, 10, pad_id=999)
    b = merge_text_encoder(sd, [pad_to_rank4(l) for l in loras], alphas, prompts, 10, pad_id=999)
    assert len(a) == 2 * 6
    _same_weights(a, b, 'text-encoder stage, rank r vs zero-padded rank 4')


def _spatial_case(ranks):
    from oracle import inject
    from oracle import unet as ou
    u0 = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in u0.state_dict().items()}
    loras = [inject.random_lora_state(u0, seed=10 + c, rank=r, where='Transformer2DModel', up_std=0.05)
             for c, r in enumerate(ranks)]
    spatial = [{k: v for k, v in l.items() if 'attn2.to_k' not in k and 'attn2.to_v' not in k} for l in loras]
    embeds = [torch.randn(1, 16, 77, 768, generator=torch.Generator().manual_seed(20 + c)) for c in range(len(ranks))]
    return sd, spatial, embeds


def test_spatial_fusion_rank_r_equals_padded(cuda):
    from gradient_fusion import merge_spatial_attention
    from oracle import unet as ou
    sd, spatial, embeds = _spatial_case(FUSION_RANKS)
    kw = dict(latent_hw=(16, 16), num_inference_steps=2, seed=0, block_out=ou.TINY['block_out_channels'], layers=1)
    a = merge_spatial_attention(sd, spatial, [1.0, 0.8, 1.0], embeds, 5, **kw)
    b = merge_spatial_attention(sd, [pad_to_rank4(l) for l in spatial], [1.0, 0.8, 1.0], embeds, 5, **kw)
    assert len(a) == 4 * 10
    _same_weights(a, b, 'spatial stage, rank r vs zero-padded rank 4')


# ================================================================================================ (g) launch audits
AUDIT_T0 = time.time()


def test_rank2_training_step_audited(cuda):
    """a rank-2 TrainEngine step (tiny topology, 16 x 16, B = 2, whole-block LoRA, regulariser on) and its optimiser step
    (AdamW + lora_pack) under the GEMM, attention and norm / elementwise launch audits"""
    import attention_audit
    import gemm_audit
    import norm_audit
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import inject
    from oracle import unet as ou
    ref = ou.build_unet(0, ou.TINY)
    lora = inject.random_lora_state(ref, seed=10, rank=2, where='Transformer2DModel')
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    B, H = 2, 16
    x0, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    eng = TrainEngine(sd, B, H, H, lora=lora, attn_reg_weight=0.05, where='Transformer2DModel',
                      block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'], use_graph=False)
    n_x = len(eng.xattn_names)
    ehs = torch.randn(B, n_x, 77, 768, generator=g)
    masks = torch.zeros(B, 1, H, H)
    masks[:, :, 3:12, 4:13] = 1
    packed = [e[k] for e in eng.w.values() if isinstance(e, dict) for k in ('lora_down', 'lora_up')
              if isinstance(e.get(k), torch.Tensor)]
    failures = []
    for mod in (gemm_audit, attention_audit, norm_audit):
        stats = gemm_audit.Stats()
        with mod.Recorder(stats):
            eng.forward_backward(x0.cuda(), noise.cuda(), torch.tensor([77, 640]).cuda(),
                                 ehs_to_layer_major(ehs.cuda(), n_x), masks.cuda(), token_pos=[[4, 5], [6, 7]])
            torch.cuda.synchronize()
        with mod.Recorder(stats) as rec:
            rec.register(eng.state.params, *eng._lora_keep, *packed)
            eng.optimizer_step()
            torch.cuda.synchronize()
        assert stats.rows, mod.__name__
        print(f'\nrank-2 training step, {mod.__name__}\n' + stats.table())
        failures += stats.failures
    assert not failures, '\n'.join(failures[:30])


def test_rank1_sampling_audited(cuda):
    """a rank-1 fp16 sampling call at 64 x 64 (tiny topology, CFG batch 2, fused attention LoRA) under the GEMM,
    attention and norm / elementwise launch audits"""
    import attention_audit
    import gemm_audit
    import norm_audit
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    lora = inject.random_lora_state(unet, seed=10, rank=1, up_std=0.05)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(1, 4, 64, 64, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    eng = UNetEngine(sd, 2, 64, 64, lora=lora, lora_alpha=1.0, use_graph=False,
                     block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    nx = len(eng.xattn_names)
    failures = []
    for mod in (gemm_audit, attention_audit, norm_audit):
        stats = gemm_audit.Stats()
        with mod.Recorder(stats):
            eng.forward(torch.cat([lat, lat]).cuda(), torch.tensor([981.0, 981.0]).cuda(),
                        ehs_to_layer_major(ehs[:, :nx].cuda(), nx))
            torch.cuda.synchronize()
        assert stats.rows, mod.__name__
        print(f'\nrank-1 sampling, {mod.__name__}\n' + stats.table())
        failures += stats.failures
    assert not failures, '\n'.join(failures[:30])


def test_mixed_rank_fusion_audited(cuda):
    """the cross-K/V and text-encoder stages with concepts of ranks 1, 3 and 4 under the solver launch audit (lora_merge
    loops over each concept's own rank)"""
    import solver_audit as sa
    from gradient_fusion import merge_kv_in_cross_attention, merge_text_encoder
    stats = sa.Stats()
    sd, names, feats, tuned = _cross_kv_case(FUSION_RANKS)
    with sa.Recorder(stats):
        merge_kv_in_cross_attention(sd, names, feats, tuned, [1.0, 0.7, 1.3], 20, device='cuda')
        torch.cuda.synchronize()
    tsd, loras, prompts = _text_case(FUSION_RANKS)
    with sa.Recorder(stats):
        merge_text_encoder(tsd, loras, [1.0, 0.7, 0.9], prompts, 10, pad_id=999)
        torch.cuda.synchronize()
    print(f'\nmixed-rank fusion ({time.time() - AUDIT_T0:.0f} s of audits)\n' + stats.table())
    assert 'lora_merge' in stats.rows
    assert not stats.failures, '\n'.join(stats.failures[:30])
