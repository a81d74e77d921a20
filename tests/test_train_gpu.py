"""One ED-LoRA training step (forward, loss incl. attention regulariser, backward, AdamW) on the GPU engine vs the
fp32 oracle differentiated by torch.autograd (oracle/unet.py + oracle/train_ref.py, the latter pinned against the
reference's cal_attn_reg golden).

Tolerances: the forward is bf16 (eps rel-L2 <= 2e-2 as in test_unet_gpu); gradients pass through ~2x as many bf16
GEMMs, so per-tensor LoRA gradients are compared at rel-L2 <= 8e-2 and the whole flat gradient at cosine >= 0.995.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def _setup(reg_weight, full_identity, seed=0):
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
    loss, pred, attn = train_ref.train_loss(ref, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                            reg_full_identity=full_identity, attn_reg_weight=reg_weight)
    loss.backward()
    ehs_grad, ehs = ehs.grad.detach(), ehs.detach()
    return dict(ref=ref, lora=lora, leaves=leaves, alpha=alpha, n_layers=n_layers, x0=x0, noise=noise, t=t, ehs=ehs,
                ehs_grad=ehs_grad,
                masks=masks, pos=pos, loss=loss.detach(), pred=pred.detach(), attn=attn)


@pytest.mark.parametrize('reg_weight,full', [(None, True), (0.05, True), (0.05, False)])
def test_train_step_vs_oracle_autograd(cuda, reg_weight, full):
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import unet as ou
    S = _setup(reg_weight, full)
    eng = TrainEngine({k: v.detach() for k, v in S['ref'].state_dict().items()}, 2, 16, 16, lora=S['lora'],
                      lora_alpha=S['alpha'], attn_reg_weight=reg_weight, reg_full_identity=full,
                      block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    out = eng.forward_backward(S['x0'].cuda(), S['noise'].cuda(), S['t'].cuda(),
                               ehs_to_layer_major(S['ehs'].cuda(), S['n_layers']), S['masks'].cuda(), token_pos=S['pos'])
    torch.cuda.synchronize()
    e_pred = rel_l2(eng.out_eps, S['pred'])
    loss = out[0].item()
    print(f'[reg={reg_weight} full={full}] eps rel-L2 {e_pred:.3e}; loss {loss:.6f} vs oracle {S["loss"].item():.6f}'
          f' (attn {out[1].item():.6f} vs {0.0 if S["attn"] is None else S["attn"].item():.6f})')
    assert e_pred < 2e-2
    assert abs(loss - S['loss'].item()) < 2e-2 * abs(S['loss'].item())
    if reg_weight is not None:
        assert abs(out[1].item() - S['attn'].item()) < 3e-2 * abs(S['attn'].item())
    grads = eng.lora_grad_dict()
    flat_g, flat_r, worst = [], [], (0.0, '')
    for m, (gD, gU) in grads.items():
        rD = S['leaves'][m + '.lora_down.weight'].grad
        rU = S['leaves'][m + '.lora_up.weight'].grad
        for tag, a, b in (('down', gD, rD), ('up', gU, rU)):
            e = rel_l2(a, b)
            if e > worst[0]:
                worst = (e, f'{m}.{tag}')
            flat_g.append(a.flatten().cpu())
            flat_r.append(b.flatten())
    fg, fr = torch.cat(flat_g), torch.cat(flat_r)
    cos = torch.nn.functional.cosine_similarity(fg, fr, dim=0).item()
    print(f'    flat LoRA gradient: rel-L2 {rel_l2(fg, fr):.3e}, cosine {cos:.5f}; worst tensor {worst[1]} {worst[0]:.3e}')
    assert cos > 0.9995 and rel_l2(fg, fr) < 2e-2     # measured 8e-3 (bf16 activations, fp32 accumulation)
    assert worst[0] < 5e-2


def test_optimizer_step_changes_forward(cuda):
    """AdamW on the flat state + re-pack: the next forward sees the updated LoRA; parameters follow torch.optim.AdamW."""
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import unet as ou
    S = _setup(None, True)
    eng = TrainEngine({k: v.detach() for k, v in S['ref'].state_dict().items()}, 2, 16, 16, lora=S['lora'],
                      lora_alpha=S['alpha'], attn_reg_weight=None, lr=1e-3,
                      block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    args = (S['x0'].cuda(), S['noise'].cuda(), S['t'].cuda(), ehs_to_layer_major(S['ehs'].cuda(), S['n_layers']),
            S['masks'].cuda())
    l0 = eng.forward_backward(*args)[0].item()
    p0 = eng.state.params.clone()
    g0 = eng.state.grads[:eng.state.n].clone()
    eng.optimizer_step()
    ref_p = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref_p], lr=1e-3, weight_decay=0.01)
    ref_p.grad = g0.clone()
    opt.step()
    assert rel_l2(eng.state.params, ref_p.detach()) < 1e-5
    losses = [l0]
    for _ in range(5):
        losses.append(eng.forward_backward(*args)[0].item())
        eng.optimizer_step()
    print('    loss over 6 steps on a fixed batch:', ' '.join(f'{l:.5f}' for l in losses))
    assert losses[-1] < losses[0]


def test_train_step_full_sd15_topology(cuda):
    """BASELINE config 2 shape (SD1.5 topology, 64x64 latents; batch 2 here): loss and flat LoRA gradient vs the fp32
    oracle differentiated by autograd — the oracle runs on the GPU in true fp32 (TF32 off, conftest) to finish in
    seconds.  All 16 cross-attention layers feed the attention regulariser (4 resolution groups, as the reference)."""
    from mixofshow.utils.ptp_util import AttentionStore
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import inject, train_ref
    from oracle import unet as ou
    from oracle.schedulers import DDPMScheduler
    ref = ou.build_unet(0)
    lora = inject.random_lora_state(ref, seed=10)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    ref = ref.cuda()
    leaves = {k: v.clone().cuda().requires_grad_(True) for k, v in lora.items()}
    inject.inject_lora(ref, leaves, 1.0)
    ctl = AttentionStore(training=True)
    assert inject.install_control_processors(ref, ctl) == 16
    g = torch.Generator().manual_seed(5)
    B, H = 2, 64
    x0, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([77, 640])
    ehs = torch.randn(B, 16, 77, 768, generator=g).to(torch.bfloat16).float()
    masks = torch.zeros(B, 1, H, H)
    masks[:, :, 12:50, 16:44] = 1.0
    pos = [[4, 5], [2, 3]]
    noisy = DDPMScheduler().add_noise(x0, noise, t)
    loss, pred, attn = train_ref.train_loss(ref, ctl, noisy.cuda(), t.cuda(), ehs.cuda(), noise.cuda(), masks.cuda(),
                                            masks.cuda(), pos, reg_full_identity=True, attn_reg_weight=0.01)
    loss.backward()
    ref_grads = {k: v.grad.detach().clone() for k, v in leaves.items()}
    del ref, ctl, pred
    torch.cuda.empty_cache()
    eng = TrainEngine(sd, B, H, H, lora=lora, lora_alpha=1.0, attn_reg_weight=0.01, reg_full_identity=True)
    out = eng.forward_backward(x0.cuda(), noise.cuda(), t.cuda(), ehs_to_layer_major(ehs.cuda()), masks.cuda(),
                               token_pos=pos)
    torch.cuda.synchronize()
    print(f'full SD1.5 train step: loss {out[0].item():.6f} vs oracle {loss.item():.6f}; attn {out[1].item():.6f} vs '
          f'{attn.item():.6f}')
    assert abs(out[0].item() - loss.item()) < 2e-2 * abs(loss.item())
    assert abs(out[1].item() - attn.item()) < 3e-2 * abs(attn.item())
    fg, fr = [], []
    for m, (gD, gU) in eng.lora_grad_dict().items():
        fg += [gD.flatten(), gU.flatten()]
        fr += [ref_grads[m + '.lora_down.weight'].flatten(), ref_grads[m + '.lora_up.weight'].flatten()]
    fg, fr = torch.cat(fg), torch.cat(fr)
    cos = torch.nn.functional.cosine_similarity(fg, fr, dim=0).item()
    print(f'    flat LoRA gradient ({fg.numel()} params): rel-L2 {rel_l2(fg, fr):.3e}, cosine {cos:.5f}')
    assert fg.numel() == 797184                      # SURVEY.md §8a: UNet `where: Attention` rank-4 parameter count
    assert cos > 0.9995 and rel_l2(fg, fr) < 2e-2     # measured 8e-3 on the full topology
    # timing of the step (forward + loss + backward in one CUDA graph, + AdamW + LoRA re-pack)
    import time
    for _ in range(2):
        eng.forward_backward(x0.cuda(), noise.cuda(), t.cuda(), ehs_to_layer_major(ehs.cuda()), masks.cuda())
        eng.optimizer_step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        eng.forward_backward(x0.cuda(), noise.cuda(), t.cuda(), ehs_to_layer_major(ehs.cuda()), masks.cuda())
        eng.optimizer_step()
    torch.cuda.synchronize()
    print(f'    train step (B={B}, CUDA graph): {(time.perf_counter() - t0) / 5 * 1e3:.1f} ms')


def _tiny_trainer(reg=0.01, lr=1e-3, seed=0, lora_state=None):
    from mixofshow.pipelines.trainer_edlora import UNetLoRATrainer
    from oracle import unet as ou
    ref = ou.build_unet(0, ou.TINY)
    cfg = {'text_embedding': {'enable_tuning': False}, 'text_encoder': {'enable_tuning': False},
           'unet': {'enable_tuning': True, 'lr': lr, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}}}
    concept = {'<TOK>': {'concept_token_ids': list(range(49408, 49440)),
                         'concept_token_names': [f'<new{i}>' for i in range(32)]}}
    tr = UNetLoRATrainer({k: v.detach() for k, v in ref.state_dict().items()}, 2, new_concept_cfg=concept,
                       finetune_cfg=cfg, attn_reg_weight=reg, latent_size=(16, 16), seed=seed, lora_state=lora_state,
                       unet_topology=dict(block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block']))
    return tr, ref


def _batches(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ids = torch.full((2 * 4, 77), 49407, dtype=torch.long)
        ids[:, 0] = 49406
        for b in range(2):
            for l in range(4):
                ids[b * 4 + l, 2 + b] = 49408 + l
                ids[b * 4 + l, 5] = 49424 + l
        m = (torch.rand(2, 1, 16, 16, generator=g) > 0.5).float()
        m[:, :, 0, 0] = 0
        out.append(dict(latents=torch.randn(2, 4, 16, 16, generator=g),
                        encoder_hidden_states=torch.randn(2, 4, 77, 768, generator=g), masks=m,
                        img_masks=torch.ones(2, 1, 16, 16), text_input_ids=ids))
    return out


def test_trainer_mirror_loop_and_checkpoint(cuda):
    """EDLoRATrainer / train() mirrors (trainer_edlora.py, train_edlora.py:105-158): checkpoint keys of the reference
    recipe, linear LR decay, loss goes down on a repeated batch, delta_state_dict round trip."""
    import train_edlora as te
    from oracle import inject
    tr, ref = _tiny_trainer()
    d0 = tr.delta_state_dict()
    want = inject.lora_target_modules(ref)
    assert sorted(d0['unet']) == sorted([f'{n}.lora_{s}.weight' for n in want for s in ('down', 'up')])
    assert all(v.abs().max().item() == 0 for k, v in d0['unet'].items() if k.endswith('lora_up.weight'))   # edlora.py:239
    assert d0['new_concept_embedding'] == {} and d0['text_encoder'] == {}
    data = _batches(1) * 8
    lrs = []
    losses = te.train(tr, data, dataset_len=16, batch_size_per_gpu=2, print_freq=1,
                      log=lambda s: lrs.append(float(s.split('lr ')[1])))
    assert len(losses) == 8                                   # total_iter = 16 / (2 * 1 * 1)
    assert lrs == pytest.approx([1e-3 * (8 - k) / 8 for k in range(8)], rel=1e-3)
    print('    trainer loop losses:', ' '.join(f'{l:.4f}' for l in losses))
    d1 = tr.delta_state_dict()
    assert any(v.abs().max().item() > 0 for k, v in d1['unet'].items() if k.endswith('lora_up.weight'))
    # round trip into a fresh trainer: identical loss on a fixed batch / noise / timesteps
    tr2, _ = _tiny_trainer(seed=7)
    tr2.load_delta_state_dict(d1)
    b = data[0]
    noise, t = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(1)), torch.tensor([10, 700])
    la = tr(b['latents'], b['encoder_hidden_states'], b['masks'], b['img_masks'], text_input_ids=b['text_input_ids'],
            noise=noise, timesteps=t).item()
    lb = tr2(b['latents'], b['encoder_hidden_states'], b['masks'], b['img_masks'], text_input_ids=b['text_input_ids'],
             noise=noise, timesteps=t).item()
    assert la == lb


def test_gradient_accumulation(cuda):
    tr, _ = _tiny_trainer(reg=None)
    b1, b2 = _batches(2, seed=9)
    noise, t = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(1)), torch.tensor([10, 700])
    kw = dict(noise=noise, timesteps=t)
    n = tr.engine.state.n
    tr(b1['latents'], b1['encoder_hidden_states'], b1['masks'], b1['img_masks'], **kw)
    g1 = tr.engine.state.grads[:n].clone()
    tr(b2['latents'], b2['encoder_hidden_states'], b2['masks'], b2['img_masks'], **kw)
    g2 = tr.engine.state.grads[:n].clone()
    tr(b1['latents'], b1['encoder_hidden_states'], b1['masks'], b1['img_masks'], **kw)
    tr(b2['latents'], b2['encoder_hidden_states'], b2['masks'], b2['img_masks'], accumulate=True, **kw)
    assert rel_l2(tr.engine.state.grads[:n], g1 + g2) < 1e-6
    tr(b1['latents'], b1['encoder_hidden_states'], b1['masks'], b1['img_masks'], **kw)
    tr(b2['latents'], b2['encoder_hidden_states'], b2['masks'], b2['img_masks'], accumulate=True, **kw)   # graph replay
    assert rel_l2(tr.engine.state.grads[:n], g1 + g2) < 1e-6


@pytest.mark.parametrize('reg_weight', [None, 0.05])
def test_text_embedding_gradient(cuda, reg_weight):
    """d loss / d(encoder_hidden_states) out of the UNet backward (SURVEY.md 8d config 2: "ehs ... with grad"): the input
    gradient of the 16 text K / V projections (incl. their LoRA term), laid out like `in_ehs` so that it is the text
    encoder's output gradient.  vs autograd on the fp32 oracle; bf16 operands: rel-L2 <= 3e-2, cosine >= 0.999."""
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import unet as ou
    S = _setup(reg_weight, True)
    eng = TrainEngine({k: v.detach() for k, v in S['ref'].state_dict().items()}, 2, 16, 16, lora=S['lora'],
                      lora_alpha=S['alpha'], attn_reg_weight=reg_weight, reg_full_identity=True, text_grad=True,
                      block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    eng.forward_backward(S['x0'].cuda(), S['noise'].cuda(), S['t'].cuda(),
                         ehs_to_layer_major(S['ehs'].cuda(), S['n_layers'], torch.bfloat16), S['masks'].cuda(),
                         token_pos=S['pos'])
    torch.cuda.synchronize()
    nl = S['n_layers']
    got = eng.d_ehs[:, :768].float().view(nl, 2, 77, 768).cpu()
    ref = S['ehs_grad'].permute(1, 0, 2, 3)
    e = rel_l2(got, ref)
    cos = torch.nn.functional.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
    print(f'[reg={reg_weight}] d(ehs): rel-L2 {e:.3e}, cosine {cos:.5f}')
    assert eng.d_ehs[:, 768:].abs().max().item() == 0.0
    assert e < 3e-2 and cos > 0.999
