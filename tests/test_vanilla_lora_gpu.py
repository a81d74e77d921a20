"""Vanilla LoRA (`enable_edlora: false`) on the GPU: one text-encoder pass per sample, one [b, 77, 768] embedding read by
all 16 cross-attention layers, d(text embedding) summed over the layers in fp32 (TrainEngine(shared_ehs=True)).

- the captured step of EDLoRATrainer(enable_edlora=False) for all seven parameter-group subsets against fp32 autograd
  through transformers' CLIPTextModel over b sequences chained into the oracle UNet with the 3-D embedding (LoRA
  gradients rel-L2 <= 1e-2, concept rows <= max(4e-2, 2 x the bf16-autocast error), each widened only to twice the error
  bf16 autocast alone puts into the same autograd run);
- equivalence with ED-LoRA: fed one copy of the embedding per cross-attention layer, the ED-LoRA engine's loss and
  UNet-LoRA gradients are bit-identical to the vanilla engine's, and its bf16 d(ehs) slices summed in float64 match the
  fp32 accumulator;
- the captured vanilla step is bit-identical to its eager walk;
- the vanilla training step and a StableDiffusionPipeline call pass the GEMM / attention / norm launch audits;
- `train_edlora.py -opt` with `enable_edlora: false` end to end: lora_model-*.pth, reload, convert_edlora(enable_edlora=
  False) into StableDiffusionPipeline, CFG-7.5 latents of the first step of a 50-step schedule within 1e-3 of the fp32
  oracle (the target of test_unet_gpu.py)."""
import os

import pytest
import torch
import yaml

from test_finetune_groups import COMBOS, combo_id, finetune_cfg
from test_trainer_full_gpu import _base_dir, _cos, batch_inputs, rel_l2

pytestmark = pytest.mark.gpu

PROMPTS = ['photo of a <new0> <new1>', 'the <new0> <new1> on a beach']
BF16_U = 2.0 ** -8                       # unit roundoff of bf16 (8 significand bits)


def _trainer(base, combo, tok=None, latent=16):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', False, finetune_cfg=finetune_cfg(*combo),
                         attn_reg_weight=0.05, reg_full_identity=False, use_mask_loss=True,
                         tokenizer=tok or WordTokenizer(), latent_size=(latent, latent))


def _data(ref_unet, clip, combo, B=2):
    """-> delta, prompts, latents, noise, timesteps, masks; at B != 2 the per-sample batch of test_trainer_full_gpu"""
    from oracle import inject
    g = torch.Generator().manual_seed(5)
    d = {'new_concept_embedding': {c: torch.randn(1, 768, generator=g) * 0.02 for c in ('<c1>', '<c2>')},
         'text_encoder': {}, 'unet': {}}
    if combo[1]:
        d['text_encoder'] = inject.random_lora_state(clip, seed=3, where='CLIPAttention', up_std=0.05)
    if combo[2]:
        d['unet'] = inject.random_lora_state(ref_unet, seed=10)
    if B != 2:
        return (d, *batch_inputs(B, seed=50 + B, words=('<new0>', '<new1>')))
    H = 16
    lat, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    return d, PROMPTS, lat, noise, torch.tensor([130, 811]), masks


ALL_GROUPS = (True, True, True)
# every group subset at B = 2, and all three groups at the other batch sizes (the B = 2 ids stay the combo's)
STEP_CASES = [(2, c) for c in COMBOS] + [(b, ALL_GROUPS) for b in (1, 3, 4)]


@pytest.mark.parametrize('B,combo', STEP_CASES,
                         ids=[combo_id(c) if b == 2 else f'{combo_id(c)}-B{b}' for b, c in STEP_CASES])
def test_vanilla_step_vs_autograd(cuda, tmp_path, B, combo):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle.schedulers import DDPMScheduler
    emb_on, text_on, unet_on = combo
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    tr = _trainer(base, combo, tok)
    assert tr.get_all_concept_token_ids() == [49408, 49409]
    delta, prompts, lat, noise, t, masks = _data(ref_unet, clip, combo, B)
    tr.load_delta_state_dict(delta)
    loss = tr(lat, prompts, masks, torch.ones_like(masks), noise=noise, timesteps=t)    # warm-up + capture + replay
    torch.cuda.synchronize()
    assert tr.text_engine.n_seq == B and tuple(tr.engine.in_ehs.shape) == (1, B, 77, 768)
    assert tr.state.grads.numel() == sum(tr.flat_group_sizes()) + 2 and tr.flat_group_sizes()[0] == (2 * 768 if emb_on else 0)
    clip.resize_token_embeddings(49408 + 2)
    emb = clip.get_input_embeddings().weight
    with torch.no_grad():
        emb[49408] = delta['new_concept_embedding']['<c1>'][0]
        emb[49409] = delta['new_concept_embedding']['<c2>'][0]
    for p in list(clip.parameters()) + list(ref_unet.parameters()):
        p.requires_grad_(False)
    emb.requires_grad_(emb_on)
    t_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['text_encoder'].items()}
    u_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['unet'].items()}
    if t_leaves:
        inject.inject_lora(clip, t_leaves, 1.0)
    if u_leaves:
        inject.inject_lora(ref_unet, u_leaves, 1.0)
    ids = tok(prompts, padding='max_length', max_length=77, return_tensors='pt').input_ids       # unbound, [b, 77]
    assert torch.equal(ids, tr.tokenize(prompts))
    pos = train_ref.concept_token_positions(ids, B, tr.get_all_concept_token_ids())
    noisy = DDPMScheduler().add_noise(lat, noise, t)
    ours, order = {}, {}
    if emb_on:
        ours['rows'] = tr.text_engine.emb_grad.flatten().cpu()
    for name, on, eng in (('text', text_on, tr.text_engine), ('unet', unet_on, tr.engine)):
        if on:
            grads = eng.lora_grad_dict()
            order[name] = [(m, gd.shape, gu.shape) for m, (gd, gu) in grads.items()]
            ours[name] = torch.cat([x.flatten().cpu() for gd, gu in grads.values() for x in (gd, gu)])

    def autograd(bf16):
        for p in [emb, *t_leaves.values(), *u_leaves.values()]:
            p.grad = None
        ctl = AttentionStore(training=True)
        inject.install_control_processors(ref_unet, ctl)
        with torch.autocast('cpu', dtype=torch.bfloat16, enabled=bf16):
            ehs = clip(ids)[0]                                                  # [b, 77, 768]: no rearrange
            loss_r, _, _ = train_ref.train_loss(ref_unet, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                                reg_full_identity=False, attn_reg_weight=0.05)
        loss_r.float().backward()
        out = {}
        if emb_on:
            out['rows'] = emb.grad[49408:49410].float().flatten().clone()
        for name, leaves in (('text', t_leaves), ('unet', u_leaves)):
            if name in order:
                out[name] = torch.cat([leaves[m + f'.lora_{s}.weight'].grad.float().reshape(shp).flatten()
                                       for m, sd, su in order[name] for s, shp in (('down', sd), ('up', su))])
        return loss_r.item(), out

    loss_bf, g_bf = autograd(True)
    loss_ref, g_ref = autograd(False)
    msg = [f'{combo_id(combo)} B={B}: loss {loss.item():.6f} vs {loss_ref:.6f}']
    assert abs(loss.item() - loss_ref) < 2e-2 * abs(loss_ref)
    for name, g in ours.items():
        r, c = rel_l2(g, g_ref[name]), _cos(g, g_ref[name])
        r_bf = rel_l2(g_bf[name], g_ref[name])
        msg.append(f'{name}: rel-L2 {r:.3e} cos {c:.5f} (bf16 autocast autograd: {r_bf:.3e})')
        bound = 4e-2 if name == 'rows' else 1e-2
        assert r <= max(bound, 2 * r_bf), msg[-1]
    print('  ' + ';  '.join(msg))


def _engines(ref_unet):
    """the same UNet and LoRA as an ED-LoRA and a vanilla TrainEngine, both producing d(text embedding), eager"""
    from mos_b200.train_engine import TrainEngine
    from oracle import inject
    from oracle import unet as ou
    sd = {k: v.detach().clone() for k, v in ref_unet.state_dict().items()}
    lora = inject.random_lora_state(ref_unet, seed=10)
    kw = dict(lora=lora, lora_alpha=0.8, attn_reg_weight=0.05, reg_full_identity=False, text_grad=True,
              block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    return TrainEngine(sd, 2, 16, 16, **kw), TrainEngine(sd, 2, 16, 16, shared_ehs=True, **kw)


def test_equivalence_with_edlora(cuda, tmp_path):
    """identical layer embeddings (one per cross-attention layer: 4 in the tiny UNet, 16 in SD1.5) through the ED-LoRA
    engine = one shared embedding through the vanilla engine.
    Loss and UNet-LoRA gradients: bit-identical (the same launches on the same values).  d(text embedding): ED-LoRA writes
    each layer's slice dK W_k' + dV W_v' in bf16, rounded twice (after the dK product and after adding the dV product into
    it), each rounding off by at most u = 2^-8 of the value rounded; the vanilla engine sums the same products in fp32
    (rounding ~2^-24).  So ||sum_l S_l - acc|| <= 2u sum_l ||S_l|| (first order in u, the products' size taken as the
    slices' size), and the bound is checked on the float64 sum of the slices."""
    _, ref_unet, _ = _base_dir(tmp_path, clip_layers=1)
    ed, va = _engines(ref_unet)
    ed.use_train_graph = va.use_train_graph = False
    nx = len(ed.xattn_names)
    g = torch.Generator().manual_seed(7)
    ehs = (torch.randn(2, 77, 768, generator=g) * 0.5).to(torch.bfloat16)
    lat, noise = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 4, 16, 16, generator=g)
    masks = torch.zeros(2, 1, 16, 16)
    masks[:, :, 3:12, 2:10] = 1.0
    t = torch.tensor([250, 700])
    out = {}
    for tag, eng, e in (('ed', ed, ehs[None].expand(nx, -1, -1, -1)), ('va', va, ehs[None])):
        loss = eng.forward_backward(lat.cuda(), noise.cuda(), t.cuda(), e.cuda(), masks.cuda(), token_pos=[[4, 5], [2, 9]])
        torch.cuda.synchronize()
        out[tag] = (loss.clone(), eng.state.grads.clone())
    assert torch.isfinite(out['va'][0]).all() and out['va'][1].abs().sum() > 0
    assert torch.equal(out['ed'][0], out['va'][0])
    assert torch.equal(out['ed'][1], out['va'][1])
    assert tuple(va.d_ehs.shape) == (2 * 77, 800) and tuple(ed.d_ehs.shape) == (nx * 2 * 77, 800)
    S = ed.d_ehs.double().view(nx, 2 * 77, 800)[:, :, :768]
    acc = va.d_ehs_f32.double()[:, :768]
    err = (S.sum(0) - acc).norm().item()
    bound = 2 * BF16_U * sum(S[l].norm().item() for l in range(nx))
    print(f'\n  d(ehs): ||sum of {nx} bf16 slices - fp32 accumulator|| = {err:.3e}, bound {bound:.3e}, '
          f'||acc|| = {acc.norm().item():.3e}')
    assert 0 < acc.norm().item() and err <= bound
    assert torch.equal(va.d_ehs, va.d_ehs_f32.to(torch.bfloat16))             # rounded to bf16 once
    assert va.d_ehs_f32[:, 768:].abs().max().item() == 0                     # the 32 pad columns stay zero


def _batch():
    g = torch.Generator().manual_seed(1)
    m = torch.zeros(2, 1, 16, 16)
    m[:, :, 3:12, 4:13] = 1
    return torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 4, 16, 16, generator=g), torch.tensor([90, 600]), m


def test_captured_vanilla_step_equals_eager(cuda, tmp_path):
    base, ref_unet, clip = _base_dir(tmp_path, clip_layers=1)
    combo = (True, True, True)
    tr = _trainer(base, combo)
    tr.load_delta_state_dict(_data(ref_unet, clip, combo)[0])
    tr._build(2)
    lat, noise, t, m = _batch()
    res = {}
    for graph in (False, True):
        tr.engine.use_train_graph = graph
        loss = tr(lat, PROMPTS, m, torch.ones_like(m), noise=noise, timesteps=t)
        torch.cuda.synchronize()
        res[graph] = (loss.clone(), tr.state.grads.clone(), tr.engine.d_ehs.clone())
    assert tr.engine.tgraph is not None
    for a, b in zip(res[False], res[True]):
        assert torch.equal(a, b)


def _audit_all(walk):
    import attention_audit
    import gemm_audit
    import norm_audit
    failures = []
    for mod in (gemm_audit, attention_audit, norm_audit):
        stats = gemm_audit.Stats()
        with mod.Recorder(stats):
            walk()
            torch.cuda.synchronize()
        assert stats.rows, mod.__name__
        print(f'\n{mod.__name__}\n' + stats.table())
        failures += stats.failures
    assert not failures, '\n'.join(failures[:30])


def test_vanilla_training_step_audited(cuda, tmp_path):
    """walk: one eager vanilla step with all three groups (CLIP over b sequences, the fp32 d(ehs) accumulation and its
    bf16 rounding, the CLIP backward) under the GEMM, attention and norm / elementwise audits"""
    base, ref_unet, clip = _base_dir(tmp_path, clip_layers=1)
    combo = (True, True, True)
    tr = _trainer(base, combo)
    tr.load_delta_state_dict(_data(ref_unet, clip, combo)[0])
    tr._build(2)
    tr.engine.use_train_graph = False
    lat, noise, t, m = _batch()
    _audit_all(lambda: tr(lat, PROMPTS, m, torch.ones_like(m), noise=noise, timesteps=t))


def test_stable_diffusion_pipeline_audited(cuda, tmp_path):
    """walk: StableDiffusionPipeline on a synthetic pretrained directory, 64 x 64, 3 DPM-Solver++ steps with CFG, eager
    UNet with its default processors and the 3-D embedding"""
    from synth import make_pretrained_dir
    from mixofshow.pipelines.pipeline_edlora import StableDiffusionPipeline
    pipe = StableDiffusionPipeline.from_pretrained(make_pretrained_dir(str(tmp_path / 'base')))
    pipe.unet.use_graph = False
    _audit_all(lambda: pipe('photo of a cat', negative_prompt='blurry', height=64, width=64, num_inference_steps=3,
                            guidance_scale=7.5, output_type='latent'))


FINETUNE = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
            'text_encoder': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'CLIPAttention'}, 'lr': 1e-5},
            'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}, 'lr': 1e-4}}


def _merged(weights, lora, alpha):
    out = dict(weights)
    for k, down in lora.items():
        if k.endswith('.lora_down.weight'):
            m = k[:-len('.lora_down.weight')]
            w = out[m + '.weight']
            out[m + '.weight'] = w + alpha * (lora[m + '.lora_up.weight'].flatten(1) @ down.flatten(1)).view_as(w)
    return out


def test_train_opt_vanilla_end_to_end(cuda, tmp_path, capsys):
    import train_edlora
    from synth import make_pretrained_dir
    from transformers import CLIPTextModel
    from mixofshow.pipelines.pipeline_edlora import StableDiffusionPipeline
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    from mixofshow.utils import model_io
    from mixofshow.utils.convert_edlora_to_diffusers import convert_edlora
    from oracle import edlora_ref as er
    from oracle import unet as ou
    from oracle.schedulers import DPMSolverMultistepScheduler
    base = make_pretrained_dir(str(tmp_path / 'base'))
    g = torch.Generator().manual_seed(1)
    n = 8
    masks = torch.zeros(n, 1, 32, 32)
    masks[:, :, 4:28, 8:24] = 1.0
    data = str(tmp_path / 'data.pt')
    # the concept tokens written literally: vanilla prompts are not bound (a `<TOK>: <c1> <c2>` mapping would not train them)
    torch.save({'latents': torch.randn(n, 4, 32, 32, generator=g) * 0.8, 'prompts': ['photo of a <TOK>'] * n,
                'masks': masks}, data)
    models = tmp_path / 'lora' / 'models'
    opt = {'name': 'lora', 'manual_seed': 1, 'gradient_accumulation_steps': 1,
           'datasets': {'train': {'path': data, 'replace_mapping': {'<TOK>': '<new0> <new1>'}, 'batch_size_per_gpu': 2,
                                  'dataset_enlarge_ratio': 1}},
           'models': {'pretrained_path': base, 'enable_edlora': False, 'new_concept_token': '<c1>+<c2>',
                      'initializer_token': '<rand-0.013>+a', 'finetune_cfg': FINETUNE, 'noise_offset': 0.01,
                      'attn_reg_weight': 0.01, 'reg_full_identity': False, 'use_mask_loss': True,
                      'gradient_checkpoint': False, 'enable_xformers': True, 'latent_size': [32, 32]},
           'train': {'optim_g': {'type': 'AdamW', 'lr': 0.0, 'weight_decay': 0.01, 'betas': [0.9, 0.999]},
                     'emb_norm_threshold': 0.55},
           'val': {'val_during_save': False},
           'path': {'models': str(models)}, 'logger': {'print_freq': 1, 'save_checkpoint_freq': 2}}
    yml = tmp_path / 'lora.yml'
    yml.write_text(yaml.safe_dump(opt))
    losses = train_edlora.main(['-opt', str(yml)])
    assert len(losses) == 4 and all(x == x and x > 0 for x in losses)
    assert sorted(os.listdir(models)) == ['lora_model-2.pth', 'lora_model-4.pth', 'lora_model-latest.pth']
    ckpt = str(models / 'lora_model-latest.pth')
    params = torch.load(ckpt)['params']
    assert list(params['new_concept_embedding']) == ['<c1>', '<c2>']
    assert all(tuple(v.shape) == (1, 768) for v in params['new_concept_embedding'].values())
    assert len(params['text_encoder']) == 2 * 4 * 2 and len(params['unet']) > 0
    # reload through load_delta_state_dict: the same checkpoint comes back out
    models_cfg = {k: v for k, v in opt['models'].items() if k != 'latent_size'}
    tr = EDLoRATrainer(**models_cfg, latent_size=(32, 32))
    tr.load_delta_state_dict(params)
    tr._build(2)
    back = tr.delta_state_dict()
    for part in ('new_concept_embedding', 'text_encoder', 'unet'):
        assert set(back[part]) == set(params[part])
        for k in params[part]:
            assert torch.equal(back[part][k], params[part][k]), (part, k)
    del tr
    # merge into StableDiffusionPipeline and sample
    alpha = 0.7
    pipe = StableDiffusionPipeline.from_pretrained(base)
    pipe, cfg = convert_edlora(pipe, torch.load(ckpt), enable_edlora=False, alpha=alpha)
    assert cfg == {'<c1>': {'concept_token_ids': [49408], 'concept_token_names': ['<new0>']},
                   '<c2>': {'concept_token_ids': [49409], 'concept_token_names': ['<new1>']}}
    prompt, neg = 'a <new0> <new1> on the beach', 'blurry'
    lat0 = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(3))
    first = []
    out = pipe(prompt, negative_prompt=neg, height=64, width=64, num_inference_steps=50, guidance_scale=7.5,
               latents=lat0.clone(), output_type='latent',
               callback=lambda i, t, x: first.append(x.clone()) if i == 0 else None).images
    assert tuple(out.shape) == (1, 4, 32, 32) and torch.isfinite(out).all()
    # fp32 oracle of the first step: transformers CLIP with the concept rows and the merged text LoRA, the oracle UNet
    # with the merged UNet LoRA and its default processors on the [2, 77, 768] CFG embedding
    clip = CLIPTextModel.from_pretrained(os.path.join(base, 'text_encoder')).eval()
    clip.resize_token_embeddings(49410)
    with torch.no_grad():
        clip.get_input_embeddings().weight[49408:49410] = torch.cat([params['new_concept_embedding'][c] for c in ('<c1>', '<c2>')])
    clip.load_state_dict(_merged(clip.state_dict(), params['text_encoder'], alpha))
    ref = ou.build_unet(0, ou.TINY)
    ref.load_state_dict(_merged(model_io.load_unet(base).state_dict(), params['unet'], alpha))
    ids = pipe.tokenizer([neg, prompt], padding='max_length', max_length=77, truncation=True, return_tensors='pt').input_ids
    assert int((ids[1] == 49408).sum()) == 1 and int((ids[1] == 49409).sum()) == 1
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(50)
    t0 = int(sched.timesteps[0])
    with torch.no_grad():
        ehs = clip(ids)[0]
        eps = ref(torch.cat([lat0, lat0]), torch.tensor([t0, t0]), ehs).sample
    want = sched.step(er.cfg_combine(eps, 7.5), t0, lat0).prev_sample
    e = rel_l2(first[0], want)
    print(f'\n  losses {losses}; StableDiffusionPipeline CFG-7.5 first-step latents vs fp32 oracle: rel-L2 {e:.3e}')
    assert e < 1e-3
