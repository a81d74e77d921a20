"""The full ED-LoRA training step through the reference-shaped `EDLoRATrainer` (mixofshow/pipelines/trainer_edlora.py):
prompts -> bind_concept_prompt -> tokenizer -> CLIP text encoder (LoRA) -> UNet (LoRA) -> masked MSE + attention regulariser
-> backward through BOTH networks, against fp32 autograd through transformers' CLIPTextModel chained into the oracle UNet
(reference LoRA formula injected in both, oracle/train_ref.py loss).  Checks the three parameter groups of
trainer_edlora.py:82-139: new-concept embedding rows, CLIPAttention LoRA, UNet Attention LoRA.  At B = 1, 2, 3 and 4 with
both regulariser modes: much of the step depends on B (the loss's 1 / B, the regulariser's batch-wide maxima and zero
count, the GroupNorm partitions, the split-K and row blocking of M = B x HW, the 16 x B text sequences), and the samples of
a batch differ in prompt length, timestep and mask, so that a sample mix-up shows.

Tolerances: bf16 operands through two networks forward and backward: whole-group gradient rel-L2 <= 4e-2, cosine >= 0.998;
loss within 2 %."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.flatten().float().cpu(), b.flatten().float().cpu(), dim=0).item()


FINETUNE = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
            'text_encoder': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'CLIPAttention'}, 'lr': 1e-5},
            'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}, 'lr': 1e-4}}


def _base_dir(tmp_path, clip_layers=2):
    from transformers import CLIPTextConfig, CLIPTextModel
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    from oracle import unet as ou
    torch.manual_seed(0)
    ref_unet = ou.build_unet(0, ou.TINY)
    unet = UNet2DConditionModel(block_out_channels=ou.TINY['block_out_channels'], layers_per_block=ou.TINY['layers_per_block'])
    unet.load_state_dict(ref_unet.state_dict())
    base = str(tmp_path / 'base')
    model_io.save_unet(unet, base)
    clip = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072,
                                        num_hidden_layers=clip_layers, num_attention_heads=12,
                                        max_position_embeddings=77)).eval()
    clip.save_pretrained(os.path.join(base, 'text_encoder'))
    return base, ref_unet, clip


PREFIX = ('photo of a', 'the', 'a close photo of one', 'an old')     # sample b's concept words sit at a position of its own
SUFFIX = ('', 'on a beach', 'smiling', 'in the snow')


def batch_inputs(B, seed, words=('<c1>', '<c2>'), H=16):
    """a training batch whose samples differ where the step could mix them up: prompt length (so the concept-token
    positions), timestep (0 and 999 among them), mask; at B >= 2 the last mask is all ones, so that sample adds to the
    regulariser's zero-pixel count only through the others.  -> prompts, latents, noise, timesteps, masks"""
    g = torch.Generator().manual_seed(seed)
    prompts = [f'{PREFIX[b]} {words[0]} {words[1]} {SUFFIX[b]}'.strip() for b in range(B)]
    lat, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([0, 999, 511, 130][:B])
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    if B >= 2:
        masks[B - 1] = 1.0
    return prompts, lat, noise, t, masks


def _trainer(base, tok, reg_w, full):
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=json.loads(json.dumps(FINETUNE)),
                         noise_offset=None, attn_reg_weight=reg_w, reg_full_identity=full, use_mask_loss=True,
                         enable_xformers=True, tokenizer=tok, latent_size=(16, 16))


def _delta(ref_unet, clip):
    from oracle import inject
    g = torch.Generator().manual_seed(5)
    return {'new_concept_embedding': {'<c1>': torch.randn(16, 768, generator=g) * 0.02,
                                      '<c2>': torch.randn(16, 768, generator=g) * 0.02},
            'text_encoder': inject.random_lora_state(clip, seed=3, where='CLIPAttention', up_std=0.05),
            'unet': inject.random_lora_state(ref_unet, seed=10)}


def autograd_reference(tr, clip, ref_unet, delta, tok, batches, reg_w, full):
    """the step in fp32 autograd: transformers' CLIPTextModel chained into the oracle UNet, reference LoRA formula injected
    in both, oracle/train_ref.py loss.  The gradients of all `batches` ((prompts, latents, noise, t, masks) each, one
    backward per batch, the regulariser per batch as the reference computes it) are summed.
    -> (losses, d concept rows [32, 768], text LoRA leaves, UNet LoRA leaves); the leaves hold the gradients"""
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle.schedulers import DDPMScheduler
    clip.resize_token_embeddings(49408 + 32)
    emb = clip.get_input_embeddings().weight
    with torch.no_grad():
        emb[49408:49408 + 16] = delta['new_concept_embedding']['<c1>']
        emb[49408 + 16:49408 + 32] = delta['new_concept_embedding']['<c2>']
    emb.requires_grad_(True)
    t_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['text_encoder'].items()}
    u_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['unet'].items()}
    inject.inject_lora(clip, t_leaves, 1.0)
    inject.inject_lora(ref_unet, u_leaves, 1.0)
    ctl = AttentionStore(training=True)
    inject.install_control_processors(ref_unet, ctl)
    losses = []
    for prompts, lat, noise, t, masks in batches:
        b = len(prompts)
        ids = tok(bind_concept_prompt(prompts, tr.new_concept_cfg), padding='max_length', max_length=77,
                  return_tensors='pt').input_ids
        ehs = clip(ids)[0].view(b, 16, 77, 768)
        pos = train_ref.concept_token_positions(ids, b, tr.get_all_concept_token_ids())
        noisy = DDPMScheduler().add_noise(lat, noise, t)
        loss_ref, _, _ = train_ref.train_loss(ref_unet, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                              reg_full_identity=full, attn_reg_weight=reg_w)
        loss_ref.backward()
        losses.append(loss_ref.item())
        ctl.reset()
    return losses, emb.grad[49408:49408 + 32], t_leaves, u_leaves


def group_errors(tr, g_rows, t_leaves, u_leaves):
    """{'rows' | 'text' | 'unet': (rel-L2, cosine, size)} of the trainer's gradient against autograd's"""
    res = {'rows': (rel_l2(tr.text_engine.emb_grad, g_rows), _cos(tr.text_engine.emb_grad, g_rows), g_rows.numel())}
    for name, eng, leaves in (('text', tr.text_engine, t_leaves), ('unet', tr.engine, u_leaves)):
        fg, fr = [], []
        for m, (gd, gu) in eng.lora_grad_dict().items():
            fg += [gd.flatten().cpu(), gu.flatten().cpu()]
            fr += [leaves[m + '.lora_down.weight'].grad.reshape(gd.shape).flatten(),
                   leaves[m + '.lora_up.weight'].grad.reshape(gu.shape).flatten()]
        fg, fr = torch.cat(fg), torch.cat(fr)
        res[name] = (rel_l2(fg, fr), _cos(fg, fr), fg.numel())
    return res


def format_errors(res):
    return ';  '.join(f'{name} ({n}): rel-L2 {r:.3e} cos {c:.5f}' for name, (r, c, n) in res.items())


def test_full_trainer_step_vs_autograd(cuda, tmp_path):
    """the shipped batch, B = 2, regulariser with reg_full_identity=False"""
    _full_trainer_step_vs_autograd(tmp_path, 2, False)


# the other batch sizes and regulariser modes (the B = 2 / reg_full_identity=False case is the test above)
BATCH_CASES = [(b, f) for b in (1, 2, 3, 4) for f in (False, True) if (b, f) != (2, False)]


@pytest.mark.parametrize('B,full', BATCH_CASES,
                         ids=[f'B{b}-{"reg_full_identity" if f else "reg_subject_outside"}' for b, f in BATCH_CASES])
def test_full_trainer_step_vs_autograd_batch(cuda, tmp_path, B, full):
    _full_trainer_step_vs_autograd(tmp_path, B, full)


def _full_trainer_step_vs_autograd(tmp_path, B, full):
    from test_fusion_orchestration import WordTokenizer
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    reg_w = 0.05
    tr = _trainer(base, tok, reg_w, full)
    assert tr.new_concept_cfg['<c2>']['concept_token_names'] == [f'<new{16 + i}>' for i in range(16)]
    assert tr.get_all_concept_token_ids() == list(range(49408, 49408 + 32))
    delta = _delta(ref_unet, clip)
    tr.load_delta_state_dict(delta)
    prompts, lat, noise, t, masks = batch_inputs(B, seed=40 + B)
    loss = tr(lat, prompts, masks, torch.ones_like(masks), noise=noise, timesteps=t)
    torch.cuda.synchronize()
    assert tr.text_engine.n_seq == len(tr.engine.xattn_names) * B
    ids, _ = tr.tokenize_layerwise(prompts)
    pos = tr.concept_token_positions(ids, B)
    assert len({tuple(p) for p in pos}) == B, pos               # every sample has its concept tokens elsewhere
    (loss_ref,), g_rows, t_leaves, u_leaves = autograd_reference(tr, clip, ref_unet, delta, tok,
                                                                 [(prompts, lat, noise, t, masks)], reg_w, full)
    res = group_errors(tr, g_rows, t_leaves, u_leaves)
    print(f'full trainer step B={B} full_identity={full}: loss {loss.item():.6f} vs autograd {loss_ref:.6f};  '
          + format_errors(res))
    assert abs(loss.item() - loss_ref) < 2e-2 * abs(loss_ref)
    for name, (r, c, _) in res.items():
        assert r < 4e-2 and c > 0.998, name
    # checkpoint layout of the reference (trainer_edlora.py:358-378) and round trip
    d = tr.delta_state_dict()
    assert set(d) == {'new_concept_embedding', 'text_encoder', 'unet'} and set(d['new_concept_embedding']) == {'<c1>', '<c2>'}
    assert sorted(d['text_encoder']) == sorted(delta['text_encoder']) and sorted(d['unet']) == sorted(delta['unet'])
    for k in delta['text_encoder']:
        assert rel_l2(d['text_encoder'][k], delta['text_encoder'][k]) < 1e-6
    assert rel_l2(d['new_concept_embedding']['<c2>'], delta['new_concept_embedding']['<c2>']) < 1e-6


def test_train_loop_three_groups(cuda, tmp_path):
    """train() (train_edlora.py:105-158 mirror) with the full trainer: all three groups move, the learning rates decay
    linearly, the loss on a repeated batch goes down, the embedding rows freeze once Norm_mean crosses the threshold."""
    import train_edlora as te
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    base, _, _ = _base_dir(tmp_path, clip_layers=1)
    tr = EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.013>+<rand-0.013>', True, finetune_cfg=json.loads(json.dumps(FINETUNE)),
                       attn_reg_weight=0.01, reg_full_identity=False, tokenizer=WordTokenizer(), latent_size=(16, 16))
    g = torch.Generator().manual_seed(1)
    m = torch.zeros(2, 1, 16, 16)
    m[:, :, 3:12, 4:13] = 1
    batch = {'images': torch.randn(2, 4, 16, 16, generator=g), 'prompts': ['photo of a <c1> <c2>', 'a <c1> <c2> smiling'],
             'masks': m, 'img_masks': torch.ones(2, 1, 16, 16)}
    logs = []
    losses = te.train(tr, [batch] * 12, dataset_len=24, batch_size_per_gpu=2, print_freq=1, log=logs.append,
                      emb_norm_threshold=0.41)
    assert len(losses) == 12
    d = tr.delta_state_dict()
    assert any(v.abs().max().item() > 0 for k, v in d['unet'].items() if k.endswith('lora_up.weight'))
    assert any(v.abs().max().item() > 0 for k, v in d['text_encoder'].items() if k.endswith('lora_up.weight'))
    norms = [float(l.split('Norm_mean ')[1]) for l in logs]
    print('    losses', ' '.join(f'{x:.4f}' for x in losses), '| Norm_mean', ' '.join(f'{x:.4f}' for x in norms))
    assert norms[0] != norms[1]                                   # the rows train (lr 1e-3) ...
    crossed = [i for i, n in enumerate(norms) if n >= 0.41]
    if crossed:                                                   # ... and freeze for good after crossing the threshold
        assert all(abs(n - norms[crossed[0]]) < 1e-6 for n in norms[crossed[0]:])
