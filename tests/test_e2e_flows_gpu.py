"""The reference's user workflows driven through their ENTRY POINTS on one GPU, with a synthetic model directory (tiny UNet,
2-layer CLIP, tiny VAE, a character-level CLIP tokenizer loaded by transformers' own CLIPTokenizer):

    python train_edlora.py -opt <yml>                     (train_edlora.py:174-180)       x 2 concepts
    EDLoRAPipeline.from_pretrained + convert_edlora + pipe(prompt).images[0]              (test_edlora.py)
    python gradient_fusion.py --concept_cfg ... --pretrained_models ...                   (gradient_fusion.py:816-841)
    python regionally_controlable_sampling.py --pretrained_model <fused> --prompt_rewrite ...

Integration smoke: shapes, finiteness, files on disk and that the trained / fused parameters actually changed.  The numerics
of every stage have their own parity tests."""
import json
import os

import pytest
import torch
import yaml

from synth import make_pretrained_dir

pytestmark = pytest.mark.gpu

FINETUNE = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
            'text_encoder': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'CLIPAttention'}, 'lr': 1e-5},
            'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}, 'lr': 1e-4}}


def _train_one(tmp_path, base, tag, concept_token, init_token, caption, seed, batch_size_per_gpu=2,
               gradient_accumulation_steps=1):
    import train_edlora
    g = torch.Generator().manual_seed(seed)
    n = 8
    masks = torch.zeros(n, 1, 32, 32)
    masks[:, :, 4:28, 8:24] = 1.0
    data = str(tmp_path / f'{tag}_data.pt')
    torch.save({'latents': torch.randn(n, 4, 32, 32, generator=g) * 0.8, 'prompts': [caption] * n, 'masks': masks}, data)
    out_dir = str(tmp_path / f'{tag}_models')
    opt = {'name': tag, 'manual_seed': seed, 'gradient_accumulation_steps': gradient_accumulation_steps,
           'datasets': {'train': {'path': data, 'replace_mapping': {'<TOK>': concept_token.replace('+', ' ')},
                                  'batch_size_per_gpu': batch_size_per_gpu, 'dataset_enlarge_ratio': 1}},
           'models': {'pretrained_path': base, 'enable_edlora': True, 'new_concept_token': concept_token,
                      'initializer_token': init_token, 'finetune_cfg': FINETUNE, 'noise_offset': 0.01, 'attn_reg_weight': 0.01,
                      'reg_full_identity': False, 'use_mask_loss': True, 'gradient_checkpoint': False, 'enable_xformers': True,
                      'latent_size': [32, 32]},
           'train': {'optim_g': {'type': 'AdamW', 'lr': 0.0, 'weight_decay': 0.01, 'betas': [0.9, 0.999]},
                     'emb_norm_threshold': 0.55},
           'path': {'models': out_dir}, 'logger': {'print_freq': 1}}
    yml = str(tmp_path / f'{tag}.yml')
    yaml.safe_dump(opt, open(yml, 'w'))
    losses = train_edlora.main(['-opt', yml])
    steps = train_edlora.total_iterations(n, batch_size_per_gpu, 1, gradient_accumulation_steps)
    assert len(losses) == steps == n // (batch_size_per_gpu * gradient_accumulation_steps)   # 8 / (2 x 1) = 4 by default
    assert all(l == l and l > 0 for l in losses)
    ckpt = os.path.join(out_dir, 'edlora_model-latest.pth')
    params = torch.load(ckpt)['params']
    words = concept_token.split('+')
    assert list(params['new_concept_embedding']) == words
    assert all(tuple(v.shape) == (16, 768) and torch.isfinite(v).all() for v in params['new_concept_embedding'].values())
    assert len(params['text_encoder']) == 2 * 4 * 2                            # 2 layers x q/k/v/out x (down, up)
    ups = [v for k, v in params['unet'].items() if k.endswith('lora_up.weight')]
    assert ups and all(torch.isfinite(v).all() for v in ups) and sum(float(v.abs().sum()) for v in ups) > 0   # up starts at 0
    return ckpt


def test_reference_workflows_end_to_end(cuda, tmp_path):
    import gradient_fusion
    import regionally_controlable_sampling as rcs
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from mixofshow.utils import model_io
    from mixofshow.utils.convert_edlora_to_diffusers import convert_edlora
    base = make_pretrained_dir(str(tmp_path / 'base'))
    # ---- 1. train two concepts from yml files (two concept words each: the attention regulariser needs exactly two)
    ck_cat = _train_one(tmp_path, base, 'cat', '<cat1>+<cat2>', '<rand-0.013>+a', 'photo of a <TOK>', seed=1)
    ck_dog = _train_one(tmp_path, base, 'dog', '<dog1>+<dog2>', '<rand-0.013>+<rand-0.013>', 'a <TOK> in the snow', seed=2)
    # ---- 2. single-concept sampling as test_edlora.py does
    pipe = EDLoRAPipeline.from_pretrained(base)
    pipe, new_cfg = convert_edlora(pipe, torch.load(ck_cat), enable_edlora=True, alpha=0.7)
    pipe.set_new_concept_cfg(new_cfg)
    assert new_cfg['<cat2>']['concept_token_ids'] == list(range(49408 + 16, 49408 + 32))
    img = pipe('a <cat1> <cat2> on the beach', negative_prompt='blurry', height=64, width=64, num_inference_steps=4,
               guidance_scale=7.5, generator=torch.Generator().manual_seed(3)).images[0]
    assert img.size == (64, 64)
    lat = pipe('a <cat1> <cat2> on the beach', negative_prompt='blurry', height=64, width=64, num_inference_steps=4,
               guidance_scale=7.5, generator=torch.Generator().manual_seed(3), output_type='latent').images
    assert tuple(lat.shape) == (1, 4, 32, 32) and torch.isfinite(lat).all()
    # ---- 3. gradient fusion of the two checkpoints through the CLI entry
    cfg_json = str(tmp_path / 'concepts.json')
    json.dump([{'lora_path': ck_cat, 'unet_alpha': 1.0, 'text_encoder_alpha': 1.0, 'concept_name': '<cat1> <cat2>'},
               {'lora_path': ck_dog, 'unet_alpha': 0.8, 'text_encoder_alpha': 0.8, 'concept_name': '<dog1> <dog2>'}],
              open(cfg_json, 'w'))
    out_dir, fused_cfg = gradient_fusion.main(['--concept_cfg', cfg_json, '--save_path', str(tmp_path / 'fused'),
                                               '--pretrained_models', base, '--optimize_textenc_iters', '10',
                                               '--optimize_unet_iters', '3', '--suffix', 'e2e'])
    assert os.path.basename(out_dir) == 'combined_model_e2e' and list(fused_cfg) == ['<cat1>', '<cat2>', '<dog1>', '<dog2>']
    for sub in ('unet', 'text_encoder', 'tokenizer', 'new_concept_cfg.json'):
        assert os.path.exists(os.path.join(out_dir, sub)), sub
    w0 = model_io.load_unet(base).state_dict()
    w1 = model_io.load_unet(out_dir).state_dict()
    k = 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight'
    assert torch.isfinite(w1[k]).all() and not torch.equal(w0[k], w1[k])
    # ---- 4. regional multi-concept sampling of the fused model through the CLI entry
    save = str(tmp_path / 'regional')
    lat = rcs.main(['--pretrained_model', out_dir, '--height', '256', '--width', '512', '--num_inference_steps', '6',
                    '--prompt', 'two animals in the snow', '--negative_prompt', 'blurry',
                    '--prompt_rewrite', '[a <cat1> <cat2> in the snow]-*-[blurry]-*-[10,20,200,250]|'
                                        '[a <dog1> <dog2> in the snow]-*-[blurry]-*-[20,260,230,500]',
                    '--save_dir', save, '--seed', '7'])
    assert tuple(lat.shape) == (1, 4, 32, 64) and torch.isfinite(lat).all()
    assert os.path.exists(os.path.join(save, 'latents---7.pt')) and os.path.exists(os.path.join(save, 'config.json'))
