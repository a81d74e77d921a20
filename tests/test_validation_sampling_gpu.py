"""The sampling-check workflow on the GPU: `test_edlora.py -opt <yml>` and the validation pass of `train_edlora.py` on the
synthetic model directory (tests/synth.py), and the multi-prompt sampling they drive (a 4-prompt call is CFG UNet batch 8
and VAE decode batch 4) against the CPU oracle and against the same prompts sampled one at a time.

Tolerance: post-scheduler latents rel-L2 <= 1e-3, the bound of tests/test_unet_gpu.py (fp16 engine vs fp32 oracle)."""
import os

import pytest
import torch
import yaml

from synth import make_pretrained_dir

pytestmark = pytest.mark.gpu

CONCEPT = '<c1> <c2>'


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def random_edlora_checkpoint(base, path, seed=0, rank=4):
    """An ED-LoRA delta checkpoint for the model at `base`: 16 embedding rows per concept word and a random LoRA on every
    attention projection of the UNet and the text encoder."""
    from mixofshow.utils import model_io
    from mixofshow.utils.convert_edlora_to_diffusers import lora_down_name
    g = torch.Generator().manual_seed(seed)
    unet_sd = model_io.load_unet(base).state_dict()
    clip_sd = model_io.load_text_encoder(base).state_dict()
    params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) * 0.02 for w in CONCEPT.split()}}
    for part, sd, leaves in (('unet', unet_sd, ('to_q', 'to_k', 'to_v', 'to_out.0')),
                             ('text_encoder', clip_sd, ('q_proj', 'k_proj', 'v_proj', 'out_proj'))):
        lora = {}
        for k, v in sd.items():
            if v.ndim == 2 and any(k.endswith(f'.{leaf}.weight') for leaf in leaves):
                down = lora_down_name(k, part)
                lora[down] = torch.randn(rank, v.shape[1], generator=g) / v.shape[1] ** 0.5
                lora[down.replace('lora_down', 'lora_up')] = torch.randn(v.shape[0], rank, generator=g) * 0.02
        params[part] = lora
    torch.save({'params': params}, path)
    return path


@pytest.fixture(scope='module')
def base(tmp_path_factory):
    return make_pretrained_dir(str(tmp_path_factory.mktemp('base')))


@pytest.fixture(scope='module')
def ckpt(base, tmp_path_factory):
    return random_edlora_checkpoint(base, str(tmp_path_factory.mktemp('ckpt') / 'edlora_model-latest.pth'))


def _val_vis(n_samples=2, batch=4):
    # the synthetic UNet samples 64x64 latents (sample_size 64; the tiny VAE has one 2x level: 128x128 images)
    return {'name': 'PromptDataset', 'prompts': ['photo of a <TOK>', 'a <TOK> on the beach', '<TOK> in the snow'],
            'num_samples_per_prompt': n_samples, 'latent_size': [4, 64, 64], 'replace_mapping': {'<TOK>': CONCEPT},
            'batch_size_per_gpu': batch}


def test_test_edlora_writes_reference_layout(cuda, base, ckpt, tmp_path, monkeypatch):
    import test_edlora
    vis = tmp_path / 'vis'
    alphas = [0, 0.7, 1.0]
    opt = {'name': 'synthetic', 'manual_seed': 0, 'datasets': {'val_vis': _val_vis()},
           'models': {'pretrained_path': base, 'enable_edlora': True},
           'path': {'lora_path': ckpt, 'visualization': str(vis)},
           'val': {'compose_visualize': True, 'alpha_list': alphas,
                   'sample': {'num_inference_steps': 3, 'guidance_scale': 7.5}}}
    yml = tmp_path / 'test.yml'
    yml.write_text(yaml.safe_dump(opt))
    after_free = []
    free = test_edlora.free_pipeline

    def recording_free():
        free()
        torch.cuda.synchronize()
        after_free.append(torch.cuda.memory_allocated())
    monkeypatch.setattr(test_edlora, 'free_pipeline', recording_free)
    test_edlora.main(['-opt', str(yml)])
    root = vis / 'PromptDataset'
    prompts = ['photo_of_a_<c1>_<c2>', 'a_<c1>_<c2>_on_the_beach', '<c1>_<c2>_in_the_snow']
    pngs = 0
    for a in alphas:
        it = f'validation_edlora_{a}'
        names = sorted(os.listdir(root / it))
        assert names == sorted(f'{p}---G_7.5_S_3---{i}---{it}.png' for p in prompts for i in (1, 2))
        pngs += len(names)
        assert (root / f'G_7.5_S_3---{it}.jpg').exists()
    assert pngs == 18
    print(f'allocated after each alpha: {after_free}')
    assert len(after_free) == 3 and max(after_free[1:]) <= after_free[0], after_free


def test_alpha_zero_is_the_embeddings_alone(cuda, base, ckpt):
    import test_edlora
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from mixofshow.utils import model_io
    from mixofshow.utils.convert_edlora_to_diffusers import load_new_concept
    merged = test_edlora.load_pipeline(base, ckpt, 0)
    for got, want in ((merged.unet.state_dict(), model_io.load_unet(base).state_dict()),
                      (merged.text_encoder.state_dict(), model_io.load_text_encoder(base).state_dict())):
        for k, v in want.items():
            if 'token_embedding' not in k:
                assert torch.equal(got[k].cpu(), v.cpu()), k
    emb = EDLoRAPipeline.from_pretrained(base)
    emb, cfg = load_new_concept(emb, torch.load(ckpt)['params']['new_concept_embedding'], enable_edlora=True)
    emb.set_new_concept_cfg(cfg)
    lat = torch.randn(2, 4, 64, 64, generator=torch.Generator().manual_seed(1))
    kw = dict(prompt=[f'photo of a {CONCEPT}', f'a {CONCEPT} on the beach'], negative_prompt=['blurry'] * 2,
              num_inference_steps=4, guidance_scale=7.5, output_type='latent')
    a = merged(latents=lat.clone(), **kw).images
    b = emb(latents=lat.clone(), **kw).images
    assert torch.equal(a, b)


def test_four_prompt_cfg_call_matches_oracle(cuda):
    """One 4-prompt CFG call (UNet batch 8) on the tiny topology: each sample's latents after the first step of a 50-step
    schedule against the fp32 oracle."""
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from oracle import edlora_ref as er
    from oracle import inject
    from oracle import unet as ou
    from oracle.schedulers import DPMSolverMultistepScheduler
    n = 4
    ref = ou.build_unet(0, ou.TINY)
    inject.install_edlora_processors(ref)
    unet = UNet2DConditionModel(**ou.TINY)
    unet.load_state_dict(ref.state_dict())
    pipe = EDLoRAPipeline(unet=unet).to('cuda')
    pipe.set_new_concept_cfg({})
    lat = torch.randn(n, 4, 32, 32, generator=torch.Generator().manual_seed(3))
    pe = torch.randn(n, 16, 77, 768, generator=torch.Generator().manual_seed(4))
    ne = torch.randn(n, 77, 768, generator=torch.Generator().manual_seed(5))
    first = []
    pipe(prompt_embeds=pe.cuda(), negative_prompt_embeds=ne.cuda(), latents=lat.clone(), height=256, width=256,
         num_inference_steps=50, guidance_scale=7.5, output_type='latent',
         callback=lambda i, t, x: first.append(x.clone()) if i == 0 else None)
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(50)
    t0 = int(sched.timesteps[0])
    emb = torch.cat([ne.view(n, 1, 77, 768).repeat(1, 16, 1, 1), pe])
    with torch.no_grad():
        eps = ref(torch.cat([lat, lat]), torch.tensor([t0] * 2 * n), emb).sample
    want = sched.step(er.cfg_combine(eps, 7.5), t0, lat).prev_sample
    errs = [rel_l2(first[0][i], want[i]) for i in range(n)]
    print(f'4-prompt CFG call vs oracle, per-sample latents rel-L2 after step 1: {errs}')
    assert max(errs) < 1e-3


def test_four_prompt_call_matches_single_prompt_calls_sd15(cuda):
    """Full SD1.5 topology with a rank-4 ED-LoRA on every attention projection, 512x512: each sample of a 4-prompt call
    against the same prompt and latents sampled alone (UNet batch 8 vs batch 2), after 3 steps of a 50-step schedule."""
    import bench
    n, steps = 4, 3
    sd, lora, lat, ehs, cfg = bench.build_workload(images=n)
    pipe = bench.build_pipeline(sd, lora, cfg, torch.device('cuda'))
    cond, neg = ehs[n:], ehs[:n, 0]

    def run(idx):
        got = []
        pipe(prompt_embeds=cond[idx].cuda(), negative_prompt_embeds=neg[idx].cuda(), latents=lat[idx].clone(),
             num_inference_steps=50, guidance_scale=7.5, output_type='latent',
             callback=lambda i, t, x: got.append(x.clone()) if i == steps - 1 else None)
        return got[0]
    batched = run(slice(0, n))
    errs = [rel_l2(batched[i], run(slice(i, i + 1))[0]) for i in range(n)]
    print(f'SD1.5 4-prompt call vs single-prompt calls, per-sample latents rel-L2 after {steps} steps: {errs}')
    assert torch.isfinite(batched).all() and max(errs) < 1e-3


def test_vae_decode_batch4_512_vs_oracle(cuda):
    """The 4-prompt call's decode: SD1.5 VAE, 4 latents of 64x64 -> 512x512, each image against the fp32 oracle (run on the
    GPU, TF32 off) within the 5e-3 image tolerance of tests/test_vae_gpu.py."""
    from mos_b200.vae_engine import VAEEngine
    from oracle import vae as ov
    ref = ov.build_vae(0).to(cuda)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    eng = VAEEngine(sd, 4, 512, 512, block_out=ov.SD15_VAE['block_out_channels'], layers=ov.SD15_VAE['layers_per_block'])
    z = torch.randn(4, 4, 64, 64, generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        want = ref.decode(z.to(cuda))
    got = eng.decode(z.cuda())
    torch.cuda.synchronize()
    errs = [rel_l2(got[i], want[i]) for i in range(4)]
    print(f'VAE decode batch 4 at 512x512 vs oracle, per image rel-L2: {errs}')
    assert max(errs) < 5e-3


def _train_yml(tmp_path, base, tag, with_val):
    g = torch.Generator().manual_seed(1)
    n = 8
    masks = torch.zeros(n, 1, 32, 32)
    masks[:, :, 4:28, 8:24] = 1.0
    data = str(tmp_path / 'data.pt')
    if not os.path.exists(data):
        torch.save({'latents': torch.randn(n, 4, 32, 32, generator=g) * 0.8, 'prompts': ['photo of a <TOK>'] * n,
                    'masks': masks}, data)
    finetune = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
                'text_encoder': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'CLIPAttention'},
                                 'lr': 1e-5},
                'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}, 'lr': 1e-4}}
    opt = {'name': tag, 'manual_seed': 1, 'gradient_accumulation_steps': 1,
           'datasets': {'train': {'path': data, 'replace_mapping': {'<TOK>': CONCEPT}, 'batch_size_per_gpu': 2,
                                  'dataset_enlarge_ratio': 1}},
           'models': {'pretrained_path': base, 'enable_edlora': True, 'new_concept_token': CONCEPT.replace(' ', '+'),
                      'initializer_token': '<rand-0.013>+a', 'finetune_cfg': finetune, 'noise_offset': 0.01,
                      'attn_reg_weight': 0.01, 'reg_full_identity': False, 'use_mask_loss': True,
                      'gradient_checkpoint': False, 'enable_xformers': True, 'latent_size': [32, 32]},
           'train': {'optim_g': {'type': 'AdamW', 'lr': 0.0, 'weight_decay': 0.01, 'betas': [0.9, 0.999]},
                     'emb_norm_threshold': 0.55},
           'path': {'models': str(tmp_path / tag / 'models'), 'visualization': str(tmp_path / tag / 'visualization')},
           'logger': {'print_freq': 1}}
    if with_val:
        opt['datasets']['val_vis'] = _val_vis(n_samples=1)
        opt['val'] = {'val_during_save': True, 'compose_visualize': True, 'alpha_list': [0, 1.0],
                      'sample': {'num_inference_steps': 2, 'guidance_scale': 7.5}}
        opt['logger']['save_checkpoint_freq'] = 2
    yml = tmp_path / f'{tag}.yml'
    yml.write_text(yaml.safe_dump(opt))
    return str(yml)


def test_train_with_validation_does_not_perturb_training(cuda, base, tmp_path):
    import train_edlora
    plain = train_edlora.main(['-opt', _train_yml(tmp_path, base, 'plain', False)])
    val = train_edlora.main(['-opt', _train_yml(tmp_path, base, 'val', True)])
    assert len(val) == 4 and val == plain
    models = tmp_path / 'val' / 'models'
    assert sorted(os.listdir(models)) == ['edlora_model-2.pth', 'edlora_model-4.pth', 'edlora_model-latest.pth']
    assert sorted(os.listdir(tmp_path / 'plain' / 'models')) == ['edlora_model-latest.pth']
    a = torch.load(tmp_path / 'plain' / 'models' / 'edlora_model-latest.pth')['params']
    b = torch.load(models / 'edlora_model-latest.pth')['params']
    assert a.keys() == b.keys()
    for part in a:
        assert a[part].keys() == b[part].keys()
        for k in a[part]:
            assert torch.equal(a[part][k], b[part][k]), (part, k)
    root = tmp_path / 'val' / 'visualization' / 'PromptDataset'
    for step in ('2', '4', 'latest'):
        for alpha in (0, 1.0):
            it = f'Iters-{step}_Alpha-{alpha}'
            assert len(os.listdir(root / it)) == 3, it
            assert (root / f'G_7.5_S_2---{it}.jpg').exists()
