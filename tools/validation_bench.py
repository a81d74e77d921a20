"""Times the sampling-check workflow (test_edlora.py, and the validation pass train_edlora.py runs at every checkpoint) at
the size of the shipped configs: full-size SD1.5 random weights (UNet, 12-layer CLIP text encoder, VAE), 512x512, 50
DPM-Solver++ steps, guidance 7.5, an ED-LoRA checkpoint merged at alpha 0.7.

Reports, with the card's name and power limit read in the same run:
  - one alpha pass of the shipped prompt set (11 prompts x 8 samples in batches of 4: 22 pipeline calls, 1 100 UNet
    steps at CFG batch 8, 22 VAE decodes at batch 4; PNG writes and the composed grid included) and its images/s;
  - ms per denoise step (UNet graph replay + fused CFG / DPM-Solver++ update) at UNet batch 8 and at batch 2;
  - ms per VAE decode of 4 latents.

    python tools/validation_bench.py [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

PROMPTS = os.path.join(ROOT, 'tests', 'golden', 'validation', 'test_man.txt')


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return {'device': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def make_model_dir(path):
    """unet/, text_encoder/, vae/ and tokenizer/ of an SD1.5-sized model with random weights"""
    import torch
    from transformers import CLIPTextConfig, CLIPTextModel

    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.models.vae_b200 import AutoencoderKL
    from mixofshow.utils import model_io
    from oracle import vae as ov
    from synth import make_clip_tokenizer_dir
    torch.manual_seed(0)
    unet = UNet2DConditionModel()
    model_io.save_unet(unet, path)
    CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                                 num_attention_heads=12, max_position_embeddings=77, hidden_act='quick_gelu')
                  ).save_pretrained(os.path.join(path, 'text_encoder'))
    model_io.save_vae(AutoencoderKL({k: v.detach() for k, v in ov.build_vae(0).state_dict().items()}, device='cpu'), path)
    make_clip_tokenizer_dir(os.path.join(path, 'tokenizer'))
    return {k: v.detach() for k, v in unet.state_dict().items()}


def make_checkpoint(path, unet_sd):
    import torch

    import bench
    g = torch.Generator().manual_seed(3)
    emb = {w: torch.randn(16, 768, generator=g) * 0.02 for w in ('<potter1>', '<potter2>')}
    torch.save({'params': {'new_concept_embedding': emb, 'text_encoder': {}, 'unet': bench.random_unet_lora(unet_sd)}},
               path)
    return path


def time_events(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def step_ms(pipe, images, reps):
    """one denoise step of the pipeline's loop at CFG batch 2 x images (pipeline_edlora.py: graph replay + fused update)"""
    import torch

    from mos_b200 import ops
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(5)
    sess = pipe.unet.session(2 * images, 64, 64, dev, torch.randn(2 * images, 16, 77, 768, generator=g).to(dev))
    pipe.scheduler.set_timesteps(50)
    latents = torch.randn(images, 4, 64, 64, generator=g).to(dev)
    x0_prev = torch.zeros_like(latents)
    sess.latents_in.copy_(torch.cat([latents, latents]))
    sess.t_in.fill_(float(pipe.scheduler.timesteps[0]))

    def step():
        eps = sess.step()
        ops.cfg_dpmpp_step(eps, latents, x0_prev, sess.latents_in.view(-1), cfg=True, guidance=7.5,
                           coef=pipe.scheduler.coefficients(1), t_out=sess.t_in, t_next=float(pipe.scheduler.timesteps[2]))
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    return time_events(step, reps)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for the JSON result (default: print only)')
    ap.add_argument('--step-reps', type=int, default=50)
    args = ap.parse_args(argv)
    import torch
    import yaml

    import test_edlora
    from mixofshow.data.prompt_dataset import PromptDataset
    assert torch.cuda.is_available(), 'validation_bench needs a GPU'
    result = {'card': card()}
    with tempfile.TemporaryDirectory() as tmp:
        base = os.path.join(tmp, 'sd15')
        t = time.perf_counter()
        ckpt = make_checkpoint(os.path.join(tmp, 'edlora.pth'), make_model_dir(base))
        result['setup_s'] = round(time.perf_counter() - t, 1)
        opt = {'name': 'bench', 'path': {'visualization': os.path.join(tmp, 'vis')},
               'datasets': {'val_vis': {'name': 'PromptDataset', 'prompts': PROMPTS, 'num_samples_per_prompt': 8,
                                        'latent_size': [4, 64, 64], 'replace_mapping': {'<TOK>': '<potter1> <potter2>'},
                                        'batch_size_per_gpu': 4}},
               'val': {'compose_visualize': True, 'sample': {'num_inference_steps': 50, 'guidance_scale': 7.5}}}
        dataset = PromptDataset(opt['datasets']['val_vis'])
        pipe = test_edlora.load_pipeline(base, ckpt, 0.7)
        # warm-up: engines and graphs for the full and the short batch are built on their first call
        warm = yaml.safe_load(yaml.safe_dump(opt))
        warm['val']['sample']['num_inference_steps'] = 2
        warm['path']['visualization'] = os.path.join(tmp, 'warm')
        test_edlora.visual_validation(pipe, dataset, 'warm', warm)
        torch.cuda.synchronize()
        t = time.perf_counter()
        test_edlora.visual_validation(pipe, dataset, 'validation_edlora_0.7', opt)
        torch.cuda.synchronize()
        pass_s = time.perf_counter() - t
        n = len(dataset)
        result['alpha_pass'] = {'images': n, 'pipeline_calls': -(-n // 4), 'unet_steps_batch8': 50 * -(-n // 4),
                                'seconds': round(pass_s, 2), 'images_per_s': round(n / pass_s, 3)}
        result['step_ms'] = {'unet_batch8': round(step_ms(pipe, 4, args.step_reps), 3),
                             'unet_batch2': round(step_ms(pipe, 1, args.step_reps), 3)}
        z = torch.randn(4, 4, 64, 64, generator=torch.Generator().manual_seed(6)).cuda()
        pipe.vae.decode(z)
        torch.cuda.synchronize()
        result['vae_decode_batch4_ms'] = round(time_events(lambda: pipe.vae.decode(z), 10), 2)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'validation_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
