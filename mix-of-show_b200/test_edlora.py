"""GPU mirror of the reference's sampling entry point (test_edlora.py): `python test_edlora.py -opt <yml>` samples the
`datasets.val_vis` prompt set (a `PromptDataset`) with a trained ED-LoRA checkpoint (`path.lora_path`) once per alpha of
the alpha list, writes one PNG per (prompt, sample) and, with `val.compose_visualize`, one JPEG grid per alpha.

Output: `<visualization>/<val_vis.name>/validation_edlora_<alpha>/{prompt}---G_{guidance}_S_{steps}---{index}---
validation_edlora_<alpha>.png` and `<visualization>/<val_vis.name>/G_{guidance}_S_{steps}---validation_edlora_<alpha>.jpg`,
where `<visualization>` is `path.visualization` or `results/<name>/visualization`.  `train_edlora.py` runs the same
`visual_validation` on every checkpoint it saves when `val.val_during_save` is set.

One process per GPU (launch with torchrun to shard the prompt set): rank r samples batches r, r + W, r + 2W, ... of the
set, so every image is written exactly once.
"""
import gc
import os

import torch
import torch.distributed as dist

from mixofshow.data.prompt_dataset import PromptDataset
from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
from mixofshow.pipelines.trainer_edlora import VANILLA_LORA_UNSUPPORTED
from mixofshow.utils.convert_edlora_to_diffusers import convert_edlora
from mixofshow.utils.util import NEGATIVE_PROMPT, compose_visualize, pil_imwrite
from mos_b200.scheduler import DPMSolverPP2M


def rank_batches(n, batch_size, rank=0, world=1):
    """Index lists of the batches of range(n) that `rank` of `world` samples: batches of `batch_size` in order (the last
    one may be short), every world-th one starting at `rank`."""
    batches = [list(range(s, min(s + batch_size, n))) for s in range(0, n, batch_size)]
    return batches[rank::world]


def alpha_list(opt):
    """`val.alpha_list`, or `models.alpha_list` for configs that keep it there (the shipped anime test config)."""
    val = opt.get('val') or {}
    return list(val['alpha_list'] if 'alpha_list' in val else opt['models']['alpha_list'])


def check_edlora(opt):
    if not opt['models'].get('enable_edlora', True):
        raise NotImplementedError(VANILLA_LORA_UNSUPPORTED)


def load_pipeline(pretrained_path, lora_path, alpha):
    """A freshly loaded pipeline with the ED-LoRA checkpoint at `lora_path` merged at `alpha` (test_edlora.py:90-95)."""
    pipe = EDLoRAPipeline.from_pretrained(pretrained_path,
                                          scheduler=DPMSolverPP2M.from_pretrained(pretrained_path, subfolder='scheduler'))
    pipe, new_concept_cfg = convert_edlora(pipe, torch.load(lora_path, map_location='cpu'), enable_edlora=True,
                                           alpha=alpha)
    pipe.set_new_concept_cfg(new_concept_cfg)
    return pipe


def free_pipeline():
    """Returns the memory of a pipeline whose last reference the caller has dropped, before the next one loads."""
    gc.collect()
    torch.cuda.empty_cache()


def visual_validation(pipe, dataset, current_iter, opt, rank=0, world=1):
    """Samples this rank's batches of `dataset` into `<visualization>/<dataset name>/<current_iter>/`, then (rank 0,
    after every rank has finished) composes the grid when `val.compose_visualize` is set.  Returns that directory."""
    sample = opt['val']['sample']
    guidance_scale = sample.get('guidance_scale', 7.5)
    steps = sample.get('num_inference_steps', 50)
    out_dir = os.path.join(opt['path']['visualization'], dataset.opt.get('name', 'PromptDataset'), f'{current_iter}')
    for idx in rank_batches(len(dataset), dataset.opt['batch_size_per_gpu'], rank, world):
        items = [dataset[i] for i in idx]
        prompts = [it['prompts'] for it in items]
        latents = torch.stack([it['latents'] for it in items])
        images = pipe(prompt=prompts, latents=latents.to(dtype=torch.float16),
                      negative_prompt=[NEGATIVE_PROMPT] * len(prompts), num_inference_steps=steps,
                      guidance_scale=guidance_scale).images
        for img, prompt, it in zip(images, prompts, items):
            img_name = f"{prompt.replace(' ', '_')}---G_{guidance_scale}_S_{steps}---{it['indices']}"
            pil_imwrite(img, os.path.join(out_dir, f'{img_name}---{current_iter}.png'))
        del images
    if world > 1:
        dist.barrier()
    if opt['val'].get('compose_visualize') and rank == 0:
        compose_visualize(out_dir)
    return out_dir


def main(argv=None):
    import argparse

    import yaml
    parser = argparse.ArgumentParser()
    parser.add_argument('-opt', type=str, required=True)
    args = parser.parse_args(argv)
    with open(args.opt) as f:
        opt = yaml.safe_load(f)
    check_edlora(opt)
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    opt['path'] = dict(opt.get('path') or {})
    opt['path']['visualization'] = opt['path'].get('visualization') or os.path.join('results', opt['name'],
                                                                                    'visualization')
    dataset = PromptDataset(opt['datasets']['val_vis'])
    for alpha in alpha_list(opt):
        pipe = load_pipeline(opt['models']['pretrained_path'], opt['path']['lora_path'], alpha)
        if rank == 0:
            print(f'Start validation sample lora({alpha}):')
        visual_validation(pipe, dataset, f'validation_edlora_{alpha}', opt, rank, world)
        del pipe
        free_pipeline()
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
