"""GPU mirror of the reference's `regionally_controlable_sampling.py` entry script (BASELINE config 4): region-string
parsing, model loading from a fused `combined_model_*` directory, and the sampling call.  Host logic only; the UNet loop runs
on `RegionallyT2IAdapterPipeline` (mixofshow/pipelines/pipeline_regionally_t2iadapter.py).

Conditions are condition images (`--keypose_condition` / `--sketch_condition`, as in the reference) run through T2I-Adapters
loaded from LOCAL directories (`--keypose_adapter` / `--sketch_adapter`: the reference downloads them from the hub), or
pre-computed adapter feature maps (`--keypose_adapter_state` / `--sketch_adapter_state file.pt`: the 4 maps a T2IAdapter
returns).  Out of scope here (SURVEY.md §8f): the VAE, so the result is written as latents."""
import argparse
import ast
import json
import os

import torch


def prepare_text(prompt, region_prompts, height, width):
    """regionally_controlable_sampling.py:67-94.  region_prompts:
    '[subject1]-*-[negative1]-*-[h0, w0, h1, w1]|[subject2]-*-[negative2]-*-[...]' (pixel boxes; '[]' = whole image) ->
    (prompt, [(region prompt, region negative prompt, [h0/H, w0/W, h1/H, w1/W]), ...]).  The box arithmetic is Python
    float division exactly as in the reference (the fractions feed the bit-exact ceil/floor of the region masks)."""
    region_collection = []
    for region in region_prompts.split('|'):
        if region == '':
            break
        prompt_region, neg_prompt_region, pos = region.split('-*-')
        prompt_region = prompt_region.replace('[', '').replace(']', '')
        neg_prompt_region = neg_prompt_region.replace('[', '').replace(']', '')
        pos = list(ast.literal_eval(pos))          # the reference uses eval(); the strings are list literals
        if len(pos) == 0:
            pos = [0, 0, 1, 1]
        else:
            pos[0], pos[2] = pos[0] / height, pos[2] / height
            pos[1], pos[3] = pos[1] / width, pos[3] / width
        region_collection.append((prompt_region, neg_prompt_region, pos))
    return (prompt, region_collection)


def build_model(pretrained_model, device='cuda', tokenizer=None):
    """reference :55-64: pipeline + new_concept_cfg.json from a fused model directory."""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionallyT2IAdapterPipeline
    from mixofshow.utils import model_io
    assert os.path.exists(os.path.join(pretrained_model, 'new_concept_cfg.json'))
    unet = model_io.load_unet(pretrained_model)
    text_encoder = model_io.load_text_encoder(pretrained_model, device=device)
    if tokenizer is None:
        from transformers import CLIPTokenizer
        tokenizer = CLIPTokenizer.from_pretrained(pretrained_model, subfolder='tokenizer')
    new_concept_cfg = model_io.load_new_concept_cfg(pretrained_model)
    model_io.ensure_concept_tokens(tokenizer, new_concept_cfg)      # the fused model's added `<new{k}>` tokens
    pipe = RegionallyT2IAdapterPipeline(text_encoder=text_encoder, tokenizer=tokenizer, unet=unet).to(device)
    pipe.set_new_concept_cfg(new_concept_cfg)
    return pipe


def sample_image(pipe, input_prompt, input_neg_prompt=None, generator=None, num_inference_steps=50, guidance_scale=7.5,
                 **extra_kargs):
    """reference :14-52 (adapter states / weights travel in extra_kargs: keypose_adapter_state=..., sketch_adaptor_weight=...)."""
    return pipe(prompt=input_prompt, negative_prompt=input_neg_prompt, generator=generator, guidance_scale=guidance_scale,
                num_inference_steps=num_inference_steps, **extra_kargs).images


def parse_args(argv=None):
    parser = argparse.ArgumentParser('', add_help=False)
    parser.add_argument('--pretrained_model', required=True, type=str)
    parser.add_argument('--sketch_adapter_state', default=None, type=str, help='torch file: 4 pre-computed sketch adapter maps')
    parser.add_argument('--sketch_adaptor_weight', default=1.0, type=float)
    parser.add_argument('--region_sketch_adaptor_weight', default='', type=str)
    parser.add_argument('--keypose_adapter_state', default=None, type=str, help='torch file: 4 pre-computed keypose adapter maps')
    parser.add_argument('--keypose_adaptor_weight', default=1.0, type=float)
    parser.add_argument('--region_keypose_adaptor_weight', default='', type=str)
    parser.add_argument('--height', default=768, type=int)
    parser.add_argument('--width', default=1536, type=int)
    parser.add_argument('--save_dir', default=None, type=str)
    parser.add_argument('--prompt', default='photo of a toy', type=str)
    parser.add_argument('--negative_prompt', default='', type=str)
    parser.add_argument('--prompt_rewrite', default='', type=str)
    parser.add_argument('--seed', default=16141, type=int)
    parser.add_argument('--suffix', default='', type=str)
    parser.add_argument('--num_inference_steps', default=50, type=int)       # the reference samples with 50 steps (:38)
    parser.add_argument('--sketch_condition', default=None, type=str, help='sketch condition image (opened as L)')
    parser.add_argument('--keypose_condition', default=None, type=str, help='key-pose condition image (opened as RGB)')
    parser.add_argument('--sketch_adapter', default=None, type=str, help='local T2I-Adapter directory for --sketch_condition')
    parser.add_argument('--keypose_adapter', default=None, type=str,
                        help='local T2I-Adapter directory for --keypose_condition')
    return parser.parse_args(argv)


CONDITION_ARGS = ('sketch_condition', 'keypose_condition', 'sketch_adapter', 'keypose_adapter')
_MODES = {'sketch': 'L', 'keypose': 'RGB'}           # reference :118-130


def load_conditions(args):
    """reference :118-135: open the condition images (sketch as 'L', key pose as 'RGB'); when any is given, height and width
    become its size (two conditions must agree) and are written back to `args`.  -> {kind: PIL image}.  A condition needs
    its adapter directory (the reference's hub downloads are not made here) and excludes a precomputed state."""
    from PIL import Image
    conds = {}
    for kind, mode in _MODES.items():
        path = getattr(args, f'{kind}_condition')
        if path is None:
            continue
        if getattr(args, f'{kind}_adapter') is None:
            raise ValueError(f'--{kind}_condition needs --{kind}_adapter (a local T2I-Adapter directory)')
        if getattr(args, f'{kind}_adapter_state') is not None:
            raise ValueError(f'--{kind}_condition and --{kind}_adapter_state both give the {kind} adapter features')
        conds[kind] = Image.open(path).convert(mode)
    sizes = {im.size for im in conds.values()}
    if len(sizes) > 1:
        raise ValueError(f'conditions should be same size, got (width, height) {sorted(sizes)}')
    if sizes:
        args.width, args.height = sizes.pop()
    return conds


def main(argv=None):
    """`python regionally_controlable_sampling.py ...`, or `torchrun --nproc_per_node 2 ...`: the two ranks sample the one
    image together, each running one classifier-free-guidance half (RegionallyT2IAdapterPipeline's `cfg_group`), and
    rank 0 alone writes the outputs."""
    import torch.distributed as dist
    from mos_b200 import dp
    args = parse_args(argv)
    conds = load_conditions(args)
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world not in (1, 2):
        raise ValueError(f'regional sampling runs on 1 process, or on 2 under torchrun (one classifier-free-guidance '
                         f'half each); got WORLD_SIZE={world}')
    rank, world, device = dp.init_distributed()
    try:
        return _sample(args, conds, rank, torch.device(device), dist.group.WORLD if world == 2 else None)
    finally:
        if world > 1:
            dist.destroy_process_group()


def _sample(args, conds, rank, device, cfg_group):
    pipe = build_model(args.pretrained_model, device)
    kwargs = {'height': args.height, 'width': args.width, 'output_type': 'latent', 'cfg_group': cfg_group}
    for kind in ('sketch', 'keypose'):
        path = getattr(args, f'{kind}_adapter_state')
        if path is not None:
            kwargs[f'{kind}_adapter_state'] = torch.load(path)
        if kind in conds:
            from mixofshow.models.adapter_b200 import T2IAdapter
            setattr(pipe, f'{kind}_adapter', T2IAdapter.from_pretrained(getattr(args, f'{kind}_adapter'), device=device))
            kwargs[f'{kind}_adapter_input'] = [conds[kind]]
        kwargs[f'{kind}_adaptor_weight'] = getattr(args, f'{kind}_adaptor_weight')
        kwargs[f'region_{kind}_adaptor_weight'] = getattr(args, f'region_{kind}_adaptor_weight')
    input_prompt = [prepare_text(args.prompt, args.prompt_rewrite, args.height, args.width)]
    latents = sample_image(pipe, input_prompt=input_prompt, input_neg_prompt=[args.negative_prompt],
                           generator=torch.Generator('cpu').manual_seed(args.seed),
                           num_inference_steps=args.num_inference_steps, **kwargs)
    if args.save_dir is not None and rank == 0:
        os.makedirs(args.save_dir, exist_ok=True)
        out = os.path.join(args.save_dir, f'latents---{args.seed}{"---" + args.suffix if args.suffix else ""}.pt')
        # condition options that were not given are left out, so an unconditioned run records what it always did
        config = {k: v for k, v in vars(args).items() if not (k in CONDITION_ARGS and v is None)}
        torch.save({'latents': latents.cpu(), 'config': config}, out)
        with open(os.path.join(args.save_dir, 'config.json'), 'w') as f:
            json.dump(config, f)
        print(f'save to: {out}')
    return latents


if __name__ == '__main__':
    main()
