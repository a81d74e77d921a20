"""GPU mirror of the reference training entry point (train_edlora.py): `python train_edlora.py -opt <yml>` ->
`EDLoRATrainer(**opt['models'])` -> the loop of train_edlora.py:105-158.

One process per GPU (launch with torchrun for data parallelism), the batch sharded across ranks, ONE NCCL all-reduce per
optimiser step on the flat fp32 gradient buffer [concept embedding rows | CLIP LoRA | UNet LoRA | loss, Norm_mean]
(SURVEY.md 8e; the reference's DDP moves the whole 152 MB embedding gradient, train_edlora.py:70,128), fused flat AdamW with
the learning rates of the groups trainer_edlora.py:82-139 enables, linear learning-rate decay to zero (diffusers
get_scheduler('linear', warmup 0), train_edlora.py:85-90), the `Norm_mean >= emb_norm_threshold` embedding freeze
(:138-143).  The reference's "restore every non-concept row after the step" (:133-136) needs no code here: only the concept
rows are parameters of the flat state.

Data: the image pipeline (LoraDataset transforms, VAE encoder) is outside the hot path (SURVEY.md 8f); the yml's
`datasets.train` is read as a `LatentDataset`: `path` = a torch file {'latents' [n,4,h,w] (VAE latents x 0.18215),
'prompts' [n str], 'masks' [n,1,h,w], optional 'img_masks'}; `replace_mapping`, `batch_size_per_gpu` and
`dataset_enlarge_ratio` keep their reference meaning.

Checkpoints and validation (train_edlora.py:157-189): `edlora_model-{step}.pth` every `logger.save_checkpoint_freq` steps
and `edlora_model-latest.pth` at the end; with `val.val_during_save`, each saved checkpoint is sampled over
`datasets.val_vis` for every alpha of `val.alpha_list` by test_edlora.py's `visual_validation`, sharded across ranks.

With `models.enable_edlora: false` the trainer is vanilla LoRA (one embedding per concept) and the checkpoints are
`lora_model-{step}.pth` / `lora_model-latest.pth` (train_edlora.py:166-168).  Such a checkpoint cannot be validated through
EDLoRAPipeline, so `val.val_during_save: true` is refused at startup, before anything is built or trained (the reference
only fails after its first checkpoint).
"""
import functools
import os

import torch
import torch.distributed as dist

from mos_b200.dp import allreduce_flat, optimizer_step


def total_iterations(dataset_len, batch_size_per_gpu, world_size, gradient_accumulation_steps=1):
    """train_edlora.py:73-75 (a float, compared with `global_step < total_iter`)."""
    return dataset_len / (batch_size_per_gpu * world_size * gradient_accumulation_steps)


def linear_lr(base_lr, step, num_training_steps):
    """LambdaLR of diffusers' linear schedule with 0 warm-up: lr_k = base * max(0, (T - k) / T)."""
    return base_lr * max(0.0, float(num_training_steps - step) / float(max(1.0, num_training_steps)))


def train(trainer, batches, *, dataset_len, batch_size_per_gpu, gradient_accumulation_steps=1, print_freq=0,
          log=print, emb_norm_threshold=5.5e-1, save_checkpoint_freq=0, save=None):
    """Runs the loop of train_edlora.py:105-158; returns the list of per-step mean losses (rank-averaged).
    `batches`: dicts with either ('images' = latents, 'prompts', 'masks', 'img_masks') for EDLoRATrainer or ('latents',
    'encoder_hidden_states', 'masks', 'img_masks'[, 'text_input_ids']) for UNetLoRATrainer.  `save(global_step)` is
    called after every `save_checkpoint_freq`-th optimiser step (train_edlora.py:157-158)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    total_iter = total_iterations(dataset_len, batch_size_per_gpu, world, gradient_accumulation_steps)
    sched_steps = total_iter * gradient_accumulation_steps
    it = iter(batches)
    global_step, micro, sched_k = 0, 0, 0
    losses = []
    stop_emb_update = False
    base_lrs = norm_buf = None
    while global_step < total_iter:
        batch = next(it)
        masks = batch['masks'] if 'masks' in batch else batch['img_masks']
        if 'prompts' in batch:
            loss = trainer(batch['images'], batch['prompts'], masks, batch['img_masks'], accumulate=micro > 0)
        else:
            loss = trainer(batch['latents'], batch['encoder_hidden_states'], masks, batch['img_masks'],
                           text_input_ids=batch.get('text_input_ids'), accumulate=micro > 0)
        state = trainer.engine.state
        if base_lrs is None:
            base_lrs = tuple(state.lrs)
            norm_buf = torch.zeros(1, device=state.params.device)
        micro += 1
        # accelerate steps the optimiser (and the scheduler) on every micro-batch call but only applies it when
        # gradients are synchronised; the schedule therefore advances once per micro-step (train_edlora.py:128-130)
        if micro == gradient_accumulation_steps:
            lrs = [linear_lr(b, sched_k, sched_steps) for b in base_lrs]
            if stop_emb_update:
                lrs[0] = 0.0                       # frozen embedding rows (:141-143): lr 0 also switches the decay off
            state.lrs = tuple(lrs)
            grad_scale, mean_loss, _ = allreduce_flat(state, loss_value=float(loss))
            optimizer_step(state, grad_scale / gradient_accumulation_steps, norm_out=norm_buf if state.has_rows else None)
            refresh = getattr(trainer, 'refresh', None) or trainer.engine.refresh_lora
            refresh()
            micro = 0
            global_step += 1
            losses.append(mean_loss)
            norm_mean = float(norm_buf) if state.has_rows else None
            # the freeze only matters while the rows train (lr 0 on an empty group changes nothing)
            if state.emb_rows and not stop_emb_update and norm_mean >= emb_norm_threshold:
                stop_emb_update = True
            if print_freq and global_step % print_freq == 0:
                # lr_scheduler.get_last_lr(): the groups present, in the order embedding -> text LoRA -> UNet LoRA
                lr = ','.join(f'{x:.3e}' for x, n in zip(state.lrs, state.group_sizes) if n)
                extra = '' if norm_mean is None else f' Norm_mean {norm_mean:.4f}'
                log(f'iter {global_step}: loss {mean_loss:.5f} lr {lr}{extra}')
            if save is not None and save_checkpoint_freq and global_step % save_checkpoint_freq == 0:
                save(global_step)
        sched_k += 1
    return losses


# ------------------------------------------------------------------------------------------------ `-opt <yml>` entry point
class LatentDataset:
    """Pre-encoded training set (see the module docstring).  Mirrors what LoraDataset yields per sample after the VAE:
    `images` (latents), `prompts` (with `replace_mapping` applied, mixofshow/data/lora_dataset.py), `masks`,
    `img_masks`; `dataset_enlarge_ratio` repeats the set."""

    def __init__(self, cfg):
        blob = torch.load(cfg['path'], map_location='cpu')
        self.latents, self.prompts = blob['latents'].float(), list(blob['prompts'])
        n = len(self.prompts)
        self.masks = blob['masks'].float() if 'masks' in blob else torch.ones(n, 1, *self.latents.shape[-2:])
        self.img_masks = blob['img_masks'].float() if 'img_masks' in blob else torch.ones_like(self.masks)
        for k, v in (cfg.get('replace_mapping') or {}).items():
            self.prompts = [p.replace(k, v) for p in self.prompts]
        self.n = n
        self.enlarge = int(cfg.get('dataset_enlarge_ratio', 1))

    def __len__(self):
        return self.n * self.enlarge

    def batches(self, batch_size, rank=0, world=1, seed=0):
        """endless shuffled batches (DataLoader(shuffle=True, drop_last=True) + the data yielder of train_edlora.py:92-97);
        every rank draws from the same permutation and takes its own slice (accelerate's sharded sampler)."""
        g = torch.Generator().manual_seed(seed)
        while True:
            perm = torch.randperm(len(self), generator=g) % self.n
            per_step = batch_size * world
            for s in range(0, len(perm) - per_step + 1, per_step):
                idx = perm[s + rank * batch_size:s + (rank + 1) * batch_size]
                yield {'images': self.latents[idx], 'prompts': [self.prompts[i] for i in idx.tolist()],
                       'masks': self.masks[idx], 'img_masks': self.img_masks[idx]}


def main(argv=None):
    import argparse

    import yaml
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    parser = argparse.ArgumentParser()
    parser.add_argument('-opt', type=str, required=True)
    args = parser.parse_args(argv)
    with open(args.opt) as f:
        opt = yaml.safe_load(f)
    check_options(opt)
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    seed = opt.get('manual_seed')
    models = dict(opt['models'])
    trainer = EDLoRATrainer(**models, device=f'cuda:{local}', seed=0 if seed is None else seed)   # every rank: same init
    train_opt = opt['train']
    optim = dict(train_opt['optim_g'])
    assert optim.pop('type') == 'AdamW', 'only support AdamW now'                          # train_edlora.py:54-55
    assert abs(optim.get('weight_decay', 0.01) - 0.01) < 1e-12 and tuple(optim.get('betas', (0.9, 0.999))) == (0.9, 0.999), \
        'the fused flat AdamW is built for weight_decay 0.01, betas (0.9, 0.999) (every shipped config)'
    tcfg = opt['datasets']['train']
    dataset = LatentDataset(tcfg)
    bs = int(tcfg['batch_size_per_gpu'])
    accum = int(opt.get('gradient_accumulation_steps', 1))
    log = print if rank == 0 else (lambda *a, **k: None)
    log(f'***** Running training *****  examples {len(dataset)}, batch/GPU {bs}, world {world}, accumulation {accum}')
    name = opt.get('name', 'edlora')
    paths = dict(opt.get('path') or {})
    paths['models'] = paths.get('models') or os.path.join('experiments', name, 'models')
    paths['visualization'] = paths.get('visualization') or os.path.join('experiments', name, 'visualization')
    val_opt = opt.get('val') or {}
    val_dataset = None
    if val_opt.get('val_during_save'):
        from mixofshow.data.prompt_dataset import PromptDataset
        val_dataset = PromptDataset(opt['datasets']['val_vis'])
    save = functools.partial(save_and_validation, trainer, dict(opt, path=paths), val_dataset, rank=rank, world=world,
                             log=log)
    losses = train(trainer, dataset.batches(bs, rank, world, seed=(seed or 0)), dataset_len=len(dataset),
                   batch_size_per_gpu=bs, gradient_accumulation_steps=accum,
                   print_freq=int(opt.get('logger', {}).get('print_freq', 10)), log=log,
                   emb_norm_threshold=float(train_opt.get('emb_norm_threshold', 5.5e-1)),
                   save_checkpoint_freq=int((opt.get('logger') or {}).get('save_checkpoint_freq', 0)), save=save)
    save('latest')
    if world > 1:
        dist.destroy_process_group()
    return losses


def check_options(opt):
    """Refuses (NotImplementedError) what the run could only fail at later: validating vanilla LoRA checkpoints."""
    from mixofshow.pipelines.trainer_edlora import VANILLA_LORA_UNSUPPORTED
    if not opt['models'].get('enable_edlora', True) and (opt.get('val') or {}).get('val_during_save'):
        raise NotImplementedError(f'val.val_during_save: {VANILLA_LORA_UNSUPPORTED}; set val_during_save: false')


def checkpoint_path(opt, global_step):
    """train_edlora.py:166-168: `edlora_model-{step}.pth`, or `lora_model-{step}.pth` for vanilla LoRA"""
    lora_type = 'edlora' if opt['models'].get('enable_edlora', True) else 'lora'
    return os.path.join(opt['path']['models'], f'{lora_type}_model-{global_step}.pth')


def save_and_validation(trainer, opt, val_dataset, global_step, *, rank=0, world=1, log=print):
    """train_edlora.py:165-189: rank 0 writes `checkpoint_path(opt, global_step)`; then every rank waits for it and, when
    `val_dataset` is given, samples its share of the set from that file for each alpha of `val.alpha_list` into
    `Iters-{global_step}_Alpha-{alpha}` (test_edlora.py's `visual_validation`).  The pipeline is loaded fresh from the
    pretrained directory and the checkpoint file, so validation reads nothing of the trainer."""
    save_path = checkpoint_path(opt, global_step)
    if rank == 0:
        os.makedirs(opt['path']['models'], exist_ok=True)
        torch.save({'params': trainer.delta_state_dict()}, save_path)
        log(f'Save state to {save_path}')
    if world > 1:
        dist.barrier()
    if val_dataset is None:
        return
    import test_edlora
    log(f'Start validation {save_path}:')
    for alpha in test_edlora.alpha_list(opt):
        pipe = test_edlora.load_pipeline(opt['models']['pretrained_path'], save_path, alpha)
        test_edlora.visual_validation(pipe, val_dataset, f'Iters-{global_step}_Alpha-{alpha}', opt, rank, world)
        del pipe
        test_edlora.free_pipeline()


if __name__ == '__main__':
    main()
