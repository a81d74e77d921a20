"""Training-step throughput of the H100 ED-LoRA path (BASELINE configs 2 and 5): SD1.5 topology, 64x64 latents,
synthetic data, random-init weights.  One process per GPU; the batch is sharded (weak scaling: --batch per GPU) and the
ONLY collective is one NCCL all-reduce of the flat LoRA gradient (3.19 MB) per step.

  python tools/train_bench.py --batch 4                      # config 2 (1 GPU, batch 4)
  python tools/train_bench.py --batch 4 --where Transformer2DModel   # LoRA on whole transformer blocks
  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/train_bench.py --batch 8   # config 5
Timed region: K x (forward + loss + backward CUDA graph, all-reduce, AdamW + LoRA re-pack), CUDA events, max over ranks.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--no-reg', action='store_true')
    ap.add_argument('--where', default='Attention', choices=('Attention', 'Transformer2DModel'),
                    help='UNet LoRA placement (lora_cfg.where)')
    a = ap.parse_args()
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    from mos_b200 import dp
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    import bench
    sd, lora = bench.build_workload(False)[:2]
    if a.where != 'Attention':          # the wider placement adds pairs for proj_in / proj_out / ff.net.0.proj / ff.net.2
        from mixofshow.pipelines.trainer_edlora import _NameProbe
        gl = torch.Generator().manual_seed(11)
        for m in TrainEngine.lora_module_names.__get__(_NameProbe({}, a.where))():
            if f'{m}.lora_down.weight' not in lora:
                w = sd[m + '.weight']
                n, k = w.shape[0], w[0].numel()
                lora[f'{m}.lora_down.weight'] = (torch.rand(4, k, generator=gl) * 2 - 1) / k ** 0.5
                lora[f'{m}.lora_up.weight'] = torch.randn(n, 4, generator=gl) * 0.02
    B = a.batch
    eng = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=None if a.no_reg else 0.01, where=a.where)
    g = torch.Generator().manual_seed(100 + rank)
    x0 = torch.randn(B, 4, 64, 64, generator=g).cuda()
    noise = torch.randn(B, 4, 64, 64, generator=g).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    ehs = ehs_to_layer_major(torch.randn(B, 16, 77, 768, generator=g).cuda())
    masks = torch.zeros(B, 1, 64, 64)
    masks[:, :, 12:50, 16:44] = 1.0
    masks = masks.cuda()
    pos = [[4, 5]] * B

    def step():
        out = eng.forward_backward(x0, noise, t, ehs, masks, token_pos=pos)
        scale = dp.allreduce_flat_device(eng.state, out[0:1])
        dp.optimizer_step(eng.state, scale)
        eng.refresh_lora()

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device='cuda')
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = ms.item() / a.steps
    loss = eng.state.grads[eng.state.n].item() / world
    if rank == 0:
        print(json.dumps({'metric': 'ED-LoRA train samples/sec (SD1.5 UNet @512^2, bf16, UNet-LoRA group)',
                          'value': round(B * world / ms * 1e3, 2), 'unit': 'samples/s', 'n_gpus': world,
                          'ms_per_step': round(ms, 3), 'batch_per_gpu': B, 'global_batch': B * world,
                          'scaling': 'weak', 'allreduce_bytes_per_step': (eng.state.n + 2) * 4,
                          'lora_params': eng.state.n, 'loss': round(loss, 5), 'data': 'synthetic',
                          'attn_reg': not a.no_reg, 'where': a.where}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
