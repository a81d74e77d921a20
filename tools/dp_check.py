"""SURVEY.md 8d config-5 check on real GPUs (run under torchrun, one rank per GPU, NCCL):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tools/dp_check.py

Every rank runs one data-parallel ED-LoRA step (UNet-LoRA group) on ITS shard: forward + loss + backward, ONE NCCL all-reduce
of the flat gradient buffer, fused AdamW with grad_scale 1/world.  Checked:
  (1) the parameters after the step are BIT-identical on every rank;
  (2) they equal - to fp32 summation-order tolerance - a single-GPU run that accumulates the same `world` shards into one
      gradient buffer (forward_backward(accumulate=True)) and applies the same optimiser step (the reference's
      gradient-accumulation equivalence, train_edlora.py:73-75,120-130).
Prints one JSON line on rank 0."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200')):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402


def shard_data(rank, B, nx, dev):
    from mos_b200.engine import ehs_to_layer_major
    g = torch.Generator().manual_seed(100 + rank)
    x0 = torch.randn(B, 4, 64, 64, generator=g).to(dev)
    noise = torch.randn(B, 4, 64, 64, generator=g).to(dev)
    t = torch.randint(0, 1000, (B,), generator=g).to(dev)
    ehs = ehs_to_layer_major(torch.randn(B, 16, 77, 768, generator=g)[:, :nx].to(dev), nx, torch.bfloat16)
    masks = torch.zeros(B, 1, 64, 64)
    masks[:, :, 8:56, 16:48] = 1.0
    return x0, noise, t, ehs, masks.to(dev)


def main():
    from mos_b200 import dp
    from mos_b200.train_engine import TrainEngine
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    dist.init_process_group('nccl', device_id=dev)
    tiny = '--full' not in sys.argv
    sd, lora, _, _, cfg = bench.build_workload(tiny)
    kw = dict(block_out=cfg['block_out_channels'], layers=cfg['layers_per_block']) if cfg else {}
    B = 2
    pos = [[2, 3]] * B
    # ---- data-parallel step
    eng = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=0.01, device=dev, **kw)
    nx = len(eng.xattn_names)
    x0, noise, t, ehs, masks = shard_data(rank, B, nx, dev)
    out = eng.forward_backward(x0, noise, t, ehs, masks, token_pos=pos)
    scale = dp.allreduce_flat_device(eng.state, out[0:1])
    g_dp = eng.state.grads[:eng.state.n].clone()          # summed over ranks by the collective
    dp.optimizer_step(eng.state, scale)
    p_dp = eng.state.params.clone()
    hi, lo = p_dp.clone(), p_dp.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    identical = bool(torch.equal(hi, lo))
    # ---- the same global batch on ONE GPU by gradient accumulation (every rank repeats it; rank 0 reports)
    ref = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=0.01, device=dev, **kw)
    p0 = ref.state.params.clone()
    for r in range(world):
        d = shard_data(r, B, nx, dev)
        ref.forward_backward(*d, token_pos=pos, accumulate=r > 0)
    g_acc = ref.state.grads[:ref.state.n].clone()
    dp.optimizer_step(ref.state, 1.0 / world)
    p_acc = ref.state.params
    upd_dp, upd_acc = (p_dp - p0).double(), (p_acc - p0).double()
    rel = ((upd_dp - upd_acc).norm() / upd_acc.norm()).item()
    grel = ((g_dp.double() - g_acc.double()).norm() / g_acc.double().norm()).item()
    if rank == 0:
        print(json.dumps({'check': 'config 5: data-parallel step == single-GPU gradient accumulation', 'world': world,
                          'batch_per_gpu': B, 'topology': 'tiny' if tiny else 'sd15',
                          'params_bit_identical_across_ranks': identical,
                          'grad_rel_l2_vs_accumulation': grel, 'update_rel_l2_vs_accumulation': rel, 'update_norm': upd_acc.norm().item(),
                          'n_params': int(p_dp.numel())}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    assert identical and grel < 1e-5 and rel < 1e-3, (identical, grel, rel)


if __name__ == '__main__':
    main()
