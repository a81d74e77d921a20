"""The compute side of CFG-split sampling on one H100: the denoise step of regional sampling at batch 2 (both CFG halves
in one UNet call, as one process samples) against the batch-1 step of each half (what one rank of a two-rank
`cfg_group` call runs), synthetic SD1.5-topology weights, 3 regions and 4 adapter maps.

  python tools/cfg_split_bench.py [--steps 20] [--rounds 2]

A batch-2 step is one graph replay + the fused CFG / DPM-Solver++ kernel writing both copies of the next UNet input.  A
batch-1 step is one graph replay + a copy of the rank's eps into its half of the [2, 4, h, w] buffer (the local part of
the all-gather) + the fused kernel + the copy of the latents into the session's single input.  The exchange itself,
and the wall time per image on two GPUs, need two GPUs and are reported as not measured.  Prints one JSON line per
size, with the card's name, power limit and clocks read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

import bench  # noqa: E402  (synthetic SD1.5-topology weights)

SIZES = {'config4_768x1536': (768, 1536), 'regional_1024x2048': (1024, 2048)}
BOXES = [(3, 5, 768, 368), (11, 368, 768, 690), (2, 977, 768, 1494)]     # config 4's pixel boxes at 768 x 1536
ADAPTER = [(320, 1), (640, 2), (1280, 4), (1280, 8)]


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True)
    return dict(zip(q.split(','), [v.strip() for v in r.stdout.strip().splitlines()[0].split(',')]))


def engines(sd, height, width):
    """-> {'b2': batch-2 engine, 'b1_uncond', 'b1_cond': batch-1 engines}, each with its embeddings, regions and adapter
    maps set as the pipelines set them"""
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    h, w = height // 8, width // 8
    g = torch.Generator().manual_seed(20)
    ctx = torch.randn(2, 16, 77, 768, generator=g)
    regs = [torch.randn(2, 16, 77, 768, generator=g) for _ in BOXES]
    boxes = [(a / 768, b / 1536, c / 768, d / 1536) for a, b, c, d in BOXES]
    ad = [torch.randn(1, c, -(-h // s), -(-w // s), generator=g) * 0.1 for c, s in ADAPTER]
    out = {}
    for name, rows in (('b2', slice(0, 2)), ('b1_uncond', slice(0, 1)), ('b1_cond', slice(1, 2))):
        B = rows.stop - rows.start
        eng = UNetEngine(sd, B, h, w)
        eng.set_regions([(ehs_to_layer_major(r[rows].cuda()), bx) for r, bx in zip(regs, boxes)], (height, width))
        eng.set_adapters([torch.cat([a] * B).cuda().permute(0, 2, 3, 1).reshape(-1, a.shape[1]).to(eng.ACT)
                          for a in ad])
        eng.in_ehs.copy_(ehs_to_layer_major(ctx[rows].cuda()))
        out[name] = eng
    return out


def time_steps(eng, steps, half=None):
    """mean ms per denoise step over `steps` steps (CUDA events); half = None: batch 2, else the batch-1 step of that half"""
    from mos_b200 import ops
    from mos_b200.scheduler import DPMSolverPP2M
    sched = DPMSolverPP2M()
    sched.set_timesteps(steps)
    ts = [float(t) for t in sched.timesteps]
    shape = (1,) + tuple(eng.in_latents.shape[1:])
    latents = torch.randn(shape, generator=torch.Generator().manual_seed(14)).cuda()
    x0_prev = torch.zeros_like(latents)
    both = torch.zeros((2,) + shape[1:], device='cuda')
    eng.in_latents.copy_(latents.expand_as(eng.in_latents))
    eng.in_t.fill_(ts[0])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        eng.run()
        nxt = ts[i + 1] if i + 1 < steps else 0.0
        if half is None:
            ops.cfg_dpmpp_step(eng.out_eps, latents, x0_prev, eng.in_latents.view(-1), cfg=True, guidance=7.5,
                               coef=sched.coefficients(i), t_out=eng.in_t, t_next=nxt)
        else:
            both[half].copy_(eng.out_eps[0])
            ops.cfg_dpmpp_step(both, latents, x0_prev, None, cfg=True, guidance=7.5, coef=sched.coefficients(i),
                               t_out=eng.in_t, t_next=nxt)
            eng.in_latents.copy_(latents)
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(latents).all()
    return e0.elapsed_time(e1) / steps


def time_copy(n, reps=1000):
    """µs per copy of the next batch-1 UNet input (the step's one extra launch)"""
    a, b = torch.randn(n, device='cuda'), torch.empty(n, device='cuda')
    for _ in range(10):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        b.copy_(a)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--sizes', default=','.join(SIZES))
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'the benchmark needs a GPU'
    sd = bench.build_workload(False)[0]
    for key in a.sizes.split(','):
        height, width = SIZES[key]
        engs = engines(sd, height, width)
        for name, eng in engs.items():                      # warm-up + graph capture
            time_steps(eng, 2, None if name == 'b2' else int(name == 'b1_cond'))
        ms = {name: [] for name in engs}
        for _ in range(a.rounds):                           # alternate the three engines within each round
            for name, eng in engs.items():
                ms[name].append(round(time_steps(eng, a.steps, None if name == 'b2' else int(name == 'b1_cond')), 3))
        h, w = height // 8, width // 8
        b2 = min(ms['b2'])
        print(json.dumps({
            'size': key, 'latent': [h, w], 'steps_per_round': a.steps, 'gpu': gpu_info(),
            'b2_step_ms': ms['b2'], 'b1_uncond_step_ms': ms['b1_uncond'], 'b1_cond_step_ms': ms['b1_cond'],
            'b1_over_b2': {n: round(min(ms[n]) / b2, 3) for n in ('b1_uncond', 'b1_cond')},
            'next_input_copy_us': round(time_copy(4 * h * w), 2),
            'exchange_bytes_per_step': 2 * 4 * h * w * 4,
            'two_gpu_wall_per_image': 'not measured', 'nccl_exchange_time': 'not measured',
            'data': 'synthetic (random-init SD1.5 weights, random embeddings / adapter maps)'}), flush=True)
        del engs
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
