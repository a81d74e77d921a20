"""Device time of the two T2I-Adapters (key pose: 3 input channels, sketch: 1) at 768 x 1536 next to one config-4 denoise
step (BASELINE.json config 4: 768 x 1536, CFG batch 2, 3 regions + 4 adapter maps; UNet graph replay + the fused CFG /
DPM-Solver++ update).  The adapters run once per image, the step once per denoising step.

  python tools/adapter_bench.py [--iters 20]

Synthetic weights (random, fan-in scaled); time = CUDA events around `iters` back-to-back calls after 3 warm-up calls.
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

import bench  # noqa: E402  (synthetic SD1.5-topology UNet weights)


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def adapter_ms(cin, iters):
    from mos_b200.adapter_engine import AdapterEngine, adapter_param_shapes
    g = torch.Generator().manual_seed(cin)
    sd = {}
    for k, s in adapter_param_shapes(cin, (320, 640, 1280, 1280), 2).items():
        fan_in = 1
        for d in s[1:]:
            fan_in *= d
        sd[k] = torch.randn(s, generator=g) * (fan_in ** -0.5 if len(s) > 1 else 0.01)
    eng = AdapterEngine(sd, 1, 768, 1536, in_channels=cin)
    img = torch.rand(1, cin, 768, 1536, generator=g).cuda()
    ms = timed(lambda: eng.forward(img), iters)
    return ms, eng.launches


def step_ms(iters):
    from mos_b200 import ops
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from mos_b200.scheduler import DPMSolverPP2M
    sd = bench.build_workload(False)[0]
    H, W, B = 96, 192, 2
    eng = UNetEngine(sd, B, H, W)
    g = torch.Generator().manual_seed(20)
    px = [[3, 5, 768, 368], [11, 368, 768, 690], [2, 977, 768, 1494]]
    eng.set_regions([(ehs_to_layer_major(torch.randn(B, 16, 77, 768, generator=g).cuda()),
                      (h0 / 768, w0 / 1536, h1 / 768, w1 / 1536)) for h0, w0, h1, w1 in px], (768, 1536))
    shapes = [(320, 96, 192), (640, 48, 96), (1280, 24, 48), (1280, 12, 24)]
    eng.set_adapters([(torch.randn(B * h * w, c, generator=g) * 0.1).to(eng.ACT).cuda() for c, h, w in shapes])
    eng.in_ehs.copy_(ehs_to_layer_major(torch.randn(B, 16, 77, 768, generator=g).cuda()))
    sched = DPMSolverPP2M()
    sched.set_timesteps(30)
    latents = torch.randn(1, 4, H, W, generator=g).cuda()
    x0_prev = torch.zeros_like(latents)
    eng.in_latents.copy_(torch.cat([latents, latents]))
    eng.in_t.fill_(float(sched.timesteps[0]))

    def step():
        eng.run()
        ops.cfg_dpmpp_step(eng.out_eps, latents, x0_prev, eng.in_latents.view(-1), cfg=True, guidance=7.5,
                           coef=sched.coefficients(1), t_out=eng.in_t, t_next=float(sched.timesteps[1]))
    return timed(step, iters)


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--iters', type=int, default=20)
    a = p.parse_args()
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    q = subprocess.run(['nvidia-smi', '-i', f'GPU-{props.uuid}', '--query-gpu=name,power.limit',
                        '--format=csv,noheader,nounits'], capture_output=True, text=True, check=True).stdout
    name, power = [f.strip() for f in q.strip().split(',')]
    kp, n = adapter_ms(3, a.iters)
    sk, _ = adapter_ms(1, a.iters)
    st = step_ms(a.iters)
    print(json.dumps({'gpu': name, 'power_limit_w': float(power), 'size': '768x1536',
                      'keypose_adapter_ms': round(kp, 3), 'sketch_adapter_ms': round(sk, 3), 'adapter_launches': n,
                      'config4_step_ms': round(st, 3), 'adapters_over_step': round((kp + sk) / st, 3),
                      'data': 'synthetic (random weights, random image / embeddings / adapter maps)'}))


if __name__ == '__main__':
    main()
