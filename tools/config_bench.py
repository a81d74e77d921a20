"""Wall-clock numbers for BASELINE.json configs 3 and 4 at full size on one H100 (synthetic data, SURVEY.md 8d).

  python tools/config_bench.py regional      # config 4: 768x1536, 3 regions + 4 adapter maps, 30 DPM-Solver++ steps, CFG 7.5
  python tools/config_bench.py fusion        # config 3: UNet half of gradient fusion, 5 synthetic ED-LoRAs, 500 / 50 iters
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

import bench  # noqa: E402  (synthetic SD1.5-topology weights / LoRAs; no oracle on this path)


def regional(steps=30):
    from mos_b200 import ops
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from mos_b200.scheduler import DPMSolverPP2M
    sd = bench.build_workload(False)[0]
    H, W = 96, 192                      # latent size of 768 x 1536
    B = 2                               # CFG
    eng = UNetEngine(sd, B, H, W)       # fused checkpoint: LoRA already merged into the weights (regional :56-63)
    g = torch.Generator().manual_seed(20)
    ctx = torch.randn(B, 16, 77, 768, generator=g)
    px = [[3, 5, 768, 368], [11, 368, 768, 690], [2, 977, 768, 1494]]      # regionally_sample.sh:66-74 scaled x0.75
    regions = []
    for r, (h0, w0, h1, w1) in enumerate(px):
        emb = torch.randn(B, 16, 77, 768, generator=torch.Generator().manual_seed(21 + r))
        regions.append((ehs_to_layer_major(emb.cuda()), (h0 / 768, w0 / 1536, h1 / 768, w1 / 1536)))
    eng.set_regions(regions, (768, 1536))
    shapes = [(320, 96, 192), (640, 48, 96), (1280, 24, 48), (1280, 12, 24)]
    eng.set_adapters([(torch.randn(B * h * w, c, generator=g) * 0.1).to(eng.ACT).cuda() for c, h, w in shapes])
    eng.in_ehs.copy_(ehs_to_layer_major(ctx.cuda()))
    sched = DPMSolverPP2M()
    sched.set_timesteps(steps)
    ts = [float(t) for t in sched.timesteps]
    lat0 = torch.randn(1, 4, H, W, generator=torch.Generator().manual_seed(14)).cuda()
    latents, x0_prev = lat0.clone(), torch.zeros_like(lat0)

    def run():
        latents.copy_(lat0)
        x0_prev.zero_()
        eng.in_latents.copy_(torch.cat([latents, latents]))
        eng.in_t.fill_(ts[0])
        for i in range(steps):
            eng.run()
            nxt = ts[i + 1] if i + 1 < steps else 0.0
            ops.cfg_dpmpp_step(eng.out_eps, latents, x0_prev, eng.in_latents.view(-1), cfg=True, guidance=7.5,
                               coef=sched.coefficients(i), t_out=eng.in_t, t_next=nxt)

    run()                               # warm-up + graph capture
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    assert torch.isfinite(latents).all()
    print(json.dumps({'config': 'regionally_controlable_sampling 3-region 768x1536, 30 DPMSolver steps, 1xH100',
                      'seconds_per_image_unet_loop': round(ms / 1e3, 4), 'ms_per_step': round(ms / steps, 3),
                      'steps_per_s': round(steps / ms * 1e3, 2), 'launches_per_step': eng.launches,
                      'algorithmic_tflop_per_step': 11.11, 'tflops': round(11.11 * steps / ms * 1e3, 1),
                      'data': 'synthetic (random-init SD1.5 weights, random embeddings / adapter maps)'}))


def fusion():
    import gradient_fusion as gf
    sd = bench.build_workload(False)[0]
    loras = [bench.random_unet_lora(sd, None, seed=10 + c) for c in range(5)]
    spatial = [{k: v for k, v in l.items() if 'attn2.to_k' not in k and 'attn2.to_v' not in k} for l in loras]
    crosskv = [{k: v for k, v in l.items() if 'attn2.to_k' in k or 'attn2.to_v' in k} for l in loras]
    alphas = [1.0] * 5
    out = {'config': 'gradient_fusion merge of 5 ED-LoRAs into SD1.5-topology UNet weights on 1xH100 (UNet half)',
           'workers': gf.FUSION_WORKERS, 'native_driver': gf.FUSION_NATIVE}
    solve_s = []
    _solve_all = gf.solve_all

    def timed_solve_all(jobs, iters, workers=None):      # how much of a stage is the L-BFGS solves themselves
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = _solve_all(jobs, iters, workers)
        torch.cuda.synchronize()
        solve_s.append(round(time.perf_counter() - t, 2))
        return r

    gf.solve_all = timed_solve_all
    # ---- cross-attention K/V: 32 layers, X = 6 text-feature rows per concept (3 positions x 2 prompts), 500 iterations
    kv_names = sorted({k.replace('.lora_down', '').replace('.lora_up', '') for k in crosskv[0]})
    from mos_b200.engine import cross_attention_names
    order = {n: i for i, n in enumerate(cross_attention_names())}
    layer_list = [(order[n.rsplit('.to_', 1)[0]], n) for n in kv_names]
    feats = [{i: torch.randn(6, 768, generator=torch.Generator().manual_seed(100 + 16 * c + i)) for i in range(16)}
             for c in range(5)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    w_kv = gf.merge_kv_in_cross_attention(sd, layer_list, feats, crosskv, alphas, 500)
    torch.cuda.synchronize()
    out['cross_kv_seconds'] = round(time.perf_counter() - t0, 2)
    out['cross_kv_layers'] = len(w_kv)
    out['cross_kv_solve_seconds'] = solve_s[-1]
    # ---- spatial attention: 96 layers, 5 x 20 recorded UNet forwards (Gram accumulation on the GPU), 50 iterations
    embeds = [torch.randn(1, 16, 77, 768, generator=torch.Generator().manual_seed(30 + c)) for c in range(5)]
    t0 = time.perf_counter()
    w_sp = gf.merge_spatial_attention(sd, spatial, alphas, embeds, 50, latent_hw=(64, 64), num_inference_steps=20)
    torch.cuda.synchronize()
    out['spatial_seconds'] = round(time.perf_counter() - t0, 2)
    out['spatial_layers'] = len(w_sp)
    out['spatial_solve_seconds'] = solve_s[-1]
    name = 'down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q.weight'
    out['example_delta_rel'] = round(((w_sp[name] - sd[name]).norm() / sd[name].norm()).item(), 5)
    out['data'] = 'synthetic (random-init weights, 5 random ED-LoRAs up~N(0,0.02^2), random text features)'
    print(json.dumps(out))


if __name__ == '__main__':
    {'regional': regional, 'fusion': fusion}[sys.argv[1]]()
