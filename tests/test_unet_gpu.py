"""End-to-end parity of the GPU UNet engine against the fp32 CPU oracle (oracle/unet.py + oracle/inject.py).

Metric: rel-L2 = ||a-b||_2 / ||b||_2.  The sampling engine runs fp16 operands (weights and activations; fp32 accumulation,
fp32 statistics) - the reference's own sampling precision - the oracle is fp32.  Tolerances: eps (UNet output) rel-L2 <=
5e-3 (tests/numerics_emulation.py predicts ~1e-3); post-scheduler latents (one DPM-Solver++ step from a 50-step schedule,
SURVEY.md §8d) rel-L2 <= 1e-3 — the target BASELINE.json states — BOTH for BASELINE config 1 (guidance <= 1) and for
classifier-free guidance 7.5, which is what bench.py times (the scheduler input u + 7.5 (c - u) amplifies the activation
rounding noise of the two halves ~10x: 2.8e-3 with bf16 activations in round 1, 4.6e-4 predicted with fp16).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _setup(cfg, B, H, W, lora_mode, seed=0):
    from oracle import inject, unet as ou
    unet = ou.build_unet(seed, cfg)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10) if lora_mode else None
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    if lora is not None:
        inject.inject_lora(unet, lora, alpha=1.0)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(B, 4, H, W, generator=g)
    ehs = torch.randn(B, 16, 77, 768, generator=torch.Generator().manual_seed(2))
    return unet, sd, lora, lat, ehs


def _engine(sd, lora, B, H, W, cfg, merge=False):
    from mos_b200.engine import UNetEngine
    kw = {}
    if cfg:
        kw = dict(block_out=cfg['block_out_channels'], layers=cfg['layers_per_block'])
    return UNetEngine(sd, B, H, W, lora=lora, lora_alpha=1.0, merge_lora=merge, **kw)


@pytest.mark.parametrize('lora_mode', ['none', 'fused', 'merged'])
def test_unet_tiny(cuda, lora_mode):
    from mos_b200.engine import ehs_to_layer_major
    from oracle import unet as ou
    B, H, W = 2, 32, 32
    unet, sd, lora, lat, ehs = _setup(ou.TINY, B, H, W, lora_mode != 'none')
    t = torch.tensor([981.0, 981.0])
    with torch.no_grad():
        ref = unet(lat, torch.tensor([981, 981]), ehs).sample
    eng = _engine(sd, lora, B, H, W, ou.TINY, merge=(lora_mode == 'merged'))
    n_x = len(eng.xattn_names)
    out = eng.forward(lat.cuda(), t.cuda(), ehs_to_layer_major(ehs[:, :n_x].cuda(), n_x)).clone()
    torch.cuda.synchronize()
    e1 = rel_l2(out, ref)
    out2 = eng.forward(lat.cuda(), t.cuda(), ehs_to_layer_major(ehs[:, :n_x].cuda(), n_x))  # graph replay
    torch.cuda.synchronize()
    assert torch.equal(out2, out), 'CUDA-graph replay must be bitwise reproducible'
    print(f'tiny unet [{lora_mode}] eps rel-L2 = {e1:.3e}, launches = {eng.launches}')
    assert e1 < 5e-3


def test_unet_sd15_step(cuda):
    """BASELINE config 1 shape on the GPU: one CFG denoise step (batch 2) of the full SD1.5 topology with un-merged
    ED-LoRA on all 128 attention linears, then CFG + DPM-Solver++ update; compared with the fp32 oracle."""
    from mos_b200 import ops
    from mos_b200.engine import ehs_to_layer_major
    from oracle import edlora_ref as er
    from oracle.schedulers import DPMSolverMultistepScheduler
    B, H, W = 2, 64, 64
    unet, sd, lora, lat1, ehs = _setup(None, B, H, W, True)
    lat1 = lat1[:1]
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(50)
    t0 = int(sched.timesteps[0])
    lat2 = torch.cat([lat1, lat1])
    with torch.no_grad():
        eps_ref = unet(lat2, torch.tensor([t0, t0]), ehs).sample
    prev_ref = sched.step(er.cfg_combine(eps_ref, 7.5), t0, lat1).prev_sample
    eng = _engine(sd, lora, B, H, W, None)
    eps = eng.forward(lat2.cuda(), torch.tensor([float(t0)] * 2).cuda(), ehs_to_layer_major(ehs.cuda()))
    torch.cuda.synchronize()
    e_eps = rel_l2(eps, eps_ref)
    latents = lat1.cuda().clone()
    x0_prev = torch.zeros_like(latents)
    ops.cfg_dpmpp_step(eps, latents, x0_prev, None, cfg=True, guidance=7.5, coef=sched.coefficients(0))
    torch.cuda.synchronize()
    e_lat = rel_l2(latents, prev_ref)
    # BASELINE config 1: no guidance (conditional half only)
    prev_ref1 = DPMSolverMultistepScheduler()
    prev_ref1.set_timesteps(50)
    ref1 = prev_ref1.step(eps_ref[1:], t0, lat1).prev_sample
    lat_ng = lat1.cuda().clone()
    ops.cfg_dpmpp_step(eps[1:].contiguous(), lat_ng, torch.zeros_like(lat_ng), None, cfg=False, guidance=1.0,
                       coef=sched.coefficients(0))
    torch.cuda.synchronize()
    e_lat1 = rel_l2(lat_ng, ref1)
    print(f'sd1.5 unet eps rel-L2 = {e_eps:.3e}; post-scheduler latents rel-L2: guidance 1 = {e_lat1:.3e}, '
          f'guidance 7.5 = {e_lat:.3e}; launches = {eng.launches}')
    assert e_eps < 5e-3
    assert e_lat1 < 1e-3
    assert e_lat < 1e-3
