"""Sampling at image sizes that are multiples of 8 pixels but not of 64, and at the regional sampler's own 1024 x 2048,
against the fp32 oracle (oracle/unet.py, oracle/vae.py) run ON THE GPU (TF32 off).

diffusers' UNet samples at any latent size: Downsample2D (3x3, stride 2, pad 1) rounds up, and each non-final up block
interpolates (nearest, explicit size) to the size of the skip it is concatenated with.  The engine works out its level
sizes with the same rule (engine.level_sizes), so a 65 x 49 latent runs 65 x 49 -> 33 x 25 -> 17 x 13 -> 9 x 7 and back.

Tolerances as tests/test_unet_gpu.py: eps rel-L2 <= 5e-3, latents after one CFG-7.5 DPM-Solver++ step <= 1e-3;
3-step pipeline loops <= 5e-3 (tests/test_regional_gpu.py); the VAE <= 5e-3 (tests/test_vae_gpu.py).  The oracle's
self-attention runs in query chunks (`chunked_sdpa`): at 1024 x 2048 the 2 x 8 x 32768^2 fp32 score tensor alone would be
68 GB.
"""
import copy
import gc

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# latent sizes (pixel size / 8): every level odd in both sides (520 x 392), even on top then odd (528 x 528), odd on top
# and exact below (1000 x 1000), exact halving with an 81-token mid level (576 x 576), and a one-pixel-wide strip
SD15_LATENTS = [(65, 49), (66, 66), (125, 125), (72, 72), (8, 1)]
REGION_BOXES = [(0.0, 0.0, 1.0, 0.3), (0.0, 0.3, 1.0, 0.62), (0.0, 0.62, 1.0, 1.0)]    # three full-height columns


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _chunked(q, k, v, attn_mask=None, dropout_p=0.0, is_causal=False, scale=None, **kw):
    """softmax(q k^T scale) v in fp32, a block of queries at a time (at most ~1 GB of scores per block)"""
    assert attn_mask is None and not is_causal and dropout_p == 0.0
    scale = q.shape[-1] ** -0.5 if scale is None else scale
    bh = q.numel() // (q.shape[-2] * q.shape[-1])
    step = max(1, (1 << 28) // (bh * k.shape[-2]))
    out = torch.empty(*q.shape[:-1], v.shape[-1], device=q.device, dtype=q.dtype)
    for s in range(0, q.shape[-2], step):
        p = (torch.matmul(q[..., s:s + step, :], k.transpose(-1, -2)) * scale).softmax(-1)
        out[..., s:s + step, :] = torch.matmul(p, v)
    return out


@pytest.fixture
def chunked_sdpa(monkeypatch):
    monkeypatch.setattr(torch.nn.functional, 'scaled_dot_product_attention', _chunked)


@pytest.fixture(scope='module')
def sd15_edlora(cuda):
    """the SD1.5 oracle with ED-LoRA processors and an un-merged random LoRA, on the GPU, and its state / LoRA"""
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, None)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    inject.inject_lora(unet.to(cuda), {k: v.to(cuda) for k, v in lora.items()}, alpha=1.0)
    yield unet, sd, lora
    _free()


def _sched(steps=50):
    from oracle.schedulers import DPMSolverMultistepScheduler
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(steps)
    return sched, int(sched.timesteps[0])


def _cfg_step_ref(eps_ref, lat1, steps=50):
    """the oracle's latents after the first CFG-7.5 DPM-Solver++ step of a `steps`-step schedule"""
    from oracle import edlora_ref as er
    sched, t0 = _sched(steps)
    return sched.step(er.cfg_combine(eps_ref.cpu(), 7.5), t0, lat1).prev_sample


def _engine_step(eng, lat2, t0, ehs_lm):
    """eager walk, then the captured graph twice: all three bit-identical; returns eps"""
    t = torch.tensor([float(t0)] * lat2.shape[0]).cuda()
    eng.use_graph = False
    eager = eng.forward(lat2.cuda(), t, ehs_lm).clone()
    eng.use_graph = True
    g1 = eng.forward(lat2.cuda(), t, ehs_lm).clone()
    g2 = eng.forward(lat2.cuda(), t, ehs_lm).clone()
    torch.cuda.synchronize()
    assert torch.equal(eager, g1), 'captured graph differs from the eager walk'
    assert torch.equal(g1, g2), 'graph replay is not bitwise reproducible'
    return g1


@pytest.mark.parametrize('h,w', SD15_LATENTS, ids=[f'{h}x{w}' for h, w in SD15_LATENTS])
def test_sd15_cfg_step(cuda, sd15_edlora, chunked_sdpa, h, w):
    """one CFG denoise step (batch 2) of the full SD1.5 topology with un-merged ED-LoRA, then CFG 7.5 + DPM-Solver++"""
    from mos_b200 import ops
    from mos_b200.engine import UNetEngine, ehs_to_layer_major, level_sizes
    unet, sd, lora = sd15_edlora
    g = torch.Generator().manual_seed(h * 1000 + w)
    lat1 = torch.randn(1, 4, h, w, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    lat2 = torch.cat([lat1, lat1])
    sched, t0 = _sched()
    with torch.no_grad():
        eps_ref = unet(lat2.cuda(), torch.tensor([t0, t0]).cuda(), ehs.cuda()).sample.cpu()
    prev_ref = _cfg_step_ref(eps_ref, lat1)
    eng = UNetEngine(sd, 2, h, w, lora=lora, lora_alpha=1.0)
    assert eng.level_hw == level_sizes(h, w, 4)
    eps = _engine_step(eng, lat2, t0, ehs_to_layer_major(ehs.cuda()))
    latents = lat1.cuda().clone()
    ops.cfg_dpmpp_step(eps, latents, torch.zeros_like(latents), None, cfg=True, guidance=7.5, coef=sched.coefficients(0))
    torch.cuda.synchronize()
    e_eps, e_lat = rel_l2(eps, eps_ref), rel_l2(latents, prev_ref)
    print(f'SD1.5 {h}x{w} latent (levels {eng.level_hw}): eps rel-L2 {e_eps:.3e}, CFG-7.5 latents rel-L2 {e_lat:.3e}')
    del eng
    _free()
    assert e_eps < 5e-3 and e_lat < 1e-3


@pytest.mark.parametrize('mode', ['fused', 'merged'])
def test_tiny_33(cuda, mode):
    """TINY (two levels) at a 33 x 33 latent: 33 -> 17 -> 33, with the LoRA in the GEMM epilogue or merged"""
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, ou.TINY)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    inject.inject_lora(unet.to(cuda), {k: v.to(cuda) for k, v in lora.items()}, alpha=1.0)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(2, 4, 33, 33, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    with torch.no_grad():
        ref = unet(lat.cuda(), torch.tensor([981, 981]).cuda(), ehs.cuda()).sample
    eng = UNetEngine(sd, 2, 33, 33, lora=lora, lora_alpha=1.0, merge_lora=mode == 'merged', block_out=(320, 640),
                     layers=1)
    n_x = len(eng.xattn_names)
    out = _engine_step(eng, lat, 981, ehs_to_layer_major(ehs[:, :n_x].cuda(), n_x))
    e = rel_l2(out, ref)
    print(f'TINY 33x33 [{mode}]: eps rel-L2 {e:.3e}')
    assert e < 5e-3


# --------------------------------------------------------------------------------------------- the two kernels alone
@pytest.mark.parametrize('B,H,W,Ho,Wo,C', [(2, 9, 7, 17, 13, 1280), (2, 33, 25, 65, 49, 640), (1, 32, 32, 63, 63, 320),
                                           (2, 1, 1, 2, 1, 1280), (3, 5, 3, 9, 5, 16)])
def test_upsample_to_size_kernel(cuda, B, H, W, Ho, Wo, C):
    """mos_upsample2x at an explicit output size against F.interpolate(size=...) bit for bit, read at a pitched row,
    nothing written past y"""
    from gpu_helpers import canary, same_bits
    from mos_b200 import ops
    ld = C + 16
    x = torch.randn(B * H * W, ld, generator=torch.Generator().manual_seed(H * W), dtype=torch.float32)
    x = x.to(torch.float16).cuda()
    y = canary((B * Ho * Wo + 64, C), cuda, torch.float16)
    ops.upsample2x(x, y, B=B, H=H, W=W, C=C, ldx=ld, Ho=Ho, Wo=Wo)
    torch.cuda.synchronize()
    xs = x[:, :C].reshape(B, H, W, C).permute(0, 3, 1, 2)
    want = F.interpolate(xs, size=(Ho, Wo), mode='nearest').permute(0, 2, 3, 1).reshape(-1, C)
    assert same_bits(y[:B * Ho * Wo], want.contiguous())
    assert same_bits(y[B * Ho * Wo:], canary((64, C), cuda, torch.float16))


@pytest.mark.parametrize('B,H,W,C', [(2, 65, 49, 320), (2, 33, 25, 640), (1, 17, 13, 1280), (2, 1, 1, 16), (2, 8, 1, 320)])
def test_im2col_s2_odd_extents(cuda, B, H, W, C):
    """mos_im2col_s2 (pad 1) at odd sides: ceil(H / 2) x ceil(W / 2) output pixels whose 9 taps, times a weight, are
    F.conv2d(stride=2, padding=1) in float64"""
    from gpu_helpers import canary, same_bits
    from mos_b200 import ops
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    x = torch.randn(B * H * W, C, generator=torch.Generator().manual_seed(H + W)).to(torch.float16).cuda()
    col = canary((B * Ho * Wo + 8, 9 * C), cuda, torch.float16)
    ops.im2col_s2(x, col, B=B, H=H, W=W, C=C)
    torch.cuda.synchronize()
    xs = x.double().view(B, H, W, C).permute(0, 3, 1, 2)
    wt = torch.randn(4, C, 3, 3, generator=torch.Generator().manual_seed(5), dtype=torch.float64).cuda()
    got = torch.einsum('ptc,otc->po', col[:B * Ho * Wo].double().view(-1, 9, C), wt.permute(0, 2, 3, 1).reshape(4, 9, C))
    want = F.conv2d(xs, wt, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, 4)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10)
    assert same_bits(col[B * Ho * Wo:], canary((8, 9 * C), cuda, torch.float16))


# ----------------------------------------------------------------------------------------------------- pipelines
@pytest.fixture(scope='module')
def sd15_plain(cuda):
    from oracle import unet as ou
    ref = ou.build_unet(0, None)
    sd = {k: v.clone() for k, v in ref.state_dict().items()}
    yield ref, sd
    _free()


def _b200(sd):
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    u = UNet2DConditionModel()
    u.load_state_dict(sd)
    return u


def _oracle_loop(ref, lat, emb, steps, gs, kw=None):
    from oracle import edlora_ref as er
    from oracle.schedulers import DPMSolverMultistepScheduler
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(steps)
    x = lat.clone()
    for t in sched.timesteps:
        with torch.no_grad():
            eps = ref(torch.cat([x, x]).cuda(), torch.tensor([int(t)] * 2).cuda(), emb.cuda(),
                      cross_attention_kwargs=kw).sample.cpu()
        x = sched.step(er.cfg_combine(eps, gs), int(t), x).prev_sample
    return x


@pytest.mark.parametrize('kind', ['edlora', 'sd'])
def test_pipeline_520x392(cuda, sd15_plain, chunked_sdpa, kind):
    """EDLoRAPipeline (layer-wise embeddings) and StableDiffusionPipeline (one embedding) at 520 x 392, 3 CFG steps"""
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline, StableDiffusionPipeline
    from oracle import inject
    ref, sd = sd15_plain
    ref = copy.deepcopy(ref)
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(1, 4, 65, 49, generator=g)
    ne = torch.randn(1, 77, 768, generator=g)
    steps, gs = 3, 7.5
    if kind == 'edlora':
        inject.install_edlora_processors(ref)
        pe = torch.randn(1, 16, 77, 768, generator=g)
        pipe = EDLoRAPipeline(unet=_b200(sd)).to('cuda')
        pipe.set_new_concept_cfg({})
        emb = torch.cat([ne.view(1, 1, 77, 768).repeat(1, 16, 1, 1), pe])
    else:
        pe = torch.randn(1, 77, 768, generator=g)
        pipe = StableDiffusionPipeline(unet=_b200(sd)).to('cuda')
        emb = torch.cat([ne, pe])
    res = pipe(prompt_embeds=pe.cuda(), negative_prompt_embeds=ne.cuda(), latents=lat.clone(), height=520, width=392,
               num_inference_steps=steps, guidance_scale=gs, output_type='latent').images
    want = _oracle_loop(ref.cuda(), lat, emb, steps, gs)
    e = rel_l2(res, want)
    print(f'{type(pipe).__name__} 520x392, 3 CFG steps vs oracle loop: latents rel-L2 {e:.3e}')
    del pipe, ref
    _free()
    assert e < 5e-3


def _regional_inputs(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(1, 4, h, w, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    regs = [(torch.randn(2, 16, 77, 768, generator=g), b) for b in REGION_BOXES]
    return lat, ehs, regs


def test_regional_pipeline_640x448(cuda, sd15_plain, chunked_sdpa):
    """RegionallyT2IAdapterPipeline without adapters at 640 x 448 (levels 80 x 56 ... 10 x 7), 3 CFG steps vs the oracle
    loop; at 520 x 520 the call refuses (the region rule reads the 33 x 33 level as 32 x 32)"""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionallyT2IAdapterPipeline
    from oracle import inject
    ref, sd = sd15_plain
    ref = copy.deepcopy(ref)
    inject.install_region_processors(ref)
    pipe = RegionallyT2IAdapterPipeline(unet=_b200(sd)).to('cuda')
    pipe.set_new_concept_cfg({})
    lat, ehs, regs = _regional_inputs(80, 56, 9)
    steps, gs = 3, 7.5
    res = pipe(prompt_embeds=ehs.cuda(), region_list=[(r.cuda(), b) for r, b in regs], latents=lat.clone(), height=640,
               width=448, num_inference_steps=steps, guidance_scale=gs, output_type='latent').images
    kw = {'region_list': [(r.cuda(), b) for r, b in regs], 'height': 640, 'width': 448}
    want = _oracle_loop(ref.cuda(), lat, ehs, steps, gs, kw)
    e = rel_l2(res, want)
    print(f'RegionallyT2IAdapterPipeline 640x448, 3 regions, 3 CFG steps vs oracle loop: latents rel-L2 {e:.3e}')
    lat5, ehs5, regs5 = _regional_inputs(65, 65, 10)
    with pytest.raises(ValueError, match='520 x 520'):
        pipe(prompt_embeds=ehs5.cuda(), region_list=[(r.cuda(), b) for r, b in regs5], latents=lat5, height=520,
             width=520, num_inference_steps=steps, guidance_scale=gs, output_type='latent')
    del pipe, ref
    _free()
    assert e < 5e-3


def test_regional_step_1024x2048(cuda, sd15_plain, chunked_sdpa):
    """the reference regional sampler's shipped size: latent 128 x 256 (32768 tokens at level 0), three full-height boxes,
    one CFG step of the full SD1.5 UNet, then CFG 7.5 + DPM-Solver++"""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import revise_regionally_t2iadapter_attention_forward
    from mos_b200 import ops
    from mos_b200.scheduler import DPMSolverPP2M
    from oracle import inject
    ref, sd = sd15_plain
    lat1, ehs, regs = _regional_inputs(128, 256, 11)
    lat2 = torch.cat([lat1, lat1])
    _, t0 = _sched(30)
    kw = {'region_list': [(r.cuda(), b) for r, b in regs], 'height': 1024, 'width': 2048}
    oracle = copy.deepcopy(ref)
    inject.install_region_processors(oracle)
    oracle = oracle.cuda()
    with torch.no_grad():
        eps_ref = oracle(lat2.cuda(), torch.tensor([t0, t0]).cuda(), ehs.cuda(), cross_attention_kwargs=kw).sample.cpu()
    del oracle
    _free()
    prev_ref = _cfg_step_ref(eps_ref, lat1, steps=30)
    unet = _b200(sd)
    revise_regionally_t2iadapter_attention_forward(unet)
    eps = unet(lat2.cuda(), torch.tensor([float(t0)] * 2).cuda(), ehs.cuda(), cross_attention_kwargs=kw).sample
    s2 = DPMSolverPP2M()
    s2.set_timesteps(30)
    latents = lat1.cuda().clone()
    ops.cfg_dpmpp_step(eps.float().contiguous(), latents, torch.zeros_like(latents), None, cfg=True, guidance=7.5,
                       coef=s2.coefficients(0))
    torch.cuda.synchronize()
    e_eps, e_lat = rel_l2(eps, eps_ref), rel_l2(latents, prev_ref)
    print(f'regional 1024x2048, 3 boxes: eps rel-L2 {e_eps:.3e}, CFG-7.5 latents rel-L2 {e_lat:.3e}')
    del unet
    _free()
    assert e_eps < 5e-3 and e_lat < 1e-3


# ------------------------------------------------------------------------------------------------------------ VAE
def _vae(cuda):
    from mos_b200.vae_engine import VAEEngine
    from oracle import vae as ov
    ref = ov.build_vae(0, None)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    return ref.to(cuda), sd, VAEEngine


def test_vae_520x392(cuda):
    """encode (posterior mean, logvar, sampled latents) and decode at 520 x 392: a 65 x 49 latent, 3185 mid-block tokens"""
    ref, sd, VAEEngine = _vae(cuda)
    eng = VAEEngine(sd, 1, 520, 392)
    g = torch.Generator().manual_seed(12)
    img = torch.rand(1, 3, 520, 392, generator=g) * 2 - 1
    noise = torch.randn(1, 4, 65, 49, generator=g)
    z = torch.randn(1, 4, 65, 49, generator=g)
    with torch.no_grad():
        mean_ref, logvar_ref = ref.moments(img.cuda())
        lat_ref = ref.encode_sample(img.cuda(), noise.cuda()) * 0.18215
        dec_ref = ref.decode(z.cuda())
    mean, logvar, lat = eng.encode(img.cuda(), noise=noise.cuda())
    dec = eng.decode(z.cuda())
    torch.cuda.synchronize()
    errs = [rel_l2(mean, mean_ref), rel_l2(logvar, logvar_ref), rel_l2(lat, lat_ref), rel_l2(dec, dec_ref)]
    print(f'VAE 520x392: mean / logvar / latents / decode rel-L2 {["%.3e" % e for e in errs]}')
    del eng, ref
    _free()
    assert max(errs) < 5e-3


def test_vae_decode_1024x2048(cuda):
    """decode of one 128 x 256 latent: 32768 mid-block tokens, a 32768 x 32800 fp32 score matrix, 1024 x 2048 x 128
    activations at the top level"""
    ref, sd, VAEEngine = _vae(cuda)
    eng = VAEEngine(sd, 1, 1024, 2048)
    z = torch.randn(1, 4, 128, 256, generator=torch.Generator().manual_seed(13))
    dec = eng.decode(z.cuda()).cpu()
    del eng
    _free()
    with torch.no_grad():
        dec_ref = ref.decode(z.cuda()).cpu()
    e = rel_l2(dec, dec_ref)
    print(f'VAE decode 1024x2048: rel-L2 {e:.3e}')
    del ref
    _free()
    assert e < 5e-3


# -------------------------------------------------------------------------------------------------- launch audits
def test_launch_audits_sd15_65x49(cuda, sd15_edlora):
    """every GEMM, attention and norm / elementwise launch of one SD1.5 CFG step at a 65 x 49 latent passes its float64
    bound and write window; the sized nearest upsample is among them"""
    import attention_audit as aa
    import gemm_audit as ga
    import norm_audit as na
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    _, sd, lora = sd15_edlora
    g = torch.Generator().manual_seed(14)
    lat = torch.randn(1, 4, 65, 49, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    eng = UNetEngine(sd, 2, 65, 49, lora=lora, lora_alpha=1.0, use_graph=False)
    stats = {}
    for name, mod in (('gemm', ga), ('attention', aa), ('norm', na)):
        st = mod.Stats()
        with mod.Recorder(st):
            eng.forward(torch.cat([lat, lat]).cuda(), torch.tensor([981.0, 981.0]).cuda(), ehs_to_layer_major(ehs.cuda()))
            torch.cuda.synchronize()
        stats[name] = st
        print(f'\n{name} launch audit, SD1.5 at 65 x 49:\n' + st.table())
    del eng
    _free()
    for name, st in stats.items():
        assert not st.failures, f'{name}: ' + '\n'.join(st.failures[:20])
        assert st.rows, name
    assert 'upsample2x|sized' in stats['norm'].rows
    assert 'im2col|pad=1' in stats['norm'].rows


def test_train_engine_refuses_65x65(cuda, sd15_edlora):
    from mos_b200.train_engine import TrainEngine
    _, sd, lora = sd15_edlora
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match='multiples of 8'):
        TrainEngine(sd, 2, 65, 65, lora=lora)
    assert torch.cuda.memory_allocated() == before
