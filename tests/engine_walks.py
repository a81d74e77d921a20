"""Eager engine walks shared by the launch audits (test_gemm_engine_launches_gpu.py, test_attention_engine_launches_gpu.py,
test_norm_engine_launches_gpu.py, test_solver_engine_launches_gpu.py).

Each walk builds its engine outside the audit and runs one engine call inside `audit()`, a zero-argument callable that
returns the recorder's context manager.  The product-shape walks (train_sd15_full, validation_sd15) build through
bench.py's workload and are built the same way by test_graph_replay_gpu.py, which holds the captured graphs bit-identical
to these eager walks.
"""
import os

import torch


def sd15_pair():
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, None)
    inject.install_edlora_processors(unet)
    return unet, {k: v.clone() for k, v in unet.state_dict().items()}


def _run(audit, fn, register=()):
    """register: tensors that device pointer tables of the call may point into"""
    with audit() as rec:
        rec.register(*register)
        out = fn()
        torch.cuda.synchronize()
    return out


def sample_64(sd15, audit, regions=None, emit_probs=False):
    """fp16 SD1.5 UNet at 64 x 64, CFG batch 2, fused attention LoRA; regions: 3 boxes of per-region embeddings"""
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    unet, sd = sd15
    lora = inject.random_lora_state(unet, seed=10)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(1, 4, 64, 64, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=torch.Generator().manual_seed(2))
    eng = UNetEngine(sd, 2, 64, 64, lora=lora, lora_alpha=1.0, use_graph=False, emit_probs=emit_probs)
    if regions:
        gr = torch.Generator().manual_seed(4)
        eng.set_regions([(ehs_to_layer_major(torch.randn(2, 16, 77, 768, generator=gr).cuda()), b) for b in regions],
                        (512, 512))
    return _run(audit, lambda: eng.forward(torch.cat([lat, lat]).cuda(), torch.tensor([981.0, 981.0]).cuda(),
                                           ehs_to_layer_major(ehs.cuda())).clone())


def sample_96x192_whole_block(sd15, audit):
    """fp16 at 96 x 192 (18432 / 4608 / 1152 / 288 tokens) with a fused whole-block LoRA"""
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    unet, sd = sd15
    lora = inject.random_lora_state(unet, seed=11, where='Transformer2DModel', up_std=0.05)
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(2, 4, 96, 192, generator=g)
    ehs = torch.randn(2, 16, 77, 768, generator=g)
    eng = UNetEngine(sd, 2, 96, 192, lora=lora, lora_alpha=0.8, use_graph=False)
    _run(audit, lambda: eng.forward(lat.cuda(), torch.tensor([501.0, 501.0]).cuda(), ehs_to_layer_major(ehs.cuda())))


def train_sd15_channels_whole_block(audit, attn_reg_weight=None, optimizer_step=False):
    """bf16 TrainEngine.forward_backward at the SD1.5 channels, one layer per block, 16 x 16, B = 2, whole-block LoRA;
    with attn_reg_weight the regulariser runs (pcols / pos / gcols) on a box mask with concept tokens at 4, 5 / 6, 7;
    with optimizer_step the AdamW step and the LoRA re-pack (its table points into the flat state and the GEMM
    operands, registered with the audit) follow"""
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import inject
    from oracle import unet as ou
    cfg = dict(block_out_channels=(320, 640, 1280, 1280), layers_per_block=1)
    ref = ou.build_unet(0, cfg)
    lora = inject.random_lora_state(ref, seed=10, where='Transformer2DModel')
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    B, H = 2, 16
    x0, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    eng = TrainEngine(sd, B, H, H, lora=lora, attn_reg_weight=attn_reg_weight, where='Transformer2DModel',
                      block_out=cfg['block_out_channels'], layers=1, use_graph=False)
    n_x = len(eng.xattn_names)
    ehs = torch.randn(B, n_x, 77, 768, generator=g)
    masks, pos = torch.ones(B, 1, H, H), None
    if attn_reg_weight is not None:
        masks = torch.zeros(B, 1, H, H)
        masks[:, :, 3:12, 4:13] = 1
        pos = [[4, 5], [6, 7]]
    _run(audit, lambda: eng.forward_backward(x0.cuda(), noise.cuda(), torch.tensor([77, 640]).cuda(),
                                             ehs_to_layer_major(ehs.cuda(), n_x), masks.cuda(), token_pos=pos))
    if optimizer_step:
        packed = [e[k] for e in eng.w.values() if isinstance(e, dict) for k in ('lora_down', 'lora_up')
                  if isinstance(e.get(k), torch.Tensor)]
        _run(audit, eng.optimizer_step, register=[eng.state.params, *eng._lora_keep, *packed])


def build_train_sd15_full(use_graph=True, B=2):
    """The training step of bench.py `train_leg` at batch B (2 = the shipped configs' batch_size_per_gpu): SD1.5 UNet at
    64 x 64 with a rank-4 `where: Attention` LoRA, the attention regulariser on all 16 cross layers (weight 0.01,
    reg_full_identity=False) and a 12-layer CLIPTrainEngine over 16 * B layer-major sequences attached (text_grad), all in
    one shared dp.FlatTrainState.  -> SimpleNamespace(eng, text, state, B, nx, concept_ids)"""
    import math
    from types import SimpleNamespace

    from mos_b200 import dp
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from mos_b200.train_engine import TrainEngine
    import bench
    sd, lora, _, _, _ = bench.build_workload()
    dev = torch.device('cuda')
    tsd = bench.synthetic_clip_state()
    g0 = torch.Generator().manual_seed(12)
    tlora = {}                                      # the CLIPAttention LoRA train_leg builds
    for i in range(12):
        for pj in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
            m = f'text_model.encoder.layers.{i}.self_attn.{pj}'
            tlora[m + '.lora_down.weight'] = (torch.rand(4, 768, generator=g0) * 2 - 1) / math.sqrt(768)
            tlora[m + '.lora_up.weight'] = torch.randn(768, 4, generator=g0) * 0.02
    concept_ids = list(range(49408, 49408 + 32))
    n_text = CLIPTrainEngine.lora_param_count(12, 768, 960)
    n_unet = sum(v.numel() for v in lora.values())
    state = dp.FlatTrainState(len(concept_ids), 768, n_text, n_unet, lrs=(1e-3, 1e-5, 1e-4), device=dev)
    eng = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=0.01, reg_full_identity=False, state=state,
                      state_offset=state.group_end[1], text_grad=True, device=dev, use_graph=use_graph)
    nx = len(eng.xattn_names)
    text = CLIPTrainEngine(tsd, nx * B, lora=tlora, lora_alpha=1.0, concept_token_ids=concept_ids, state=state,
                           emb_offset=0, lora_offset=state.group_end[0], device=dev)
    eng.attach_text_engine(text)
    return SimpleNamespace(eng=eng, text=text, state=state, B=B, nx=nx, concept_ids=concept_ids)


def train_sd15_full_inputs(w, seed):
    """one batch of the bench leg's kind: x0, noise, t, box masks and layer-major token ids [16 * B, 77] (BOS, 8 words with
    the two concept tokens of each layer at positions 2 and 3, EOS padding); the box moves with the seed.  At B != 2 the
    prompts have 9 words and sample b carries its concept tokens at positions 1 + b and 3 + 2b, so that they differ
    per sample"""
    B, nx = w.B, w.nx
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, 64, 64, generator=g).cuda()
    noise = torch.randn(B, 4, 64, 64, generator=g).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    ids = torch.randint(1000, 40000, (nx, B, 77), generator=g)
    ids[:, :, 0] = 49406
    ids[:, :, 9 if B == 2 else 10:] = 49407
    pos = [[2, 3]] * B if B == 2 else [[1 + b, 3 + 2 * b] for b in range(B)]
    for l in range(nx):
        for b, (p0, p1) in enumerate(pos):
            ids[l, b, p0], ids[l, b, p1] = w.concept_ids[l % 16], w.concept_ids[16 + l % 16]
    r0, c0 = (int(v) for v in torch.randint(0, 17, (2,), generator=g))
    masks = torch.zeros(B, 1, 64, 64)
    masks[:, :, r0:r0 + 48, c0:c0 + 32] = 1.0
    return dict(latents=x0, noise=noise, timesteps=t, ehs_layers=None, masks=masks.cuda(), token_pos=pos,
                text_ids=ids.reshape(nx * B, 77))


def train_optimizer_step(w):
    """the bench leg's optimiser step: the loss onto the flat buffer, flat AdamW, both LoRA re-packs"""
    from mos_b200 import dp
    scale = dp.allreduce_flat_device(w.state, w.eng.loss_out[0:1])
    dp.optimizer_step(w.state, scale)
    w.eng.refresh_lora()
    w.text.refresh_lora()


def _packed_lora(ents):
    return [e[k] for e in ents if isinstance(e, dict) for k in ('lora_down', 'lora_up')
            if isinstance(e.get(k), torch.Tensor)]


def train_sd15_full(audit, B=2, w=None):
    """bench.py `train_leg` at batch B, eager: one forward_backward (CLIP forward, UNet forward at 64 x 64, masked MSE, the
    regulariser at 64^2 / 32^2 / 16^2 / 8^2, UNet backward with d(text embeddings), CLIP backward), then the optimiser step
    (its lora_pack tables point into the flat state and both engines' GEMM operands, registered with the audit).
    w: an eager build_train_sd15_full to run on instead of a new one"""
    w = w or build_train_sd15_full(use_graph=False, B=B)
    batch = train_sd15_full_inputs(w, 100)
    _run(audit, lambda: w.eng.forward_backward(**batch))
    text_ents = [v for ent in w.text.w.values() for v in ent.values()]
    _run(audit, lambda: train_optimizer_step(w),
         register=[w.state.params, *w.eng._lora_keep, *w.text._keep, *_packed_lora(w.eng.w.values()),
                   *_packed_lora(text_ents)])
    return w


def build_validation_sd15():
    """bench.build_workload(images=4) in bench.build_pipeline: the 4-prompt validation call of the SD1.5 UNet (CFG batch 8)
    -> (pipe, cond [4, 16, 77, 768], neg [4, 77, 768], latents [4, 4, 64, 64])"""
    import bench
    sd, lora, lat, ehs, cfg = bench.build_workload(images=4)
    pipe = bench.build_pipeline(sd, lora, cfg, torch.device('cuda'))
    return pipe, ehs[4:], ehs[:4, 0], lat


def validation_call(pipe, cond, neg, lat, steps=2, callback=None):
    return pipe(prompt_embeds=cond.cuda(), negative_prompt_embeds=neg.cuda(), latents=lat.clone(),
                num_inference_steps=steps, guidance_scale=7.5, output_type='latent', callback=callback).images


def validation_sd15(audit):
    """the validation pass at SD1.5 size: a 4-prompt CFG call (UNet batch 8, 2 DPM-Solver++ steps, eager UNet, latent
    output), then an SD1.5-width VAEEngine decode of 4 latents to 512 x 512"""
    from mos_b200.vae_engine import VAEEngine
    from oracle import vae as ov
    pipe, cond, neg, lat = build_validation_sd15()
    pipe.unet.use_graph = False
    out = _run(audit, lambda: validation_call(pipe, cond, neg, lat))
    del pipe
    ref = ov.build_vae(0, None)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    eng = VAEEngine(sd, 4, 512, 512, block_out=ov.SD15_VAE['block_out_channels'], layers=ov.SD15_VAE['layers_per_block'])
    _run(audit, lambda: eng.decode(out / 0.18215))


def vae_512(audit):
    """VAEEngine at 512 x 512 with the SD1.5 VAE widths: encode with a noise draw, then decode"""
    from mos_b200.vae_engine import VAEEngine
    from oracle import vae as ov
    ref = ov.build_vae(0, None)
    full = dict(ov.SD15_VAE)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    eng = VAEEngine(sd, 1, 512, 512, block_out=full['block_out_channels'], layers=full['layers_per_block'])
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, 512, 512, generator=g) * 2 - 1
    noise, z = torch.randn(1, 4, 64, 64, generator=g), torch.randn(1, 4, 64, 64, generator=g)
    _run(audit, lambda: eng.encode(img.cuda(), noise=noise.cuda()))
    _run(audit, lambda: eng.decode(z.cuda()))


def sampling_loop(audit, tmp_dir):
    """EDLoRAPipeline on a synthetic pretrained directory: 64 x 64, 3 DPM-Solver++ steps with CFG, latent output, eager
    UNet (the CFG / DPM update with the next timestep written for the following UNet call)"""
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from synth import make_pretrained_dir
    pipe = EDLoRAPipeline.from_pretrained(make_pretrained_dir(str(tmp_dir)))
    pipe.set_new_concept_cfg({})                     # no concept tokens: every layer reads the plain prompt
    pipe.unet.use_graph = False
    _run(audit, lambda: pipe('photo of a cat', negative_prompt='blurry', height=64, width=64, num_inference_steps=3,
                             guidance_scale=7.5, output_type='latent'))


def clip_text_and_train(audit, device):
    """CLIPTextEngine (12 layers, fused CLIPAttention LoRA) and CLIPTrainEngine forward + backward (CLIPEncoderLayer LoRA)"""
    from transformers import CLIPTextConfig, CLIPTextModel
    from mos_b200.clip_engine import CLIPTextEngine
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from oracle import inject
    cfg = CLIPTextConfig(vocab_size=49408 + 32, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                         num_attention_heads=12, max_position_embeddings=77)
    torch.manual_seed(0)
    model = CLIPTextModel(cfg).eval()
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 49407, (16, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 9:] = 49407
    concept_ids = list(range(49408, 49408 + 32))
    ids[:, 4] = torch.tensor(concept_ids[:16])
    ids[:, 5] = torch.tensor(concept_ids[16:])
    lora_a = inject.random_lora_state(model, seed=7, where='CLIPAttention', up_std=0.05)
    eng = CLIPTextEngine(sd, 16, lora=lora_a, lora_alpha=0.8)
    _run(audit, lambda: eng(ids))
    lora_l = inject.random_lora_state(model, seed=8, where='CLIPEncoderLayer', up_std=0.05)
    tr = CLIPTrainEngine(sd, 16, lora=lora_l, lora_alpha=0.8, concept_token_ids=concept_ids)
    dy = (torch.randn(16 * 77, 768, generator=g) * 0.05).to(device).to(torch.bfloat16)

    def fwd_bwd():
        tr.forward_train(ids)
        tr.backward(dy)
    _run(audit, fwd_bwd)


# ------------------------------------------------------------------------------------------------ gradient fusion
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden.pt')


def fusion_golden(audit):
    """update_quasi_newton on both golden cases (K [30, 64] / [400, 48], 50 iterations) and merge_lora_into_weight on the
    golden state dict"""
    import gradient_fusion as gf
    gold = torch.load(GOLDEN, weights_only=False)
    g = gold['quasi_newton']
    for case in ('', '2'):
        _run(audit, lambda: gf.update_quasi_newton(g['K' + case], g['V' + case], g['W0' + case].clone(), 50, 'cuda'))
    m = gold['merge_lora']
    _run(audit, lambda: gf.merge_lora_into_weight(m['sd'], m['lora'], list(m['sd'].keys()), 'unet', m['alpha'], 'cuda'))


def fusion_cross_kv(audit):
    """merge_kv_in_cross_attention, 2 concepts x 6 text positions, K / V at the SD1.5 widths (320 / 640 / 1280 x 768)"""
    import gradient_fusion as gf
    g = torch.Generator().manual_seed(21)
    names = [(0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight', 320),
             (0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_v.weight', 320),
             (1, 'down_blocks.1.attentions.0.transformer_blocks.0.attn2.to_k.weight', 640),
             (2, 'mid_block.attentions.0.transformer_blocks.0.attn2.to_v.weight', 1280)]
    sd = {n: torch.randn(c, 768, generator=g) * 768 ** -0.5 for _, n, c in names}
    feats = [{i: torch.randn(6, 768, generator=g) for i in range(3)} for _ in range(2)]
    tuned = []
    for _ in range(2):
        t = {}
        for _, n, c in names:
            dn = n.replace('.weight', '.lora_down.weight')
            t[dn] = torch.randn(4, 768, generator=g) * 768 ** -0.5
            t[dn.replace('lora_down', 'lora_up')] = torch.randn(c, 4, generator=g) * 0.1
        tuned.append(t)
    _run(audit, lambda: gf.merge_kv_in_cross_attention(sd, [(i, n) for i, n, _ in names], feats, tuned, [1.0, 0.7], 20))


def fusion_text_encoder(audit):
    """merge_text_encoder with two CLIPEncoderLayer LoRAs on a 2-layer CLIP (768 / 3072): gram_small at d = 3072"""
    from transformers import CLIPTextConfig, CLIPTextModel
    import gradient_fusion as gf
    from oracle import inject
    cfg = CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                         num_attention_heads=12, max_position_embeddings=77, eos_token_id=999, bos_token_id=998,
                         pad_token_id=999)
    torch.manual_seed(0)
    base = CLIPTextModel(cfg).eval()
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    loras = [inject.random_lora_state(base, seed=40 + c, where='CLIPEncoderLayer', up_std=0.05) for c in range(2)]
    g = torch.Generator().manual_seed(9)
    prompts = [[torch.cat([torch.tensor([998]), torch.randint(0, 990, (n,), generator=g), torch.tensor([999])])
                for n in (5, 2, 5, 2)] for _ in range(2)]
    _run(audit, lambda: gf.merge_text_encoder(sd, loras, [1.0, 0.7], prompts, 10, pad_id=999))


def fusion_spatial_whole_block_tiny(audit):
    """merge_spatial_attention on the tiny topology with two Transformer2DModel LoRAs (2 sampling steps, 5 iterations):
    the Gram recorder's transposes of strided activations, sgemm at in = 4C (ff.net.2), 4-D proj_in / proj_out"""
    import gradient_fusion as gf
    from oracle import inject
    from oracle import unet as ou
    u0 = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in u0.state_dict().items()}
    loras = [inject.random_lora_state(u0, seed=10 + c, where='Transformer2DModel', up_std=0.05) for c in range(2)]
    spatial = [{k: v for k, v in l.items() if 'attn2.to_k' not in k and 'attn2.to_v' not in k} for l in loras]
    embeds = [torch.randn(1, 16, 77, 768, generator=torch.Generator().manual_seed(20 + c)) for c in range(2)]
    _run(audit, lambda: gf.merge_spatial_attention(sd, spatial, [1.0, 1.0], embeds, 5, latent_hw=(16, 16),
                                                   num_inference_steps=2, seed=0,
                                                   block_out=ou.TINY['block_out_channels'], layers=1))


def fusion_sd15_solves(audit, iters=3):
    """the two largest SD1.5 solves of a whole-block fusion, ff.net.0.proj [10240, 1280] and ff.net.2 [1280, 5120]
    (13.1 M-element vectors, a 5120^2 Gram matrix), from Gram matrices of 6000 random feature rows"""
    import gradient_fusion as gf
    jobs = []
    for name, out_f, in_f in (('ff.net.0.proj', 10240, 1280), ('ff.net.2', 1280, 5120)):
        g = torch.Generator(device='cuda').manual_seed(out_f)
        X = torch.randn(6000, in_f, device='cuda', generator=g)
        W0 = torch.randn(out_f, in_f, device='cuda', generator=g) * in_f ** -0.5
        Wt = W0 + 0.01 * torch.randn(out_f, in_f, device='cuda', generator=g)
        G = X.t() @ X
        Cm = Wt @ G
        vv = float((Wt.double() * (Wt.double() @ G.double())).sum())
        jobs.append((name, G, Cm, vv, 6000, W0, (out_f, in_f)))
    return _run(audit, lambda: gf.solve_all(jobs, iters))
