"""Eager engine walks shared by the launch audits (test_gemm_engine_launches_gpu.py, test_attention_engine_launches_gpu.py).

Each walk builds its engine outside the audit and runs one engine call inside `audit()`, a zero-argument callable that
returns the recorder's context manager.
"""
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
